"""Stage A against a float64 reference: the two track heads on designed cost maps, and
query-feature sampling, through the C ABI.

Designed maps (tests/stage_a_designs.py) reach the heads through tapir_cost_volume_tracks_batched:
query n's feature is one-hot on channel n mod 256 and its map is that channel of the grid, so the
split-bf16 GEMM returns the map exactly.  Queries n >= 256 repeat query n mod 256 and must repeat
its outputs bit for bit.  The reference is oracle.tapir_oracle.tracks_from_cost_volume, run once
per clip in float64 (query points stay float32, so the passthrough frame rounds as the reference's
does).  Per map:

  * arg-max equal wherever the fp64 top two tie exactly or their gap is clear of fp32 rounding
    (D.MARGIN); the rest is counted as skipped;
  * points bit-exact on passthrough frames (the query's own coordinates) and on saturated maps
    (the peak cell centre scaled by init / g in the kernels' operation order), within 1e-3 px
    elsewhere wherever the arg-max agrees;
  * logits within 1e-4 (synthetic head) or 1e-4 * max(1, |ref|) (identity head, large logits).

Output buffers carry NaN guards."""
import functools
import math
from typing import NamedTuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import tapir_oracle as O  # noqa: E402
from tapnet_b200 import _lib  # noqa: E402
from tests import gpu_util as U  # noqa: E402
from tests import stage_a_designs as D  # noqa: E402

STRIDE = 8   # initial-resolution pixels per cost-map cell
SAMPLE_TOL = 1e-5


class Case(NamedTuple):
  B: int
  N: int
  T: int
  gh: int
  gw: int
  kind: str          # head weights: 'synth' or 'identity'
  temp: float
  queries: bool      # False: query_tyx = NULL (no passthrough)
  source: str = 'designed'  # or 'unit': random unit features, queries near grid features

  @property
  def id(self):
    s = f'{self.gh}x{self.gw}-b{self.B}_n{self.N}_t{self.T}-{self.source}-{self.kind}-temp{self.temp:g}'
    return s if self.queries else s + '-noquery'


def _cases_32():
  out = []
  # 120 maps (fewer than the 132 persistent CTAs) and 600 maps (the next-map prefetch and the
  # persistent loop); three clips read query b * N + n
  for B, N in ((1, 24), (3, 8), (3, 40)):
    for kind in D.HEAD_KINDS:
      for temp in D.TEMPERATURES:
        out.append(Case(B, N, 5, 32, 32, kind, temp, True))
  out.append(Case(1, 24, 5, 32, 32, 'synth', 20.0, False))
  out.append(Case(3, 8, 5, 32, 32, 'identity', 20.0, False))
  # B * N = 65535: the largest query count a call with 32 x 32 maps accepts
  out += [Case(1, 65535, 1, 32, 32, kind, 20.0, True) for kind in D.HEAD_KINDS]
  out += [Case(1, 40, 6, 32, 32, 'synth', temp, True, 'unit') for temp in (20.0, 1.0)]
  return out


# (gh, gw) -> (B, N, T): 2 x 2 and 7 x 64 run more maps than the generic head has CTAs (528)
_GENERIC_SHAPES = {(2, 2): (1, 200, 3), (3, 5): (2, 30, 5), (5, 3): (1, 40, 5), (7, 64): (1, 120, 5),
                   (64, 7): (2, 20, 5), (31, 32): (1, 30, 5), (32, 31): (1, 30, 5),
                   (33, 33): (3, 12, 5), (96, 128): (1, 8, 5)}


def _cases_generic():
  out = []
  for (gh, gw), (B, N, T) in _GENERIC_SHAPES.items():
    for kind in D.HEAD_KINDS:
      for temp in D.TEMPERATURES:
        out.append(Case(B, N, T, gh, gw, kind, temp, True))
  out.append(Case(3, 12, 5, 33, 33, 'synth', 20.0, False))
  out.append(Case(1, 40, 5, 33, 33, 'synth', 20.0, True, 'unit'))
  return out


CASES_32 = _cases_32()
CASES_GENERIC = _cases_generic()


# ------------------------------------------------------------------------- inputs and reference
@functools.lru_cache(maxsize=None)
def _inputs(B, N, T, gh, gw, source):
  """grid [B, T, gh, gw, 256], query features [B, N, 256], query points [B, N, 3] (fp32) and the
  design index of every map [B, n, T] for the n = min(N, 256) distinct queries."""
  n = min(N, D.C)
  ih, iw = gh * STRIDE, gw * STRIDE
  g = torch.Generator().manual_seed(1000 * B + 7 * n + 11 * T + 13 * gh + gw)
  grid = torch.randn(B, T, gh, gw, D.C, generator=g)  # channels no query reads: any finite values
  design = torch.full((B, n, T), -1, dtype=torch.int64)
  if source == 'designed':
    ds = D.designs(gh, gw)
    k = 0
    for b in range(B):
      for q in range(n):
        for t in range(T):
          design[b, q, t] = k % len(ds)
          grid[b, t, :, :, q] = torch.from_numpy(ds[k % len(ds)].map)
          k += 1
    qf = torch.zeros(B, n, D.C)
    qf[:, torch.arange(n), torch.arange(n)] = 1.0
  else:
    grid = grid / grid.norm(dim=-1, keepdim=True)
    idx = torch.randint(0, T * gh * gw, (B, n), generator=g)
    qf = grid.reshape(B, -1, D.C)[torch.arange(B)[:, None], idx] + 0.05 * torch.randn(B, n, D.C, generator=g)
    qf = qf / qf.norm(dim=-1, keepdim=True)
  qp = D.query_points(B, n, T, ih, iw, seed=17 + n)
  rep = torch.arange(N) % n
  return dict(grid=grid, qf=qf[:, rep].contiguous(), qp=qp[:, rep].contiguous(), design=design, n=n)


@functools.lru_cache(maxsize=None)
def _reference(case):
  inp = _inputs(case.B, case.N, case.T, case.gh, case.gw, case.source)
  n, T, gh, gw = inp['n'], case.T, case.gh, case.gw
  sd64 = {k: v.double() for k, v in D.head_state_dict(case.kind).items()}
  temp = float(np.float32(case.temp))  # the kernels receive the temperature as a float
  cfg = O.Config(softmax_temperature=temp, initial_resolution=(gh * STRIDE, gw * STRIDE))
  grid64, qf64 = inp['grid'].double(), inp['qf'][:, :n].double()
  acc = {k: [] for k in ('pts', 'occ', 'expd', 'am', 'gap', 'tie', 'scale')}
  for b in range(case.B):
    qp = inp['qp'][b:b + 1, :n] if case.queries else None  # float32, as the reference rounds it
    with torch.no_grad():
      pts, occ, expd, am, cv = O.tracks_from_cost_volume(sd64, cfg, qf64[b:b + 1], grid64[b:b + 1], qp,
                                                         return_debug=True)
    assert pts.dtype == torch.float64 and occ.dtype == torch.float64 and cv.dtype == torch.float64
    heat, scale = D.heat_fp64(sd64, cv.permute(1, 0, 2, 3).reshape(n * T, gh, gw), temp)
    gap, tie = D.top_two(heat)
    for k, v in (('pts', pts[0]), ('occ', occ[0]), ('expd', expd[0]), ('am', am[0]),
                 ('gap', gap.view(n, T)), ('tie', tie.view(n, T)), ('scale', scale.view(n, T))):
      acc[k].append(v)
  return {k: torch.stack(v) for k, v in acc.items()}


# ------------------------------------------------------------------------- kernels
_HEADS = {}


def _head_weights(kind):
  """A HeadWeights built from CUDA tensors kept alive here for every later call."""
  if kind not in _HEADS:
    sd = {k: v.float().contiguous().cuda() for k, v in D.head_state_dict(kind).items()}
    hw = _lib.HeadWeights()
    for name, key in (('hid1', 'hid1'), ('hid2', 'hid2'), ('hid3', 'hid3'), ('hid4', 'hid4'),
                      ('occ', 'occ_out')):
      setattr(hw, name + '_w', sd[D.HEAD_PREFIX + key + '.weight'].data_ptr())
      setattr(hw, name + '_b', sd[D.HEAD_PREFIX + key + '.bias'].data_ptr())
    _HEADS[kind] = (hw, sd)
  return _HEADS[kind][0]


def _run(case):
  """Runs one case through tapir_cost_volume_tracks_batched; returns CPU outputs."""
  inp = _inputs(case.B, case.N, case.T, case.gh, case.gw, case.source)
  B, N, T, gh, gw = case.B, case.N, case.T, case.gh, case.gw
  grid, qf = inp['grid'].cuda().contiguous(), inp['qf'].cuda().contiguous()
  qp = inp['qp'].cuda().contiguous() if case.queries else None
  shape = {'pts': (B, N, T, 2), 'occ': (B, N, T), 'expd': (B, N, T), 'am': (B, N, T)}
  outs = {name: U.guarded(math.prod(shape[name]), dt) for name, dt in
          (('pts', torch.float32), ('occ', torch.float32), ('expd', torch.float32), ('am', torch.int32))}
  ws = torch.empty(_lib.cost_volume_workspace_bytes(qf, grid), dtype=torch.uint8, device='cuda')
  _lib.cost_volume_tracks(_head_weights(case.kind), qf, grid, qp, case.temp, (gh * STRIDE, gw * STRIDE),
                          *(body.view(shape[name]) for name, (_, body) in outs.items()), ws)
  torch.cuda.synchronize()
  for name, (buf, _) in outs.items():
    assert U.guards_intact(buf), f'{case.id}: {name}: bytes outside the output were written'
  return {name: body.view(shape[name]).cpu() for name, (_, body) in outs.items()}


# ------------------------------------------------------------------------- comparison
def _check(case, head, got):
  B, N, T, gh, gw = case.B, case.N, case.T, case.gh, case.gw
  inp = _inputs(B, N, T, gh, gw, case.source)
  ref = _reference(case)
  n = inp['n']
  if N > n:  # query n repeats query n mod 256
    rep = torch.arange(N) % n
    for name, v in got.items():
      assert torch.equal(v.view(torch.int32), v[:, rep].view(torch.int32)), f'{name}: repeated queries differ'
  g = {k: v[:, :n] for k, v in got.items()}

  if case.source == 'designed':
    ds = D.designs(gh, gw)
    family = np.array([ds[i].family for i in inp['design'].flatten().tolist()]).reshape(B, n, T)
    designed_tie = torch.tensor([case.kind in ds[i].tie_heads for i in inp['design'].flatten().tolist()])
    designed_tie = designed_tie.view(B, n, T)
    bad = designed_tie & ~ref['tie']
    assert not bad.any(), f'{int(bad.sum())} designed ties do not tie in the reference'
  else:
    family = np.full((B, n, T), 'unit')

  clear = ref['gap'] > D.MARGIN * ref['scale']
  asserted = ref['tie'] | clear
  am_ok = g['am'].long() == ref['am']
  wrong = asserted & ~am_ok
  if wrong.any():
    where = wrong.nonzero()[:8].tolist()
    detail = [(tuple(w), family[tuple(w)], int(g['am'][tuple(w)]), int(ref['am'][tuple(w)])) for w in where]
    pytest.fail(f'{int(wrong.sum())} arg-max cells differ from the reference '
                f'((b, n, t), family, got, want): {detail}')

  qp = inp['qp'][:, :n]
  passed = D.passthrough(qp, T) if case.queries else torch.zeros(B, n, T, dtype=torch.bool)
  saturated = (ref['gap'] > D.SATURATED_GAP) & ~passed
  pts = g['pts']
  # passthrough frames: the query's own (x, y), bit for bit
  want_q = qp[..., [2, 1]][:, :, None].expand(B, n, T, 2)
  assert torch.equal(pts[passed], want_q[passed]), 'passthrough frames'
  assert torch.equal(ref['pts'][passed], want_q[passed].double())
  # saturated maps: the peak cell centre scaled by init / g, in the kernels' fp32 operation order
  am = g['am'].long().numpy()
  cx = ((am % gw).astype(np.float32) + np.float32(0.5)) * np.float32(gw * STRIDE) / np.float32(gw)
  cy = ((am // gw).astype(np.float32) + np.float32(0.5)) * np.float32(gh * STRIDE) / np.float32(gh)
  want_sat = torch.from_numpy(np.stack([cx, cy], -1))
  assert torch.equal(pts[saturated], want_sat[saturated]), 'saturated maps'
  # everywhere else the arg-max agrees: the track budget
  free = am_ok & ~passed & ~saturated
  perr = (pts.double() - ref['pts']).abs().amax(-1)
  assert bool((perr[free] < D.POINT_TOL).all()), f'points: max error {perr[free].max().item():.3e} px'
  assert bool((perr[saturated] < D.POINT_TOL).all())

  # the identity head's logits are large (its hid3 input is map + 64): a relative budget there
  rel = (lambda r: r.abs().clamp(min=1.0)) if case.kind == 'identity' else (lambda r: torch.ones_like(r))
  e_occ = (g['occ'].double() - ref['occ']).abs()
  e_exp = (g['expd'].double() - ref['expd']).abs()
  rel_occ, rel_exp = e_occ / rel(ref['occ']), e_exp / rel(ref['expd'])

  rec = dict(maps=B * n * T, skipped=int((~asserted).sum()), ties=int(ref['tie'].sum()),
             saturated=int(saturated.sum()), passthrough=int(passed.sum()),
             occ_err=e_occ.max(), expd_err=e_exp.max(), occ_rel=rel_occ.max(), expd_rel=rel_exp.max())
  for fam in sorted(set(family.flatten().tolist())):
    m = torch.from_numpy(family == fam)
    if (m & free).any():
      rec[f'pts_err_{fam}'] = perr[m & free].max()
    rec[f'skipped_{fam}'] = int((m & ~asserted).sum())
  U.record(f'stage_a_{head}_{case.id}', **rec)
  assert bool((rel_occ < D.LOGIT_TOL).all()) and bool((rel_exp < D.LOGIT_TOL).all()), \
      f'logits: occ {rel_occ.max().item():.3e}, expd {rel_exp.max().item():.3e}'


@pytest.mark.parametrize('case', CASES_32, ids=[c.id for c in CASES_32])
def test_head_32x32_tc(case):
  """The tensor-core head: every 32 x 32 map."""
  _check(case, 'tc', _run(case))


@pytest.mark.parametrize('case', CASES_GENERIC, ids=[c.id for c in CASES_GENERIC])
def test_head_any_map_size(case):
  """The generic head: every map size other than 32 x 32."""
  _check(case, 'generic', _run(case))


# ------------------------------------------------------------------------- query sampling
def _sample_queries(N, vT, vH, vW, gh, gw, seed):
  """[N, 3] float32 (t, y, x) in video coordinates, and how many leading rows are designed: cell
  centres, the frame border, points outside the frame in y and in x, each at t < 0, t = T - 0.5,
  t > T and inside; random points (some outside the video) after those."""
  g = torch.Generator().manual_seed(seed)
  ymid, xmid = vH * 0.37, vW * 0.61
  yx = [(0.5 * vH / gh, 0.5 * vW / gw), ((gh - 0.5) * vH / gh, (gw - 0.5) * vW / gw),
        ((gh // 2 + 0.5) * vH / gh, (gw // 3 + 0.5) * vW / gw),
        (0.0, 0.0), (vH, vW), (0.0, vW), (vH, 0.0),
        (-5.25, xmid), (vH + 9.0, xmid), (ymid, -3.5), (ymid, vW + 20.0), (-40.0, vW + 40.0)]
  ts = [0.0, min(1.0, vT - 1.0), -1.25, -0.5, vT - 0.5, vT + 2.0, vT - 1.0, 0.7 * vT]
  special = torch.tensor([(t, y, x) for t in ts for (y, x) in yx], dtype=torch.float32)
  rnd = torch.rand(N, 3, generator=g) * torch.tensor([vT + 2.0, vH + 20.0, vW + 20.0]) - \
      torch.tensor([1.0, 10.0, 10.0])
  rnd[:len(special)] = special
  return rnd, len(special)


def _sample_reference(grid64, q, vT, vH, vW):
  """sample_3d with float64 features: the normalised coordinates are formed in fp32 exactly as
  oracle.tapir_oracle.sample_3d does, then F.grid_sample runs in float64 (border padding)."""
  T, gh, gw, _ = grid64.shape
  pos = O.scale_coords(q[None], (vT, vH, vW), (T, gh, gw))
  y = pos[:, :, None, None, :].float().clone()
  y[..., 0] += 0.5
  y = 2 * (y / torch.tensor([T, gh, gw], dtype=torch.float32)) - 1
  y = torch.flip(y, dims=(-1,)).double()
  out = F.grid_sample(grid64.permute(3, 0, 1, 2)[None], y, mode='bilinear', align_corners=False,
                      padding_mode='border')
  return out[0, :, :, 0, 0].t()


# (T, gh, gw, (vT, vH, vW), N): 70000 queries is more than the 65535 the other stage-A launches
# accept (this kernel puts N on grid.x); 17 x 9 from 136 x 72 is not a multiple-of-8 grid
SAMPLE_CASES = [(1, 32, 32, (1, 256, 256), 3000), (3, 24, 40, (3, 192, 320), 3000),
                (5, 60, 60, (5, 480, 480), 70000), (7, 17, 9, (7, 136, 72), 3000)]


@pytest.mark.parametrize('C', [128, 256])
@pytest.mark.parametrize('case', SAMPLE_CASES, ids=[f'T{c[0]}_{c[1]}x{c[2]}_N{c[4]}' for c in SAMPLE_CASES])
def test_sample_query_features(case, C):
  T, gh, gw, (vT, vH, vW), N = case
  lib = _lib.load()
  g = torch.Generator().manual_seed(T * 100 + gh + C)
  grid = torch.randn(T, gh, gw, C, generator=g)
  grid = grid / grid.norm(dim=-1, keepdim=True)  # unit features, as the backbone's grids
  q, n_special = _sample_queries(N, vT, vH, vW, gh, gw, seed=C + N)
  grid_d, q_d = grid.cuda().contiguous(), q.cuda().contiguous()
  buf, out = U.guarded(N * C)
  _lib.check(lib.tapir_sample_query_features(U.ptr(grid_d), T, gh, gw, C, U.ptr(q_d), N, vT, vH, vW,
                                             U.ptr(out), U.stream()), 'sample_query_features')
  torch.cuda.synchronize()
  assert U.guards_intact(buf), 'bytes outside the output were written'
  ref = _sample_reference(grid.double(), q, vT, vH, vW)
  err = (out.view(N, C).cpu().double() - ref).abs()
  U.record(f'sample_query_T{T}_{gh}x{gw}_C{C}_N{N}', err=err.max(), err_special=err[:n_special].max())
  assert err.max().item() < SAMPLE_TOL
