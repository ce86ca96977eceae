"""CPU checks of tests/refine_refs.py: the float64 references agree with the oracle at fp32, the
fp32 error bounds hold for numpy emulations of the kernels' operation order on the designs the
GPU tests use, the same emulations with one deliberate slip each exceed them, the designs contain
the edges they claim, and the refinement entry points of the C ABI reject bad arguments (status 1)
before any CUDA call, so none of this needs a GPU."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import tapir_oracle as O
from tapnet_b200 import _lib
from tests import refine_refs as R

f32 = np.float32


# ------------------------------------------------------------------------------- designs
def unit_grid(B, T, h, w, C, seed):
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(B, T, h, w, C, generator=g)
  return x / x.norm(dim=-1, keepdim=True)


def pyramid(B, T, hires_hw, lowres_hw, pyramid_level, seed):
  """[hires (C 128), lowres (C 256), then pyramid_level avg-pooled copies of lowres]."""
  levels = [unit_grid(B, T, *hires_hw, 128, seed), unit_grid(B, T, *lowres_hw, 256, seed + 1)]
  for _ in range(pyramid_level):
    prev = levels[-1]
    levels.append(R.pool_emulate(prev.reshape(-1, *prev.shape[2:])).reshape(
        B, T, prev.shape[2] // 2, prev.shape[3] // 2, 256))
  return levels


def overflow_positions(h, init, count=4, span=64):
  """fp32 coordinates p (in init-pixel units, along an axis with h cells) whose seven sample rows
  span 8 + 1 cells in the kernel's fp32 chain: the first row's position rounds to just below an
  integer and the last one's to that integer + 6 or above, so the last sample's lower corner
  leaves the 8-row box.  Found by scanning the fp32 values next to each such boundary."""
  found = []
  for k in range(-2, h + 2):
    centre = f32((k + 3.5) * init / h)
    p = centre
    for _ in range(span):
      p = np.nextafter(p, f32(-np.inf))
    for _ in range(2 * span):
      arr = np.array([p], f32)
      y0 = np.floor(R.pix_f32(arr, h, init, h, h, -3))[0]
      y6 = np.floor(R.pix_f32(arr, h, init, h, h, 3))[0]
      if y6 - y0 >= R.BOX_ROWS - 1:
        found.append(float(p))
        if len(found) >= count:
          return found
      p = np.nextafter(p, f32(np.inf))
  return found


def box17_positions(h, w, init_w):
  """x coordinates where the box is 16 and 17 columns wide (w / h = 29 / 12: the 49 samples span
  14.5 cells in x)."""
  xs = np.arange(0, init_w, init_w / 97.0, dtype=np.float64).astype(f32)
  _, _, bw = R.kernel_box(np.zeros_like(xs), xs, h, w, (8 * h, init_w))
  return xs, bw


def corr_positions(Q, T, init_hw, lowres_hw, seed):
  """Random positions over the image and a margin, plus designed rows: corners of the image,
  positions whose samples sit exactly on cell edges, ones partly outside the map, fully outside
  it, far outside, and (per level, along y) the box-overflow positions."""
  ih, iw = init_hw
  g = torch.Generator().manual_seed(seed)
  pos = torch.rand(Q, T, 2, generator=g) * torch.tensor([iw * 1.2, ih * 1.2]) - torch.tensor([iw * 0.1, ih * 0.1])
  gh, gw = lowres_hw
  special = [(0.0, 0.0), (iw - 0.01, ih - 0.01),
             (iw * 4.5 / gw, ih * 4.5 / gh),           # lowres cell centres: edges at every level
             (iw / 2, ih / 2),                          # exact integers
             (-3.0, ih * 0.5), (iw + 2.0, -5.0),        # partly outside
             (-iw * 0.5, ih * 2.0),                     # fully outside
             (-1e4, 3e4)]                               # far outside
  over = overflow_positions(gh, ih)
  special += [(iw * 0.37, p) for p in over]
  flat = pos.view(-1, 2)  # every other row (query-major) is a designed one, while they last
  for i, s in enumerate(special[:(flat.shape[0] + 1) // 2]):
    flat[2 * i] = torch.tensor(s)
  return pos


def corr_feats(Q, T, seed):
  g = torch.Generator().manual_seed(seed)
  return torch.randn(Q, T, 128, generator=g), torch.randn(Q, T, 256, generator=g)


# name: (batch, N, T, init_hw, hires_hw, lowres_hw, pyramid_level)
CORR_DESIGNS = {
    'pl0_32x32': (1, 13, 3, (256, 256), (64, 64), (32, 32), 0),
    'pl1_40x48': (1, 11, 3, (320, 384), (80, 96), (40, 48), 1),
    'pl2_32x32': (1, 13, 2, (256, 256), (64, 64), (32, 32), 2),
    'pl3_32x32': (1, 13, 2, (256, 256), (64, 64), (32, 32), 3),
    'pl3_192x320': (1, 13, 2, (192, 320), (48, 80), (24, 40), 3),   # pooled 12x20, 6x10, 3x5
    'pl1_1024': (1, 5, 2, (1024, 1024), (256, 256), (128, 128), 1),
    'portrait_48x16': (1, 13, 2, (384, 128), (96, 32), (48, 16), 1),
    'box17_12x29': (1, 16, 2, (96, 232), (24, 58), (12, 29), 0),
    'pano_24x72': (1, 13, 2, (192, 576), (48, 144), (24, 72), 1),
    'tiny_4x8': (1, 13, 2, (32, 64), (8, 16), (4, 8), 2),           # pooled 2x4, 1x2
    'tiny_8x8': (1, 13, 2, (64, 64), (16, 16), (8, 8), 3),          # pooled 4x4, 2x2, 1x1
    'batched_b3': (3, 6, 2, (256, 256), (64, 64), (32, 32), 1),
}
HOST_DESIGNS = [k for k in CORR_DESIGNS if k != 'pl1_1024']


def corr_design(name, seed=0):
  B, N, T, init_hw, hi, lo, pl = CORR_DESIGNS[name]
  levels = pyramid(B, T, hi, lo, pl, seed=len(name) + seed)
  pos = corr_positions(B * N, T, init_hw, lo, seed=len(name) + 7)
  feats = corr_feats(B * N, T, seed=len(name) + 9)
  return levels, pos, feats, init_hw, B


def ragged_corr_design(name, clips, T, seed=0):
  """corr_design(name)'s queries split over `clips` clips by a shuffled query_clip table (not in
  clip order; every clip has queries), the clips' grids the design's and seeded variants of it,
  frames 0..T-1.  Returns (levels [clips, T, ...], pos, feats, init_hw, query_clip int32 [Q])."""
  levels, pos, feats, init_hw, B = corr_design(name)
  assert B == 1 and T <= pos.shape[1]
  variants = [levels] + [corr_design(name, seed=100 * seed + c)[0] for c in range(1, clips)]
  levels = [torch.cat([v[li][:, :T] for v in variants]) for li in range(len(levels))]
  Q = pos.shape[0]
  g = torch.Generator().manual_seed(seed)
  table = (torch.arange(Q) % clips)[torch.randperm(Q, generator=g)].to(torch.int32)
  assert not bool((table[1:] >= table[:-1]).all())
  return levels, pos[:, :T].contiguous(), tuple(f[:, :T].contiguous() for f in feats), init_hw, table


# ------------------------------------------------------------------------------- emulations
def _fma_chain(f, q):
  """f [..., K], q [..., K] fp32 -> fp32 sum by sequential FMAs from 0 (each one rounding)."""
  acc = np.zeros(f.shape[:-1], f32)
  for k in range(f.shape[-1]):
    acc = (f[..., k].astype(np.float64) * q[..., k].astype(np.float64) + acc).astype(f32)
  return acc


def _lane_dot(f, q):
  """The kernel's C-long dot: lane l accumulates float4 v * 32 + l by FMAs, then the butterfly."""
  C = f.shape[-1]
  fl = f.reshape(*f.shape[:-1], C // 128, 32, 4).swapaxes(-3, -2).reshape(*f.shape[:-1], 32, C // 32)
  ql = np.broadcast_to(q.reshape(*q.shape[:-1], C // 128, 32, 4).swapaxes(-3, -2).reshape(*q.shape[:-1], 32, C // 32),
                       fl.shape)
  part = _fma_chain(fl, ql)
  lanes = np.arange(32)
  for s in (16, 8, 4, 2, 1):
    part = (part + part[..., lanes ^ s]).astype(f32)
  return part[..., 0]


def emulate_local_corr(levels, pos, feats, init_hw, batch, slip=None):
  """numpy fp32 emulation of local_corr_kernel's correlations [Q, T, 49 L]: the fp32 coordinate
  chain, the 8-row box (cells outside it are 0), the box / per-sample split at 16 columns.
  slip: 'x_by_w' (x normalised by w), 'box16' (box fixed at 16 columns, never per-sample)."""
  ih, iw = init_hw
  Q, T, _ = pos.shape
  N = Q // batch
  out = np.zeros((Q, T, 49 * len(levels)), f32)
  dy, dx = np.repeat(R.OFFSETS, 7), np.tile(R.OFFSETS, 7)
  for t in range(T):
    px, py = pos[:, t, 0].numpy().astype(f32), pos[:, t, 1].numpy().astype(f32)
    for li, grid in enumerate(levels):
      _, _, h, w, C = grid.shape
      g = grid[:, t].numpy().astype(f32)
      q = (feats[0] if C == 128 else feats[1])[:, t].numpy().astype(f32)
      xnorm = w if slip == 'x_by_w' else h
      iy = R.pix_f32(py[:, None], h, ih, h, h, dy[None])
      ix = R.pix_f32(px[:, None], w, iw, xnorm, w, dx[None])
      y0 = np.floor(R.pix_f32(py, h, ih, h, h, -3)).astype(np.int64)
      x0 = np.floor(R.pix_f32(px, w, iw, xnorm, w, -3)).astype(np.int64)
      bw = np.maximum(np.floor(R.pix_f32(px, w, iw, xnorm, w, 3)).astype(np.int64) + 1 - x0 + 1, 2)
      if slip == 'box16':
        bw = np.minimum(bw, R.BOX_COLS_MAX)
      fy, fx = np.floor(iy), np.floor(ix)
      wy1, wy0 = (iy - fy).astype(f32), ((fy + 1) - iy).astype(f32)
      wx1, wx0 = (ix - fx).astype(f32), ((fx + 1) - ix).astype(f32)
      for qi in range(Q):
        gb = g[qi // N]

        def dot(yy, xx):
          ok = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
          res = np.zeros(yy.shape, f32)
          if ok.any():
            res[ok] = _lane_dot(gb[yy[ok], xx[ok]], q[qi][None])
          return res

        boxed = bw[qi] <= R.BOX_COLS_MAX
        ry, rx = fy[qi].astype(np.int64), fx[qi].astype(np.int64)
        ws = [(wx0[qi] * wy0[qi]).astype(f32), (wx1[qi] * wy0[qi]).astype(f32),
              (wx0[qi] * wy1[qi]).astype(f32), (wx1[qi] * wy1[qi]).astype(f32)]
        corners = [(ry, rx), (ry, rx + 1), (ry + 1, rx), (ry + 1, rx + 1)]
        v = np.zeros(49, f32)
        for (cy, cx), wk in zip(corners, ws):
          d = dot(cy, cx)
          if boxed:
            inside = ((cy - y0[qi] >= 0) & (cy - y0[qi] < R.BOX_ROWS) &
                      (cx - x0[qi] >= 0) & (cx - x0[qi] < bw[qi]))
            d = np.where(inside, d, f32(0))
          v = (v + (d * wk).astype(f32)).astype(f32)
        out[qi, t, 49 * li:49 * (li + 1)] = v
  return torch.from_numpy(out)


def emulate_ln512(x, w):
  """ln512 (refine.cu): warp-per-row LayerNorm without bias, fp32 [rows, 512]."""
  from tests.test_backbone_refs_host import emulate_layernorm
  return emulate_layernorm(x, w, None).numpy()


def _gelu32(a):
  A, B = f32(R.GELU_A), f32(R.GELU_B)
  x2 = (a * a).astype(f32)
  inner = (x2.astype(np.float64) * np.float64(B) + np.float64(A)).astype(f32)
  u = (a * inner).astype(f32)
  with np.errstate(over='ignore'):
    e = np.exp2(u.astype(np.float64)).astype(f32)
  d = (e + f32(1)).astype(f32)
  with np.errstate(divide='ignore'):
    r = (f32(1) / d).astype(f32)
  return (a * r).astype(f32)


def _conv32(seq, w, b, causal):
  """fma(w2, v2, fma(w1, v1, fma(w0, v0, b))) over the taps, fp32 (seq [n, F, 2048])."""
  taps = R._conv_taps(torch.from_numpy(seq), causal).numpy()
  acc = np.broadcast_to(b, taps.shape[1:]).astype(f32)
  for k in range(3):
    acc = (taps[k].astype(np.float64) * w[:, k].astype(np.float64) + acc).astype(f32)
  return acc


def emulate_mixer_dw(bs, x, causal, ctx1=None, ctx2=None, slip=None):
  """numpy fp32 emulation of mixer_dw_kernel: (z, LN_1(z) w1, ctx1 out, ctx2 out).  ex2 / rcp are
  replaced by correctly rounded fp32 ones (within the bound's allowance for the MUFU versions).
  slip: 'ctx_swap' (the causal context slots swapped), 'skip_first' (+ skip before the group
  sum), 'ln_no_weight' (LN without its weight)."""
  n, T, C = x.shape
  ln_w = bs['ln_w'] if slip != 'ln_no_weight' else torch.ones(C)
  y = emulate_ln512(x.reshape(-1, C), ln_w).reshape(n, T, C)
  if causal:
    c1 = ctx1.numpy().astype(f32) if ctx1 is not None else np.zeros((n, 2, C), f32)
    c2 = ctx2.numpy().astype(f32) if ctx2 is not None else np.zeros((n, 2, 4 * C), f32)
    if slip == 'ctx_swap':
      c1, c2 = c1[:, ::-1], c2[:, ::-1]
    Y = np.concatenate([c1, y], 1)
  else:
    Y = y
  w1 = bs['w1'].numpy().reshape(4 * C, 3).astype(f32)
  w2 = bs['w2'].numpy().reshape(4 * C, 3).astype(f32)
  a = _conv32(np.repeat(Y, 4, -1), w1, bs['b1'].numpy().astype(f32), causal)
  h = _gelu32(a)
  H = np.concatenate([c2, h], 1) if causal else h
  m = _conv32(H, w2, bs['b2'].numpy().astype(f32), causal).reshape(n, T, C, 4)
  xs = x.numpy().astype(f32)
  if slip == 'skip_first':
    z = xs
    for k in range(4):
      z = (z + m[..., k]).astype(f32)
  else:
    s = (((m[..., 0] + m[..., 1]).astype(f32) + m[..., 2]).astype(f32) + m[..., 3]).astype(f32)
    z = (s + xs).astype(f32)
  p = emulate_ln512(torch.from_numpy(z.reshape(-1, C)), bs['ln1_w']).reshape(n, T, C)
  t = torch.from_numpy
  return (t(z), t(p), t(np.ascontiguousarray(Y[:, -2:])) if causal else None,
          t(np.ascontiguousarray(H[:, -2:])) if causal else None)


def mixer_input(n, T, seed, large_every=3):
  """N(0, 1) rows, every `large_every`-th query scaled by 1e3 (where the skip dominates z, so the
  order of its addition shows), plus random contexts."""
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(n, T, 512, generator=g)
  if large_every:
    x[::large_every] *= 1e3
  return x, torch.randn(n, 2, 512, generator=g), torch.randn(n, 2, 2048, generator=g)


def _ratio(got, ref, bound):
  err = (got.double() - ref.double()).abs()
  return float((err / bound.clamp(min=1e-300)).max()), float(err.max())


# ------------------------------------------------------------------------------- designs hold
def test_overflow_positions_exist_and_drop_a_weighted_corner():
  for h, init in ((40, 320), (24, 192), (12, 192), (3, 192), (48, 384)):
    ps = overflow_positions(h, init)
    assert ps, (h, init)
    arr = np.array(ps, f32)
    y0 = np.floor(R.pix_f32(arr, h, init, h, h, -3))
    y6 = R.pix_f32(arr, h, init, h, h, 3)
    assert bool((np.floor(y6) - y0 >= 7).all())
    # the dropped corner's weight is fp jitter: nonzero for some, tiny for all
    w = y6 - np.floor(y6)
    assert float(w.max()) < 1e-4


def test_box17_design_has_both_widths_and_the_per_sample_path_runs_elsewhere():
  xs, bw = box17_positions(12, 29, 232)
  assert {16, 17} <= set(bw.tolist())
  _, _, bw_pano = R.kernel_box(np.zeros(50, f32), np.linspace(0, 576, 50).astype(f32), 24, 72, (192, 576))
  assert bool((bw_pano > R.BOX_COLS_MAX).all())


def test_designs_contain_edges():
  levels, pos, feats, init_hw, B = corr_design('pl1_40x48')
  ih, iw = init_hw
  p = pos.reshape(-1, 2)
  assert bool(((p[:, 0] < 0) | (p[:, 1] < 0) | (p[:, 0] > iw) | (p[:, 1] > ih)).any())
  assert bool((p.abs() > 1e3).any())  # far outside
  # samples exactly on cell edges at the lowres level (the kernel's fp32 chain lands a rounding
  # error away from them)
  iy = R.pix_exact(p[:, 1].numpy(), 40, ih, 40, 40, 0)
  assert bool((iy == np.floor(iy)).any())
  # rows whose box overflows (a dropped corner) at the lowres level
  y0 = np.floor(R.pix_f32(p[:, 1].numpy(), 40, ih, 40, 40, -3))
  y6 = np.floor(R.pix_f32(p[:, 1].numpy(), 40, ih, 40, 40, 3))
  assert bool((y6 - y0 >= 7).any())


# ------------------------------------------------------------------------------- bounds hold
@pytest.mark.parametrize('name', HOST_DESIGNS)
def test_corr_bound_holds_for_fp32_emulation(name):
  levels, pos, feats, init_hw, B = corr_design(name)
  ref, bound = R.local_corr_ref(levels, pos, feats, init_hw, B)
  got = emulate_local_corr(levels, pos, feats, init_hw, B)
  r, err = _ratio(got, ref, bound)
  assert r <= 1.0, (r, err)


@pytest.mark.parametrize('name,slip', [('pl1_40x48', 'x_by_w'), ('portrait_48x16', 'x_by_w'),
                                       ('box17_12x29', 'box16')])
def test_corr_bound_rejects_slips(name, slip):
  levels, pos, feats, init_hw, B = corr_design(name)
  ref, bound = R.local_corr_ref(levels, pos, feats, init_hw, B)
  got = emulate_local_corr(levels, pos, feats, init_hw, B, slip=slip)
  r, _ = _ratio(got, ref, bound)
  assert r > 100, r


MIXER_HOST_CASES = [(False, 3, False), (False, 25, False), (True, 1, True), (True, 3, True),
                    (True, 26, True), (True, 3, False), (True, 1, False)]


@pytest.mark.parametrize('causal,T,with_ctx', MIXER_HOST_CASES)
def test_mixer_dw_bound_holds_for_fp32_emulation(causal, T, with_ctx):
  bs = R.block_weights(seed=T)
  x, c1, c2 = mixer_input(4, T, seed=T + causal)
  c1, c2 = (c1, c2) if with_ctx else (None, None)
  ref = R.mixer_dw_ref(bs, x, causal, c1, c2)
  z, p, o1, o2 = emulate_mixer_dw(bs, x, causal, c1, c2)
  for key, got in (('z', z), ('planes', p), ('ctx1', o1), ('ctx2', o2)):
    if key in ref:
      r, err = _ratio(got, *ref[key])
      assert r <= 1.0, (key, r, err)


@pytest.mark.parametrize('slip,key', [('ctx_swap', 'z'), ('skip_first', 'z'), ('ln_no_weight', 'planes')])
def test_mixer_dw_bound_rejects_slips(slip, key):
  bs = R.block_weights(seed=5)
  x, c1, c2 = mixer_input(6, 3, seed=5)
  ref = R.mixer_dw_ref(bs, x, True, c1, c2)
  got = emulate_mixer_dw(bs, x, True, c1, c2, slip=slip)
  got = got[0] if key == 'z' else got[1]
  r, _ = _ratio(got, *ref[key])
  assert r > 1.5, r


def test_corr_ref_clip_table_in_order_equals_batched():
  levels, pos, feats, init_hw, B = corr_design('batched_b3')
  want = R.local_corr_ref(levels, pos, feats, init_hw, B)
  table = torch.arange(pos.shape[0]) // (pos.shape[0] // B)
  got = R.local_corr_ref(levels, pos, feats, init_hw, B, query_clip=table)
  assert all(torch.equal(x, y) for x, y in zip(got, want))
  # a shuffled table reads each query's own clip: the batched result, permuted with the queries
  perm = torch.randperm(pos.shape[0], generator=torch.Generator().manual_seed(1))
  got = R.local_corr_ref(levels, pos[perm], tuple(f[perm] for f in feats), init_hw, B, query_clip=table[perm])
  assert all(torch.equal(x, y[perm]) for x, y in zip(got, want))


@pytest.mark.parametrize('T', [1, 2])
@pytest.mark.parametrize('name,clips', [('tiny_4x8', 3), ('box17_12x29', 4), ('pl3_32x32', 5)])
def test_corr_ref_sees_a_wrong_clip_table(name, clips, T):
  """On the ragged designs of tests/test_refine_ops_gpu.py, the correlations of a kernel that read
  clip 0 (or the clip in query order) for every query break the bound of the right table."""
  levels, pos, feats, init_hw, table = ragged_corr_design(name, clips, T)
  ref, bound = R.local_corr_ref(levels, pos, feats, init_hw, clips, query_clip=table)
  for wrong in (torch.zeros_like(table), table.sort().values):
    got, _ = R.local_corr_ref(levels, pos, feats, init_hw, clips, query_clip=wrong)
    r, _ = _ratio(got.float(), ref, bound)
    assert r > 100, r


# ------------------------------------------------------------------------------- vs the oracle
@pytest.mark.parametrize('name', HOST_DESIGNS)
def test_corr_ref_matches_oracle(name):
  levels, pos, feats, init_hw, B = corr_design(name)
  if B != 1:
    pytest.skip('the oracle takes one clip')
  ref, bound = R.local_corr_ref(levels, pos, feats, init_hw, B)
  cfg = O.Config(initial_resolution=init_hw)
  last = torch.cat(feats, -1)[None]
  ora = O.local_correlation(cfg, [None] * len(levels), list(levels), pos[None], last)[0]
  # the oracle is fp32 throughout (scale, offsets, grid_sample's unnormalisation): it agrees to
  # fp32 noise (1.1e-5 of the largest correlation at most over these designs)
  scale = float(ref.abs().max())
  assert float((ora.double() - ref).abs().max()) < 2e-5 * max(scale, 1.0)


@pytest.mark.parametrize('causal,with_ctx', [(True, True), (True, False), (False, False)])
def test_mixer_dw_ref_matches_oracle(causal, with_ctx):
  """The oracle's block restated up to the channel MLP: _ln_noshift, _dwconv, gelu, group sum."""
  bs = R.block_weights(seed=11)
  n, T = 3, 5
  x, c1, c2 = mixer_input(n, T, seed=12, large_every=0)
  c1, c2 = (c1, c2) if with_ctx else (None, None)
  ref = R.mixer_dw_ref(bs, x, causal, c1, c2)
  y = O._ln_noshift(x, bs['ln_w'])
  if with_ctx:
    y = torch.cat([c1, y], 1)
  h = F.gelu(O._dwconv(y, bs['w1'], bs['b1'], causal), approximate='tanh')
  if with_ctx:
    h = torch.cat([c2, h[:, 2:]], 1)
  hh = O._dwconv(h, bs['w2'], bs['b2'], causal)
  if with_ctx:
    hh = hh[:, 2:]
  z = hh[..., 0::4] + hh[..., 1::4] + hh[..., 2::4] + hh[..., 3::4] + x
  assert torch.allclose(ref['z'][0].float(), z, rtol=1e-5, atol=1e-4)
  assert torch.allclose(ref['planes'][0].float(), O._ln_noshift(z, bs['ln1_w']), rtol=1e-4, atol=1e-4)
  if with_ctx:
    assert torch.allclose(ref['ctx1'][0].float(), y[:, -2:], atol=1e-5)
    assert torch.allclose(ref['ctx2'][0].float(), h[:, -2:], atol=1e-5)


def test_pool_emulation_matches_avg_pool3d():
  g = torch.Generator().manual_seed(3)
  x = torch.randn(1, 3, 9, 11, 256, generator=g)
  ora = F.avg_pool3d(x, (2, 2, 1), (2, 2, 1))[0]
  assert torch.allclose(R.pool_emulate(x[0]), ora, atol=1e-6)


def test_update_emulation_matches_refine_pips_update_lines():
  """O.refine_pips' last lines: scale_coords(res[:2], (rw, rh), (iw, ih)) + pos, res[2] + occ,
  res[3] + expd, res[4:] + feats; train2orig: scale_coords(pos, init, video)."""
  g = torch.Generator().manual_seed(4)
  Q, T = 5, 3
  res = torch.randn(Q, T, 388, generator=g)
  pos = torch.rand(Q, T, 2, generator=g) * 300
  occ, expd = torch.randn(Q, T, generator=g), torch.randn(Q, T, generator=g)
  feats = torch.randn(Q, T, 384, generator=g)
  init_hw, resize_hw, video_hw = (192, 320), (384, 640), (480, 854)
  p, o, e, f, trk = R.update_emulate(res, pos, occ, expd, feats, init_hw, resize_hw, video_hw)
  dpos = O.scale_coords(res[..., :2], resize_hw[::-1], init_hw[::-1])
  assert torch.equal(p, dpos + pos)
  assert torch.equal(o, res[..., 2] + occ) and torch.equal(e, res[..., 3] + expd)
  assert torch.equal(f, res[..., 4:] + feats)
  assert torch.equal(trk, O.scale_coords(p, init_hw[::-1], video_hw[::-1]))


def test_update_emulation_per_query_sizes_equal_per_clip_calls():
  """update_emulate with one (h, w) per query, from an in-order clip table, equals the batched form
  clip by clip; with a shuffled table, each query is scaled to its own clip's size."""
  g = torch.Generator().manual_seed(5)
  counts, T = [4, 1, 6], 2
  Q = sum(counts)
  res = torch.randn(Q, T, 392, generator=g)
  pos = torch.rand(Q, T, 2, generator=g) * 300
  occ, expd = torch.randn(Q, T, generator=g), torch.randn(Q, T, generator=g)
  feats = torch.randn(Q, T, 384, generator=g)
  sizes = [(480, 640), (200, 200), (1080, 1920)]
  args = ((256, 256), (320, 384))
  for table in (torch.tensor([b for b, n in enumerate(counts) for _ in range(n)]),
                torch.tensor([2, 0, 1, 2, 2, 0, 2, 0, 2, 0, 2])):
    got = R.update_emulate(res, pos, occ, expd, feats, *args, np.array(sizes)[table.numpy()])
    for b in range(len(sizes)):
      m = table == b
      want = R.update_emulate(res[m], pos[m], occ[m], expd[m], feats[m], *args, sizes[b])
      assert all(torch.equal(x[m], y) for x, y in zip(got, want)), b


# ------------------------------------------------------------------------------- bad arguments
def _p(addr):
  return ctypes.c_void_p(addr)


A = 1 << 20  # a 16-byte aligned fake device address: every call below fails before using it


def corr_args(**kw):
  ca = _lib.CorrArgs()
  for i in range(3):
    ca.levels[i].grid, ca.levels[i].h, ca.levels[i].w = A, 32 >> i, 32 >> i
    ca.levels[i].C = 128 if i == 0 else 256
  ca.num_levels, ca.num_points, ca.num_frames = 3, 4, 2
  ca.init_h = ca.init_w = 256
  ca.planes = 2
  ca.pos = ca.occ = ca.expd = A
  ca.feat_hi, ca.feat_hi_stride_n, ca.feat_hi_stride_t = A, 128, 0
  ca.feat_lo, ca.feat_lo_stride_n, ca.feat_lo_stride_t = A, 256, 0
  ca.ld = 576
  ca.out_planes, ca.out_plane_stride = A, 8 * 576
  for k, v in kw.items():
    if k.startswith('level'):
      i, field = k[5], k[7:]
      setattr(ca.levels[int(i)], field, v)
    else:
      setattr(ca, k, v)
  return ca


CORR_BAD = {'grid align': dict(level1_grid=A + 4), 'level h': dict(level2_h=0), 'level w': dict(level0_w=0),
            'init_h': dict(init_h=0), 'init_w': dict(init_w=-1), 'feat_hi align': dict(feat_hi=A + 8),
            'feat_lo align': dict(feat_lo=A + 4), 'feat stride_n': dict(feat_lo_stride_n=258),
            'feat stride_t': dict(feat_hi_stride_t=130), 'feat stride negative': dict(feat_hi_stride_t=-128),
            'planes overlap': dict(out_plane_stride=576), 'out align': dict(out_planes=A + 2),
            'levels': dict(num_levels=6), 'null pos': dict(pos=None)}


@pytest.mark.parametrize('batched', [False, True])
@pytest.mark.parametrize('case', list(CORR_BAD))
def test_local_corr_rejects_bad_arguments(case, batched):
  lib = _lib.load()
  ca = corr_args(**CORR_BAD[case])
  rc = (lib.tapir_local_corr_batched(ctypes.byref(ca), 2, None) if batched
        else lib.tapir_local_corr(ctypes.byref(ca), None))
  assert rc == 1, (case, rc, lib.tapir_last_error())
  assert b'local_corr' in lib.tapir_last_error()


def update_args(**kw):
  ua = _lib.UpdateArgs()
  ua.res, ua.ld_res, ua.num_points, ua.num_frames = A, 388, 4, 2
  ua.init_h = ua.init_w = ua.resize_h = ua.resize_w = ua.video_h = ua.video_w = 256
  ua.feat_hi, ua.feat_hi_stride_n, ua.feat_hi_stride_t = A, 128, 0
  ua.feat_lo, ua.feat_lo_stride_n, ua.feat_lo_stride_t = A, 256, 0
  ua.pos = ua.occ_in = ua.expd_in = ua.occ_out = ua.expd_out = ua.feat_out = ua.tracks_out = A
  for k, v in kw.items():
    setattr(ua, k, v)
  return ua


UPDATE_BAD = {'null feat_hi': dict(feat_hi=None), 'null feat_lo': dict(feat_lo=None),
              'null occ_in': dict(occ_in=None), 'null expd_in': dict(expd_in=None),
              'null res': dict(res=None), 'num_points': dict(num_points=0), 'num_frames': dict(num_frames=-1),
              'rows 2^31': dict(num_points=1 << 16, num_frames=1 << 15), 'ld_res': dict(ld_res=387),
              'resize_w': dict(resize_w=0), 'video_h with tracks': dict(video_h=0)}


@pytest.mark.parametrize('case', list(UPDATE_BAD))
def test_refine_update_rejects_bad_arguments(case):
  lib = _lib.load()
  ua = update_args(**UPDATE_BAD[case])
  rc = lib.tapir_refine_update(ctypes.byref(ua), None)
  assert rc == 1, (case, rc, lib.tapir_last_error())
  assert lib.tapir_last_error().startswith(b'tapir_refine_update:')


POOL_BAD = {'null': (None, 1, 4, 4, 256, _p(A)), 'grid align': (_p(A + 4), 1, 4, 4, 256, _p(A)),
            'out align': (_p(A), 1, 4, 4, 256, _p(A + 8)), 'h': (_p(A), 1, 1, 4, 256, _p(A)),
            'C': (_p(A), 1, 4, 4, 254, _p(A)), 'T': (_p(A), 0, 4, 4, 256, _p(A))}


@pytest.mark.parametrize('case', list(POOL_BAD))
def test_pool_pyramid_rejects_bad_arguments(case):
  lib = _lib.load()
  rc = lib.tapir_pool_pyramid(*POOL_BAD[case], None)
  assert rc == 1, (case, rc)
  assert lib.tapir_last_error().startswith(b'tapir_pool_pyramid:')


def mixer_block(**kw):
  blk = _lib.MixerBlock()
  blk.ln_w = blk.dw1_w = blk.dw1_b = blk.dw2_w = blk.dw2_b = blk.ln1_w = A
  for k, v in kw.items():
    setattr(blk, k, v)
  return blk


X, Z, PL, C1I, C2I, C1O, C2O = (A * k for k in (1, 64, 128, 256, 320, 384, 448))


def mixer_dw_call(blk=None, x=X, n=4, T=3, causal=1, c1i=C1I, c2i=C2I, c1o=C1O, c2o=C2O, z=Z, planes_out=PL,
                  plane_stride=4 * 3 * 512, planes=3):
  lib = _lib.load()
  blk = blk if blk is not None else mixer_block()
  return lib.tapir_mixer_dw(ctypes.byref(blk), _p(x), n, T, causal, _p(c1i) if c1i else None,
                            _p(c2i) if c2i else None, _p(c1o) if c1o else None, _p(c2o) if c2o else None,
                            _p(z) if z else None, _p(planes_out) if planes_out else None, plane_stride, planes,
                            None)


MIXER_BAD = {'null x': dict(x=0), 'null z': dict(z=0), 'null planes': dict(planes_out=0),
             'null weight': dict(blk=mixer_block(dw2_b=None)), 'n 0': dict(n=0), 'n 65536': dict(n=65536),
             'T 0': dict(T=0), 'planes 0': dict(planes=0), 'planes 4': dict(planes=4),
             'x align': dict(x=X + 4), 'z align': dict(z=Z + 8), 'ctx align': dict(c2o=C2O + 4),
             'ln_w align': dict(blk=mixer_block(ln1_w=A + 4)), 'planes align': dict(planes_out=PL + 4),
             'planes overlap': dict(plane_stride=512), 'x z overlap': dict(z=X + 4096),
             'ctx on non-causal': dict(causal=0, c1i=0, c2i=0, c2o=0),
             'ctx1 alias T 3': dict(c1o=C1I), 'ctx2 alias T 3': dict(c2o=C2I),
             'ctx2 partial alias T 1': dict(T=1, c2o=C2I + 16, plane_stride=4 * 512)}


@pytest.mark.parametrize('case', list(MIXER_BAD))
def test_mixer_dw_rejects_bad_arguments(case):
  lib = _lib.load()
  rc = mixer_dw_call(**MIXER_BAD[case])
  assert rc == 1, (case, rc, lib.tapir_last_error())
  assert lib.tapir_last_error().startswith(b'tapir_mixer_dw:')
