"""Per-stage parity of the CUDA path (through the C ABI) against the CPU oracle."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import synth  # noqa: E402
from oracle import tapir_oracle as O  # noqa: E402
from tapnet_b200 import _lib, tapir_model  # noqa: E402
from tests import gpu_util as U  # noqa: E402

_MODELS = {}


def get_model(pyramid_level=1, extra_convs=True, causal=False, precision='bf16x3'):
  key = (pyramid_level, extra_convs, causal, precision)
  if key not in _MODELS:
    sd = synth.make_state_dict(0, pyramid_level, extra_convs)
    m = tapir_model.TAPIR(pyramid_level=pyramid_level, extra_convs=extra_convs,
                          use_casual_conv=causal, precision=precision)
    m.load_state_dict(sd)
    _MODELS[key] = (m.cuda().eval(), sd,
                    O.Config(pyramid_level=pyramid_level, extra_convs=extra_convs,
                             use_casual_conv=causal))
  return _MODELS[key]


def maxerr(a, b):
  return (a.detach().float().cpu() - b.detach().float().cpu()).abs().max().item()


def test_abi_loads():
  lib = _lib.load()
  assert lib.tapir_abi_version() == 2


@pytest.mark.parametrize('shape', [(2, 256, 256), (1, 64, 96)])
def test_backbone(shape):
  T, H, W = shape
  model, sd, cfg = get_model()
  video = synth.make_video(T, H, W)
  with torch.no_grad():
    cfg2 = cfg._replace(initial_resolution=(H, W))
    ref = O.get_feature_grids(sd, cfg2, video, refinement_resolutions=[(H, W)])
  model.initial_resolution = (H, W)
  try:
    got = model.get_feature_grids(video.cuda(), False, [(H, W)])
  finally:
    model.initial_resolution = (256, 256)
  torch.cuda.synchronize()
  e_lo = maxerr(got.lowres[0], ref.lowres[0])
  e_hi = maxerr(got.hires[0], ref.hires[0])
  U.record(f'backbone_{T}x{H}x{W}', lowres_err=e_lo, hires_err=e_hi)
  assert e_lo < 2e-4 and e_hi < 2e-4


def test_backbone_resize_path():
  model, sd, cfg = get_model()
  video = synth.make_video(1, 320, 384)
  with torch.no_grad():
    ref = O.get_feature_grids(sd, cfg, video)
  got = model.get_feature_grids(video.cuda(), False)
  assert [tuple(r) for r in got.resolutions] == [tuple(r) for r in ref.resolutions]
  for i in range(len(ref.lowres)):
    e = maxerr(got.lowres[i], ref.lowres[i])
    U.record(f'backbone_resize_level{i}', lowres_err=e, hires_err=maxerr(got.hires[i], ref.hires[i]))
    assert e < 3e-4


def test_query_features():
  model, sd, cfg = get_model()
  T, N = 5, 64
  g = torch.Generator().manual_seed(3)
  lo = torch.randn(1, T, 32, 32, 256, generator=g)
  hi = torch.randn(1, T, 64, 64, 128, generator=g)
  q = synth.make_queries(N, T)
  q[0, 0] = torch.tensor([0.0, 0.0, 0.0])
  q[0, 1] = torch.tensor([T - 1.0, 255.9, 255.9])
  q[0, 2] = torch.tensor([2.5, 100.25, 3.75])  # fractional t (allowed by the API)
  grids = O.Grids((lo,), (hi,), ((256, 256),))
  ref = O.get_query_features(cfg, (1, T, 256, 256, 3), q, grids)
  fg = tapir_model.FeatureGrids((lo.cuda(),), (hi.cuda(),), ((256, 256),))
  got = model.get_query_features(torch.empty(1, T, 256, 256, 3), False, q.cuda(), fg)
  e1, e2 = maxerr(got.lowres[0], ref.lowres[0]), maxerr(got.hires[0], ref.hires[0])
  U.record('query_features', lowres_err=e1, hires_err=e2)
  assert e1 < 1e-5 and e2 < 1e-5


def _run_cost_volume(model, qf, grid, qp, init_hw, *outs):
  """Stage A of one clip (qf [1, N, 256], grid [1, T, h, w, 256], qp [1, N, 3] on the CPU) into the
  [N, T, ...] CUDA outputs (points, occ, expd, argmax)."""
  qf, grid, qp = (t.cuda().contiguous() for t in (qf, grid, qp))
  ws = torch.empty(_lib.cost_volume_workspace_bytes(qf, grid), dtype=torch.uint8, device='cuda')
  _lib.cost_volume_tracks(model._pack()['head'], qf, grid, qp, 20.0, init_hw, *(o[None] for o in outs), ws)


def _unit_grid(T, h, w, c, seed):
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(1, T, h, w, c, generator=g)
  return x / x.norm(dim=-1, keepdim=True)


def test_cost_volume_tracks():
  model, sd, cfg = get_model()
  T, N = 6, 40
  grid = _unit_grid(T, 32, 32, 256, 5)
  # queries = features sampled from the grid itself (+ noise) so heat maps are peaked
  g = torch.Generator().manual_seed(6)
  idx = torch.randint(0, T * 32 * 32, (N,), generator=g)
  qf = grid.reshape(-1, 256)[idx] + 0.05 * torch.randn(N, 256, generator=g)
  qf = (qf / qf.norm(dim=-1, keepdim=True))[None]
  qp = synth.make_queries(N, T)
  with torch.no_grad():
    pts, occ, expd, am, cv = O.tracks_from_cost_volume(sd, cfg, qf, grid, qp, return_debug=True)
  dev = 'cuda'
  o_pts = torch.empty(N, T, 2, device=dev)
  o_occ = torch.empty(N, T, device=dev)
  o_exp = torch.empty(N, T, device=dev)
  o_am = torch.empty(N, T, dtype=torch.int32, device=dev)
  _run_cost_volume(model, qf, grid, qp, (256, 256), o_pts, o_occ, o_exp, o_am)
  torch.cuda.synchronize()
  agree = (o_am.cpu().long() == am[0]).float().mean().item()
  e_p, e_o, e_e = maxerr(o_pts, pts[0]), maxerr(o_occ, occ[0]), maxerr(o_exp, expd[0])
  U.record('cost_volume_tracks', argmax_agree=agree, pts_err=e_p, occ_err=e_o, expd_err=e_e)
  assert agree == 1.0
  assert e_p < 1e-3 and e_o < 1e-4 and e_e < 1e-4


@pytest.mark.parametrize('shape', [(24, 40), (48, 16)])
def test_cost_volume_tracks_any_map_size(shape):
  """initial_resolution != (256, 256) (ctor argument, tapir_model.py:86): the cost map is not
  32 x 32 and the generic-size head runs.  Same checks as the 32 x 32 case."""
  gh, gw = shape
  model, sd, cfg = get_model()
  T, N = 3, 20
  grid = _unit_grid(T, gh, gw, 256, 15)
  g = torch.Generator().manual_seed(16)
  idx = torch.randint(0, T * gh * gw, (N,), generator=g)
  qf = grid.reshape(-1, 256)[idx] + 0.05 * torch.randn(N, 256, generator=g)
  qf = (qf / qf.norm(dim=-1, keepdim=True))[None]
  ih, iw = gh * 8, gw * 8
  qp = synth.make_queries(N, T, ih, iw)
  cfg2 = cfg._replace(initial_resolution=(ih, iw))
  with torch.no_grad():
    pts, occ, expd, am, _ = O.tracks_from_cost_volume(sd, cfg2, qf, grid, qp, return_debug=True)
  dev = 'cuda'
  o_pts = torch.empty(N, T, 2, device=dev)
  o_occ = torch.empty(N, T, device=dev)
  o_exp = torch.empty(N, T, device=dev)
  o_am = torch.empty(N, T, dtype=torch.int32, device=dev)
  _run_cost_volume(model, qf, grid, qp, (ih, iw), o_pts, o_occ, o_exp, o_am)
  torch.cuda.synchronize()
  agree = (o_am.cpu().long() == am[0]).float().mean().item()
  e_p, e_o, e_e = maxerr(o_pts, pts[0]), maxerr(o_occ, occ[0]), maxerr(o_exp, expd[0])
  U.record(f'cost_volume_tracks_{gh}x{gw}', argmax_agree=agree, pts_err=e_p, occ_err=e_o, expd_err=e_e)
  assert agree == 1.0
  assert e_p < 1e-3 and e_o < 1e-4 and e_e < 1e-4


def _run_mixer(model, x, causal, ctx=None, get_ctx=False, in_place=False):
  """in_place: the context output pointers are the context input buffers (the streaming call)."""
  pk = model._pack()
  n, T, cin = x.shape
  dev = 'cuda'
  xp = U.split(x.reshape(n * T, cin).cuda(), model._planes, pk['mixer_in'])
  out = torch.empty(n, T, 388, device=dev)
  nb = pk['num_blocks']
  c1 = c2 = o1 = o2 = None
  if ctx is not None:
    c1 = [ctx[f'block_{i}_causal_1'].cuda().contiguous() for i in range(nb)]
    c2 = [ctx[f'block_{i}_causal_2'].cuda().contiguous() for i in range(nb)]
  if get_ctx:
    if in_place:
      o1, o2 = c1, c2
    else:
      o1 = [torch.empty(n, 2, 512, device=dev) for _ in range(nb)]
      o2 = [torch.empty(n, 2, 2048, device=dev) for _ in range(nb)]
  ws = torch.empty(_lib.mixer_workspace_bytes(xp), dtype=torch.uint8, device=dev)
  _lib.mixer_forward(pk['mixer'], xp, out, causal, c1, c2, o1, o2, ws)
  torch.cuda.synchronize()
  new_ctx = None
  if get_ctx:
    new_ctx = {}
    for i in range(nb):
      new_ctx[f'block_{i}_causal_1'] = o1[i].cpu()
      new_ctx[f'block_{i}_causal_2'] = o2[i].cpu()
  return out.cpu().reshape(n, T, 388), new_ctx


@pytest.mark.parametrize('T', [1, 5, 8, 24, 50])
def test_mixer_noncausal(T):
  model, sd, cfg = get_model()
  g = torch.Generator().manual_seed(T)
  n = 9
  x = torch.randn(n, T, 535, generator=g)
  with torch.no_grad():
    ref, _ = O.mixer(sd, x, O.Ctx(), False)
  got, _ = _run_mixer(model, x, False)
  e = (got - ref).abs().max().item()
  U.record(f'mixer_noncausal_T{T}', err=e, scale=ref.abs().max().item())
  assert e < 2e-4 * max(1.0, ref.abs().max().item())


# T = 5, 7 and 8 run the several-queries-per-CTA variant with one or more unrolled interior trips
# followed by two or more checked frames, the shape that its non-causal instantiation got wrong
@pytest.mark.parametrize('T', [1, 2, 5, 7, 8, 12, 30])
def test_mixer_causal_with_context(T):
  model, sd, cfg = get_model(causal=True)
  g = torch.Generator().manual_seed(100 + T)
  n = 6
  x = torch.randn(n, T, 535, generator=g)
  ctx = {}
  for i in range(12):
    ctx[f'block_{i}_causal_1'] = torch.randn(n, 2, 512, generator=g)
    ctx[f'block_{i}_causal_2'] = torch.randn(n, 2, 2048, generator=g)
  with torch.no_grad():
    ref, ref_ctx = O.mixer(sd, x, O.Ctx(), True, {k: v.clone() for k, v in ctx.items()}, True)
    ref0, _ = O.mixer(sd, x, O.Ctx(), True, None, False)
  got, got_ctx = _run_mixer(model, x, True, ctx, True)
  got0, _ = _run_mixer(model, x, True, None, False)
  e = (got - ref).abs().max().item()
  e0 = (got0 - ref0).abs().max().item()
  ec = max((got_ctx[k] - ref_ctx[k]).abs().max().item() for k in ref_ctx)
  U.record(f'mixer_causal_T{T}', err=e, err_noctx=e0, ctx_err=ec, scale=ref.abs().max().item())
  s = max(1.0, ref.abs().max().item())
  assert e < 2e-4 * s and e0 < 2e-4 * s and ec < 2e-4 * s


def _mixer_queries_per_cta(n, T):
  """Queries per CTA of the depthwise mixer kernel: a copy of the choice in mixer_forward
  (tapnet_b200/csrc/refine.cu), with its constants kDwTileMax 24, kDwRowBudget 52, kDwHalo 4,
  kDwSmallQueries 8 and the H100's 132 SMs."""
  tt = min(T, 24)
  qb = min(max(52 // (2 * tt + 4), 1), 8)
  if qb > 1:
    per_sm = -(-n * -(-T // tt) // 132)
    if per_sm < qb:
      qb = max(per_sm, 2)
  return min(qb, n)


# (T, n) pairs giving every QB from 1 to 8, each with a partial last query group where QB > 1
MIXER_QB_CASES = [(1, 1001), (1, 801), (1, 700), (3, 531), (4, 401), (5, 301), (2, 263), (12, 5)]


def test_mixer_qb_cases_cover_every_queries_per_cta():
  qbs = [_mixer_queries_per_cta(n, T) for T, n in MIXER_QB_CASES]
  assert sorted(qbs) == list(range(1, 9)), qbs
  assert all(qb == 1 or n % qb != 0 for (T, n), qb in zip(MIXER_QB_CASES, qbs))


def _oracle_mixer(*args):
  # n ~ 1000 query rows through twelve blocks: use every core for the fp32 oracle
  threads = torch.get_num_threads()
  torch.set_num_threads(max(threads, os.cpu_count() or 1))
  try:
    with torch.no_grad():
      return O.mixer(*args)
  finally:
    torch.set_num_threads(threads)


def _random_ctx(g, n):
  ctx = {}
  for i in range(12):
    ctx[f'block_{i}_causal_1'] = torch.randn(n, 2, 512, generator=g)
    ctx[f'block_{i}_causal_2'] = torch.randn(n, 2, 2048, generator=g)
  return ctx


# The causal kernel with several queries per CTA (SMALL) at every QB: the register context window
# refill for query slots 4-7 and a partial last query group, with and without context
@pytest.mark.parametrize('T,n', MIXER_QB_CASES,
                         ids=[f'T{T}_n{n}_qb{_mixer_queries_per_cta(n, T)}' for T, n in MIXER_QB_CASES])
def test_mixer_causal_every_queries_per_cta(T, n):
  model, sd, cfg = get_model(causal=True)
  g = torch.Generator().manual_seed(7 * T + n)
  x = torch.randn(n, T, 535, generator=g)
  ctx = _random_ctx(g, n)
  ref, ref_ctx = _oracle_mixer(sd, x, O.Ctx(), True, {k: v.clone() for k, v in ctx.items()}, True)
  ref0, ref0_ctx = _oracle_mixer(sd, x, O.Ctx(), True, None, False)
  got, got_ctx = _run_mixer(model, x, True, ctx, True)
  got0, _ = _run_mixer(model, x, True, None, False)
  e = (got - ref).abs().max().item()
  e0 = (got0 - ref0).abs().max().item()
  ec = max((got_ctx[k] - ref_ctx[k]).abs().max().item() for k in ref_ctx)
  qb = _mixer_queries_per_cta(n, T)
  U.record(f'mixer_causal_qb{qb}_T{T}_n{n}', err=e, err_noctx=e0, ctx_err=ec,
           scale=ref.abs().max().item())
  s = max(1.0, ref.abs().max().item())
  assert e < 2e-4 * s and e0 < 2e-4 * s and ec < 2e-4 * s  # as test_mixer_causal_with_context


# The non-causal (generic) kernel with several queries per CTA
@pytest.mark.parametrize('T,n', [(1, 1001), (3, 531), (5, 301)])
def test_mixer_noncausal_many_queries_per_cta(T, n):
  model, sd, cfg = get_model()
  assert _mixer_queries_per_cta(n, T) >= 3
  g = torch.Generator().manual_seed(3 * T + n)
  x = torch.randn(n, T, 535, generator=g)
  ref, _ = _oracle_mixer(sd, x, O.Ctx(), False)
  got, _ = _run_mixer(model, x, False)
  e = (got - ref).abs().max().item()
  U.record(f'mixer_noncausal_qb{_mixer_queries_per_cta(n, T)}_T{T}_n{n}', err=e,
           scale=ref.abs().max().item())
  assert e < 2e-4 * max(1.0, ref.abs().max().item())  # as test_mixer_noncausal


@pytest.mark.parametrize('n', [6, 1001])
def test_mixer_causal_streaming_step_updates_context_in_place(n):
  """T = 1 with the context output buffers being the input buffers (what OnlineTracker passes)."""
  model, sd, cfg = get_model(causal=True)
  g = torch.Generator().manual_seed(n)
  x = torch.randn(n, 1, 535, generator=g)
  ctx = _random_ctx(g, n)
  ref, ref_ctx = _oracle_mixer(sd, x, O.Ctx(), True, {k: v.clone() for k, v in ctx.items()}, True)
  got, got_ctx = _run_mixer(model, x, True, ctx, True, in_place=True)
  e = (got - ref).abs().max().item()
  ec = max((got_ctx[k] - ref_ctx[k]).abs().max().item() for k in ref_ctx)
  U.record(f'mixer_causal_in_place_n{n}', err=e, ctx_err=ec, scale=ref.abs().max().item())
  s = max(1.0, ref.abs().max().item())
  assert e < 2e-4 * s and ec < 2e-4 * s


@pytest.mark.parametrize('T,n', [(1, 1001), (3, 531)])
def test_mixer_query_permutation_is_bit_exact(T, n):
  """Same n, so the same QB and GEMM schedules: permuting the queries permutes output and new
  context bit for bit (a query mixed up with its CTA slot would break this)."""
  model, sd, cfg = get_model(causal=True)
  g = torch.Generator().manual_seed(11 * T + n)
  x = torch.randn(n, T, 535, generator=g)
  ctx = _random_ctx(g, n)
  perm = torch.randperm(n, generator=g)
  got, got_ctx = _run_mixer(model, x, True, ctx, True)
  got_p, got_ctx_p = _run_mixer(model, x[perm], True, {k: v[perm] for k, v in ctx.items()}, True)
  assert torch.equal(got_p.view(torch.int32), got[perm].view(torch.int32))
  for k in got_ctx:
    assert torch.equal(got_ctx_p[k].view(torch.int32), got_ctx[k][perm].view(torch.int32)), k


def test_refine_update():
  g = torch.Generator().manual_seed(11)
  n, T = 5, 4
  res = torch.randn(n * T, 388, generator=g)
  pos = torch.rand(n, T, 2, generator=g) * 256
  occ, expd = torch.randn(n, T, generator=g), torch.randn(n, T, generator=g)
  feat = torch.randn(n, T, 384, generator=g)
  d = lambda t: t.cuda().contiguous()  # noqa: E731
  res_d, pos_d, occ_d, expd_d, feat_d = d(res), d(pos), d(occ), d(expd), d(feat)
  occ_o, expd_o = torch.empty_like(occ_d), torch.empty_like(expd_d)
  feat_o, trk = torch.empty_like(feat_d), torch.empty_like(pos_d)
  _lib.refine_update(res_d.view(n, T, 388), pos_d, occ_d, expd_d, feat_d[..., :128], feat_d[..., 128:], occ_o,
                     expd_o, feat_o, trk, (256, 256), (320, 384), (480, 640))
  torch.cuda.synchronize()
  r = res.reshape(n, T, 388)
  new_pos = pos + r[..., :2] * torch.tensor([256.0, 256.0]) / torch.tensor([384.0, 320.0])
  assert maxerr(pos_d, new_pos) < 1e-4
  assert maxerr(trk, new_pos * torch.tensor([640.0, 480.0]) / 256.0) < 1e-3
  assert maxerr(occ_o, occ + r[..., 2]) < 1e-6 and maxerr(expd_o, expd + r[..., 3]) < 1e-6
  assert maxerr(feat_o, feat + r[..., 4:]) < 1e-6
