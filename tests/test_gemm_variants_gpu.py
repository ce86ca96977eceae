"""The GEMM / implicit-conv variants the dispatcher picks in production, against exact fp64 models.

Covers what tests/test_gemm_gpu.py does not reach: the scalar epilogue branches (odd N, padded
leading dimensions, 4-byte aligned outputs, out_P of 1 / 3, plane output in conv mode, statistics
fused with bias / GELU / residual), split-K with its reduction kernel, the halo-patch convolution at
shapes that do not tile, the conv tile geometries, BLOCK_N and row-range invariance, and the
host-side argument checks."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from tapnet_b200 import _lib  # noqa: E402
from tests import gpu_util as U  # noqa: E402

IMPLS = pytest.mark.parametrize('impl', [1, 0], ids=['simt', 'tc'])


def _problem(seed, M, N, K, P, conv=None, bias=False, resid=False):
  g = torch.Generator().manual_seed(seed)
  if conv is None:
    a = torch.randn(M, K, generator=g).cuda()
    a_pl = U.split(a, P)
  else:
    Fr, H, W, C = conv
    x = torch.randn(Fr * H * W, C, generator=g).cuda()
    a_pl = U.split(x, P).reshape(P, Fr, H, W, C)
  w_pl = U.split((torch.randn(N, K, generator=g) / K ** 0.5).cuda(), P)
  b = torch.randn(N, generator=g).cuda() if bias else None
  r = torch.randn(M, N, generator=g).cuda() if resid else None
  return a_pl, w_pl, b, r


def _model(a_pl, w_pl, conv, impl, b=None, gelu=False, r=None):
  """fp64 model of the GEMM: the i+j<P plane pairs (tensor cores) or all of them (SIMT)."""
  if impl == 1:
    a_pl, w_pl = a_pl.double().sum(0, keepdim=True), w_pl.double().sum(0, keepdim=True)
  ref = U.conv_planes_fp64(a_pl, w_pl) if conv else U.planes_matmul_fp64(a_pl, w_pl)
  if b is not None:
    ref = ref + b.double().cpu()
  if gelu:
    ref = F.gelu(ref, approximate='tanh')
  if r is not None:
    ref = ref + r.double().cpu()
  return ref


def _check_out(name, out, ref, gelu, K, P):
  err = (out.double().cpu() - ref).abs().max().item()
  scale = ref.abs().max().item()
  U.record(name, max_err=err, scale=scale, rel=err / max(scale, 1.0))
  assert torch.isfinite(out).all(), name
  assert err <= U.accum_tol(K, P, scale, gelu), (name, err, scale)


def _check_planes(name, res, ref, gelu, K, P):
  """Plane outputs: the exact bf16 split of the fp32 output when there is one, else their sum
  against the model within the rounding of the last plane (2^-8 relative per plane)."""
  if res.out is not None:
    want = U.split_like_kernel(res.out, res.out_P)
    assert torch.equal(res.planes.view(torch.int16), want.view(torch.int16)), name
    return
  rec = res.planes.double().sum(0).cpu()
  err = ((rec - ref).abs() - 2.0 ** (-8 * res.out_P) * ref.abs()).max().item()
  scale = ref.abs().max().item()
  U.record(name + '_planes', max_err_beyond_rounding=err, scale=scale)
  assert err <= U.accum_tol(K, P, scale, gelu), (name, err, scale)


# ---------------------------------------------------------------------------- epilogue matrix
EPILOGUE_CASES = [
    # id, M, N, K, P, conv, bias, gelu, resid, out_f32, out_P, ld_pad, offset, stats
    ('odd_n_planes3_pad_off', 300, 389, 128, 2, None, True, True, True, True, 3, 3, 1, False),
    ('odd_n_planes1_pad', 300, 67, 192, 1, None, True, False, True, True, 1, 3, 0, False),
    ('planes2_only_pad', 257, 389, 128, 3, None, False, False, True, False, 2, 3, 0, False),
    ('odd_n_off', 300, 67, 128, 2, None, False, True, False, True, 0, 0, 1, False),
    ('even_n_off_resid', 200, 128, 64, 2, None, True, False, True, True, 0, 0, 1, False),
    ('stats_bias_gelu_resid', 384, 67, 128, 2, None, True, True, True, True, 0, 3, 1, True),
    ('conv_planes3_pad_off', None, 67, None, 2, (2, 12, 20, 64), True, True, True, True, 3, 3, 1, False),
    ('conv_planes2_only', None, 389, None, 2, (1, 9, 13, 128), True, False, False, False, 2, 0, 0, False),
    ('conv_planes1', None, 128, None, 1, (2, 10, 24, 64), False, True, True, True, 1, 3, 0, False),
    ('conv_stats_bias_gelu_resid', None, 67, None, 2, (2, 10, 24, 64), True, True, True, True, 0, 3, 1, True),
]


@IMPLS
@pytest.mark.parametrize('case', EPILOGUE_CASES, ids=[c[0] for c in EPILOGUE_CASES])
def test_epilogue_matrix(case, impl):
  cid, M, N, K, P, conv, bias, gelu, resid, of32, out_P, ld_pad, offset, want_stats = case
  if conv is not None:
    M, K = conv[0] * conv[1] * conv[2], 9 * conv[3]
  a_pl, w_pl, b, r = _problem(M + N + K, M, N, K, P, conv, bias, resid)
  stats = None
  frames = conv[0] if conv else M // 128
  if want_stats:
    stats = torch.zeros(frames, N, 2, dtype=torch.float64, device='cuda')
  res = U.gemm(a_pl, w_pl, b, r, gelu, of32, out_P, impl, conv=conv, stats=stats,
               rows_per_frame=128 if want_stats and not conv else 0, ld_pad=ld_pad, offset=offset,
               details=True)
  ref = _model(a_pl, w_pl, conv, impl, b, gelu, r)
  name = f'epilogue_{cid}_impl{impl}'
  assert U.untouched_padding(res), f'{name}: wrote outside the [M, N] output'
  if of32:
    _check_out(name, res.out, ref, gelu, K, P)
  if out_P:
    _check_planes(name, res, ref, gelu, K, P)
  if want_stats:
    out = res.out.double().reshape(frames, -1, N)
    want = torch.stack([out.sum(1), (out * out).sum(1)], -1)
    rel = ((stats - want).abs() / want.abs().clamp(min=1.0)).max().item()
    U.record(name + '_stats', rel_err=rel)
    # fp32 partial sums over a warp's 16 rows, then fp64 atomics: as test_fused_instance_norm_statistics
    assert rel < 5e-5


# ---------------------------------------------------------------------------------- split-K
def _ldw(N):
  return (N + 7) // 8 * 8  # the partial-sum row pitch gemm_tc uses


SPLITK_CASES = [
    # id, M, N, K, P, conv, bias, gelu, resid, out_P (0: fp32 out), workspace bytes (None: ample), splits
    ('down_resid_f32', 1000, 512, 2048, 2, None, True, False, True, 0, None, True),
    ('odd_n_gelu_planes', 300, 389, 2048, 2, None, True, True, False, 2, None, True),
    ('odd_n_p3_resid', 300, 389, 2048, 3, None, False, False, True, 0, None, True),
    ('ws_exactly_two_splits', 300, 389, 2048, 2, None, True, False, True, 0, 2 * 300 * _ldw(389) * 4, True),
    ('ws_too_small', 300, 389, 2048, 2, None, True, False, True, 0, 2 * 300 * _ldw(389) * 4 - 16, False),
    ('conv_gelu_planes', None, 1024, None, 2, (1, 16, 16, 256), True, True, False, 2, None, True),
    ('conv_resid_f32', None, 256, None, 2, (1, 12, 20, 1024), True, False, True, 0, None, True),
]


@IMPLS
@pytest.mark.parametrize('case', SPLITK_CASES, ids=[c[0] for c in SPLITK_CASES])
def test_splitk(case, impl):
  cid, M, N, K, P, conv, bias, gelu, resid, out_P, ws_bytes, splits = case
  if conv is not None:
    M, K = conv[0] * conv[1] * conv[2], 9 * conv[3]
  a_pl, w_pl, b, r = _problem(M + N + K + 7, M, N, K, P, conv, bias, resid)
  ws = torch.empty(ws_bytes if ws_bytes is not None else 8 * M * _ldw(N) * 4, dtype=torch.uint8,
                   device='cuda')
  runs = [U.gemm(a_pl, w_pl, b, r, gelu, out_P == 0, out_P, impl, conv=conv, ld_pad=3, offset=1,
                 splitk_ws=ws, details=True) for _ in range(2)]
  res = runs[0]
  ref = _model(a_pl, w_pl, conv, impl, b, gelu, r)
  name = f'splitk_{cid}_impl{impl}'
  # a split GEMM is one partial-sum launch plus the reduction (the SIMT path never splits)
  expect = 2 if (impl == 0 and splits) else 1
  U.record(name + '_launches', launches=res.launches, expected=expect)
  assert res.launches == expect and runs[1].launches == expect
  assert U.untouched_padding(res), name
  if out_P == 0:
    _check_out(name, res.out, ref, gelu, K, P)
    assert torch.equal(res.out_buf.view(torch.int32), runs[1].out_buf.view(torch.int32)), 'not deterministic'
  else:
    _check_planes(name, res, ref, gelu, K, P)
    assert torch.equal(res.planes_buf.view(torch.int16), runs[1].planes_buf.view(torch.int16)), 'not deterministic'


def test_splitk_workspace_must_be_aligned_tc():
  lib = _lib.load()
  a_pl, w_pl, _, _ = _problem(1, 300, 389, 2048, 2)
  out = torch.empty(300, 389, device='cuda')
  ws = torch.empty(1 << 22, dtype=torch.uint8, device='cuda')
  lin = U.make_linear(w_pl, None)
  before = U.launch_count()
  st = lib.tapir_gemm_ex(U.ptr(a_pl), 2048, 300 * 2048, ctypes.byref(lin), 300, 0, 0, 0, 0, 0,
                         None, 0, 0, U.ptr(out), 389, None, 0, 0, 0, None, 0, 0,
                         ctypes.c_void_p(ws.data_ptr() + 4), (1 << 22) - 4, U.stream())
  assert st == 1 and b'aligned' in lib.tapir_last_error()
  assert U.launch_count() == before


# ------------------------------------------------------------------------------- halo conv
# (F, H, W, P, bias, residual, stats): W not a multiple of 8 and below 8, H not a multiple of 16
HALO_CASES = [
    (1, 7, 5, 1, True, True, True),
    (3, 33, 13, 2, True, True, True),
    (3, 7, 37, 1, False, True, False),
    (1, 33, 37, 2, True, False, True),
    (3, 33, 5, 2, False, False, False),
    (1, 7, 13, 1, True, True, False),
    (3, 40, 56, 2, True, True, True),
]


def test_halo_conv_shapes_tc():
  """conv3x3_halo_kernel (C = 64 -> 64, P <= 2) against the fp64 model, and bit for bit against the
  generic implicit GEMM (TAPIR_B200_CONV_HALO=0)."""
  for i, (Fr, H, W, P, bias, resid, stats) in enumerate(HALO_CASES):
    a_pl, w_pl, b, r = _problem(100 + i, Fr * H * W, 64, 576, P, (Fr, H, W, 64), bias, resid)
    outs = {}
    for halo in (1, 0):
      st = torch.zeros(Fr, 64, 2, dtype=torch.float64, device='cuda') if stats else None
      with U.switches(TAPIR_B200_CONV_HALO=halo):
        o, _ = U.gemm(a_pl, w_pl, b, r, False, True, 0, 0, conv=(Fr, H, W, 64), stats=st)
      outs[halo] = (o, st)
    (o_h, st_h), (o_g, _) = outs[1], outs[0]
    ref = _model(a_pl, w_pl, True, 0, b, False, r)
    name = f'halo_{Fr}x{H}x{W}_P{P}'
    _check_out(name, o_h, ref, False, 576, P)
    assert torch.equal(o_h.view(torch.int32), o_g.view(torch.int32)), f'{name}: halo != generic'
    if stats:
      out = o_h.double().reshape(Fr, -1, 64)
      want = torch.stack([out.sum(1), (out * out).sum(1)], -1)
      rel = ((st_h - want).abs() / want.abs().clamp(min=1.0)).max().item()
      U.record(name + '_stats', rel_err=rel)
      assert rel < 5e-5


# --------------------------------------------------------------------------- conv tile geometry
TILE_CASES = [
    # F, H, W, C, N, P: 8 x 16 tiles (narrow, tall), a partial 128-wide tile with H = 1, W = 1
    (2, 48, 8, 64, 128, 2),
    (1, 1, 200, 64, 96, 2),
    (2, 40, 1, 128, 64, 1),
    (1, 1, 1, 64, 72, 3),
]


@IMPLS
@pytest.mark.parametrize('case', TILE_CASES, ids=['x'.join(map(str, c[:5])) for c in TILE_CASES])
def test_conv_tile_geometry(case, impl):
  Fr, H, W, C, N, P = case
  conv = (Fr, H, W, C)
  M, K = Fr * H * W, 9 * C
  a_pl, w_pl, b, r = _problem(M + N, M, N, K, P, conv, True, True)
  res = U.gemm(a_pl, w_pl, b, r, True, True, 2, impl, conv=conv, ld_pad=1, details=True)
  ref = _model(a_pl, w_pl, conv, impl, b, True, r)
  name = f'conv_tile_{Fr}x{H}x{W}x{C}to{N}_P{P}_impl{impl}'
  assert U.untouched_padding(res), name
  _check_out(name, res.out, ref, True, K, P)
  _check_planes(name, res, ref, True, K, P)


# ------------------------------------------------------------------------------- invariance
@pytest.mark.parametrize('mode', ['plain', 'conv'])
@pytest.mark.parametrize('P', [1, 2, 3])
def test_block_n_invariance_tc(P, mode):
  """An output element's K-summation order does not depend on the tile width: same bits."""
  N = 389
  conv = (2, 20, 24, 64) if mode == 'conv' else None
  M, K = (2 * 20 * 24, 576) if conv else (700, 256)
  a_pl, w_pl, b, r = _problem(P + N, M, N, K, P, conv, True, True)
  run = lambda: U.gemm(a_pl, w_pl, b, r, True, True, P, 0, conv=conv, ld_pad=3, details=True)  # noqa: E731
  with U.switches(TAPIR_B200_BLOCK_N=64):
    r64 = run()
  with U.switches(TAPIR_B200_BLOCK_N=128):
    r128 = run()
  same = torch.equal(r64.out_buf.view(torch.int32), r128.out_buf.view(torch.int32)) and \
      torch.equal(r64.planes_buf.view(torch.int16), r128.planes_buf.view(torch.int16))
  U.record(f'block_n_invariance_{mode}_P{P}', identical=int(same))
  assert same


@pytest.mark.parametrize('P', [1, 2, 3])
def test_row_range_invariance_tc(P):
  """Without split-K, rows [a, b) of a GEMM give the same bits as those rows of the full GEMM
  (the shorter problem also runs a different tile width and schedule)."""
  M, N, K = 3000, 389, 512
  a_pl, w_pl, b, r = _problem(P, M, N, K, P, None, True, True)
  full, _ = U.gemm(a_pl, w_pl, b, r, True, True, 0, 0)
  for lo, hi in ((0, 128), (136, 1000), (2048, 3000), (8, 9)):
    part, _ = U.gemm(a_pl[:, lo:hi].contiguous(), w_pl, b, r[lo:hi].contiguous(), True, True, 0, 0)
    assert torch.equal(part.view(torch.int32), full[lo:hi].view(torch.int32)), (lo, hi)


# ------------------------------------------------------------------------------ argument checks
@IMPLS
@pytest.mark.parametrize('bad', ['a_misaligned', 'b_misaligned', 'k_not_64', 'stats_with_planes'])
def test_bad_arguments_are_rejected_on_the_host(bad, impl):
  lib = _lib.load()
  M, N, K, P = 256, 128, 128, 2
  a_pl, w_pl, _, _ = _problem(3, M, N, K, P)
  a_ptr, lda, ldo = U.ptr(a_pl), K, N
  lin = U.make_linear(w_pl, None)
  out = torch.full((M, N), float('nan'), device='cuda')
  planes, out_P = None, 0
  stats, rpf = None, 0
  if bad == 'a_misaligned':
    a_ptr = ctypes.c_void_p(a_pl.data_ptr() + 2)
  elif bad == 'b_misaligned':
    lin.w = w_pl.data_ptr() + 2
  elif bad == 'k_not_64':
    w96 = U.split((torch.randn(N, 96) / 10).cuda(), P)
    a96 = U.split(torch.randn(M, 96).cuda(), P)
    lin = U.make_linear(w96, None)
    a_ptr, lda = U.ptr(a96), 96
  else:
    planes = torch.zeros(2, M, N, dtype=torch.bfloat16, device='cuda')
    out_P = 2
    stats = torch.zeros(2, N, 2, dtype=torch.float64, device='cuda')
    rpf = 128
  torch.cuda.synchronize()
  before = U.launch_count()
  st = lib.tapir_gemm_ex(a_ptr, lda, M * lda, ctypes.byref(lin), M, 0, 0, 0, 0, 0, None, 0, 0,
                         U.ptr(out), ldo, U.ptr(planes), N, M * N, out_P, U.ptr(stats), rpf, impl,
                         None, 0, U.stream())
  msg = lib.tapir_last_error()
  assert st == 1, (bad, st, msg)
  assert msg and b'gemm' in msg, msg
  assert U.launch_count() == before
  torch.cuda.synchronize()
  assert torch.isnan(out).all()
