"""The backbone's memory-bound kernels, one at a time through their C entry points, against the
float64 references of tests/backbone_refs.py on designed inputs at the shapes where they go
wrong: partial tiles, the asymmetric stem padding, single-frame block shrinking, large-mean and
constant channels, row tails, the L2 clamp, up- and down-sampling.  Every output sits between
NaN guards (before, after, and between its planes) that must be untouched.  Last, the whole
backbone against the fp64 oracle, which catches orchestration errors."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import synth  # noqa: E402
from oracle import tapir_oracle as O  # noqa: E402
from tapnet_b200 import _lib, tapir_model  # noqa: E402
from tests import backbone_refs as R  # noqa: E402
from tests import gpu_util as U  # noqa: E402
from tests.test_backbone_refs_host import (RESIZE_SHAPES, l2_rows, ln_rows,  # noqa: E402
                                           ln_weights)

GUARD = 64  # guard elements before, after and between planes (a multiple of 16 bytes)
_MODEL = {}


def get_model():
  if not _MODEL:
    sd = synth.make_state_dict(0, 1, True)
    m = tapir_model.TAPIR(pyramid_level=1, extra_convs=True)
    m.load_state_dict(sd)
    _MODEL['m'] = (m.cuda().eval(), sd)
  return _MODEL['m']


class Guarded:
  """`planes` NaN-initialised device arrays of n elements, GUARD elements before the first, between
  consecutive ones and after the last."""

  def __init__(self, n, dtype, planes=1):
    self.n, self.planes, self.stride = n, planes, n + GUARD
    self.buf = torch.full((GUARD + planes * self.stride,), float('nan'), dtype=dtype, device='cuda')

  def ptr(self):
    return ctypes.c_void_p(self.buf.data_ptr() + GUARD * self.buf.element_size())

  def body(self):
    return self.buf[GUARD:].view(self.planes, self.stride)[:, :self.n]

  def guards_untouched(self):
    rest = self.buf[GUARD:].view(self.planes, self.stride)[:, self.n:]
    return bool(torch.isnan(self.buf[:GUARD].float()).all() and torch.isnan(rest.float()).all())


def lib():
  return _lib.load()


def ratio(got, ref, bound):
  """(max error, max error / bound); an element with a zero bound must be exact."""
  err = (got.double().cpu() - ref.double()).abs()
  return float(err.max()), float((err / bound.clamp(min=1e-300)).max())


# ------------------------------------------------------------------------------- stem conv
def stem_video(Fr, H, W, u8, seed):
  g = torch.Generator().manual_seed(seed)
  n = Fr * H * W * 3
  if u8:  # every byte value, in random places; non-zero on the last two rows / columns
    v = (torch.arange(n) % 256)[torch.randperm(n, generator=g)].to(torch.uint8).view(Fr, H, W, 3)
    v[:, -2:] = torch.randint(1, 256, v[:, -2:].shape, generator=g, dtype=torch.uint8)
    v[:, :, -2:] = torch.randint(1, 256, v[:, :, -2:].shape, generator=g, dtype=torch.uint8)
    return v
  v = torch.rand(Fr, H, W, 3, generator=g) * 2 - 1
  v[:, -2:] = 0.5 + 0.5 * torch.rand(v[:, -2:].shape, generator=g)
  v[:, :, -2:] = -0.5 - 0.5 * torch.rand(v[:, :, -2:].shape, generator=g)
  return v


# 2 x 36 x 70: OH = 18, OW = 35 (a partial row tile, a 3-pixel last column tile); 64 x 96: OW = 48,
# where the second pixel of the last column tile is exactly out of range
@pytest.mark.parametrize('u8', [False, True], ids=['f32', 'u8'])
@pytest.mark.parametrize('shape', [(1, 16, 16), (2, 36, 70), (1, 64, 96), (2, 256, 256), (1, 40, 1000)],
                         ids=lambda s: 'x'.join(map(str, s)))
def test_stem_conv(shape, u8):
  Fr, H, W = shape
  model, sd = get_model()
  stem_w = model._pack()['backbone'].stem_w  # TAPIR._pack's [7][7][3][64] layout
  video = stem_video(Fr, H, W, u8, seed=H + W + u8)
  out = Guarded(Fr * (H // 2) * (W // 2) * 64, torch.float32)
  vd = video.cuda()
  _lib.check(lib().tapir_stem_conv(U.ptr(vd), int(u8), ctypes.c_void_p(stem_w), Fr, H, W, out.ptr(),
                                   U.stream()), 'tapir_stem_conv')
  torch.cuda.synchronize()
  assert out.guards_untouched()
  ref, bound = R.stem_ref(video, sd['resnet_torch.initial_conv.weight'])
  err, r = ratio(out.body().view(ref.shape), ref, bound)
  U.record(f'bb_stem_{"u8" if u8 else "f32"}_{Fr}x{H}x{W}', err=err, ratio=r)
  assert r <= 1.0, (err, r)


# ------------------------------------------------------------------------------- instance norm
def norm_input(Fr, hw, C, seed):
  """Channel c follows design c % 3: N(0, 1); mean 1e3 with std 1e-2 (fp32 sums would fail
  there); constant (a different value per channel and frame)."""
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(Fr, hw, C, generator=g)
  x[:, :, 1::3] = 1e3 + 1e-2 * x[:, :, 1::3]
  const = torch.randn(Fr, 1, C, generator=g) * 10
  x[:, :, 2::3] = const[:, :, 2::3].expand(Fr, hw, -1)
  return x


NORM_CASES = [(Fr, hw, C) for C in (64, 128, 256) for hw in (16, 60, 96, 1000, 16384)
              for Fr in (1, 48) if Fr * hw * C <= 48 * 1000 * 256]


@pytest.mark.parametrize('Fr,hw,C', NORM_CASES, ids=lambda v: str(v))
def test_instnorm_stats(Fr, hw, C):
  x = norm_input(Fr, hw, C, seed=hw + C + Fr)
  xd = x.cuda()
  sums = Guarded(Fr * C * 2, torch.float64)  # NaN inside as well: the call must clear it
  _lib.check(lib().tapir_instnorm_stats(U.ptr(xd), Fr, hw, C, sums.ptr(), U.stream()),
             'tapir_instnorm_stats')
  torch.cuda.synchronize()
  assert sums.guards_untouched()
  ref, bound = R.instnorm_stats_ref(x)
  err, r = ratio(sums.body().view(Fr, C, 2), ref, bound)
  U.record(f'bb_instnorm_stats_{Fr}x{hw}x{C}', err=err, ratio=r)
  assert r <= 1.0, (err, r)


@pytest.mark.parametrize('Fr,hw,C', NORM_CASES, ids=lambda v: str(v))
def test_instnorm_apply(Fr, hw, C):
  g = torch.Generator().manual_seed(C)
  x = norm_input(Fr, hw, C, seed=hw + C + Fr)
  # a few channels with |mu| / sigma = 1e4, where x sc + sh cancels most
  x[:, :, 4] = 1e2 + 1e-2 * torch.randn(Fr, hw, generator=g)
  w = 1 + 0.5 * torch.randn(C, generator=g)
  b = 0.5 * torch.randn(C, generator=g)
  xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
  sums = R.sums_fp64(x).cuda()
  n = Fr * hw * C
  zc = C + 64 if C < 256 else 32  # zero_channels != C, both larger and smaller
  outs = {}
  for P in (1, 2, 3):
    out = Guarded(n, torch.bfloat16, P)
    zero = Guarded(Fr * 2 * zc, torch.float64) if P == 3 else None
    _lib.check(lib().tapir_instnorm_relu_split(U.ptr(xd), U.ptr(sums), U.ptr(wd), U.ptr(bd), Fr, hw, C,
                                               out.ptr(), out.stride, P,
                                               zero.ptr() if zero else None, zc, U.stream()),
               'tapir_instnorm_relu_split')
    torch.cuda.synchronize()
    assert out.guards_untouched(), P
    outs[P] = out.body()
    if zero is not None:
      assert zero.guards_untouched()
      assert bool((zero.body() == 0).all())
  p3 = outs[3]
  for P in (1, 2):
    assert torch.equal(outs[P].view(torch.int16), p3[:P].view(torch.int16)), P
  got = p3.double().sum(0).view(Fr, hw, C)
  ref, bound = R.instnorm_apply_ref(x, w, b)
  err, r = ratio(got, ref, bound)
  U.record(f'bb_instnorm_apply_{Fr}x{hw}x{C}', err=err, ratio=r)
  assert r <= 1.0, (err, r)


# ------------------------------------------------------------------------------- im2col
@pytest.mark.parametrize('P', [1, 2, 3])
@pytest.mark.parametrize('C', [64, 128])
@pytest.mark.parametrize('taps', [1, 9])
def test_im2col_s2(taps, C, P):
  Fr, H, W = 2, 18, 10  # 9 x 5 outputs: H / 2 and W / 2 odd
  g = torch.Generator().manual_seed(taps + C + P)
  src = torch.randn(P, Fr, H, W, C, generator=g).to(torch.bfloat16)
  inp = Guarded(Fr * H * W * C, torch.bfloat16, P)
  inp.body().copy_(src.view(P, -1).cuda())
  out = Guarded(Fr * (H // 2) * (W // 2) * taps * C, torch.bfloat16, P)
  _lib.check(lib().tapir_im2col_s2(inp.ptr(), inp.stride, Fr, H, W, C, taps, out.ptr(), out.stride, P,
                                   U.stream()), 'tapir_im2col_s2')
  torch.cuda.synchronize()
  assert out.guards_untouched()
  ref = R.im2col_ref(src, taps).reshape(P, -1)
  assert torch.equal(out.body().cpu().view(torch.int16), ref.view(torch.int16))


# ------------------------------------------------------------------------------- layer norm
def ln_input(rows, C, seed):
  """Row r follows design r % 3: N(0, 1), mean 1e3 with std 1, constant."""
  parts = [ln_rows(k, rows, C, seed + i) for i, k in enumerate(('normal', 'offset', 'constant'))]
  x = torch.empty(rows, C)
  for i in range(3):
    x[i::3] = parts[i][i::3]
  return x


@pytest.mark.parametrize('rows', [1, 7, 8, 9, 4097])
@pytest.mark.parametrize('C', [256, 512])
def test_layernorm_split(C, rows):
  """C = 256: bias, fp32 y and three planes (the ExtraConvs' call); C = 512: no bias, planes only
  (the mixer's final LayerNorm)."""
  x = ln_input(rows, C, seed=rows + C)
  w, b = ln_weights(C, seed=C)
  b = b if C == 256 else None
  xd, wd = x.cuda(), w.cuda()
  bd = b.cuda() if b is not None else None
  P = 3
  y = Guarded(rows * C, torch.float32) if C == 256 else None
  pl = Guarded(rows * C, torch.bfloat16, P)
  _lib.check(lib().tapir_layernorm_split(U.ptr(xd), rows, C, U.ptr(wd), U.ptr(bd),
                                         y.ptr() if y else None, pl.ptr(), pl.stride, P, U.stream()),
             'tapir_layernorm_split')
  torch.cuda.synchronize()
  assert pl.guards_untouched() and (y is None or y.guards_untouched())
  ref, bound = R.layernorm_ref(x, w, b)
  planes = pl.body().view(P, rows, C)
  if y is not None:
    yv = y.body().view(rows, C)
    err, r = ratio(yv, ref, bound)
    assert torch.equal(planes.view(torch.int16), U.split_like_kernel(yv, P).view(torch.int16))
  else:
    # three planes hold the fp32 output to within 2^-27 of its magnitude
    err, r = ratio(planes.double().sum(0), ref, bound + 2.0 ** -26 * ref.abs())
  U.record(f'bb_layernorm_{C}x{rows}', err=err, ratio=r)
  assert r <= 1.0, (err, r)


# ------------------------------------------------------------------------------- L2 norm
@pytest.mark.parametrize('rows', [1, 7, 9, 4097])
@pytest.mark.parametrize('C', [128, 256])
def test_l2_normalize(C, rows):
  x = l2_rows(rows, C, seed=rows + C)
  xd = x.cuda()
  out = Guarded(rows * C, torch.float32)
  _lib.check(lib().tapir_l2_normalize(U.ptr(xd), rows, C, out.ptr(), U.stream()), 'tapir_l2_normalize')
  torch.cuda.synchronize()
  assert out.guards_untouched()
  got = out.body().view(rows, C).cpu()
  ref, bound = R.l2norm_ref(x)
  err, r = ratio(got, ref, bound)
  U.record(f'bb_l2norm_{C}x{rows}', err=err, ratio=r)
  assert r <= 1.0, (err, r)
  assert torch.equal(got[1::4], torch.zeros_like(got[1::4]))  # all-zero rows stay exactly 0


# ------------------------------------------------------------------------------- resize
RESIZE_CASES = ([(s, 3, 2) for s in RESIZE_SHAPES] +
                [(((64, 96), (256, 256)), 64, 1), (((320, 384), (256, 256)), 64, 1),
                 (((17, 9), (32, 40)), 64, 2), (((17, 9), (32, 40)), 256, 1),
                 (((1, 7), (5, 1)), 256, 1), (((24, 40), (24, 40)), 256, 1)])


@pytest.mark.parametrize('shape,C,Fr', RESIZE_CASES,
                         ids=lambda v: (f'{v[0][0]}x{v[0][1]}-{v[1][0]}x{v[1][1]}' if isinstance(v, tuple)
                                        else str(v)))
def test_bilinear_resize(shape, C, Fr):
  (H, W), (oH, oW) = shape
  g = torch.Generator().manual_seed(H * W + C)
  src = torch.randn(Fr, H, W, C, generator=g)
  sd_ = src.cuda()
  out = Guarded(Fr * oH * oW * C, torch.float32)
  _lib.check(lib().tapir_bilinear_resize(U.ptr(sd_), Fr, H, W, C, out.ptr(), oH, oW, U.stream()),
             'tapir_bilinear_resize')
  torch.cuda.synchronize()
  assert out.guards_untouched()
  got = out.body().view(Fr, oH, oW, C).cpu()
  if (H, W) == (oH, oW):
    assert torch.equal(got, src)
    return
  ref, bound = R.resize_ref(src, oH, oW)
  err, r = ratio(got, ref, bound)
  U.record(f'bb_resize_{H}x{W}-{oH}x{oW}_c{C}', err=err, ratio=r)
  assert r <= 1.0, (err, r)


# ------------------------------------------------------------------------------- whole backbone
# The largest error of the L2-normalised grids against the fp64 oracle on one H100 80GB HBM3
# (700 W limit), split-bf16 x3 wgmma GEMMs, over the shapes below: 1.9e-5 lowres, 7.5e-6 hires.
# 5e-5 leaves a margin of 2.6; test_stages_gpu.py's test_backbone allows 2e-4 against the fp32
# oracle.  The per-kernel tests above catch the small-effect bugs; this one catches orchestration
# errors (buffer ping-pong, the fused / unfused statistics choice, chunk offsets).
BACKBONE_TOL = 5e-5


def _oracle_grids(sd64, video, H, W):
  cfg = O.Config(pyramid_level=1, extra_convs=True, initial_resolution=(H, W))
  with torch.no_grad():
    r = O.get_feature_grids(sd64, cfg, video, refinement_resolutions=[(H, W)])
  return r.lowres[0], r.hires[0]


def _model_grids(model, video, H, W):
  model.initial_resolution = (H, W)
  try:
    got = model.get_feature_grids(video.cuda(), False, [(H, W)])
  finally:
    model.initial_resolution = (256, 256)
  torch.cuda.synchronize()
  return got.lowres[0].cpu(), got.hires[0].cpu()


# 3 x 24 x 40: 60 stride-2 outputs per frame (the unfused-statistics path); 1 x 256 x 256: split-K
# ExtraConvs and shrunken norm blocks
@pytest.mark.parametrize('shape,u8', [((1, 16, 16), False), ((3, 24, 40), False), ((2, 72, 200), False),
                                      ((1, 256, 256), False), ((2, 256, 256), True)],
                         ids=['1x16x16', '3x24x40', '2x72x200', '1x256x256', '2x256x256-u8'])
def test_backbone_vs_fp64_oracle(shape, u8):
  T, H, W = shape
  model, sd = get_model()
  sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
  if u8:
    g = torch.Generator().manual_seed(T * H)
    video = torch.randint(0, 256, (1, T, H, W, 3), dtype=torch.uint8, generator=g)
    video64 = R.normalise_u8(video).double()
  else:
    video = synth.make_video(T, H, W)
    video64 = video.double()
  lo, hi = _model_grids(model, video, H, W)
  rlo, rhi = _oracle_grids(sd64, video64, H, W)
  e_lo = float((lo.double() - rlo).abs().max())
  e_hi = float((hi.double() - rhi).abs().max())
  U.record(f'bb_backbone_fp64_{"x".join(map(str, shape))}{"_u8" if u8 else ""}', lowres_err=e_lo,
           hires_err=e_hi, tol=BACKBONE_TOL)
  assert e_lo <= BACKBONE_TOL and e_hi <= BACKBONE_TOL, (e_lo, e_hi)


def test_backbone_frame_chunks_are_independent():
  """A 5-frame clip in 2-frame backbone passes (2 + 2 + 1) equals the one-pass result bit for bit
  in the frames of the full chunks, and the last frame equals a pass over that frame alone (a
  single-frame pass may split K in the ExtraConvs, which changes the summation order)."""
  model, _ = get_model()
  T, H, W = 5, 24, 40
  video = synth.make_video(T, H, W, seed=3)
  lo, hi = _model_grids(model, video, H, W)
  lo1, hi1 = _model_grids(model, video[:, 4:], H, W)
  saved = tapir_model._MAX_BACKBONE_PIXELS
  tapir_model._MAX_BACKBONE_PIXELS = 2 * H * W
  try:
    clo, chi = _model_grids(model, video, H, W)
  finally:
    tapir_model._MAX_BACKBONE_PIXELS = saved
  assert torch.equal(clo[:, :4], lo[:, :4]) and torch.equal(chi[:, :4], hi[:, :4])
  assert torch.equal(clo[:, 4:], lo1) and torch.equal(chi[:, 4:], hi1)
