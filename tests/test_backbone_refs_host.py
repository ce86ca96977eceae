"""CPU checks of tests/backbone_refs.py: the float64 references agree with the oracle's functions
at fp32, the fp32 error bounds hold for numpy emulations of the kernels' operation order on
every design the GPU tests use, and the backbone building blocks of the C ABI reject bad
arguments (status 1) before any CUDA call, so none of this needs a GPU."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import tapir_oracle as O
from oracle.frames_io_oracle import preprocess_frames
from tapnet_b200 import _lib
from tests import backbone_refs as R

f32 = np.float32


# ------------------------------------------------------------------------------- designs
def ln_rows(kind, rows, C, seed):
  """Row designs of the LayerNorm test: N(0, 1), offset (mean 1e3, std 1), constant rows (values
  whose row sum is exact, so the centred values are exactly 0)."""
  g = torch.Generator().manual_seed(seed)
  if kind == 'normal':
    return torch.randn(rows, C, generator=g)
  if kind == 'offset':
    return 1e3 + torch.randn(rows, C, generator=g)
  vals = torch.tensor([0.0, 0.5, -3.0, 1024.0, 0.125])
  return vals[torch.arange(rows) % len(vals)][:, None].expand(rows, C).contiguous()


def l2_rows(rows, C, seed):
  """N(0, 1) rows, all-zero rows, rows with sum x^2 = 1e-13 (clamped) and 4e-12 (just above the
  clamp), in turn."""
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(rows, C, generator=g)
  for i in range(rows):
    if i % 4 == 1:
      x[i] = 0
    elif i % 4 in (2, 3):
      target = 1e-13 if i % 4 == 2 else 4e-12
      x[i] *= float(np.sqrt(target / float((x[i].double() ** 2).sum())))
  return x


def ln_weights(C, seed):
  g = torch.Generator().manual_seed(seed)
  return 1 + 0.5 * torch.randn(C, generator=g), 0.3 * torch.randn(C, generator=g)


RESIZE_SHAPES = [((1080, 1920), (256, 256)), ((64, 96), (256, 256)), ((17, 9), (32, 40)),
                 ((320, 384), (256, 256)), ((1, 7), (5, 1)), ((6, 1), (1, 9)), ((1, 1), (3, 4)),
                 ((24, 40), (24, 40))]


def resize_src(H, W, C, seed):
  g = torch.Generator().manual_seed(seed)
  return torch.randn(1, H, W, C, generator=g)


# ------------------------------------------------------------------------------- emulations
def _warp_sum(v):
  """[rows, 32] -> [rows]: the xor-butterfly of warp_sum (every lane ends with the same value)."""
  lanes = np.arange(32)
  for o in (16, 8, 4, 2, 1):
    v = (v + v[:, lanes ^ o]).astype(f32)
  return v[:, 0]


def _lane_chunks(x):
  """[rows, C] -> [rows, V, 32, 4]: lane l holds float4 i * 32 + l."""
  rows, C = x.shape
  return x.reshape(rows, C // 128, 32, 4)


def emulate_layernorm(x, w, b):
  x = x.numpy().astype(f32)
  rows, C = x.shape
  v = _lane_chunks(x)
  s = np.zeros((rows, 32), f32)
  for i in range(C // 128):
    q = v[:, i]
    s = (s + (((q[..., 0] + q[..., 1]) + q[..., 2]) + q[..., 3])).astype(f32)
  mean = (_warp_sum(s) * f32(1.0 / C)).astype(f32)[:, None, None, None]
  d = (v - mean).astype(f32)
  sq = (d * d).astype(f32)
  ss = np.zeros((rows, 32), f32)
  for i in range(C // 128):
    q = sq[:, i]
    ss = (ss + (((q[..., 0] + q[..., 1]) + q[..., 2]) + q[..., 3])).astype(f32)
  var = (_warp_sum(ss) * f32(1.0 / C)).astype(f32)
  rstd = (f32(1.0) / np.sqrt((var + f32(1e-5)).astype(f32))).astype(f32)[:, None, None, None]
  o = ((d * rstd).astype(f32) * _lane_chunks(w.numpy()[None].astype(f32))).astype(f32)
  if b is not None:
    o = (o + _lane_chunks(b.numpy()[None].astype(f32))).astype(f32)
  return torch.from_numpy(o.reshape(rows, C))


def emulate_l2norm(x):
  x = x.numpy().astype(f32)
  rows, C = x.shape
  sq = (_lane_chunks(x) ** 2).astype(f32)
  s = np.zeros((rows, 32), f32)
  for i in range(C // 128):
    q = sq[:, i]
    s = (s + (((q[..., 0] + q[..., 1]) + q[..., 2]) + q[..., 3])).astype(f32)
  d = np.sqrt(np.maximum(_warp_sum(s), f32(1e-12))).astype(f32)
  return torch.from_numpy((x / d[:, None]).astype(f32))


def emulate_resize(src, oH, oW, fma):
  """The kernel's fp32 arithmetic, with its coordinate computed by one FMA or by two roundings."""
  s = src.numpy().astype(f32)
  H, W = s.shape[1:3]

  def coord(o, n):
    scale = f32(n) / f32(o)
    i = np.arange(o, dtype=f32) + f32(0.5)
    c = (np.float64(scale) * i.astype(np.float64) - 0.5).astype(f32) if fma else (scale * i - f32(0.5)).astype(f32)
    return np.maximum(c, f32(0))

  fy, fx = coord(oH, H), coord(oW, W)
  y0, x0 = fy.astype(np.int64), fx.astype(np.int64)
  y1, x1 = y0 + (y0 < H - 1), x0 + (x0 < W - 1)
  ly, lx = (fy - y0.astype(f32)).astype(f32), (fx - x0.astype(f32)).astype(f32)
  hy, hx = (f32(1) - ly).astype(f32), (f32(1) - lx).astype(f32)
  hx_, lx_ = hx[None, None, :, None], lx[None, None, :, None]
  top = ((hx_ * s[:, y0][:, :, x0]).astype(f32) + (lx_ * s[:, y0][:, :, x1]).astype(f32)).astype(f32)
  bot = ((hx_ * s[:, y1][:, :, x0]).astype(f32) + (lx_ * s[:, y1][:, :, x1]).astype(f32)).astype(f32)
  out = ((hy[None, :, None, None] * top).astype(f32) + (ly[None, :, None, None] * bot).astype(f32)).astype(f32)
  return torch.from_numpy(out)


def _ratio(got, ref, bound):
  err = (got.double() - ref.double()).abs()
  return float((err / bound.clamp(min=1e-300)).max()), float(err.max())


# ------------------------------------------------------------------------------- bounds hold
@pytest.mark.parametrize('C,bias', [(256, True), (512, False)])
@pytest.mark.parametrize('kind', ['normal', 'offset', 'constant'])
def test_layernorm_bound_holds_for_fp32_emulation(C, bias, kind):
  x = ln_rows(kind, 257, C, seed=C + len(kind))
  w, b = ln_weights(C, seed=C)
  b = b if bias else None
  ref, bound = R.layernorm_ref(x, w, b)
  got = emulate_layernorm(x, w, b)
  ratio, err = _ratio(got, ref, bound)
  assert ratio <= 1.0, (ratio, err)
  if kind == 'constant':  # centred values are exactly 0: the output is b (or 0) exactly
    assert torch.equal(got, (b if b is not None else torch.zeros(C)).expand_as(got))


@pytest.mark.parametrize('C', [128, 256])
def test_l2norm_bound_holds_for_fp32_emulation(C):
  x = l2_rows(64, C, seed=C)
  ref, bound = R.l2norm_ref(x)
  got = emulate_l2norm(x)
  ratio, err = _ratio(got, ref, bound)
  assert ratio <= 1.0, (ratio, err)
  assert torch.equal(got[1::4], torch.zeros_like(got[1::4]))
  # the clamp is what the rows with sum x^2 = 1e-13 see; the 4e-12 rows are above it
  assert float(ref[2::4].double().pow(2).sum(-1).max()) < 0.2
  assert float(ref[3::4].double().pow(2).sum(-1).min()) > 0.99


@pytest.mark.parametrize('shape', RESIZE_SHAPES, ids=lambda s: f'{s[0][0]}x{s[0][1]}-{s[1][0]}x{s[1][1]}')
def test_resize_bound_holds_for_fp32_emulation(shape):
  (H, W), (oH, oW) = shape
  C = 3
  src = resize_src(H, W, C, seed=H * W)
  ref, bound = R.resize_ref(src, oH, oW)
  for fma in (False, True):
    got = emulate_resize(src, oH, oW, fma)
    ratio, err = _ratio(got, ref, bound)
    assert ratio <= 1.0, (fma, ratio, err)
  if (H, W) == (oH, oW):
    assert torch.equal(emulate_resize(src, oH, oW, True), src)


def test_resize_bound_rejects_the_unclamped_coordinate():
  """Upsampling: without the fy < 0 clamp the first output row extrapolates; the bound must be
  far below that change, or the GPU test could not see it."""
  src = resize_src(64, 96, 3, seed=5)
  _, bound = R.resize_ref(src, 256, 256)
  # fy = 0.25 * 0.5 - 0.5 = -0.375 for output row 0: unclamped, y0 = (int)fy = 0 and the row
  # becomes 1.375 src[0] - 0.375 src[1] instead of src[0] (before the blend along x)
  change = 0.375 * (src[:, 1] - src[:, 0]).double().abs()
  assert float(change.max()) > 1e3 * float(bound[:, 0].max())


def test_stem_and_instnorm_bounds_are_tight_enough():
  """The stem bound is far below the change of a one-pixel shift of the window, and the apply
  bound far below an eps change 1e-5 -> 1e-4 on unit-variance channels."""
  g = torch.Generator().manual_seed(0)
  video = torch.rand(1, 16, 16, 3, generator=g) * 2 - 1
  w = torch.randn(64, 3, 7, 7, generator=g) * 0.1
  ref, bound = R.stem_ref(video, w)
  shifted = F.conv2d(F.pad(video.double().permute(0, 3, 1, 2), (3, 3, 3, 3)), w.double(), stride=2)
  assert float(bound.max()) < 1e-3 * float((shifted.permute(0, 2, 3, 1) - ref).abs().max())
  x = torch.randn(2, 96, 64, generator=g)
  wn, bn = 1 + 0.1 * torch.randn(64, generator=g), 0.1 * torch.randn(64, generator=g)
  r5, b5 = R.instnorm_apply_ref(x, wn, bn)
  r4, _ = R.instnorm_apply_ref(x, wn, bn, eps=1e-4)
  assert float(((r4 - r5).abs() / b5.clamp(min=1e-30)).max()) > 10


# ------------------------------------------------------------------------------- vs the oracle
def _close32(a, b, rtol=1e-5, atol=1e-5):
  return torch.allclose(a.float(), b.float(), rtol=rtol, atol=atol)


def test_stem_ref_matches_oracle_stem():
  """The oracle's resnet() begins with the stem conv; capture its output through the Ctx hook."""
  g = torch.Generator().manual_seed(1)
  video = torch.randint(0, 256, (2, 18, 22, 3), dtype=torch.uint8, generator=g)
  w = torch.randn(64, 3, 7, 7, generator=g) * 0.1
  captured = []

  class Stop(Exception):
    pass

  class Capture(O.Ctx):
    def conv2d(self, x, wt, b=None, stride=1, padding=0):
      captured.append(super().conv2d(x, wt, b, stride=stride, padding=padding))
      raise Stop

  x = preprocess_frames(video).permute(0, 3, 1, 2)
  with pytest.raises(Stop):
    O.resnet({'resnet_torch.initial_conv.weight': w}, x, Capture())
  ref32, _ = R.stem_ref(video, w, dtype=torch.float32)
  assert torch.equal(R.normalise_u8(video), preprocess_frames(video))
  assert _close32(ref32, captured[0].permute(0, 2, 3, 1))
  ref64, bound = R.stem_ref(video, w)
  assert float(((ref64 - captured[0].permute(0, 2, 3, 1).double()).abs() - bound).max()) <= 0


def test_instnorm_ref_matches_oracle():
  g = torch.Generator().manual_seed(2)
  x = torch.randn(3, 60, 64, generator=g) * 2 + 0.5
  w, b = torch.randn(64, generator=g), torch.randn(64, generator=g)
  ref32, _ = R.instnorm_apply_ref(x, w, b, dtype=torch.float32)
  nchw = x.reshape(3, 6, 10, 64).permute(0, 3, 1, 2)
  ora = O._inorm_relu(nchw, w, b).permute(0, 2, 3, 1).reshape(3, 60, 64)
  assert _close32(ref32, ora)
  sums, bound = R.instnorm_stats_ref(x)
  assert torch.allclose(sums[..., 0] / 60, x.double().mean(1))
  assert bool((bound > 0).all())


def test_layernorm_ref_matches_oracle():
  g = torch.Generator().manual_seed(3)
  x = torch.randn(9, 256, generator=g) * 3 + 1
  w, b = ln_weights(256, seed=4)
  ref32, _ = R.layernorm_ref(x, w, b, dtype=torch.float32)
  assert _close32(ref32, F.layer_norm(x, (256,), w, b))  # extra_convs' call
  x5 = torch.randn(9, 512, generator=g)
  w5, _ = ln_weights(512, seed=5)
  assert _close32(R.layernorm_ref(x5, w5, None, dtype=torch.float32)[0], O._ln_noshift(x5, w5))


def test_l2norm_ref_matches_oracle():
  x = l2_rows(16, 256, seed=6)
  ref32, _ = R.l2norm_ref(x, dtype=torch.float32)
  assert _close32(ref32, O._l2norm(x), atol=1e-6)


@pytest.mark.parametrize('shape', RESIZE_SHAPES, ids=lambda s: f'{s[0][0]}x{s[0][1]}-{s[1][0]}x{s[1][1]}')
def test_resize_ref_matches_oracle(shape):
  (H, W), (oH, oW) = shape
  src = resize_src(H, W, 3, seed=H + W)
  ref32, _ = R.resize_ref(src, oH, oW, dtype=torch.float32)
  ora = O.resize_video(src[None], (oH, oW))[0]
  assert _close32(ref32, ora, atol=2e-6)


def test_im2col_ref_is_the_stride2_conv_input():
  """A stride-2 3x3 conv over F.pad(x, (0, 2, 0, 2)) equals the im2col rows times the weight."""
  g = torch.Generator().manual_seed(7)
  x = torch.randn(2, 10, 6, 8, generator=g)
  w = torch.randn(16, 8, 3, 3, generator=g)
  conv = F.conv2d(F.pad(x.permute(0, 3, 1, 2).double(), (0, 2, 0, 2)), w.double(), stride=2)
  cols = R.im2col_ref(x[None], 9)[0].double()  # [F, 5, 3, 9, C]
  mm = torch.einsum('fyxtc,otc->foyx', cols, w.double().permute(0, 2, 3, 1).reshape(16, 9, 8))
  assert torch.allclose(conv, mm)
  assert torch.equal(R.im2col_ref(x[None], 1)[0][..., 0, :], x[:, ::2, ::2])


# ------------------------------------------------------------------------------- bad arguments
def _p(addr):
  return ctypes.c_void_p(addr)


A = 1 << 20  # a 16-byte aligned fake device address: every call below fails before using it
BAD = [
    ('stem null', 'tapir_stem_conv', (None, 0, _p(A), 1, 16, 16, _p(A), None)),
    ('stem odd H', 'tapir_stem_conv', (_p(A), 0, _p(A), 1, 15, 16, _p(A), None)),
    ('stem odd W', 'tapir_stem_conv', (_p(A), 1, _p(A), 1, 16, 17, _p(A), None)),
    ('stem frames', 'tapir_stem_conv', (_p(A), 0, _p(A), 65536, 16, 16, _p(A), None)),
    ('stem out align', 'tapir_stem_conv', (_p(A), 0, _p(A), 1, 16, 16, _p(A + 4), None)),
    ('stats null', 'tapir_instnorm_stats', (_p(A), 1, 16, 64, None, None)),
    ('stats C', 'tapir_instnorm_stats', (_p(A), 1, 16, 96, _p(A), None)),
    ('stats frames', 'tapir_instnorm_stats', (_p(A), 65536, 16, 64, _p(A), None)),
    ('stats x align', 'tapir_instnorm_stats', (_p(A + 8), 1, 16, 64, _p(A), None)),
    ('apply null', 'tapir_instnorm_relu_split', (_p(A), _p(A), None, _p(A), 1, 16, 64, _p(A), 1024, 1, None, 0, None)),
    ('apply C 2048', 'tapir_instnorm_relu_split', (_p(A), _p(A), _p(A), _p(A), 1, 16, 2048, _p(A), 1 << 20, 1, None, 0, None)),
    ('apply C 32', 'tapir_instnorm_relu_split', (_p(A), _p(A), _p(A), _p(A), 1, 16, 32, _p(A), 1024, 1, None, 0, None)),
    ('apply planes 0', 'tapir_instnorm_relu_split', (_p(A), _p(A), _p(A), _p(A), 1, 16, 64, _p(A), 1024, 0, None, 0, None)),
    ('apply planes 4', 'tapir_instnorm_relu_split', (_p(A), _p(A), _p(A), _p(A), 1, 16, 64, _p(A), 1024, 4, None, 0, None)),
    ('apply frames', 'tapir_instnorm_relu_split', (_p(A), _p(A), _p(A), _p(A), 65536, 16, 64, _p(A), 1 << 30, 1, None, 0, None)),
    ('apply stride align', 'tapir_instnorm_relu_split', (_p(A), _p(A), _p(A), _p(A), 1, 16, 64, _p(A), 1026, 2, None, 0, None)),
    ('apply overlap', 'tapir_instnorm_relu_split', (_p(A), _p(A), _p(A), _p(A), 1, 16, 64, _p(A), 512, 2, None, 0, None)),
    ('apply x align', 'tapir_instnorm_relu_split', (_p(A + 4), _p(A), _p(A), _p(A), 1, 16, 64, _p(A), 1024, 1, None, 0, None)),
    ('apply zero_next', 'tapir_instnorm_relu_split', (_p(A), _p(A), _p(A), _p(A), 1, 16, 64, _p(A), 1024, 1, _p(A), 0, None)),
    ('im2col null', 'tapir_im2col_s2', (None, 0, 1, 8, 8, 64, 9, _p(A), 0, 1, None)),
    ('im2col taps', 'tapir_im2col_s2', (_p(A), 4096, 1, 8, 8, 64, 4, _p(A), 4096, 1, None)),
    ('im2col C', 'tapir_im2col_s2', (_p(A), 4096, 1, 8, 8, 60, 9, _p(A), 4096, 1, None)),
    ('im2col odd H', 'tapir_im2col_s2', (_p(A), 4096, 1, 9, 8, 64, 9, _p(A), 4096, 1, None)),
    ('im2col odd W', 'tapir_im2col_s2', (_p(A), 4096, 1, 8, 7, 64, 9, _p(A), 4096, 1, None)),
    ('im2col planes', 'tapir_im2col_s2', (_p(A), 4096, 1, 8, 8, 64, 9, _p(A), 4096, 4, None)),
    ('im2col stride align', 'tapir_im2col_s2', (_p(A), 4100, 1, 8, 8, 64, 9, _p(A), 4096, 2, None)),
    ('im2col out align', 'tapir_im2col_s2', (_p(A), 4096, 1, 8, 8, 64, 9, _p(A + 8), 4096, 1, None)),
    ('ln null', 'tapir_layernorm_split', (_p(A), 4, 256, None, None, _p(A), None, 0, 1, None)),
    ('ln no output', 'tapir_layernorm_split', (_p(A), 4, 256, _p(A), None, None, None, 0, 1, None)),
    ('ln C', 'tapir_layernorm_split', (_p(A), 4, 384, _p(A), None, _p(A), None, 0, 1, None)),
    ('ln planes', 'tapir_layernorm_split', (_p(A), 4, 256, _p(A), None, None, _p(A), 1024, 4, None)),
    ('ln overlap', 'tapir_layernorm_split', (_p(A), 4, 256, _p(A), None, None, _p(A), 512, 2, None)),
    ('ln b align', 'tapir_layernorm_split', (_p(A), 4, 256, _p(A), _p(A + 4), _p(A), None, 0, 1, None)),
    ('l2 null', 'tapir_l2_normalize', (_p(A), 4, 128, None, None)),
    ('l2 C', 'tapir_l2_normalize', (_p(A), 4, 64, _p(A), None)),
    ('l2 rows', 'tapir_l2_normalize', (_p(A), 0, 128, _p(A), None)),
    ('l2 align', 'tapir_l2_normalize', (_p(A), 4, 256, _p(A + 8), None)),
]


@pytest.mark.parametrize('name,fn,args', BAD, ids=[b[0] for b in BAD])
def test_building_blocks_reject_bad_arguments(name, fn, args):
  lib = _lib.load()
  rc = getattr(lib, fn)(*args)
  msg = lib.tapir_last_error().decode()
  assert rc == 1, (name, rc, msg)
  assert msg.startswith(fn + ':'), msg
