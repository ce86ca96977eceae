"""Float64 references of the backbone's memory-bound kernels and the error bounds of their fp32
arithmetic (tests/test_backbone_ops_gpu.py compares the kernels with them; the CPU tests in
tests/test_backbone_refs_host.py check the bounds against fp32 emulations of the kernels'
operation order and the references against the oracle).

Every reference takes CPU tensors and returns float64 (or `dtype`) tensors; every bound is an
absolute, per-element tolerance derived from the kernel's own arithmetic in the standard model
fl(a op b) = (a op b)(1 + e), |e| <= u, with gamma(n) = n u / (1 - n u) for a sum of n terms in any
order.  Layouts are the kernels' (channel-last)."""
import torch
import torch.nn.functional as F

U32 = 2.0 ** -24
U64 = 2.0 ** -53
EPS_F32 = float(torch.tensor(1e-5, dtype=torch.float32))  # the kernels' 1e-5f


def gamma(n, u=U32):
  return n * u / (1 - n * u)


def warp_row_depth(C):
  """Additions on the path of one element to a row sum of the one-warp-per-row kernels: three
  inside its float4, one per float4 a lane accumulates (C / 128) and five butterfly levels.  An
  fp32 sum in that order is within gamma(depth) sum |x| (the bound of a summation tree)."""
  return 3 + C // 128 + 5


def normalise_u8(video_u8):
  """uint8 [0, 255] -> fp32 [-1, 1] exactly as preprocess_frames: three rounded fp32 operations."""
  return video_u8.float() / 255 * 2 - 1


# ------------------------------------------------------------------------------- stem conv
def stem_ref(video, weight, dtype=torch.float64):
  """video [F, H, W, 3] fp32 or uint8, weight [64, 3, 7, 7] -> (ref [F, H/2, W/2, 64], bound).

  F.pad(x, (2, 4, 2, 4)) then the stride-2 7x7 conv.  The kernel sums 147 products per output
  with fp32 FMAs: |err| <= gamma(147) * sum |w x| (plus the fp64 reference's own rounding)."""
  x = normalise_u8(video) if video.dtype == torch.uint8 else video.float()
  x = x.to(dtype).permute(0, 3, 1, 2)
  w = weight.to(dtype)
  ref = F.conv2d(F.pad(x, (2, 4, 2, 4)), w, stride=2).permute(0, 2, 3, 1)
  mag = F.conv2d(F.pad(x.abs(), (2, 4, 2, 4)), w.abs(), stride=2).permute(0, 2, 3, 1)
  return ref, (gamma(147) + gamma(147, U64)) * mag


# ------------------------------------------------------------------------------- instance norm
def instnorm_stats_ref(x):
  """x [F, hw, C] fp32 -> (sums [F, C, 2] fp64, bound).  Any fp64 summation order of hw terms is
  within gamma_64(hw) * sum |term|; the reference's own sum is as well, hence the factor 2."""
  x = x.double()
  sums = torch.stack([x.sum(1), (x * x).sum(1)], -1)
  mag = torch.stack([x.abs().sum(1), (x * x).sum(1)], -1)
  return sums, 2 * gamma(x.shape[1], U64) * mag


def instnorm_apply_ref(x, w, b, eps=1e-5, dtype=torch.float64):
  """x [F, hw, C] fp32, w, b [C] -> (ref [F, hw, C], bound) of relu((x - mu) / sqrt(var + eps) w + b)
  with biased variance.

  The kernel forms sc = w / sqrt(var + eps) and sh = b - mu sc in fp64 from the fp64 sums, rounds
  both to fp32 and computes relu(fma(x, sc, sh)); each plane of the split is the fp32 residual of
  the ones before, so three planes sum to y within 2^-27 |y|.  Per element
    |err| <= 4 u (|x sc| + |sh|)                              fp32 sc, sh, fma, split
           + |sc| (|x - mu| e_var + e_mu)                     fp64 statistics
  with e_var = 4 gamma_64(hw + 2) E[x^2] / (var + eps) (the E[x^2] - mu^2 cancellation) and
  e_mu = 2 gamma_64(hw) E|x|.  ReLU is 1-Lipschitz, so the bound carries through it."""
  hw = x.shape[1]
  x64 = x.double()
  mu = x64.mean(1, keepdim=True)
  var = ((x64 - mu) ** 2).mean(1, keepdim=True)
  sc = w.double() / torch.sqrt(var + eps)
  sh = b.double() - mu * sc
  xd = x.to(dtype)
  ref = torch.relu((xd - mu.to(dtype)) / torch.sqrt(var.to(dtype) + eps) * w.to(dtype) + b.to(dtype))
  e_var = 4 * gamma(hw + 2, U64) * (x64 * x64).mean(1, keepdim=True) / (var + eps)
  e_mu = 2 * gamma(hw, U64) * x64.abs().mean(1, keepdim=True)
  bound = 4 * U32 * ((x64 * sc).abs() + sh.abs()) + sc.abs() * ((x64 - mu).abs() * e_var + e_mu)
  return ref, bound


def sums_fp64(x):
  """The fp64 (sum, sum of squares) the apply kernel reads, [F, C, 2]."""
  return instnorm_stats_ref(x)[0]


# ------------------------------------------------------------------------------- im2col
def im2col_ref(planes, taps):
  """planes [P, F, H, W, C] -> [P, F, H/2, W/2, taps, C]: tap (ky, kx) of a stride-2 conv over
  F.pad(x, (0, 2, 0, 2)) (taps 9), or in[2y, 2x] (taps 1)."""
  P, Fr, H, W, C = planes.shape
  x = F.pad(planes.float(), (0, 0, 0, 2, 0, 2)).to(planes.dtype)  # pad W then H by 2 at the end
  k = 3 if taps == 9 else 1
  cols = [x[:, :, ky:ky + H:2, kx:kx + W:2] for ky in range(k) for kx in range(k)]
  return torch.stack(cols, 4)


# ------------------------------------------------------------------------------- layer norm
def layernorm_ref(x, w, b=None, eps=1e-5, dtype=torch.float64):
  """x [rows, C] fp32 -> (ref, bound) of LayerNorm over C (biased variance, eps 1e-5).

  The kernel (one warp per row) is two-pass fp32: mu^ = fl(sum x) / C, d^ = fl(x - mu^),
  v = fl(sum d^2) / C, r = 1 / sqrt(v + 1e-5f), o = fl(fl(d^ r) w) (+ b).  With
    dmu  = gamma(C) sum|x| / C                           the mean's error
    dd   = dmu (1 + u) + u |d|                           the centred value's error
    dvar = gamma(C + 1) var + (2 dmu sum|d| + 2 u sum d^2 + C dd_max^2) / C
    e_r  = (dvar + u (var + eps) + |1e-5f - 1e-5|) / (2 (var + eps)) + 2 u    rstd's relative error
  the error of every output is |w| rstd (dd + (|d| + dd)(e_r + 3u)) + 2 u (|ref| + |b|), where
  n = warp_row_depth(C) is the depth of the kernel's summation tree."""
  C = x.shape[-1]
  x64 = x.double()
  mu = x64.mean(-1, keepdim=True)
  d = x64 - mu
  var = (d * d).mean(-1, keepdim=True)
  rstd = 1 / torch.sqrt(var + eps)
  w64 = w.double()
  b64 = b.double() if b is not None else torch.zeros_like(w64)
  ref = F.layer_norm(x.to(dtype), (C,), w.to(dtype), None if b is None else b.to(dtype), eps=eps)
  n = warp_row_depth(C)
  dmu = gamma(n) * x64.abs().sum(-1, keepdim=True) / C
  dd = dmu * (1 + U32) + U32 * d.abs()
  dd_max = dd.amax(-1, keepdim=True)
  dvar = (gamma(n + 1) * var + (2 * dmu * d.abs().sum(-1, keepdim=True) + 2 * U32 * (d * d).sum(-1, keepdim=True)
                                + C * dd_max ** 2) / C)
  e_r = (dvar + U32 * (var + eps) + abs(EPS_F32 - eps)) / (2 * (var + eps)) + 2 * U32
  bound = w64.abs() * rstd * (dd + (d.abs() + dd) * (e_r + 3 * U32)) + 2 * U32 * (
      (d * rstd * w64 + b64).abs() + b64.abs())
  return ref, bound


# ------------------------------------------------------------------------------- L2 norm
def l2norm_ref(x, dtype=torch.float64):
  """x [rows, C] fp32 -> (ref, bound) of x / sqrt(max(sum x^2, 1e-12)).

  fl(sum x^2) in the kernel's order has relative error gamma(n + 1), n = warp_row_depth(C); sqrtf
  and the division each round once; the clamp constant 1e-12f differs from 1e-12 by 4e-9
  relative: |err| <= |ref| (gamma(n + 1) / 2 + 3 u)."""
  C = x.shape[-1]
  xd = x.to(dtype)
  ref = xd / torch.sqrt(torch.clamp((xd * xd).sum(-1, keepdim=True), min=1e-12))
  return ref, ref.double().abs() * (gamma(warp_row_depth(C) + 1) / 2 + 3 * U32)


# ------------------------------------------------------------------------------- bilinear resize
def _source_coord(out_size, in_size, fma):
  """fp32 source coordinate of every output row / column, as F.interpolate computes it on fp32
  tensors (scale = in / out, src = scale (i + 0.5) - 0.5, clamped at 0), or with the product and
  the subtraction fused into one rounding (fma=True, what nvcc emits)."""
  scale = torch.tensor(in_size, dtype=torch.float32) / torch.tensor(out_size, dtype=torch.float32)
  i = torch.arange(out_size, dtype=torch.float32) + 0.5
  if fma:
    src = (scale.double() * i.double() - 0.5).float()
  else:
    src = scale * i - 0.5
  return torch.clamp(src, min=0.0)


def _blend(src, fy, fx, dtype):
  """src [F, H, W, C]; fy [oH], fx [oW] (float64 positions) -> [F, oH, oW, C] in dtype, with the
  weights computed in fp32 from fp32 positions as the kernel and F.interpolate do."""
  H, W = src.shape[1:3]
  fy32, fx32 = fy.float(), fx.float()
  y0 = torch.clamp(torch.floor(fy32).long(), max=H - 1)
  x0 = torch.clamp(torch.floor(fx32).long(), max=W - 1)
  y1 = torch.clamp(y0 + 1, max=H - 1)
  x1 = torch.clamp(x0 + 1, max=W - 1)
  ly = (fy32 - y0.float()).to(dtype)
  lx = (fx32 - x0.float()).to(dtype)
  hy, hx = (1 - ly.float()).to(dtype), (1 - lx.float()).to(dtype)
  s = src.to(dtype)
  r0 = s[:, y0]
  r1 = s[:, y1]
  hx_, lx_ = hx[None, None, :, None], lx[None, None, :, None]
  top = hx_ * r0[:, :, x0] + lx_ * r0[:, :, x1]
  bot = hx_ * r1[:, :, x0] + lx_ * r1[:, :, x1]
  return hy[None, :, None, None] * top + ly[None, :, None, None] * bot


def resize_ref(src, oH, oW, dtype=torch.float64):
  """src [F, H, W, C] fp32 -> (ref [F, oH, oW, C], bound): bilinear, align_corners=False, no
  antialias; source coordinates in fp32 as F.interpolate computes them on fp32 tensors, blend in
  `dtype`.

  The kernel's coordinate may differ from this one: nvcc fuses s (i + 0.5) - 0.5 into one FMA, so
  the two agree to |dy| <= 2 u (|fy| + 1).  The bound takes the largest change of the fp64 blend
  under that shift (the blend is continuous, so a shift across a pixel boundary is covered), plus
  the fp32 blend's own rounding: weights 1 - l round once, four products and three sums, all of
  magnitude <= M = max |tap|, within 6 u M."""
  H, W = src.shape[1:3]
  fy = _source_coord(oH, H, False).double()
  fx = _source_coord(oW, W, False).double()
  ref = _blend(src, fy, fx, dtype)
  if dtype != torch.float64:
    return ref, None
  r64 = ref
  dy = 2 * U32 * (fy.abs() + 1)
  dx = 2 * U32 * (fx.abs() + 1)
  shift = torch.zeros_like(r64)
  for sy, sx in ((1, 0), (-1, 0), (0, 1), (0, -1)):
    fy2 = torch.clamp(fy + sy * dy, min=0.0)
    fx2 = torch.clamp(fx + sx * dx, min=0.0)
    shift = torch.maximum(shift, (_blend_exact(src, fy2, fx2) - r64).abs())
  taps = _tap_max(src, fy, fx)
  return ref, shift + 6 * U32 * taps


def _blend_exact(src, fy, fx):
  """The bilinear blend at float64 positions (weights in float64, no fp32 rounding)."""
  H, W = src.shape[1:3]
  y0 = torch.clamp(torch.floor(fy).long(), max=H - 1)
  x0 = torch.clamp(torch.floor(fx).long(), max=W - 1)
  y1 = torch.clamp(y0 + 1, max=H - 1)
  x1 = torch.clamp(x0 + 1, max=W - 1)
  ly, lx = fy - y0.double(), fx - x0.double()
  s = src.double()
  r0, r1 = s[:, y0], s[:, y1]
  lx_ = lx[None, None, :, None]
  top = (1 - lx_) * r0[:, :, x0] + lx_ * r0[:, :, x1]
  bot = (1 - lx_) * r1[:, :, x0] + lx_ * r1[:, :, x1]
  ly_ = ly[None, :, None, None]
  return (1 - ly_) * top + ly_ * bot


def _tap_max(src, fy, fx):
  H, W = src.shape[1:3]
  y0 = torch.clamp(torch.floor(fy.float()).long(), max=H - 1)
  x0 = torch.clamp(torch.floor(fx.float()).long(), max=W - 1)
  y1, x1 = torch.clamp(y0 + 1, max=H - 1), torch.clamp(x0 + 1, max=W - 1)
  a = src.double().abs()
  r = torch.maximum(a[:, y0], a[:, y1])
  return torch.maximum(r[:, :, x0], r[:, :, x1])
