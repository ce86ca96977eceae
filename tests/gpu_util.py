"""Helpers for the -m gpu tests: everything goes through the C ABI (tapnet_b200._lib)."""
import atexit
import contextlib
import ctypes
import json
import os

import torch

from tapnet_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REPORT = {}


def _dump_report():
  if not REPORT:
    return
  out = os.path.join(ROOT, 'gpurun_out')
  try:
    os.makedirs(out, exist_ok=True)
    path = os.path.join(out, 'test_report.json')
    old = {}
    if os.path.exists(path):
      with open(path) as fh:
        old = json.load(fh)
    old.update(REPORT)
    with open(path, 'w') as fh:
      json.dump(old, fh, indent=1, sort_keys=True)
  except Exception:  # pylint: disable=broad-except
    pass


atexit.register(_dump_report)


def record(name, **vals):
  REPORT[name] = {k: (float(v) if hasattr(v, '__float__') else v) for k, v in vals.items()}
  print(f'[report] {name}: ' + ', '.join(f'{k}={v}' for k, v in REPORT[name].items()))


ptr, stream = _lib.ptr, _lib.stream


def split(x, planes, kpad=None):
  """fp32 [rows, cols] (cuda) -> bf16 planes [P, rows, kpad] through tapir_split_planes."""
  x = x.contiguous().float()
  rows, cols = x.shape
  out = torch.empty(planes, rows, kpad or cols, dtype=torch.bfloat16, device=x.device)
  _lib.split_planes(x, out)
  return out


GUARD = 16  # elements of NaN fill before and after every guarded() output


def guarded(n, dtype=torch.float32):
  """A NaN-filled buffer (-7 for integers) with GUARD elements either side of an n-element body."""
  fill = -7 if not dtype.is_floating_point else float('nan')
  buf = torch.full((n + 2 * GUARD,), fill, dtype=dtype, device='cuda')
  return buf, buf[GUARD:GUARD + n]


def guards_intact(buf):
  g = torch.cat([buf[:GUARD], buf[-GUARD:]])
  return bool(torch.isnan(g.float()).all()) if buf.dtype.is_floating_point else bool((g == -7).all())


def planes_matmul_fp64(a_pl, b_pl):
  """sum_{i+j<P} A_i @ B_j^T in float64 on the CPU (exact model of the tensor-core math)."""
  a = a_pl.double().cpu()
  b = b_pl.double().cpu()
  P = a.shape[0]
  acc = None
  for i in range(P):
    for j in range(P - i):
      t = a[i] @ b[j].t()
      acc = t if acc is None else acc + t
  return acc


def make_linear(w_pl, bias):
  P, n, k = w_pl.shape
  return _lib.Linear(w=w_pl.data_ptr(), bias=(bias.data_ptr() if bias is not None else None), N=n,
                     K=k, planes=P, k_logical=k)


def conv_planes_fp64(x_pl, w_pl):
  """sum_{i+j<P} conv3x3(X_i, W_j) in float64 on the CPU: the conv counterpart of
  planes_matmul_fp64.  x_pl [P, F, H, W, C] (NHWC), w_pl [P, N, 9*C] with K ordered (ky, kx, c);
  returns [F*H*W, N] (stride 1, zero padding 1)."""
  x = x_pl.double().cpu().permute(0, 1, 4, 2, 3)  # [P, F, C, H, W]
  P, _, C = x.shape[:3]
  wt = w_pl.double().cpu().reshape(P, -1, 3, 3, C).permute(0, 1, 4, 2, 3)  # [P, N, C, 3, 3]
  acc = None
  for i in range(P):
    for j in range(P - i):
      t = torch.nn.functional.conv2d(x[i], wt[j], padding=1)
      acc = t if acc is None else acc + t
  return acc.permute(0, 2, 3, 1).reshape(-1, wt.shape[1])


def accum_tol(k, planes, scale, gelu=False):
  """Absolute tolerance of a split-bf16 GEMM / conv output against its exact fp64 model.

  The bf16 products are exact, so what is left is fp32 accumulation error.  The wgmma accumulator
  does not round to nearest, so that error grows about linearly with the number of products summed
  into one accumulator, k * P (P + 1) / 2.  Measured on one H100 80GB HBM3 (max error / scale):
  6.1e-6 at 3456 products, 8.1e-6 at 6912, 2.3e-5 at 27648 (single pass, conv 1024 -> 256).
  The bound is 2e-5 up to 6144 products and grows in proportion beyond: margin >= 2.5x.
  tanh-GELU adds the error of its ex2 / rcp approximations (3e-5)."""
  terms = k * planes * (planes + 1) // 2
  return 2e-5 * max(1.0, terms / 6144) * max(scale, 1.0) + (3e-5 if gelu else 0.0)


def split_like_kernel(v, planes):
  """fp32 tensor -> the bf16 planes the GEMM epilogue stores: plane q = bf16(v - sum_{s<q} plane s)."""
  out, r = [], v.float().clone()
  for _ in range(planes):
    h = r.to(torch.bfloat16)
    r = r - h.float()
    out.append(h)
  return torch.stack(out)


def launch_count():
  return int(_lib.load().tapir_launch_count())


@contextlib.contextmanager
def switches(**kv):
  """Sets the library's environment switches (tapnet_b200/csrc/gemm.cuh, read on every GEMM call)
  for the body of the with block; None unsets one.  The previous values come back on exit."""
  old = {k: os.environ.get(k) for k in kv}

  def put(env):
    for k, v in env.items():
      if v is None:
        os.environ.pop(k, None)
      else:
        os.environ[k] = str(v)
  put(kv)
  try:
    yield
  finally:
    put(old)


def kernels(fn, pattern):
  """Names of the CUDA kernels that fn() runs whose names contain `pattern` (torch.profiler)."""
  from torch.profiler import ProfilerActivity, profile  # pylint: disable=g-import-not-at-top
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    fn()
    torch.cuda.synchronize()
  return [e.name for e in prof.events() if pattern in e.name]


class GemmResult:
  """What gemm(..., details=True) returns.  out / planes are [M, N] views of out_buf / planes_buf;
  everything else in those buffers (leading offset, ld padding, tail) was NaN before the call."""

  def __init__(self, **kw):
    self.__dict__.update(kw)


def gemm(a_pl, w_pl, bias=None, residual=None, gelu=False, out_f32=True, out_planes=0, impl=0,
         conv=None, stats=None, rows_per_frame=0, ld_pad=0, offset=0, splitk_ws=None,
         details=False):
  """Runs tapir_gemm_ex. a_pl: [P, M, K] (plain) or [P, F, H, W, C] (conv=(F,H,W,C)), unit
  stride in K (plain) or dense within a plane (conv); its plane stride and, plain, its row stride
  are passed as they are, so a view may space its planes and rows further apart.

  ld_pad: the output, residual and plane leading dimensions are N + ld_pad.  offset: the fp32
  output and the residual start `offset` floats into their allocations (offset 1 gives 4-byte but
  not 8-byte aligned rows).  splitk_ws: a uint8 / float cuda tensor used as split-K workspace
  (None: no split-K).  details=True returns a GemmResult with the padded buffers and the number of
  kernel launches the call made; otherwise (out [M, N] fp32 or None, planes [out_P, M, N] or None)."""
  lib = _lib.load()
  P, n, k = w_pl.shape
  dev = w_pl.device
  if conv is None:
    assert a_pl.stride(2) == 1, a_pl.stride()
    m = a_pl.shape[1]
    lda, aps = a_pl.stride(1), a_pl.stride(0)
    f = h = w = c = 0
  else:
    assert a_pl[0].is_contiguous(), a_pl.stride()
    f, h, w, c = conv
    m = f * h * w
    lda, aps = 0, a_pl.stride(0)
  ld = n + ld_pad
  tail = 8  # guard elements after the last row
  lin = make_linear(w_pl, bias)
  nan = float('nan')
  out_buf = o32 = None
  if out_f32:
    out_buf = torch.full((offset + m * ld + tail,), nan, dtype=torch.float32, device=dev)
    o32 = out_buf[offset:offset + m * ld].view(m, ld)[:, :n]
  res_buf = rp = None
  if residual is not None:
    res_buf = torch.full((offset + m * ld + tail,), nan, dtype=torch.float32, device=dev)
    res_buf[offset:offset + m * ld].view(m, ld)[:, :n] = residual
    rp = ctypes.c_void_p(res_buf.data_ptr() + 4 * offset)
  planes_buf = opl = None
  if out_planes:
    planes_buf = torch.full((out_planes * m * ld + tail,), nan, dtype=torch.bfloat16, device=dev)
    opl = planes_buf[:out_planes * m * ld].view(out_planes, m, ld)[:, :, :n]
  ws, ws_bytes = None, 0
  if splitk_ws is not None:
    ws, ws_bytes = ptr(splitk_ws), splitk_ws.numel() * splitk_ws.element_size()
  op = ctypes.c_void_p(out_buf.data_ptr() + 4 * offset) if out_f32 else None
  torch.cuda.synchronize()
  before = launch_count()
  st = lib.tapir_gemm_ex(ptr(a_pl), lda, aps, ctypes.byref(lin), m, 1 if conv else 0, f, h, w, c,
                         rp, ld if residual is not None else 0, int(gelu), op, ld, ptr(planes_buf),
                         ld, m * ld, out_planes, ptr(stats), rows_per_frame, impl, ws, ws_bytes,
                         stream())
  _lib.check(st, 'tapir_gemm_ex')
  torch.cuda.synchronize()
  launches = launch_count() - before
  if not details:
    return o32, opl
  return GemmResult(out=o32, planes=opl, out_buf=out_buf, planes_buf=planes_buf, ld=ld,
                    offset=offset, launches=launches, m=m, n=n, out_P=out_planes)


def untouched_padding(res):
  """True if every element of res's buffers outside its [M, N] views still holds its NaN fill."""
  for buf, off, planes in ((res.out_buf, res.offset, 1), (res.planes_buf, 0, res.out_P)):
    if buf is None:
      continue
    end = off + planes * res.m * res.ld
    body = buf[off:end].float().view(planes, res.m, res.ld)
    outside = torch.cat([buf[:off].float(), body[:, :, res.n:].reshape(-1), buf[end:].float()])
    if not bool(torch.isnan(outside).all()):
      return False
  return True
