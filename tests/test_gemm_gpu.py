"""wgmma split-bf16 GEMM / implicit 3x3 conv vs an exact fp64 model of the same planes."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from tests import gpu_util as U  # noqa: E402


def _gelu(x):
  return F.gelu(x, approximate='tanh')


CASES = [
    # M, N, K, P, bias, gelu, residual, out_planes
    (128, 128, 64, 1, False, False, False, 0),
    (300, 200, 128, 1, True, False, False, 0),
    (300, 200, 128, 2, True, False, True, 0),
    (300, 200, 128, 3, False, False, False, 0),
    (1000, 512, 2048, 2, True, False, True, 0),
    (4096, 2048, 512, 2, True, True, False, 2),
    (777, 388, 512, 2, True, False, False, 0),
    (520, 64, 576, 2, False, False, False, 0),
    (16, 8192, 256, 3, False, False, False, 0),
    (20000, 512, 576, 2, True, False, False, 0),
    # shapes whose persistent schedule ends in a partial round (mixer `up` and `down`; linear_out:
    # an odd number of row tiles and a last column tile that reaches beyond N = 388)
    (12288, 2048, 512, 2, True, True, False, 2),
    (12288, 512, 2048, 2, True, False, True, 0),
    (9600, 388, 512, 2, True, False, False, 0),
]


@pytest.mark.parametrize('impl', [1, 0], ids=['simt', 'tc'])
@pytest.mark.parametrize('case', CASES)
def test_gemm(case, impl):
  M, N, K, P, bias, gelu, resid, opl = case
  g = torch.Generator().manual_seed(M + N + K + P)
  a = torch.randn(M, K, generator=g).cuda()
  w = (torch.randn(N, K, generator=g) / K ** 0.5).cuda()
  b = torch.randn(N, generator=g).cuda() if bias else None
  r = torch.randn(M, N, generator=g).cuda() if resid else None
  a_pl, w_pl = U.split(a, P), U.split(w, P)
  o32, op = U.gemm(a_pl, w_pl, b, r, gelu, True, opl, impl)
  if impl == 0:
    ref = U.planes_matmul_fp64(a_pl, w_pl)
  else:  # SIMT path keeps every cross term
    ref = a_pl.double().sum(0).cpu() @ w_pl.double().sum(0).cpu().t()
  if b is not None:
    ref = ref + b.double().cpu()
  if gelu:
    ref = _gelu(ref)
  if r is not None:
    ref = ref + r.double().cpu()
  err = (o32.double().cpu() - ref).abs().max().item()
  scale = ref.abs().max().item()
  U.record(f'gemm_impl{impl}_{M}x{N}x{K}_P{P}', max_err=err, scale=scale)
  assert torch.isfinite(o32).all()
  assert err <= 2e-5 * max(scale, 1.0) + (3e-5 if gelu else 0.0)
  if opl:
    rec = op.double().sum(0).cpu()
    perr = (rec - ref).abs().max().item()
    U.record(f'gemm_impl{impl}_{M}x{N}x{K}_P{P}_planes', max_err=perr)
    assert perr <= 1e-4 * max(scale, 1.0)


CONV_CASES = [
    # frames, H, W, Cin, Cout, P, bias, gelu, residual
    (2, 32, 32, 64, 64, 2, False, False, False),
    (3, 32, 32, 256, 1024, 2, True, True, False),
    (1, 64, 64, 128, 128, 2, False, False, True),
    (2, 40, 48, 64, 128, 2, True, False, False),
    (1, 128, 128, 64, 64, 3, False, False, False),
    (2, 20, 24, 64, 64, 1, False, False, False),
]


@pytest.mark.parametrize('impl', [1, 0], ids=['simt', 'tc'])
@pytest.mark.parametrize('case', CONV_CASES)
def test_conv3x3(case, impl):
  Fr, H, W, Ci, Co, P, bias, gelu, resid = case
  g = torch.Generator().manual_seed(H * W + Ci + Co)
  x = torch.randn(Fr, H, W, Ci, generator=g).cuda()
  w = (torch.randn(Co, Ci, 3, 3, generator=g) / (9 * Ci) ** 0.5).cuda()
  b = torch.randn(Co, generator=g).cuda() if bias else None
  r = torch.randn(Fr * H * W, Co, generator=g).cuda() if resid else None
  x_pl = U.split(x.reshape(-1, Ci), P).reshape(P, Fr, H, W, Ci)
  w2d = w.permute(0, 2, 3, 1).reshape(Co, 9 * Ci)
  w_pl = U.split(w2d, P)
  o32, _ = U.gemm(x_pl, w_pl, b, r, gelu, True, 0, impl, conv=(Fr, H, W, Ci))
  if impl == 0:  # exact model of the tensor-core math: the i+j<P plane pairs only
    ref = U.conv_planes_fp64(x_pl, w_pl)
  else:  # SIMT path keeps every cross term: conv of the plane sums
    ref = U.conv_planes_fp64(x_pl.double().sum(0, keepdim=True), w_pl.double().sum(0, keepdim=True))
  if b is not None:
    ref = ref + b.double().cpu()
  if gelu:
    ref = _gelu(ref)
  if r is not None:
    ref = ref + r.double().cpu()
  err = (o32.double().cpu() - ref).abs().max().item()
  scale = ref.abs().max().item()
  U.record(f'conv_impl{impl}_{Fr}x{H}x{W}x{Ci}to{Co}_P{P}', max_err=err, scale=scale)
  assert torch.isfinite(o32).all()
  # against the exact model only fp32 accumulation error is left, whatever P
  assert err <= U.accum_tol(9 * Ci, P, scale, gelu)


@pytest.mark.parametrize('impl', [1, 0], ids=['simt', 'tc'])
@pytest.mark.parametrize('mode', ['conv', 'plain'])
def test_fused_instance_norm_statistics(mode, impl):
  """Epilogue-fused per-(frame, channel) sum / sum of squares of the GEMM output."""
  g = torch.Generator().manual_seed(5)
  Fr, H, W, Ci, Co, P = 3, 24, 32, 64, 128, 2
  w = (torch.randn(Co, Ci * (9 if mode == 'conv' else 1), generator=g) / 8).cuda()
  stats = torch.zeros(Fr, Co, 2, dtype=torch.float64, device='cuda')
  x = torch.randn(Fr * H * W, Ci, generator=g).cuda()
  x_pl = U.split(x, P)
  if mode == 'conv':
    o32, _ = U.gemm(x_pl.reshape(P, Fr, H, W, Ci), U.split(w, P), impl=impl, conv=(Fr, H, W, Ci), stats=stats)
  else:
    o32, _ = U.gemm(x_pl, U.split(w, P), impl=impl, stats=stats, rows_per_frame=H * W)
  out = o32.double().reshape(Fr, H * W, Co)
  ref = torch.stack([out.sum(1), (out * out).sum(1)], -1)
  err = ((stats - ref).abs() / ref.abs().clamp(min=1.0)).max().item()
  U.record(f'gemm_stats_{mode}_impl{impl}', rel_err=err)
  assert err < 5e-5

