"""Every GEMM epilogue path bit for bit, on operands whose accumulators are exact (tests/gemm_exact.py).

Each case runs on the tensor cores under every layout (aligned: whole tiles take epilogue_full;
odd leading dimension and 4-byte aligned output: every tile takes the general loop), both tile
widths (TAPIR_B200_BLOCK_N) and both schedules (TAPIR_B200_GEMM_SCHEDULE; ping-pong only for
P <= 2), and once on the SIMT kernel.  Every run writes NaN-filled buffers and must leave their
padding alone.  Without GELU every output bit and every fused statistic must equal the emulation.
With GELU every path must give the bits of one general-loop run with fp32 and three-plane outputs,
which lies within the tanh-GELU error bound, and its planes must be the split of its fp32 output;
GELU followed by a residual, which no model layer runs, is checked against the bound only, because
the last GELU multiply may be fused with the residual add differently on different paths.

tapir_split_planes, which makes the GEMM operands everywhere else, is checked bit for bit against
torch's round-to-nearest-even split here as well."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tapnet_b200 import _lib  # noqa: E402
from tests import gemm_exact as E  # noqa: E402
from tests import gpu_util as U  # noqa: E402

CASES = {c.cid: c for c in E.CASES}


def _tc_runs(P):
  """(label, ld_pad, offset, env) of every tensor-core run of a case."""
  for layout, (ld_pad, offset) in E.LAYOUTS.items():
    for bn in (64, 128):
      for sched in (('coop', 'pingpong') if P <= 2 else ('coop',)):
        yield (f'{layout}_bn{bn}_{sched}', ld_pad, offset,
               dict(TAPIR_B200_BLOCK_N=bn, TAPIR_B200_GEMM_SCHEDULE=sched))


def _dev(d):
  if not hasattr(d, 'dev'):
    d.dev = dict(a=d.a_pl.cuda(), w=d.w_pl.cuda(), bias=d.bias.cuda(), resid=d.resid.cuda())
  return d.dev


def _run(case, opts, impl, ld_pad=0, offset=0, env=None, splitk=False):
  d = case.design()
  t = _dev(d)
  bias, gelu, resid, f32_out, out_P, stats = opts
  frames = d.M // d.rows_per_frame
  st = torch.zeros(frames, d.N, 2, dtype=torch.float64, device='cuda') if stats else None
  ws = None
  if splitk:
    ws = torch.empty(8 * d.M * ((d.N + 7) // 8 * 8) * 4, dtype=torch.uint8, device='cuda')
  with U.switches(**(env or {})):
    res = U.gemm(t['a'], t['w'], t['bias'] if bias else None, t['resid'] if resid else None, gelu,
                 f32_out, out_P, impl, conv=case.conv, stats=st,
                 rows_per_frame=d.rows_per_frame if stats and case.conv is None else 0,
                 ld_pad=ld_pad, offset=offset, splitk_ws=ws, details=True)
  assert U.untouched_padding(res), 'wrote outside the [M, N] output'
  if splitk and impl == 0:
    assert res.launches == 2, res.launches
  return res, st


def _bits(x):
  return x.view(torch.int16 if x.element_size() == 2 else torch.int32)


def _mismatch(got, want):
  """Number of elements whose bits differ (got on the GPU, want on the CPU)."""
  got = got.cpu()
  want = torch.from_numpy(want) if isinstance(want, np.ndarray) else want
  return int((_bits(got.contiguous()) != _bits(want.contiguous())).sum())


def _check_exact(name, case, opts, res, st):
  bias, _, resid, f32_out, out_P, stats = opts
  want = E.emulate(case.design(), bias, resid, out_P, stats)
  bad = {}
  if f32_out:
    bad['out'] = _mismatch(res.out, want['out'])
  if out_P:
    bad['planes'] = _mismatch(res.planes, want['planes'])
  if stats:
    bad['stats'] = int((st.cpu().numpy() != want['stats']).sum())
  assert not any(bad.values()), (name, bad)


_GELU_REF = {}


def _gelu_reference(case, bias):
  """One general-loop run (odd leading dimension) with fp32 and three-plane outputs: within the
  GELU bound, and its planes the split of its fp32 output.  Every GELU path must reproduce it."""
  key = (case.cid, bias)
  if key not in _GELU_REF:
    opts = E.option_set(bias, True, False, True, 3, False)
    res, _ = _run(case, opts, 0, ld_pad=1, offset=1)
    out = res.out.cpu()
    v = E.pre_activation(case.design(), bias)
    want, tol = E.gelu_bound(v)
    err = (out.double() - want).abs() - tol
    U.record(f'gemm_exact_{case.cid}_gelu_ref_bias{int(bias)}', worst_excess=err.max().item())
    assert (err <= 0).all(), (case.cid, 'GELU outside its error bound', err.max().item())
    assert _mismatch(res.planes, U.split_like_kernel(out, 3)) == 0, 'planes != split of fp32 output'
    _GELU_REF[key] = out
  return _GELU_REF[key]


def _check_gelu(name, case, opts, res, agree):
  bias, _, resid, f32_out, out_P, _ = opts
  if resid:
    v = E.pre_activation(case.design(), bias)
    want, tol = E.gelu_bound(v, case.design().resid.numpy())
    out = res.out.cpu()
    assert ((out.double() - want).abs() <= tol).all(), name
    agree.append(out)
    return
  ref = _gelu_reference(case, bias)
  bad = {}
  if f32_out:
    bad['out'] = _mismatch(res.out, ref)
  if out_P:
    bad['planes'] = _mismatch(res.planes, U.split_like_kernel(ref, out_P))
  assert not any(bad.values()), (name, bad)


def _check(name, case, opts, res, st, agree):
  if opts[1]:
    _check_gelu(name, case, opts, res, agree)
  else:
    _check_exact(name, case, opts, res, st)


def _record_gelu_resid_agreement(name, agree):
  if agree:
    same = all(torch.equal(_bits(agree[0]), _bits(x)) for x in agree[1:])
    U.record(name + '_gelu_resid_paths_agree', identical=int(same), runs=len(agree))


# ------------------------------------------------------------------------------ design check
DESIGN_CHECK = ['plain_r_p1', 'plain_r_p2', 'plain_r_p3', 'conv_g', 'halo_s']
PLAIN = E.option_set(False, False, False, True, 0, False)


@pytest.mark.parametrize('cid', DESIGN_CHECK)
def test_design_check_exact_accumulator_tc(cid):
  """The premise: on these operands every tensor-core path's fp32 accumulator is the exact sum."""
  case = CASES[cid]
  for label, ld_pad, offset, env in _tc_runs(case.P):
    res, st = _run(case, PLAIN, 0, ld_pad, offset, env)
    _check_exact(f'{cid}_{label}', case, PLAIN, res, st)


@pytest.mark.parametrize('cid', DESIGN_CHECK)
def test_design_check_exact_accumulator_simt(cid):
  case = CASES[cid]
  res, st = _run(case, PLAIN, 1)
  _check_exact(f'{cid}_simt', case, PLAIN, res, st)


# ------------------------------------------------------------------------------ every path
@pytest.mark.parametrize('cid', sorted(CASES))
def test_epilogue_bits_tc(cid):
  case = CASES[cid]
  for opts in case.sets:
    agree = []
    for label, ld_pad, offset, env in _tc_runs(case.P):
      for splitk in ((True, False) if case.splitk else (False,)):
        name = f'{cid}_{E.set_name(opts)}_{label}' + ('_splitk' if splitk else '')
        res, st = _run(case, opts, 0, ld_pad, offset, env, splitk)
        _check(name, case, opts, res, st, agree)
    _record_gelu_resid_agreement(f'gemm_exact_{cid}_tc', agree)


@pytest.mark.parametrize('cid', sorted(CASES))
def test_epilogue_bits_simt(cid):
  case = CASES[cid]
  for opts in case.sets:
    agree = []
    res, st = _run(case, opts, 1)
    _check(f'{cid}_{E.set_name(opts)}_simt', case, opts, res, st, agree)
    _record_gelu_resid_agreement(f'gemm_exact_{cid}_simt', agree)


# ------------------------------------------------------------------------------ split planes
def _split_inputs(rows, cols, ld_src, seed):
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(rows, ld_src, generator=g) * torch.exp2(torch.randint(-20, 21, (rows, ld_src), generator=g).float())
  special = torch.tensor([
      1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), -(1 + 3 * 2 ** -8),   # bf16 ties: to even
      1 + 2 ** -8 + 2 ** -16 + 2 ** -24, 1 - 2 ** -24,                     # ties in lower planes
      1e-40, -3e-39, 2 ** -149, 1.2e-38, -1.17549435e-38,                  # subnormals, no flush
      1.5, -3.0, 2 ** -100, 65280.0,                                       # planes 1, 2 are zero
      -0.0, 0.0, 3.0e38, -3.0e38,                                          # signed zero, large
  ], dtype=torch.float32)
  # values at or above the bf16 overflow threshold (about 3.39e38) split into (inf, -inf) and are
  # out of scope; 3.0e38 stays below it
  x.view(-1)[:special.numel() * 40] = special.repeat(40)
  x[:, cols:] = float('nan')  # columns past `cols` must never be read
  return x.float()


@pytest.mark.parametrize('P', [1, 2, 3])
def test_tc_operand_split_planes_bits(P):
  """tapir_split_planes against torch's sequential round-to-nearest-even split: padded source rows,
  zeroed padding columns, untouched guard columns, and enough rows for the grid-stride loop."""
  lib = _lib.load()
  rows, cols, cols_padded, ld_src, ld_dst = 70001, 61, 64, 67, 72
  x = _split_inputs(rows, cols, ld_src, P)
  src = x.cuda()
  plane_stride = rows * ld_dst + 8
  buf, dst = U.guarded(P * plane_stride, torch.bfloat16)
  torch.cuda.synchronize()
  st = lib.tapir_split_planes(U.ptr(src), ld_src, U.ptr(dst), ld_dst, plane_stride, rows, cols,
                              cols_padded, P, U.stream())
  _lib.check(st, 'tapir_split_planes')
  torch.cuda.synchronize()
  assert U.guards_intact(buf)
  body = dst.view(P, plane_stride)[:, :rows * ld_dst].view(P, rows, ld_dst).cpu()
  want = U.split_like_kernel(x[:, :cols], P)
  bad = int((_bits(body[:, :, :cols].contiguous()) != _bits(want)).sum())
  U.record(f'split_planes_P{P}', mismatched=bad)
  assert bad == 0
  pad = body[:, :, cols:cols_padded]
  assert _bits(pad.contiguous()).eq(0).all(), 'padding columns must be +0'
  assert torch.isnan(body[:, :, cols_padded:].float()).all(), 'guard columns were written'
  assert torch.isnan(dst.view(P, plane_stride)[:, rows * ld_dst:].float()).all()
