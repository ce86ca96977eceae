"""The C = 64 -> 64 halo convolution under both schedules (conv3x3_halo_kernel, cooperative, and
conv3x3_halo_pingpong_kernel) and the generic implicit GEMM give the same output bits, and the
fused InstanceNorm statistics are the sums of the kernel's own output.

Every output element sums its nine taps' terms in the same order on all three paths, so no
reference computation is needed for the outputs: the schedules (TAPIR_B200_GEMM_SCHEDULE) and the
generic path (TAPIR_B200_CONV_HALO=0), switches read on every call, run into NaN-filled buffers and
must match bit for bit, padding included.  The statistics are fp64 atomic sums whose order varies,
so across paths and against an fp64 sum of the output they are compared to rounding; on operands
whose every sum is exact (tests/gemm_exact.py 'S' designs) they must equal that sum exactly."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests import gemm_exact as E  # noqa: E402
from tests import gpu_util as U  # noqa: E402

SCHEDULE = 'TAPIR_B200_GEMM_SCHEDULE'
HALO = 'TAPIR_B200_CONV_HALO'

# (frames, H, W, P): 128 x 128 is the first ResNet group of a 256 x 256 clip; the others have partial
# tiles (W not a multiple of 8, H not a multiple of 16, W below 8); f40_33x13 has many small
# frames (6 tiles each), so consecutive tiles of a CTA and of each warpgroup change frame.
SHAPES = {
    'f1_128': (1, 128, 128, 2),
    'f2_128': (2, 128, 128, 2),
    'f3_128': (3, 128, 128, 1),
    'f48_128': (48, 128, 128, 2),
    'f2_33x13': (2, 33, 13, 2),
    'f3_37x45': (3, 37, 45, 1),
    'f5_7x5': (5, 7, 5, 2),
    'f40_33x13': (40, 33, 13, 2),
}
OPTIONS = {'plain': (False, False), 'resid': (True, False), 'stats': (False, True),
           'resid_stats': (True, True)}


def _problem(name):
  Fr, H, W, P = SHAPES[name]
  g = torch.Generator(device='cuda').manual_seed(sum(map(ord, name)))
  a_pl = U.split(torch.randn(Fr * H * W, 64, generator=g, device='cuda'), P).reshape(P, Fr, H, W, 64)
  w_pl = U.split(torch.randn(64, 576, generator=g, device='cuda') / 24.0, P)
  r = torch.randn(Fr * H * W, 64, generator=g, device='cuda')
  return a_pl, w_pl, r


def _run(name, opt, schedule=None, halo=1):
  """One case on the halo kernel (halo=1) under `schedule` (None: the dispatcher's choice), or on
  the generic implicit GEMM (halo=0)."""
  Fr, H, W, _ = SHAPES[name]
  resid, stats = OPTIONS[opt]
  a_pl, w_pl, r = _problem(name)
  st = torch.zeros(Fr, 64, 2, dtype=torch.float64, device='cuda') if stats else None
  with U.switches(**{SCHEDULE: schedule, HALO: halo}):
    res = U.gemm(a_pl, w_pl, None, r if resid else None, conv=(Fr, H, W, 64), stats=st, details=True)
  assert res.launches == 1
  assert U.untouched_padding(res), (name, opt, schedule, halo)
  return res, st


def _stats_close(got, want, what):
  torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-9 * want.abs().max().item(), msg=what)


@pytest.mark.parametrize('name', sorted(SHAPES))
def test_halo_schedules_and_generic_conv_agree_bit_for_bit(name):
  Fr = SHAPES[name][0]
  for opt, (_, stats) in OPTIONS.items():
    coop, st_c = _run(name, opt, 'coop')
    pp, st_p = _run(name, opt, 'pingpong')
    gen, st_g = _run(name, opt, halo=0)
    what = f'{name}/{opt}'
    assert torch.equal(coop.out_buf.view(torch.int32), pp.out_buf.view(torch.int32)), what
    assert torch.equal(gen.out_buf.view(torch.int32), pp.out_buf.view(torch.int32)), \
        f'{what}: halo != generic implicit GEMM'
    if stats:
      # the two halo schedules share their fp32 partials (same 16-row groups): fp64 order only
      _stats_close(st_p, st_c, what)
      out = pp.out.double().reshape(Fr, -1, 64)
      want = torch.stack([out.sum(1), (out * out).sum(1)], -1)
      # fp32 sums over a warp's 16 rows, then fp64: rounding of the fp32 partials only.  The
      # generic path's warps hold other 16-pixel groups, so it is held to the same bound.
      for got in (st_p, st_g):
        rel = ((got - want).abs() / want.abs().clamp(min=1.0)).max().item()
        assert rel < 5e-5, (what, rel)


@pytest.mark.parametrize('schedule', ['coop', 'pingpong'])
@pytest.mark.parametrize('conv', [(16, 64, 64, 64), (3, 33, 13, 64)])
def test_halo_stats_are_exact_sums_on_exact_operands(conv, schedule):
  """Integer outputs below 1000: every fp32 and fp64 sum is exact, whatever its order.  16 frames
  of 64 x 64: 512 tiles, 3-4 per CTA, so each ping-pong warpgroup runs more than one."""
  case = E.Case(f'halo_pp_{conv[0]}x{conv[1]}x{conv[2]}', 'S', None, 64, None, 2, E.S_SETS, conv=conv)
  d = case.design()
  Fr = conv[0]
  for resid in (False, True):
    st = torch.zeros(Fr, 64, 2, dtype=torch.float64, device='cuda')
    with U.switches(**{SCHEDULE: schedule, HALO: 1}):
      o, _ = U.gemm(d.a_pl.cuda(), d.w_pl.cuda(), None, d.resid.cuda() if resid else None, conv=conv, stats=st)
    want = E.emulate(d, False, resid, 0, True)
    assert np.array_equal(o.cpu().numpy(), want['out']), (conv, schedule, resid)
    out = o.double().cpu().reshape(Fr, -1, 64)
    own = torch.stack([out.sum(1), (out * out).sum(1)], -1)
    assert torch.equal(st.cpu(), own), (conv, schedule, resid)
    assert np.array_equal(st.cpu().numpy(), want['stats']), (conv, schedule, resid)


def test_halo_dispatch_and_forced_schedules():
  # 48 frames: 6144 tiles, many per CTA -> ping-pong; one frame: 128 tiles -> cooperative
  want = {('f48_128', None): True, ('f1_128', None): False,
          ('f48_128', 'coop'): False, ('f1_128', 'pingpong'): True}
  with U.switches(TAPIR_B200_BLOCK_N=None):
    for (name, schedule), pingpong in want.items():
      names = set(U.kernels(lambda: _run(name, 'plain', schedule), 'conv3x3_halo'))
      assert len(names) == 1, (name, schedule, names)
      assert ('pingpong' in next(iter(names))) == pingpong, (name, schedule, names)


def test_halo_switch_takes_effect_on_every_call():
  """TAPIR_B200_CONV_HALO is read on every call: off, on and off again in one process (each run is
  one launch)."""
  for halo in (0, 1, 0):
    names = set(U.kernels(lambda: _run('f1_128', 'plain', halo=halo), 'conv3x3_halo'))
    assert len(names) == halo, (halo, names)


def test_halo_schedule_switch_rejects_unknown_values():
  with pytest.raises(Exception, match=SCHEDULE):
    _run('f5_7x5', 'plain', 'ping-pong')
