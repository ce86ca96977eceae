"""The ping-pong and cooperative wgmma GEMM schedules give bit-identical outputs, and the dispatcher
picks ping-pong for the offline clip's long GEMMs and the cooperative kernel for its short mixer
linears and for the streaming ones.  Batched GEMMs always run the cooperative kernel (the only one
is the P = 3 cost volume), so there is no batched case here.

Both schedules sum every output element's K terms in the same order, so no reference computation
is needed: each case runs once per schedule (TAPIR_B200_GEMM_SCHEDULE, read on every call) into
NaN-filled buffers and the two results must match bit for bit, guard elements included.  Fused
InstanceNorm statistics are fp64 atomic sums whose order varies between runs, so they are compared
to fp64 rounding.  Last, every switch rejects a value outside its set, on every call."""
import zlib

import pytest
import torch

pytestmark = pytest.mark.gpu

from tapnet_b200 import _lib  # noqa: E402
from tests import gpu_util as U  # noqa: E402

SCHEDULE = 'TAPIR_B200_GEMM_SCHEDULE'


def _sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


def _problem(seed, M, N, K, P, conv=None, bias=False, resid=False):
  g = torch.Generator(device='cuda').manual_seed(seed)
  if conv is None:
    a_pl = U.split(torch.randn(M, K, generator=g, device='cuda'), P)
  else:
    f, h, w, c = conv
    M = f * h * w
    a_pl = U.split(torch.randn(M, c, generator=g, device='cuda'), P).reshape(P, f, h, w, c)
  w_pl = U.split(torch.randn(N, K, generator=g, device='cuda') / K ** 0.5, P)
  b = torch.randn(N, generator=g, device='cuda') if bias else None
  r = torch.randn(M, N, generator=g, device='cuda') if resid else None
  return a_pl, w_pl, b, r


def _run(schedule, a_pl, w_pl, stats_shape=None, **kw):
  stats = torch.zeros(stats_shape, dtype=torch.float64, device='cuda') if stats_shape else None
  with U.switches(**{SCHEDULE: schedule}):
    res = U.gemm(a_pl, w_pl, stats=stats, details=True, **kw)
  assert res.launches == 1
  return res, stats


def _same_bits(x, y):
  if x is None:
    return y is None
  bits = torch.int16 if x.element_size() == 2 else torch.int32
  return torch.equal(x.view(bits), y.view(bits))


def _compare(name, M, N, K, P=2, conv=None, bias=False, resid=False, gelu=False, out_f32=True,
             out_planes=0, ld_pad=0, stats=False, rows_per_frame=0):
  a_pl, w_pl, b, r = _problem(zlib.crc32(name.encode()), M, N, K, P, conv, bias, resid)
  frames = conv[0] if conv else (M // rows_per_frame if rows_per_frame else 1)
  kw = dict(bias=b, residual=r, gelu=gelu, out_f32=out_f32, out_planes=out_planes, ld_pad=ld_pad,
            conv=conv, rows_per_frame=rows_per_frame)
  st_shape = (frames, N, 2) if stats else None
  coop, st_c = _run('coop', a_pl, w_pl, st_shape, **kw)
  pp, st_p = _run('pingpong', a_pl, w_pl, st_shape, **kw)
  assert _same_bits(coop.out_buf, pp.out_buf), name
  assert _same_bits(coop.planes_buf, pp.planes_buf), name
  assert U.untouched_padding(pp), name
  out = pp.out if pp.out is not None else pp.planes[0]
  assert torch.isfinite(out).all(), name
  if stats:
    torch.testing.assert_close(st_p, st_c, rtol=1e-12, atol=1e-9 * st_c.abs().max().item(), msg=name)


# every GEMM of the offline clip step (48 frames of 256 x 256, 256 queries): the mixer at 12288 rows,
# the extra convolutions at 48 x 32 x 32, the ResNet groups 1-3 (3x3 convolutions with fused
# InstanceNorm statistics, and the 1x1 projections)
STEP = {
    'mixer.linear_in': dict(M=12288, N=512, K=576, bias=True, out_planes=2),
    'mixer.up': dict(M=12288, N=2048, K=512, bias=True, gelu=True, out_f32=False, out_planes=2),
    'mixer.down': dict(M=12288, N=512, K=2048, bias=True, resid=True),
    'mixer.linear_out': dict(M=12288, N=388, K=512, bias=True),
    'extra_conv.up': dict(M=0, N=1024, K=9 * 256, conv=(48, 32, 32, 256), bias=True, gelu=True,
                          out_f32=False, out_planes=2),
    'extra_conv.down': dict(M=0, N=256, K=9 * 1024, conv=(48, 32, 32, 1024), bias=True, resid=True),
    'resnet.g1.conv_0': dict(M=0, N=128, K=9 * 64, conv=(48, 64, 64, 64), stats=True),
    'resnet.g1.conv': dict(M=0, N=128, K=9 * 128, conv=(48, 64, 64, 128), stats=True),
    'resnet.g1.proj': dict(M=48 * 64 * 64, N=128, K=64),
    'resnet.g2.conv_0': dict(M=0, N=256, K=9 * 128, conv=(48, 32, 32, 128), stats=True),
    'resnet.g2.conv': dict(M=0, N=256, K=9 * 256, conv=(48, 32, 32, 256), stats=True),
    'resnet.g2.proj': dict(M=48 * 32 * 32, N=256, K=128),
    'resnet.g3.proj': dict(M=48 * 32 * 32, N=256, K=256),
}


@pytest.mark.parametrize('name', sorted(STEP))
def test_tc_schedules_agree_on_step_gemms(name):
  _compare(name, **STEP[name])


EDGES = {
    'ragged_m_odd_n': dict(M=40000, N=257, K=192, bias=True, gelu=True, out_planes=2),
    'ld_pad_resid': dict(M=33000, N=300, K=128, bias=True, resid=True, ld_pad=5, out_planes=1),
    'p1_planes1': dict(M=34000, N=2048, K=256, P=1, bias=True, gelu=True, out_f32=False, out_planes=1),
    'p1_n64': dict(M=70000, N=64, K=320, P=1, bias=True),
    'n64_planes2': dict(M=70000, N=64, K=128, bias=True, resid=True, out_planes=2),
    'plain_stats': dict(M=48 * 1024, N=192, K=256, stats=True, rows_per_frame=1024),
    'conv_ragged_w': dict(M=0, N=320, K=9 * 128, conv=(5, 37, 45, 128), bias=True, gelu=True,
                          out_planes=2),
    'conv_ragged_stats': dict(M=0, N=128, K=9 * 64, conv=(7, 21, 50, 64), stats=True),
    'few_tiles': dict(M=1000, N=200, K=128, bias=True, out_planes=2),
}


@pytest.mark.parametrize('name', sorted(EDGES))
def test_tc_schedules_agree_on_edge_cases(name):
  _compare(name, **EDGES[name])


@pytest.mark.parametrize('per_cta', ['2', '2+1', '3'])
def test_tc_schedules_agree_at_tile_counts(per_cta):
  """Exactly two tiles per CTA, one CTA with a third, and an odd count everywhere (the second
  consumer warpgroup has one tile fewer and idles at the end)."""
  sms = _sms()
  tiles = {'2': 2 * sms, '2+1': 2 * sms + 1, '3': 3 * sms}[per_cta]
  _compare(f'tiles_{per_cta}', M=tiles * 128 - 3, N=128, K=256, bias=True, gelu=True, out_planes=2)


def _kernels(fn):
  return set(U.kernels(fn, 'gemm_tc'))


def test_tc_dispatch_picks_pingpong_for_long_clip_gemms_and_coop_otherwise():
  """The dispatcher's own choice: no schedule or tile width forced, the halo path allowed."""
  with U.switches(TAPIR_B200_GEMM_SCHEDULE=None, TAPIR_B200_BLOCK_N=None, TAPIR_B200_CONV_HALO=1):
    ws = torch.empty(64 << 20, dtype=torch.uint8, device='cuda')
    clip = ['mixer.up', 'mixer.down', 'extra_conv.up', 'resnet.g2.conv']
    stream = {  # one frame per step, 1024 points: the split-K and small-problem paths
        'mixer.up': dict(M=1024, N=2048, K=512, bias=True, gelu=True, out_f32=False, out_planes=2),
        'mixer.down': dict(M=1024, N=512, K=2048, bias=True, resid=True, splitk_ws=ws),
        'extra_conv.up': dict(M=0, N=1024, K=9 * 256, conv=(1, 32, 32, 256), bias=True, gelu=True,
                              out_f32=False, out_planes=2),
    }
    for name in clip + ['mixer.linear_in', 'mixer.linear_out']:
      c = dict(STEP[name])
      a_pl, w_pl, b, r = _problem(1, c.pop('M'), c.pop('N'), c.pop('K'), 2, c.get('conv'),
                                  c.pop('bias', False), c.pop('resid', False))
      c.pop('stats', None)
      names = _kernels(lambda: U.gemm(a_pl, w_pl, bias=b, residual=r, **c))
      if name in clip:
        assert names and all('pingpong' in n for n in names), (name, names)
      else:  # under four tiles per CTA of short mainloops ping-pong is slower
        assert names and not any('pingpong' in n for n in names), (name, names)
    for name, c in stream.items():
      c = dict(c)
      a_pl, w_pl, b, r = _problem(2, c.pop('M'), c.pop('N'), c.pop('K'), 2, c.get('conv'),
                                  c.pop('bias', False), c.pop('resid', False))
      names = _kernels(lambda: U.gemm(a_pl, w_pl, bias=b, residual=r, **c))
      assert names and not any('pingpong' in n for n in names), (name, names)


def test_tc_schedule_switch_rejects_unknown_values():
  """Also on a split-K GEMM, which always runs the cooperative kernel and so never uses the switch."""
  a_pl, w_pl, _, _ = _problem(3, 256, 128, 128, 2)
  with pytest.raises(Exception, match=SCHEDULE):
    _run('ping-pong', a_pl, w_pl)
  a_pl, w_pl, _, _ = _problem(4, 1000, 512, 2048, 2)
  ws = torch.empty(64 << 20, dtype=torch.uint8, device='cuda')
  with pytest.raises(Exception, match=SCHEDULE):
    _run('ping-pong', a_pl, w_pl, splitk_ws=ws)


# a value outside each switch's set; the empty string is rejected as well
BAD_VALUES = {'TAPIR_B200_GEMM': 'wgmma', 'TAPIR_B200_BLOCK_N': '96',
              'TAPIR_B200_GEMM_SCHEDULE': 'ping-pong', 'TAPIR_B200_CONV_HALO': 'yes'}


@pytest.mark.parametrize('value', ['bad', 'empty'])
@pytest.mark.parametrize('switch', sorted(BAD_VALUES))
def test_tc_switches_reject_values_outside_their_set(switch, value):
  """Every GEMM call reads all four switches, whether it uses them or not, and fails before any
  launch on a value outside a switch's set.  The cost volume reaches the GEMM through gemm()."""
  a_pl, w_pl, _, _ = _problem(3, 256, 128, 128, 2)
  with U.switches(**{switch: BAD_VALUES[switch] if value == 'bad' else ''}):
    torch.cuda.synchronize()
    before = U.launch_count()
    with pytest.raises(_lib.TapirB200Error, match=switch):
      U.gemm(a_pl, w_pl)
    assert U.launch_count() == before
    if value == 'bad':
      from tests.test_stage_a_gpu import _head_weights  # pylint: disable=g-import-not-at-top
      G, n, T = 1, 8, 2
      qf = torch.randn(G, n, 256, device='cuda')
      grid = torch.randn(G, T, 32, 32, 256, device='cuda')
      pts = torch.empty(G, n, T, 2, device='cuda')
      occ, expd = torch.empty(G, n, T, device='cuda'), torch.empty(G, n, T, device='cuda')
      ws = torch.empty(_lib.cost_volume_workspace_bytes(qf, grid), dtype=torch.uint8, device='cuda')
      with pytest.raises(_lib.TapirB200Error, match=switch):
        _lib.cost_volume_tracks(_head_weights('synth'), qf, grid, None, 20.0, (256, 256), pts, occ,
                                expd, None, ws)
