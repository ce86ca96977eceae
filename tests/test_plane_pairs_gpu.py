"""The plane pairs each GEMM kernel sums, bit for bit, on the designs of tests/plane_pairs.py.

Every tensor-core kernel must return the fp32 model of the pairs i + j < P, and the SIMT kernel
the model of all P^2 pairs, on operands whose planes are independent integer tensors: every plane
pair then contributes its own term, and the models are exact.  A's planes sit in a NaN-filled
buffer with gaps between planes and past each row's K columns, and every output buffer is
NaN-filled outside its [M, N] view and must stay so.  When an output differs, the test names the
wrong pair set of plane_pairs.wrong_sets that reproduces it, if one does.

Runs: the plain GEMM under the cooperative schedule (P = 1, 2, 3) and the ping-pong one (P = 1, 2)
at BLOCK_N 64 and 128; the generic 3 x 3 convolution (TAPIR_B200_CONV_HALO=0, P = 1, 2, 3, C = 64
and 128); the halo convolution under both schedules (P = 1, 2, C = 64); split-K (P = 2, 3, K >=
2048, the partial-sum kernel then splitk_reduce_kernel); the SIMT kernel (P = 1, 2, 3); one run per
kernel with three bf16 output planes.  Last, the stage-A cost volume, the one batched and the one
grouped P = 3 GEMM, through tapir_cost_volume_tracks_batched and tapir_cost_volume_tracks_ragged
(tensor cores and SIMT): its designed maps must pick the cells plane_pairs.CvDesign emulates."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tapnet_b200 import _lib  # noqa: E402
from tests import gpu_util as U  # noqa: E402
from tests import plane_pairs as PP  # noqa: E402
from tests.test_stage_a_gpu import _head_weights  # noqa: E402


def _dev(d):
  if not hasattr(d, 'dev'):
    d.dev = dict(a=PP.gapped_a(d.a_pl, d.conv), w=d.w_pl.cuda())
  return d.dev


def _run(d, impl=0, env=None, splitk=False, out_planes=0):
  t = _dev(d)
  ws = None
  if splitk:
    ws = torch.empty(8 * d.M * ((d.N + 7) // 8 * 8), dtype=torch.float32, device='cuda')
  a_buf, a = t['a']
  with U.switches(**(env or {})):
    res = U.gemm(a, t['w'], out_planes=out_planes, impl=impl, conv=d.conv, splitk_ws=ws, details=True)
  assert U.untouched_padding(res), 'wrote outside the [M, N] output'
  assert torch.isnan(a_buf.float()).sum() == a_buf.numel() - a.numel(), 'A was written'
  return res


def _check(label, d, res, simt=False, out_planes=0):
  pairs = PP.all_pairs(d.P) if simt else PP.tc_pairs(d.P)
  want = d.model(pairs)
  got = res.out.cpu().numpy()
  bad = PP.fp32_bits(got) != PP.fp32_bits(want)
  if bad.any():
    nan = int(np.isnan(got).sum())
    same = PP.matching_sets(got, d, PP.wrong_sets(d.P, simt=simt))
    pytest.fail(f'{label}: {int(bad.sum())} of {bad.size} outputs differ from the {"all" if simt else "i + j < P"} '
                f'pair model ({nan} NaN); the output is that of: {same or "no listed wrong set"}')
  if out_planes:
    planes = U.split_like_kernel(torch.from_numpy(want.numpy().astype(np.float32)), out_planes)
    pb = res.planes.cpu().contiguous().view(torch.int16) != planes.view(torch.int16)
    assert not pb.any(), f'{label}: {int(pb.sum())} bf16 output plane elements differ'


def _env(bn=None, sched=None, halo=None):
  env = {}
  if bn is not None:
    env['TAPIR_B200_BLOCK_N'] = bn
  if sched is not None:
    env['TAPIR_B200_GEMM_SCHEDULE'] = sched
  if halo is not None:
    env['TAPIR_B200_CONV_HALO'] = halo
  return env


# ------------------------------------------------------------------------------ plain
@pytest.mark.parametrize('bn', [64, 128])
@pytest.mark.parametrize('P', [1, 2, 3])
def test_plain_cooperative(P, bn):
  names = [f'small_p{P}', f'multi_p{P}'] + (['longk_p3'] if P == 3 else [])
  for name in names:
    d = PP.design(name)
    _check(f'{name}_bn{bn}_coop', d, _run(d, env=_env(bn, 'coop')))


@pytest.mark.parametrize('bn', [64, 128])
@pytest.mark.parametrize('P', [1, 2])
def test_plain_pingpong(P, bn):
  for name in (f'small_p{P}', f'multi_p{P}'):
    d = PP.design(name)
    _check(f'{name}_bn{bn}_pingpong', d, _run(d, env=_env(bn, 'pingpong')))


# ------------------------------------------------------------------------------ convolutions
@pytest.mark.parametrize('C', [64, 128])
@pytest.mark.parametrize('P', [1, 2, 3])
def test_conv_generic(P, C):
  d = PP.design(f'conv{C}_p{P}')
  for bn in (64, 128):
    _check(f'{d.name}_bn{bn}_generic', d, _run(d, env=_env(bn, halo=0)))


@pytest.mark.parametrize('sched', ['coop', 'pingpong'])
@pytest.mark.parametrize('P', [1, 2])
def test_conv_halo(P, sched):
  for name in (f'conv64_p{P}', f'conv64_multi_p{P}'):
    d = PP.design(name)
    _check(f'{name}_halo_{sched}', d, _run(d, env=_env(sched=sched, halo=1)))


# ------------------------------------------------------------------------------ split-K
@pytest.mark.parametrize('name', ['splitk_p2', 'splitk_p3', 'longk_p3'])
def test_splitk(name):
  d = PP.design(name)
  res = _run(d, splitk=True)
  assert res.launches == 2, f'{name}: K was not split ({res.launches} launches)'
  _check(f'{name}_splitk', d, res)


# ------------------------------------------------------------------------------ SIMT
@pytest.mark.parametrize('P', [1, 2, 3])
def test_simt_sums_all_pairs(P):
  for name in (f'small_p{P}', f'conv64_p{P}', f'conv128_p{P}'):
    d = PP.design(name)
    _check(f'{name}_simt', d, _run(d, impl=1), simt=True)


# ------------------------------------------------------------------------------ plane outputs
PLANE_RUNS = {  # kernel -> (design, impl, env, split-K)
    'coop': ('small_p3', 0, _env(128, 'coop'), False),
    'pingpong': ('multi_p2', 0, _env(64, 'pingpong'), False),
    'conv_generic': ('conv128_p2', 0, _env(halo=0), False),
    'splitk': ('splitk_p3', 0, {}, True),
    'simt': ('small_p2', 1, {}, False),
}


@pytest.mark.parametrize('kernel', sorted(PLANE_RUNS))
def test_plane_output(kernel):
  """fp32 and three bf16 planes out: the planes are the split of the exact accumulator."""
  name, impl, env, splitk = PLANE_RUNS[kernel]
  d = PP.design(name)
  res = _run(d, impl, env, splitk, out_planes=3)
  _check(f'{name}_{kernel}_planes', d, res, simt=impl == 1, out_planes=3)


# ------------------------------------------------------------------------------ kernels reached
REACH = [  # (design, impl, env, split-K, the kernel the run must reach)
    ('small_p3', 0, _env(64, 'coop'), False, 'gemm_tc_kernel<64, 3>'),
    ('small_p2', 0, _env(128, 'pingpong'), False, 'gemm_tc_pingpong_kernel<128, 2>'),
    ('conv128_p3', 0, _env(128, halo=0), False, 'gemm_tc_kernel<128, 3>'),
    ('conv64_p2', 0, _env(sched='coop', halo=1), False, 'conv3x3_halo_kernel<2>'),
    ('conv64_p1', 0, _env(sched='pingpong', halo=1), False, 'conv3x3_halo_pingpong_kernel<1>'),
    ('splitk_p3', 0, {}, True, 'splitk_reduce_kernel'),
    ('small_p1', 1, {}, False, 'gemm_simt_kernel'),
]


def test_switches_reach_the_kernels_under_test():
  """The switches the runs above set select the kernels they test.  One profiler session for all:
  the other tests run without it."""
  names = set(U.kernels(lambda: [_run(PP.design(n), impl, env, sk) for n, impl, env, sk, _ in REACH], ''))
  bare = [n.replace(' ', '') for n in names]
  missing = [k for *_, k in REACH if not any(k.replace(' ', '') in n for n in bare)]
  assert not missing, (missing, sorted(names))


# ------------------------------------------------------------------------------ cost volume
COUNTS_64 = [(1, 63, 64, 65, 129)[b % 5] for b in range(64)]  # one grouped call of 64 clips
# id: (entry, counts, T, gh, gw).  Batched: N = 40 queries per clip, so an m-tile reads the next
# clip's rows; 2925 cells (25 x 39 x 3) are no multiple of either tile width.  Ragged: counts around
# the 128-row m-tile (a clip's last tile holds 1, 40, 127, 0 or 1 rows), a one-query clip between
# two of more than 128, and 64 clips, at T = 1 and 3 on the tensor-core head's 32 x 32 maps and the
# generic head's 25 x 39.
CV_CASES = {'32x32': ('batched', [40] * 2, 2, 32, 32), '25x39': ('batched', [40] * 2, 3, 25, 39)}
for _name, _counts in (('5', [1, 40, 127, 128, 129]), ('3', [200, 1, 129]), ('64', COUNTS_64)):
  for _T in (1, 3):
    for _gh, _gw in ((32, 32), (25, 39)):
      CV_CASES[f'ragged{_name}_T{_T}_{_gh}x{_gw}'] = ('ragged', _counts, _T, _gh, _gw)
_DESIGNS_CV = {}


def _cv_design(case):
  if case not in _DESIGNS_CV:
    _DESIGNS_CV[case] = PP.CvDesign(*CV_CASES[case][1:])
  return _DESIGNS_CV[case]


def _run_cost_volume(cv, entry, gemm, bn=None):
  """One stage-A call on the design's maps with the identity head at temperature 1 (the heat is
  the map, exactly); every output between NaN guards.  The workspace has one m-tile of cost-volume
  rows (128 T gh gw floats) past what the call asks for, filled with a sentinel that must survive:
  for 32 x 32 maps cv is the workspace's last buffer, so a store of the rows of the last clip's last
  m-tile past its count lands there (other maps: past the generic head's scratch, which follows
  cv).  It does not see such stores for inner clips, whose extra rows land on the next clip's rows;
  there the designs and the repeated queries n >= 64 may see them."""
  B, T, gh, gw, Q = cv.B, cv.T, cv.gh, cv.gw, cv.Q
  qf, grid = cv.qf.cuda(), cv.grid.cuda()
  outs = {k: U.guarded(Q * T * (2 if k == 'pts' else 1), torch.int32 if k == 'am' else torch.float32)
          for k in ('pts', 'occ', 'expd', 'am')}
  if entry == 'batched':
    N = cv.counts[0]
    assert cv.counts == [N] * B
    need = _lib.cost_volume_workspace_bytes((B, N), grid.shape)
    view = lambda k: outs[k][1].view((B, N, T, 2) if k == 'pts' else (B, N, T))  # noqa: E731
  else:
    need = _lib.cost_volume_ragged_workspace_bytes(B, Q, grid.shape)
    view = lambda k: outs[k][1].view((Q, T, 2) if k == 'pts' else (Q, T))  # noqa: E731
  tail = 128 * T * gh * gw * 4
  ws = torch.full((need + tail,), 0xA5, dtype=torch.uint8, device='cuda')
  with U.switches(TAPIR_B200_GEMM=gemm, TAPIR_B200_BLOCK_N=bn):
    if entry == 'batched':
      _lib.cost_volume_tracks(_head_weights('identity'), qf.view(B, N, -1), grid, None, 1.0,
                              (gh * 8, gw * 8), view('pts'), view('occ'), view('expd'), view('am'), ws)
    else:
      _lib.cost_volume_tracks_ragged(_head_weights('identity'), qf, cv.counts, grid, None, 1.0,
                                     (gh * 8, gw * 8), view('pts'), view('occ'), view('expd'),
                                     view('am'), ws)
  torch.cuda.synchronize()
  for k, (buf, body) in outs.items():
    assert U.guards_intact(buf), f'{k}: wrote outside the output'
    assert not (body.isnan().any() if body.is_floating_point() else (body == -7).any()), f'{k}: not written'
  changed = int((ws[need:] != 0xA5).sum())
  assert changed == 0, f'{changed} workspace bytes past the cost-volume arena were written'
  return {k: outs[k][1].cpu().view((Q, T, 2) if k == 'pts' else (Q, T)) for k in outs}


def _check_cost_volume(cv, got, simt):
  """The arg-max cells are the design's winners, and each query n >= 64 of a clip repeats every
  output of query n mod 64 bit for bit."""
  for k, x in got.items():
    same = x.view(torch.int32)[cv.rank >= PP.CV_GROUPS]
    src = x.view(torch.int32)[(torch.arange(cv.Q) - cv.rank + cv.group)[cv.rank >= PP.CV_GROUPS]]
    assert torch.equal(same, src), f'{k}: a query n >= 64 differs from query n mod 64'
  am, want = got['am'].long(), cv.winner()
  heat = cv.heat_simt() if simt else cv.heat(PP.tc_pairs(3))
  assert torch.equal(PP.CvDesign.argmax(heat), want)
  bad = am != want
  if bad.any():
    same = [] if simt else [name for name, pairs in PP.wrong_sets(3).items()
                            if torch.equal(PP.CvDesign.argmax(cv.heat(pairs)), am)]
    kinds = sorted({PP.CV_KINDS[k] for k in cv.kind[bad].tolist()})
    clips = sorted(set(cv.clip[bad.any(-1)].tolist()))
    pytest.fail(f'{int(bad.sum())} of {bad.numel()} arg-max cells differ (kinds {kinds}, clips '
                f'{clips[:16]}); they are those of: {same or "no listed wrong set"}')


@pytest.mark.parametrize('bn', [64, 128])
@pytest.mark.parametrize('case', list(CV_CASES))
def test_cost_volume_pairs(case, bn):
  """The stage-A cost volume, the one batched and the one grouped P = 3 GEMM, through
  tapir_cost_volume_tracks_batched or tapir_cost_volume_tracks_ragged."""
  cv = _cv_design(case)
  _check_cost_volume(cv, _run_cost_volume(cv, CV_CASES[case][0], 'tc', bn), simt=False)


@pytest.mark.parametrize('case', [c for c in CV_CASES if c.endswith('32x32')])
def test_cost_volume_pairs_simt(case):
  """The SIMT kernel's batched and grouped modes (blockIdx.z the clip): its all-pairs sum with
  rounded products keeps every designed winner (tests/test_plane_pairs_host.py)."""
  cv = _cv_design(case)
  _check_cost_volume(cv, _run_cost_volume(cv, CV_CASES[case][0], 'simt'), simt=True)
