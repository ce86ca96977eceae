"""windowed.track_video on the GPU: the windows it yields, concatenated, equal model(video, queries)
bit for bit for every reader format; the reader is asked for each frame once, one window ahead,
and its results are let go; memory does not grow with the video's length; bad frames raise."""
import weakref

import pytest
import torch

pytestmark = pytest.mark.gpu

from tapnet_b200 import live, tapir_model, windowed  # noqa: E402
from tests.test_stages_gpu import get_model  # noqa: E402
from tests.test_windowed_gpu import _assert_equal, _queries, _video, _whole  # noqa: E402
from tests.test_yuv_gpu import make_frames  # noqa: E402

_KEYS = ('occlusion', 'tracks', 'expected_dist')


def _reader(clip, kind='device', log=None):
  """read_frames over a one-clip video [1, T, H, W, 3] on the device, returning `kind` frames:
  'pinned' / 'pageable' host uint8, 'device' (the clip's own dtype), 'float' (device float32 in
  [-1, 1] made from uint8)."""
  def read(a, z):
    if log is not None:
      log.append(('read', a, z))
    x = clip[0, a:z]
    if kind == 'pinned':
      return x.cpu().pin_memory()
    if kind == 'pageable':
      return x.cpu()
    if kind == 'float':
      return x.float() / 127.5 - 1
    return x.clone()
  return read


def _yuv_reader(clip, log=None):
  def read(a, z):
    if log is not None:
      log.append(('read', a, z))
    return live.YUV420Frames(clip.y[:, a:z], clip.u[:, a:z], clip.v[:, a:z], clip.matrix,
                             clip.full_range, clip.window)
  return read


def _collect(model, read, T, q, log=None, **kw):
  """The yields of track_video concatenated along the frame axis."""
  parts, covered = [], 0
  for start, stop, out in windowed.track_video(model, read, T, q, **kw):
    assert start == covered and stop > start
    covered = stop
    if log is not None:
      log.append(('yield', start, stop))
    parts.append(out)
  assert covered == T
  got = {k: torch.cat([p[k] for p in parts], dim=2) for k in parts[0] if k in _KEYS}
  for k in parts[0]:
    if k not in _KEYS:
      got[k] = [torch.cat([p[k][i] for p in parts], dim=2) for i in range(len(parts[0][k]))]
  return got


def _check(model, video, q, read=None, unrefined=False, want=None, **kw):
  want = _whole(model, video, q) if want is None else want
  if not unrefined:
    want = {k: want[k] for k in _KEYS}
  got = _collect(model, read or _reader(video), video.shape[1], q, unrefined=unrefined, **kw)
  _assert_equal(got, want)
  return want


_T256 = 300
_TIMES256 = [0, _T256 - 1, 31, 32, 99, 100, 64, 95, 96, 97, 131, 196, 204, 12.5, 150.49, 150.5,
             200.7, 33.3, 299.4, 0.49, 250, 275]


@pytest.fixture(scope='module')
def clip256():
  return _video(_T256, 256, 256), _queries(_TIMES256, 256, 256)


@pytest.mark.parametrize('pyramid_level', [0, 1])
def test_matches_whole_clip_256(clip256, pyramid_level):
  model = get_model(pyramid_level=pyramid_level)[0]
  video, q = clip256
  want = _check(model, video, q, window_frames=32, unrefined=True)
  _check(model, video, q, window_frames=100, want=want)
  # queries as [N, 3], on the host
  _check(model, video, q[0].cpu(), window_frames=100, want=want)


def test_matches_windowed_forward(clip256):
  model = get_model()[0]
  video, q = clip256
  want = windowed.windowed_forward(model, video, q, window_frames=64)
  _check(model, video, q, window_frames=64, unrefined=True, want=want)


def test_automatic_core(clip256):
  model = get_model()[0]
  video, q = clip256
  _check(model, video, q)


def test_causal(clip256):
  model = get_model(causal=True)[0]
  video, q = clip256
  _check(model, video, q, window_frames=64, unrefined=True)


def test_two_levels_512():
  model = get_model()[0]
  T = 400
  video = _video(T, 512, 512, seed=3)
  q = _queries([0, T - 1, 100, 101, 288, 300.5, 350.25, 399.2] + list(range(5, T, 40)), 512, 512)
  _check(model, video, q, window_frames=120, unrefined=True)  # 4 windows, the last one short


def test_non_square_resampled_and_direct_pass():
  model = get_model()[0]
  plan = tapir_model._pass_plan((256, 384), model.initial_resolution)
  assert [st.direct for st in plan if st.new] == [False, True]
  T = 97  # the last frame runs alone in the whole clip's 256 x 256 pass
  video = _video(T, 256, 384, seed=19)
  q = _queries([0, 96, 40, 41, 12.5, 80, 95.5], 256, 384)
  _check(model, video, q, window_frames=40, unrefined=True)


# C = 1 (every slide adds one frame, the ring wraps on every window), C not dividing T, and T = 97,
# whose last frame the whole-clip call runs alone through the 256 x 256 pass
@pytest.mark.parametrize('T, C, causal', [(97, 1, False), (97, 1, True), (97, 40, False),
                                          (129, 32, False)])
def test_one_frame_calls(T, C, causal):
  model = get_model(causal=causal)[0]
  video = _video(T, 256, 256, seed=11)
  q = _queries([0, T - 1, T - 2, 1, T // 2, 30.5, C, C - 1, T - 1.4], 256, 256)
  _check(model, video, q, window_frames=C)


@pytest.mark.parametrize('T', [97, 98])
def test_queries_on_the_last_frame(T):
  model = get_model()[0]
  video = _video(T, 256, 256, seed=13)
  _check(model, video, _queries([T - 1] * 6, 256, 256), window_frames=40)


@pytest.mark.parametrize('kind', ['pinned', 'pageable', 'device', 'float'])
def test_reader_formats(kind):
  model = get_model()[0]
  T = 150
  video = _video(T, 256, 256, seed=21)
  q = _queries([0, 149, 60, 61.5, 100, 3.25], 256, 256)
  clip = video.float() / 127.5 - 1 if kind == 'float' else video
  _check(model, clip, q, read=_reader(video, kind), window_frames=48)


@pytest.mark.parametrize('layout', ['nv12', 'i420'])
def test_yuv_readers(layout):
  """A crop window of 256 x 384 out of 270 x 400 frames: a resampled and a direct pass."""
  model = get_model()[0]
  T = 97
  clip, _ = make_frames(1, T, 270, 400, layout, seed=23, matrix='bt709', window=(6, 9, 256, 384))
  q = _queries([0, 96, 33, 34.5, 70, 12.25], 256, 384)
  want = _check(model, clip, q, read=_yuv_reader(clip), window_frames=40, unrefined=True)
  _assert_equal(want, {k: v for k, v in _whole(model, live.yuv420_to_rgb(clip), q).items()})


def test_call_pattern():
  """The pre-pass reads only tap frames, each once; the sweep reads consecutive ranges covering
  the video once, window w + 1's before window w is yielded; no host chunk outlives the next read."""
  model = get_model()[0]
  T, C = 300, 40
  video = _video(T, 256, 256, seed=25)
  times = [150, 10, 11.5, 290, 299, 200.25]
  q = _queries(times, 256, 256)
  log, refs = [], []

  def read(a, z):
    assert all(r() is None for r in refs)  # the driver let go of every chunk it was handed
    x = _reader(video, 'pinned', log)(a, z)
    refs.append(weakref.ref(x))
    return x

  got = _collect(model, read, T, q, log=log, window_frames=C)
  _assert_equal(got, {k: v for k, v in _whole(model, video, q).items() if k in _KEYS})
  reads = [(a, z) for e, a, z in log if e == 'read']
  plan = tapir_model._pass_plan((256, 256), model.initial_resolution)
  halos = windowed.halo_frames(model, (256, 256))
  sweep = windowed.sweep_reads(T, C, halos, plan)
  nonempty = [r for r in sweep if r[0] < r[1]]
  prepass = reads[:len(reads) - len(nonempty)]
  assert reads[len(prepass):] == nonempty
  # the six queries' tap frames fit one pre-pass chunk
  assert prepass == windowed.prepass_reads(times, T, 64)
  taps = {int(f) for t in windowed.query_tap_frames(times, T) for f in (t, t + 1) if f < T}
  read_frames = [f for a, z in prepass for f in range(a, z)]
  assert sorted(read_frames) == sorted(taps)  # tap frames only, each once
  # read-ahead: window w's frames are read after window w - 2's yield and before window w - 1's
  windows = windowed.window_plan(T, C, halos, plan)
  pos = {e: i for i, e in enumerate(log)}  # sweep reads come after the pre-pass's
  for w, (a, z) in enumerate(sweep):
    if a == z:
      continue
    i = pos[('read', a, z)]
    if w >= 1:
      assert i < pos[('yield', windows[w - 1].start, windows[w - 1].stop)]
    if w >= 2:
      assert i > pos[('yield', windows[w - 2].start, windows[w - 2].stop)]


def test_memory_is_bounded():
  """Peak allocated bytes at T and 2T (same C, queries on the same frames, yields dropped) differ by
  at most 2 MiB, a margin for the caching allocator's 512-byte rounding of the per-window tensors
  and the pre-pass chunking; windowed_forward's grow by its full-length outputs."""
  model = get_model()[0]
  T, C = 512, 64  # T >= C + 2 H_1: every buffer at full size for both lengths
  times = [0, 1, 5.5, 40] * 16

  def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base

  def run(video):
    for _ in windowed.track_video(model, _reader(video), video.shape[1], q, window_frames=C):
      pass

  v1, v2 = _video(T, 512, 512, seed=9), _video(2 * T, 512, 512, seed=9)
  q = _queries(times, 512, 512)
  run(v1)  # grows the model's workspaces
  p1, p2 = peak(lambda: run(v1)), peak(lambda: run(v2))
  w1 = peak(lambda: windowed.windowed_forward(model, v1, q, window_frames=C))
  w2 = peak(lambda: windowed.windowed_forward(model, v2, q, window_frames=C))
  growth = (windowed.output_bytes(model, v2.shape, len(times))
            - windowed.output_bytes(model, v1.shape, len(times)))
  print(f'peak bytes: track_video T {p1}, 2T {p2}; windowed_forward T {w1}, 2T {w2}; '
        f'output growth {growth}')
  assert abs(p2 - p1) <= 2 << 20
  assert w2 - w1 >= growth // 2


@pytest.mark.parametrize('bad', ['shape', 'size', 'dtype', 'format', 'count'])
def test_bad_frames_mid_stream(bad):
  model = get_model()[0]
  T = 120
  video = _video(T, 256, 256, seed=27)
  q = _queries([0, 50], 256, 256)
  good = _reader(video)
  calls = []

  def read(a, z):
    calls.append((a, z))
    x = good(a, z)
    if a < 100:
      return x
    if bad == 'shape':
      return x[..., :2]
    if bad == 'size':
      return torch.nn.functional.pad(x, (0, 0, 0, 8))
    if bad == 'dtype':
      return x.float()
    if bad == 'format':
      return make_frames(1, z - a, 256, 256, 'nv12', seed=1)[0]
    return x[:-1]

  with pytest.raises(ValueError, match=r'read_frames\((\d+), 120\)'):
    for _ in windowed.track_video(model, read, T, q, window_frames=20):
      pass
  assert calls[-1][0] >= 100


def test_reader_errors_propagate_and_early_exit():
  model = get_model()[0]
  T = 200
  video = _video(T, 256, 256, seed=29)
  q = _queries([0, 120, 199], 256, 256)
  want = _whole(model, video, q)

  def failing(a, z):
    if z > 150:
      raise KeyError('decoder gave up')
    return video[0, a:z]
  with pytest.raises(KeyError, match='decoder'):
    for _ in windowed.track_video(model, failing, T, q, window_frames=32):
      pass
  # leave the loop after the first window, with the next window's frames in flight
  for _, _, out in windowed.track_video(model, _reader(video, 'pinned'), T, q, window_frames=32):
    break
  del out
  _assert_equal(_whole(model, video, q), want)
