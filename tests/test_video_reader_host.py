"""Host logic of windowed.track_video: the frame ranges it asks the reader for, the device ring's
span, its byte model, the checks of what a reader returns and the argument checks.  No GPU needed."""
import numpy as np
import pytest
import torch

from tapnet_b200 import tapir_model
from tapnet_b200 import windowed


@pytest.fixture(scope='module')
def models():
  return tapir_model.TAPIR(), tapir_model.TAPIR(use_casual_conv=True)


def _case(model, T, C, hw):
  plan = tapir_model._pass_plan(hw, model.initial_resolution)
  halos = windowed.halo_frames(model, hw)
  return windowed.window_plan(T, C, halos, plan), halos, plan


def _pass_runs(windows):
  """What _slide computes, counted pass by pass: for each window, each pass's new frames."""
  held = [(0, 0)] * len(windows[0].passes)
  out = []
  for win in windows:
    runs = []
    for p, (a, z) in enumerate(win.passes):
      runs.append(range(max(a, held[p][1]), z))
      held[p] = (a, z)
    out.append(runs)
  return out


_CASES = [(1, 1), (7, 3), (300, 32), (300, 100), (1000, 300), (50, 64), (97, 1), (2000, 100)]


@pytest.mark.parametrize('T, C', _CASES)
@pytest.mark.parametrize('causal', [False, True])
@pytest.mark.parametrize('hw', [(256, 256), (1024, 1024)])
def test_sweep_reads(models, T, C, causal, hw):
  """Consecutive ranges that cover [0, T) once, in order; each window's new frames are read by the
  time it runs them through a pass, and not before the window they are first needed in."""
  windows, halos, plan = _case(models[causal], T, C, hw)
  reads = windowed.sweep_reads(T, C, halos, plan)
  assert len(reads) == len(windows)
  assert reads[0][0] == 0 and reads[-1][1] == T
  assert all(a <= z for a, z in reads)
  assert all(r[1] == s[0] for r, s in zip(reads, reads[1:]))
  for (a, z), runs in zip(reads, _pass_runs(windows)):
    needed = [f for r in runs for f in r]
    assert max(needed, default=-1) < z
    if a < z:
      assert max(needed) == z - 1


@pytest.mark.parametrize('T, C', _CASES)
@pytest.mark.parametrize('causal', [False, True])
@pytest.mark.parametrize('hw', [(256, 256), (1024, 1024), (1080, 1920)])
def test_ring_span(models, T, C, causal, hw):
  """Counting the passes' ranges directly: the frames read but not yet through every pass that
  needs them never exceed the ring, occupy distinct slots (frame % S) at every window, including
  the next window's frames read ahead, and fill the ring at some window."""
  windows, halos, plan = _case(models[causal], T, C, hw)
  S = windowed.ring_frames(T, C, halos, plan)
  reads = windowed.sweep_reads(T, C, halos, plan)
  last_use = {}
  for w, runs in enumerate(_pass_runs(windows)):
    for r in runs:
      for f in r:
        last_use[f] = w
  read_at = {f: w for w, (a, z) in enumerate(reads) for f in range(a, z)}
  most = 0
  for w in range(len(windows)):
    live = [f for f, u in last_use.items() if read_at[f] <= w <= u]
    most = max(most, len(live))
    assert len({f % S for f in live}) == len(live)
    # read ahead: window w + 1's frames land while the frames window w + 1 still needs are held
    ahead = [f for f, u in last_use.items() if read_at[f] <= w + 1 and u >= w + 1]
    assert len({f % S for f in ahead}) == len(ahead)
  assert most == S
  if not causal and T >= C + 2 * halos[0][0] + C:
    # the first window computes every pass from frame 0: C + H_1 frames; later ones C + H_1 - H_L
    assert S == C + halos[0][1]


@pytest.mark.parametrize('seed', range(6))
@pytest.mark.parametrize('max_frames', [2, 4, 16, 512])
def test_prepass_reads(seed, max_frames):
  """Only tap frames, each once, first the first tap pair; every chunk's frames are on the device
  (read, or kept from the chunk before) when it runs."""
  rng = np.random.default_rng(seed)
  T = int(rng.integers(1, 400))
  t = np.concatenate([rng.integers(0, T, 20), rng.random(10) * T, [T - 1, 0]]).astype(np.float32)
  reads = windowed.prepass_reads(t, T, max_frames)
  t0 = windowed.query_tap_frames(t, T)
  taps = sorted({int(f) for a in t0 for f in (a, a + 1) if f < T})
  frames = [f for a, z in reads for f in range(a, z)]
  assert sorted(frames) == taps
  assert reads[0] == (taps[0], min(taps[0] + 2, T))
  chunks = windowed._prepass_chunks(t0, T, max_frames)
  _, per_chunk = windowed._prepass_reads(t0, T, max_frames)
  kept = set(range(*reads[0]))
  for (fl, _), rs in zip(chunks, per_chunk):
    got = kept | {f for a, z in rs for f in range(a, z)}
    assert set(fl) <= got
    kept = {fl[-1]}


def test_byte_model(models):
  """Grows with C, does not grow with T once T > C + 2 H_1, and counts the ring and two windows'
  outputs on top of the sweep's buffers."""
  for model in models:
    for hw, fb in (((256, 256), None), ((1024, 1024), None), ((1080, 1920), 1080 * 1920 * 3 // 2)):
      b = [windowed.reader_sweep_bytes(model, (1, 4000, *hw), 256, c, frame_bytes=fb)
           for c in (1, 2, 8, 64, 200, 512)]
      assert all(x < y for x, y in zip(b, b[1:]))
      H1 = windowed.halo_frames(model, hw)[0][0]
      for C in (1, 64):
        base = windowed.reader_sweep_bytes(model, (1, C + 2 * H1 + 1, *hw), 256, C, frame_bytes=fb)
        for T in (C + 2 * H1 + 2, 3000, 100000):
          assert windowed.reader_sweep_bytes(model, (1, T, *hw), 256, C, frame_bytes=fb) == base
  model = models[0]
  shape = (1, 2000, 1024, 1024)
  plan = tapir_model._pass_plan((1024, 1024), model.initial_resolution)
  halos = windowed.halo_frames(model, (1024, 1024))
  ring = windowed.ring_frames(2000, 100, halos, plan) * 1024 * 1024 * 3
  outs = 2 * windowed.output_bytes(model, (1, 100, 1024, 1024), 256)
  # windowed_forward's sweep on a device clip stages the frames its resampled passes read; the ring
  # path reads them in place and adds a lone frame's pair (2 frames and 2 x 66 MB of grids) instead
  sweep = windowed.sweep_bytes(model, shape, 256, 100)
  got = windowed.reader_sweep_bytes(model, shape, 256, 100)
  assert 0.95 * (ring + outs + sweep) <= got <= ring + outs + sweep + 2 * (66 + 3) * 2 ** 20


def test_choose_reader_window_frames(models):
  model = models[0]
  shape = (1, 100000, 1024, 1024)
  need = lambda c: windowed.reader_sweep_bytes(model, shape, 256, c)  # noqa: E731
  assert windowed.choose_reader_window_frames(model, shape, 256, need(300) + 1) == 300
  assert windowed.choose_reader_window_frames(model, (1, 100, 256, 256), 16, 80e9) == 100
  with pytest.raises(ValueError, match='bytes'):
    windowed.choose_reader_window_frames(model, shape, 256, need(1) - 1)
  # no full-length term: a 100000-frame 1080p NV12 video with 8192 points fits 70 GB
  c = windowed.choose_reader_window_frames(model, (1, 100000, 1080, 1920), 8192, 70e9,
                                           frame_bytes=1080 * 1920 * 3 // 2)
  assert c > 64
  with pytest.raises(ValueError):
    windowed.choose_window_frames(model, (1, 100000, 1080, 1920), 8192, 70e9)


def _never(a, z):
  raise AssertionError('the reader must not be called')


def test_argument_errors(models):
  """Bad arguments raise when track_video is called, before any frame is read."""
  model = models[0]  # on the CPU
  q = torch.zeros(2, 3)
  for T in (0, -3, 2.5, True, None):
    with pytest.raises(ValueError, match='num_frames'):
      windowed.track_video(model, _never, T, q)
  with pytest.raises(ValueError, match='window_frames'):
    windowed.track_video(model, _never, 10, q, window_frames=0)
  with pytest.raises(ValueError, match='read_frames'):
    windowed.track_video(model, 'frames.mp4', 10, q)
  for bad in (torch.zeros(2, 2, 3), torch.zeros(2, 2), torch.zeros(0, 3), torch.zeros(1, 0, 3),
              np.zeros((2, 3))):
    with pytest.raises(ValueError, match='query_points'):
      windowed.track_video(model, _never, 10, bad)
  with pytest.raises(RuntimeError, match='CUDA'):
    windowed.track_video(model, _never, 10, q)


def test_frame_checks():
  """The first result fixes the format; a later one of another length, size, dtype, device or
  format raises ValueError naming the requested range; reader errors propagate."""
  dev = torch.device('cuda:0')
  frames = torch.zeros(10, 32, 48, 3, dtype=torch.uint8)
  bad = {}

  def read(a, z):
    return bad.pop('x', frames[a:z])
  src = windowed._FrameSource(read, dev)
  assert src(0, 4).shape == (4, 32, 48, 3)
  assert src.hw == (32, 48) and src.host and src.itemsize == 1 and src.yuv is None
  assert src.frame_bytes == 32 * 48 * 3
  for x, what in ((frames[:3], 'frames, expected 4'), (frames[:4].float(), 'first call'),
                  (torch.zeros(4, 32, 40, 3, dtype=torch.uint8), 'first call'),
                  (frames[:4, ..., :2], r'\(4, 32, 48, 2\)'), (frames[:4].numpy(), 'ndarray')):
    bad['x'] = x
    with pytest.raises(ValueError, match=r'read_frames\(4, 8\) returned .*' + what):
      src(4, 8)
  assert src(4, 8).shape == (4, 32, 48, 3)

  f32 = windowed._FrameSource(lambda a, z: frames[a:z].double(), dev)
  f32(0, 2)
  assert f32.itemsize == 4 and f32.frame_bytes == 32 * 48 * 12

  def failing(a, z):
    raise KeyError('decoder')
  with pytest.raises(KeyError):
    windowed._FrameSource(failing, dev)(0, 1)
