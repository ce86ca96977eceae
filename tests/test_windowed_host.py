"""Host logic of tapnet_b200.windowed: halos, the window plan, the byte model, the float32 mirror of
the query sampler's tap frames and the argument checks.  No GPU needed."""
import numpy as np
import pytest
import torch

from tapnet_b200 import tapir_model
from tapnet_b200 import windowed


@pytest.fixture(scope='module')
def models():
  return tapir_model.TAPIR(), tapir_model.TAPIR(use_casual_conv=True)


@pytest.mark.parametrize('hw, want', [
    ((256, 256), [96]),
    ((1024, 1024), [288, 192, 96]),
    ((1080, 1920), [384, 288, 192, 96]),
])
def test_halo_frames(models, hw, want):
  model, causal = models
  assert windowed.halo_frames(model, hw) == [(h, h) for h in want]
  # causal: each convolution reaches k - 1 frames back, none forward
  assert windowed.halo_frames(causal, hw) == [(2 * h, 0) for h in want]


def test_halo_frames_custom_resolutions(models):
  model, causal = models
  res = [(256, 256), (384, 384)]
  assert windowed.halo_frames(model, (512, 512), res) == [(192, 192), (96, 96)]
  assert windowed.halo_frames(causal, (512, 512), [(512, 512)]) == [(192, 0)]


def test_halo_frames_follow_the_model():
  model = tapir_model.TAPIR(num_pips_iter=2)
  assert windowed.halo_frames(model, (512, 512)) == [(96, 96), (48, 48)]


def _plan_case(model, T, C, hw):
  plan = tapir_model._pass_plan(hw, model.initial_resolution)
  halos = windowed.halo_frames(model, hw)
  return windowed.window_plan(T, C, halos, plan), halos, plan


@pytest.mark.parametrize('T, C', [(1, 1), (7, 3), (300, 32), (300, 100), (1000, 300), (50, 64)])
@pytest.mark.parametrize('causal', [False, True])
def test_window_plan(models, T, C, causal):
  model = models[causal]
  wins, halos, plan = _plan_case(model, T, C, (1024, 1024))
  covered = np.zeros(T, np.int64)
  for w in wins:
    assert 0 <= w.start < w.stop <= T and w.stop - w.start <= C
    covered[w.start:w.stop] += 1
    prev = None
    for (a, z), (left, right) in zip(w.levels, halos):
      a0, z0 = max(0, w.start - left), min(T, w.stop + right)
      # a one-frame range widens to two frames (the mixer splits K for one-frame calls only)
      assert (a, z) == ((a0, z0) if z0 - a0 > 1 or T == 1 else (a0 - 1, z0) if a0 else (0, 2))
      assert z - a >= min(T, 2)
      if prev is not None:  # nested, each narrower by the next level's halo where not clipped
        assert prev[0] <= a and z <= prev[1]
      prev = (a, z)
    # each pass's buffer range is the range of the widest level it serves
    for (a, z), lvl in zip(w.passes, windowed.pass_levels(plan)):
      assert (a, z) == w.levels[lvl - 1]
  assert (covered == 1).all()
  assert [w.start for w in wins] == list(range(0, T, C))


def test_window_plan_level_steps(models):
  wins, _, _ = _plan_case(models[0], 2000, 100, (1024, 1024))
  w = wins[10]
  assert w.levels == ((1000 - 288, 1100 + 288), (1000 - 192, 1100 + 192), (1000 - 96, 1100 + 96))
  with pytest.raises(ValueError):
    windowed.window_plan(10, 0, [(96, 96)], tapir_model._pass_plan((256, 256), (256, 256)))


def test_byte_model_grows_with_the_core(models):
  model = models[0]
  shape = (1, 2000, 1024, 1024)
  b = [windowed.sweep_bytes(model, shape, 256, c) for c in (1, 2, 64, 512, 2000)]
  assert all(x < y for x, y in zip(b, b[1:]))
  # the pass buffers alone: (C + 2 H) frames of each pass's grids, 48 bytes per input pixel
  C = 512
  grids = sum((C + 2 * h) * 48 * s * s for h, s in ((288, 256), (192, 512), (96, 1024)))
  assert grids < windowed.sweep_bytes(model, shape, 256, C) < grids * 1.25
  # clipped at the clip's length: a longer core than the clip changes nothing
  assert windowed.sweep_bytes(model, (1, 50, 256, 256), 8, 50) == \
      windowed.sweep_bytes(model, (1, 50, 256, 256), 8, 500)
  out = windowed.output_bytes(model, shape, 256)
  assert out == 2000 * 256 * 16 * (4 * 3 + 1 + 3 + 1)


def test_choose_window_frames(models):
  model = models[0]
  shape = (1, 2000, 1024, 1024)
  need = lambda c: (windowed.output_bytes(model, shape, 256)  # noqa: E731
                    + windowed.sweep_bytes(model, shape, 256, c))
  free = need(300) + 1
  c = windowed.choose_window_frames(model, shape, 256, free)
  assert c == 300
  assert windowed.choose_window_frames(model, (1, 100, 256, 256), 16, 80e9) == 100
  with pytest.raises(ValueError, match='bytes'):
    windowed.choose_window_frames(model, shape, 256, need(1) - 1)


def _kernel_steps_torch(t, T):
  """sample_query_kernel's time-axis steps restated with torch float32 CPU ops."""
  f = torch.tensor(float(T), dtype=torch.float32)
  c = torch.div(torch.mul(t, f), f)
  c = torch.add(c, torch.tensor(0.5, dtype=torch.float32))
  g = torch.sub(torch.mul(torch.tensor(2.0), torch.div(c, f)), 1.0)
  pix = torch.div(torch.sub(torch.mul(torch.add(g, 1.0), f), 1.0), 2.0)
  pix = torch.clamp(pix, min=0.0, max=float(T - 1))
  return torch.floor(pix).to(torch.int64).numpy()


def test_tap_frames_every_integer_time():
  bad = 0
  for T in range(1, 2049):
    t = torch.arange(T, dtype=torch.float32)
    got = windowed.query_tap_frames(t.numpy(), T)
    bad += int((got != _kernel_steps_torch(t, T)).sum())
    # the query frame is always one of the two taps
    assert ((got == np.arange(T)) | (got + 1 == np.arange(T))).all()
  assert bad == 0


def test_tap_frames_other_times():
  g = torch.Generator().manual_seed(0)
  for T in (1, 2, 3, 17, 300, 1999, 2048):
    t = torch.cat([torch.rand(500, generator=g) * T, -torch.rand(50, generator=g) * 5,
                   T + torch.rand(50, generator=g) * 5, torch.tensor([-0.5, T - 0.5, T, T + 1e-3])])
    got = windowed.query_tap_frames(t.numpy(), T)
    assert (got == _kernel_steps_torch(t, T)).all()
    assert ((got >= 0) & (got <= T - 1)).all()
    # stage A's query frame: rint(t * T / T), as the whole clip computes it
    want = torch.round(t * torch.tensor(float(T)) / torch.tensor(float(T))).to(torch.int64).numpy()
    assert (windowed.query_frames(t.numpy(), T) == want).all()


def test_argument_errors(models):
  model = models[0]  # on the CPU
  video = torch.zeros(1, 4, 256, 256, 3, dtype=torch.uint8)
  q = torch.zeros(1, 2, 3)
  with pytest.raises(ValueError, match='window_frames'):
    windowed.windowed_forward(model, video, q, window_frames=0)
  with pytest.raises(ValueError, match='video'):
    windowed.windowed_forward(model, video[0], q)
  with pytest.raises(ValueError, match='video'):
    windowed.windowed_forward(model, video[..., :2], q)
  with pytest.raises(ValueError, match='query_points'):
    windowed.windowed_forward(model, video, q[0])
  with pytest.raises(ValueError, match='query_points'):
    windowed.windowed_forward(model, video, torch.zeros(2, 2, 3))
  with pytest.raises(ValueError, match='video'):
    windowed.windowed_forward(model, video.to(torch.int32), q)
  with pytest.raises(RuntimeError, match='CUDA'):
    windowed.windowed_forward(model, video, q)


def test_alone_frames():
  """The frames the whole-clip call runs through a pass in one-frame backbone chunks."""
  p256, p1080 = (tapir_model.PassStep(h, w, True, True) for h, w in ((256, 256), (1080, 1920)))
  assert windowed._backbone_chunk(p256) == 96 and windowed._backbone_chunk(p1080) == 3
  assert list(np.nonzero(windowed._alone_frames(p256, 1, 97, 0, range(97)))[0]) == [96]
  assert not windowed._alone_frames(p256, 1, 96, 0, range(96)).any()
  assert not windowed._alone_frames(p256, 1, 98, 0, range(98)).any()
  # batches chunk their B * T frames in order: only the batch's last frame can be left over
  assert not windowed._alone_frames(p256, 2, 97, 0, range(97)).any()
  assert list(np.nonzero(windowed._alone_frames(p256, 5, 77, 4, range(77)))[0]) == [76]
  assert not windowed._alone_frames(p256, 5, 77, 3, range(77)).any()
  assert windowed._alone_frames(p256, 1, 1, 0, [0]).all()
  assert list(np.nonzero(windowed._alone_frames(p1080, 1, 7, 0, range(7)))[0]) == [6]


@pytest.mark.parametrize('alone', [[], [0], [6], [3], [0, 1, 2], [2, 4], [1, 3, 5], list(range(9))])
@pytest.mark.parametrize('n', [1, 2, 5, 9])
def test_run_frames_calls(monkeypatch, alone, n):
  """_run_frames computes every frame, the marked ones in one-frame calls and every other frame in
  calls of 2 .. chunk frames (the chunk is 4 frames here)."""
  step = tapir_model.PassStep(8, 8, True, True)
  monkeypatch.setattr(tapir_model, '_MAX_BACKBONE_PIXELS', 4 * 64)
  calls = []

  def run_pass(model, pk, video, st, a, z, out, dev):
    calls.append((video.shape[1], a, z))
    for t in out:
      t.copy_(video[:, a:z, :1, :1, 0].float().reshape(t.shape[:2] + (1,) * (t.dim() - 2)).expand_as(t))

  monkeypatch.setattr(windowed, '_run_pass', run_pass)
  video = torch.arange(n, dtype=torch.uint8).view(1, n, 1, 1, 1).expand(1, n, 8, 8, 3).contiguous()
  mask = np.zeros(n, bool)
  mask[[i for i in alone if i < n]] = True
  out = (torch.full((1, n, 1, 1, 4), -1.0), torch.full((1, n, 2, 2, 2), -1.0))
  windowed._run_frames(None, None, video, step, out, mask, 'cpu')
  for t in out:
    assert torch.equal(t[0, :, 0, 0, 0], torch.arange(n, dtype=torch.float32))
  for frames, a, z in calls:
    if z - a == 1:
      assert mask[a] and frames == n
    else:
      assert 2 <= z - a <= 4 and (frames == 2 or not mask[a:z].any())
