"""tapnet_b200.windowed on the GPU: every output of windowed_forward equals model(video, queries) bit
for bit, the halos are tight, memory stays bounded, and tapir_sample_query_features_ex samples a
partial grid exactly as the whole one."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tapnet_b200 import _lib, tapir_model, windowed  # noqa: E402
from tests.test_stages_gpu import get_model  # noqa: E402


def _video(T, H, W, seed=0, B=1):
  """A uint8 clip [B, T, H, W, 3] on the GPU: a smooth texture drifting across the frame, plus noise."""
  g = torch.Generator().manual_seed(seed)
  clips = []
  for _ in range(B):
    base = torch.rand(1, 3, H // 8 + 10, W // 8 + 10, generator=g) * 255
    base = torch.nn.functional.interpolate(base, scale_factor=8, mode='bilinear', align_corners=False)
    base = base[0].permute(1, 2, 0).cuda()
    noise = torch.rand(T, H, W, 3, generator=g).cuda() * 24
    frames = [base[(t * 2) % 71:(t * 2) % 71 + H, (t * 3) % 73:(t * 3) % 73 + W] for t in range(T)]
    clips.append((torch.stack(frames) * 0.9 + noise).clamp(0, 255).to(torch.uint8))
  return torch.stack(clips).contiguous()


def _queries(times, H, W, seed=1, B=1):
  g = torch.Generator().manual_seed(seed)
  t = torch.tensor(times, dtype=torch.float32)[None, :, None].expand(B, -1, -1)
  yx = torch.rand(B, len(times), 2, generator=g) * torch.tensor([H - 1.0, W - 1.0])
  return torch.cat([t, yx], dim=-1).contiguous().cuda()


def _assert_equal(got, want):
  assert set(got) == set(want)
  for k, v in want.items():
    if isinstance(v, (list, tuple)):
      assert len(got[k]) == len(v), k
      for i, (a, b) in enumerate(zip(got[k], v)):
        assert a.shape == b.shape and torch.equal(a, b), f'{k}[{i}] differs'
    else:
      assert got[k].shape == v.shape and torch.equal(got[k], v), f'{k} differs'


def _whole(model, video, q):
  with torch.no_grad():
    return model(video, q)


_T256 = 300
# t = 0, T - 1, core edges of C = 32 and 100, inside halos, fractional times (halves included)
_TIMES256 = [0, _T256 - 1, 31, 32, 99, 100, 64, 95, 96, 97, 131, 196, 204, 12.5, 150.49, 150.5,
             200.7, 33.3, 299.4, 0.49] + list(np.linspace(1, 298, 12).round(1))


@pytest.fixture(scope='module')
def clip256():
  video = _video(_T256, 256, 256)
  return video, _queries(_TIMES256, 256, 256)


@pytest.mark.parametrize('pyramid_level', [0, 1])
def test_matches_whole_clip_256(clip256, pyramid_level):
  model = get_model(pyramid_level=pyramid_level)[0]
  video, q = clip256
  want = _whole(model, video, q)
  for C in (32, 100):
    _assert_equal(windowed.windowed_forward(model, video, q, window_frames=C), want)


def test_one_window_and_automatic_core(clip256):
  model = get_model()[0]
  video, q = clip256
  want = _whole(model, video, q)
  _assert_equal(windowed.windowed_forward(model, video, q, window_frames=_T256 + 5), want)
  _assert_equal(windowed.windowed_forward(model, video, q), want)


def test_two_levels_512():
  model = get_model()[0]
  T = 600
  assert windowed.halo_frames(model, (512, 512)) == [(192, 192), (96, 96)]
  video = _video(T, 512, 512, seed=3)
  q = _queries([0, T - 1, 100, 101, 288, 300.5, 450.25, 599.2] + list(range(5, 600, 40)), 512, 512)
  want = _whole(model, video, q)
  _assert_equal(windowed.windowed_forward(model, video, q, window_frames=120), want)  # 5 windows


def test_causal(clip256):
  model = get_model(causal=True)[0]
  video, q = clip256
  assert windowed.halo_frames(model, (256, 256)) == [(192, 0)]
  _assert_equal(windowed.windowed_forward(model, video, q, window_frames=64),
                _whole(model, video, q))


def test_two_clips():
  model = get_model()[0]
  T = 200
  video = _video(T, 256, 256, seed=5, B=2)
  q = _queries([0, 199, 50, 51, 120.5, 7.25, 160, 99], 256, 256, B=2)
  q[1, :, 0] = q[1, :, 0].flip(0)
  _assert_equal(windowed.windowed_forward(model, video, q, window_frames=50),
                _whole(model, video, q))


def test_pinned_host_clip():
  model = get_model()[0]
  T = 260
  video = _video(T, 512, 512, seed=7)
  q = _queries([0, 259, 64, 130.5, 200, 3.7], 512, 512)
  want = _whole(model, video, q)
  host = video.cpu().pin_memory()
  _assert_equal(windowed.windowed_forward(model, host, q.cpu(), window_frames=64), want)


# One-frame backbone chunks (whose ExtraConv GEMMs split K) and one-frame mixer calls: C = 1 (every
# slide adds one frame; a causal model's first window is one frame), a last slide of one frame
# (T = 129, C = 32), and clips whose last frame the whole-clip call runs alone (T = 97, 289 at
# 256 x 256: 96 frames per chunk) while the windows run it with others.
@pytest.mark.parametrize('T, C, causal', [(97, 1, False), (97, 1, True), (129, 32, False),
                                          (289, 100, False)])
def test_one_frame_calls(T, C, causal):
  model = get_model(causal=causal)[0]
  video = _video(T, 256, 256, seed=11)
  q = _queries([0, T - 1, T - 2, 1, T // 2, 30.5, C, C - 1, T - 1.4], 256, 256)
  _assert_equal(windowed.windowed_forward(model, video, q, window_frames=C), _whole(model, video, q))


# every query on the last frame: its tap pair is that frame alone, run alone by the whole-clip call
# at T = 97 and inside its last chunk at T = 98
@pytest.mark.parametrize('T', [97, 98])
def test_queries_on_the_last_frame(T):
  model = get_model()[0]
  video = _video(T, 256, 256, seed=13)
  q = _queries([T - 1] * 6, 256, 256)
  _assert_equal(windowed.windowed_forward(model, video, q, window_frames=40), _whole(model, video, q))


def test_float_clips():
  """float32 clips in [-1, 1]: on the device at 512 x 512 (a resampled and a direct pass; 97 frames
  leave the last one alone in both passes' chunks), and as a pinned host clip at 256 x 256."""
  model = get_model()[0]
  video = _video(97, 512, 512, seed=15).float() / 127.5 - 1
  q = _queries([0, 96, 40, 41, 12.5, 80], 512, 512)
  _assert_equal(windowed.windowed_forward(model, video, q, window_frames=40), _whole(model, video, q))
  video = _video(97, 256, 256, seed=17).float() / 127.5 - 1
  q = _queries([0, 96, 31, 32, 50.5], 256, 256)
  want = _whole(model, video, q)
  host = video.cpu().pin_memory()
  _assert_equal(windowed.windowed_forward(model, host, q.cpu(), window_frames=32), want)


@pytest.mark.parametrize('side', [0, 2])
def test_halo_is_tight(clip256, side):
  """A halo one frame short changes the core's outputs; the formula's halo keeps them equal.

  With trained or random weights the influence of the frame at the halo's far edge reaches the
  core attenuated by every block's LayerNorm, below one fp32 ulp, so the model here is built to
  carry it: one iteration per level (halo 24 frames at 256 x 256) and depthwise taps that are a
  pure shift with gain (tap 0: from the frame before, tap 2: from the frame after)."""
  model = tapir_model.TAPIR(pyramid_level=1, num_pips_iter=1)
  model.load_state_dict(get_model()[0].state_dict())
  with torch.no_grad():
    for name, p in model.named_parameters():
      if name.startswith('torch_pips_mixer.blocks.') and '.mlp1_up' in name and name.endswith('weight'):
        p.zero_()
        p[..., side] = 10.0
  model = model.cuda().eval()
  assert windowed.halo_frames(model, (256, 256)) == [(24, 24)]
  video, q = clip256
  want = _whole(model, video, q)
  assert all(torch.isfinite(want[k]).all() for k in ('tracks', 'occlusion', 'expected_dist'))
  _assert_equal(windowed.windowed_forward(model, video, q, window_frames=100), want)
  got = windowed.windowed_forward(model, video, q, window_frames=100, _halo_trim=[1])
  assert not torch.equal(got['tracks'], want['tracks'])


def test_memory_is_bounded():
  model = get_model()[0]
  T, C = 512, 64  # T >= C + 2 H_1: the window buffers are at full size for both lengths
  times = [0, 1, 5.5, 40]

  def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    p = torch.cuda.max_memory_allocated() - base
    del out
    return p

  v1, v2 = _video(T, 512, 512, seed=9), _video(2 * T, 512, 512, seed=9)
  q = _queries(times, 512, 512)
  windowed.windowed_forward(model, v1, q, window_frames=C)  # grows the model's workspaces
  p1 = peak(lambda: windowed.windowed_forward(model, v1, q, window_frames=C))
  p2 = peak(lambda: windowed.windowed_forward(model, v2, q, window_frames=C))
  whole = peak(lambda: _whole(model, v2, q))
  growth = (windowed.output_bytes(model, v2.shape, len(times))
            - windowed.output_bytes(model, v1.shape, len(times)))
  print(f'peak bytes: windowed T {p1}, windowed 2T {p2}, whole 2T {whole}')
  assert abs(p2 - p1) <= growth + (64 << 20)
  assert p1 < whole and p2 < whole


@pytest.mark.parametrize('T', [1, 2, 5, 33, 300])
def test_sample_query_features_ex(T):
  g = torch.Generator().manual_seed(T)
  gh, gw, C, H, W = 32, 32, 256, 256, 256
  grid = torch.randn(T, gh, gw, C, generator=g).cuda()
  N = 600
  t = torch.cat([torch.randint(0, T, (N // 2,), generator=g).float(),
                 torch.rand(N // 2 - 4, generator=g) * (T + 2) - 1, torch.tensor([-3.0, T, T - 0.5, 0.5])])
  qp = torch.stack([t, torch.rand(N, generator=g) * H, torch.rand(N, generator=g) * W], 1).cuda()
  full = torch.empty(N, C, device='cuda')
  _lib.sample_query_features(grid, qp, (T, H, W), full)

  # the ex entry with a NULL table is the old call: same launch count, same results
  lib = _lib.load()
  ex = torch.empty_like(full)
  n0 = lib.tapir_launch_count()
  _lib.check(lib.tapir_sample_query_features_ex(_lib.ptr(grid), T, gh, gw, C, _lib.ptr(qp), N, T, H, W,
                                                None, _lib.ptr(ex), _lib.stream()), 'ex')
  n1 = lib.tapir_launch_count()
  _lib.sample_query_features(grid, qp, (T, H, W), full)
  assert lib.tapir_launch_count() - n1 == n1 - n0 == 1
  assert torch.equal(ex, full)

  # a grid of about half the frames, in a shuffled slot order
  keep = torch.nonzero(torch.rand(T, generator=g) < 0.5).flatten()
  if keep.numel() == 0:
    keep = torch.tensor([0])
  keep = keep[torch.randperm(keep.numel(), generator=g)]
  slot = torch.full((T,), -1, dtype=torch.int32)
  slot[keep] = torch.arange(keep.numel(), dtype=torch.int32)
  part = torch.empty_like(full)
  _lib.sample_query_features(grid[keep.cuda()].contiguous(), qp, (T, H, W), part,
                             frame_slot=slot.cuda())
  t0 = windowed.query_tap_frames(t.numpy(), T)
  held = set(keep.tolist())
  # the second tap has a nonzero weight unless the time lands on t0 exactly
  f = np.float32(T)
  c = (t.numpy().astype(np.float32) * f) / f + np.float32(0.5)
  pix = np.fmin(np.fmax(((np.float32(2) * (c / f) - 1 + 1) * f - 1) / 2, np.float32(0)), f - 1)
  need2 = (pix - t0.astype(np.float32) != 0) & (t0 + 1 < T)
  ok = np.array([t0[i] in held and (not need2[i] or t0[i] + 1 in held) for i in range(N)])
  part, ok = part.cpu(), torch.from_numpy(ok)
  assert ok.any()
  assert torch.equal(part[ok], full.cpu()[ok])
  assert torch.isnan(part[~ok]).all()

  # every argument is checked at the entry point
  for args in ((T, gh, gw, C, 0, T, H, W), (T, gh, gw, C, N, 0, H, W), (0, gh, gw, C, N, T, H, W)):
    Tg, a, b, c_, n, vt, vh, vw = args
    assert lib.tapir_sample_query_features_ex(_lib.ptr(grid), Tg, a, b, c_, _lib.ptr(qp), n, vt, vh, vw,
                                              None, _lib.ptr(ex), _lib.stream()) == 1
  assert lib.tapir_sample_query_features_ex(_lib.ptr(grid), T, gh, gw, C, _lib.ptr(qp), N, T, H, W,
                                            None, _lib.ptr(grid), _lib.stream()) == 1
