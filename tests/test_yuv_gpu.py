"""-m gpu: YUV 4:2:0 frames (NV12 / I420).  The conversion kernel equals the integer oracle on
every (Y, U, V) triple, and every model path fed YUV equals, bit for bit, the same path fed the
uint8 RGB frames the conversion produces (stem loader, ingest + resize, end to end, streaming)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tapnet_b200 import _lib, live, streaming  # noqa: E402
from tests.test_stages_gpu import get_model  # noqa: E402
from tests.test_yuv_host import frames_oracle, yuv_to_rgb_oracle  # noqa: E402

MATRICES = [('bt601', False), ('bt709', False), ('bt601', True), ('bt709', True)]


def _planes(y, u, v, layout, pad):
  """Device copies of numpy planes [B, T, rows, cols] in `layout`, rows padded by `pad` bytes."""
  B, T, H, W = y.shape
  ch, cw = u.shape[2:]
  yd = torch.zeros(B, T, H, W + pad, dtype=torch.uint8, device='cuda')[..., :W]
  yd.copy_(torch.from_numpy(y))
  if layout == 'nv12':
    uv = torch.zeros(B, T, ch, cw + pad, 2, dtype=torch.uint8, device='cuda')[:, :, :, :cw]
    uv.copy_(torch.from_numpy(np.stack([u, v], -1)))
    return yd, uv
  ud = torch.zeros(B, T, ch, cw + pad, dtype=torch.uint8, device='cuda')[..., :cw]
  vd = torch.zeros(B, T, ch, cw + 2 * pad, dtype=torch.uint8, device='cuda')[..., :cw]
  ud.copy_(torch.from_numpy(u))
  vd.copy_(torch.from_numpy(v))
  return yd, ud, vd


def make_frames(B, T, H, W, layout='nv12', pad=24, seed=0, **kw):
  """Random YUV420Frames on the device plus the numpy planes."""
  rng = np.random.default_rng(seed)
  y = rng.integers(0, 256, (B, T, H, W), dtype=np.uint8)
  u = rng.integers(0, 256, (B, T, (H + 1) // 2, (W + 1) // 2), dtype=np.uint8)
  v = rng.integers(0, 256, u.shape, dtype=np.uint8)
  planes = _planes(y, u, v, layout, pad)
  make = live.YUV420Frames.nv12 if layout == 'nv12' else live.YUV420Frames.i420
  return make(*planes, **kw), (y, u, v)


@pytest.mark.parametrize('layout', ['nv12', 'i420'])
@pytest.mark.parametrize('matrix,full_range', MATRICES)
def test_conversion_is_exact_on_every_triple(layout, matrix, full_range):
  """64 frames of 512^2 luma: each 2x2 block carries one of the 256^2 chroma pairs and frame f
  block pixel q has Y = 4f + q, so the clip holds all 2^24 (Y, U, V) triples once."""
  F, S = 64, 512
  u = np.broadcast_to((np.arange(256 * 256) // 256).astype(np.uint8).reshape(256, 256), (1, F, 256, 256))
  v = np.broadcast_to((np.arange(256 * 256) % 256).astype(np.uint8).reshape(256, 256), (1, F, 256, 256))
  q = (np.arange(S)[:, None] % 2) * 2 + (np.arange(S)[None, :] % 2)
  y = (4 * np.arange(F)[:, None, None] + q[None]).astype(np.uint8)[None]
  frames = (live.YUV420Frames.nv12 if layout == 'nv12' else live.YUV420Frames.i420)(
      *_planes(np.ascontiguousarray(y), np.ascontiguousarray(u), np.ascontiguousarray(v), layout, 40),
      matrix=matrix, full_range=full_range)
  got = live.yuv420_to_rgb(frames).cpu().numpy()
  up = lambda p: np.repeat(np.repeat(p, 2, 2), 2, 3)  # noqa: E731
  for f0 in range(0, F, 8):
    sl = slice(f0, f0 + 8)
    ref = yuv_to_rgb_oracle(y[:, sl], up(u[:, sl]), up(v[:, sl]), matrix, full_range)
    np.testing.assert_array_equal(got[:, sl], ref)


@pytest.mark.parametrize('layout', ['nv12', 'i420'])
@pytest.mark.parametrize('matrix,full_range', MATRICES)
def test_conversion_odd_window_and_sizes(layout, matrix, full_range):
  frames, (y, u, v) = make_frames(2, 3, 37, 53, layout, pad=13, seed=1, matrix=matrix,
                                  full_range=full_range, window=(3, 5, 31, 41))
  got = live.yuv420_to_rgb(frames).cpu().numpy()
  np.testing.assert_array_equal(got, frames_oracle(y, u, v, (3, 5, 31, 41), matrix, full_range))


def test_ingest_equals_uint8_ingest():
  frames, _ = make_frames(1, 4, 97, 131, 'nv12', seed=2, matrix='bt709', window=(7, 11, 80, 100))
  rgb = live.yuv420_to_rgb(frames)
  for res in [(256, 256), (64, 48), None]:
    assert torch.equal(live.ingest_frames(frames, None, res), live.ingest_frames(rgb, None, res))
  # a window passed to the helper replaces the clip's own (full-frame coordinates)
  full = live.yuv420_to_rgb(frames.with_window(None))
  assert torch.equal(live.ingest_frames(frames, (1, 3, 90, 120), (64, 64)),
                     live.ingest_frames(full, (1, 3, 90, 120), (64, 64)))


def _assert_grids_equal(a, b):
  assert len(a.lowres) == len(b.lowres)
  for x, y in zip(a.lowres + a.hires, b.lowres + b.hires):
    assert torch.equal(x, y)
  assert tuple(a.resolutions) == tuple(b.resolutions)


@pytest.mark.parametrize('layout', ['nv12', 'i420'])
def test_backbone_stem_loader_bit_identical(layout):
  """Frames at the model resolution: the YUV stem loader, odd frame size and odd window origin."""
  model, _, _ = get_model()
  frames, _ = make_frames(1, 3, 261, 263, layout, seed=3, window=(3, 5, 256, 256))
  _assert_grids_equal(model.get_feature_grids(frames, False),
                      model.get_feature_grids(live.yuv420_to_rgb(frames), False))


def test_backbone_resize_path_bit_identical():
  """A 480x640 camera frame, centre crop: the YUV ingest kernel (initial resolution) and the stem
  loader at the crop's own size, plus the refinement resolutions in between."""
  model, _, _ = get_model()
  frames, _ = make_frames(1, 2, 480, 640, 'nv12', seed=4, matrix='bt709',
                          window=live.center_square_window(480, 640))
  a = model.get_feature_grids(frames, False)
  assert len(a.resolutions) > 1
  _assert_grids_equal(a, model.get_feature_grids(live.yuv420_to_rgb(frames), False))


def test_end_to_end_bit_identical():
  model, _, _ = get_model()
  frames, _ = make_frames(1, 8, 256, 256, 'nv12', seed=5)
  g = torch.Generator().manual_seed(5)
  q = torch.cat([torch.randint(0, 8, (1, 16, 1), generator=g).float(),
                 torch.rand(1, 16, 2, generator=g) * 255], -1).cuda()
  a = model(frames, q)
  b = model(live.yuv420_to_rgb(frames), q)
  assert sorted(a) == sorted(b)
  for k in a:
    if isinstance(a[k], (list, tuple)):
      assert len(a[k]) == len(b[k]) > 0
      for x, y in zip(a[k], b[k]):
        assert torch.equal(x, y), k
    else:
      assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize('S', [1, 3])
def test_streaming_yuv_equals_uint8_tracker(S):
  model, _, _ = get_model(causal=True)
  H, W, N = 256, 320, 8
  window = live.center_square_window(H, W)
  clip, _ = make_frames(S, 6, H, W, 'nv12', seed=6 + S)

  def frame(t, s=None):
    sl = slice(None) if s is None else slice(s, s + 1)
    return live.YUV420Frames(clip.y[sl, t:t + 1], clip.u[sl, t:t + 1], clip.v[sl, t:t + 1],
                             window=window)

  g = torch.Generator().manual_seed(S)
  qp = torch.cat([torch.zeros(S, N, 1), torch.rand(S, N, 2, generator=g) * 255], -1).cuda()
  a = streaming.OnlineTracker(model, H, W, N, num_streams=S, yuv420=True, window=window)
  b = streaming.OnlineTracker(model, 256, 256, N, uint8_frames=True, num_streams=S)
  try:
    a.init(frame(0), qp)
    b.init(live.yuv420_to_rgb(frame(0)), qp)
    for t in range(6):
      if t == 3:
        s = S - 1
        p = torch.tensor([0., 100., 60.]).cuda()
        a.update_query(frame(t, s), p, 2, stream=s)
        b.update_query(live.yuv420_to_rgb(frame(t, s))[0, 0], p, 2, stream=s)
      ta, va = (x.clone() for x in a.step(frame(t)))
      tb, vb = (x.clone() for x in b.step(live.yuv420_to_rgb(frame(t))))
      assert torch.equal(ta, tb) and torch.equal(va, vb), t
      for x, y in zip(a.last_logits, b.last_logits):
        assert torch.equal(x, y), t
    with pytest.raises(ValueError):
      a.step(frame(0).with_window(None))        # another window than the tracker's
    with pytest.raises(ValueError):
      a.step(live.yuv420_to_rgb(frame(0)))      # not YUV
  finally:
    a.close()
    b.close()


def test_no_extra_launch_at_model_resolution():
  model, _, _ = get_model()
  lib = _lib.load()
  frames, _ = make_frames(1, 2, 256, 256, 'i420', seed=7)
  rgb = live.yuv420_to_rgb(frames)
  model.get_feature_grids(frames, False)  # workspaces and packed weights exist
  model.get_feature_grids(rgb, False)
  n0 = lib.tapir_launch_count()
  model.get_feature_grids(frames, False)
  n1 = lib.tapir_launch_count()
  model.get_feature_grids(rgb, False)
  n2 = lib.tapir_launch_count()
  assert n1 - n0 == n2 - n1 > 0


def test_c_abi_rejects_bad_descriptors():
  lib = _lib.load()
  frames, _ = make_frames(1, 1, 16, 16, 'nv12', seed=8)
  out = torch.empty(1, 16, 16, 3, dtype=torch.uint8, device='cuda')
  s = torch.cuda.current_stream().cuda_stream
  for field, value in [('chroma_step', 3), ('matrix', 2020), ('h', 0), ('x0', 1), ('full_range', 2)]:
    d = frames.c_struct()
    setattr(d, field, value)
    assert lib.tapir_yuv420_to_rgb(d, 1, out.data_ptr(), s) == 1, field
    assert lib.tapir_last_error()
  assert lib.tapir_ingest_frames_yuv420(None, 1, out.data_ptr(), 8, 8, s) == 1
