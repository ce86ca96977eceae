"""-m gpu: viz.paint_point_track (tapir_paint_point_track) against the reference-generated fixture
and the numpy oracle, bit for bit everywhere."""
import ctypes
import os
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import synth, viz_oracle  # noqa: E402
from tapnet_b200 import _lib, live, viz  # noqa: E402
from tests.test_stages_gpu import get_model  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'io_viz.npz')
CASES = [str(c) for c in np.load(GOLDEN)['cases']]


def _case(name):
  g = np.load(GOLDEN)
  return {k: g[f'{name}_{k}'] for k in ('frames', 'tracks', 'visibles', 'colors', 'out')}


def _random_case(seed, T, H, W, N, dtype):
  rng = np.random.default_rng(seed)
  frames = rng.integers(0, 256, (T, H, W, 3), dtype=np.uint8)
  tracks = np.stack([rng.uniform(-0.05 * W, 1.05 * W, (N, T)),
                     rng.uniform(-0.05 * H, 1.05 * H, (N, T))], -1).astype(dtype)
  vis = rng.uniform(size=(N, T)) < 0.8
  colors = rng.integers(0, 256, (N, 3), dtype=np.uint8)
  return frames, tracks, vis, colors


@pytest.mark.parametrize('case', CASES)
def test_fixture_numpy(case):
  g = _case(case)
  frames = g['frames'].copy()
  out = viz.paint_point_track(frames, g['tracks'], g['visibles'], g['colors'])
  assert isinstance(out, np.ndarray) and out.dtype == np.uint8
  np.testing.assert_array_equal(out, g['out'])
  np.testing.assert_array_equal(frames, g['frames'])   # the input is not modified


@pytest.mark.parametrize('case', CASES)
def test_fixture_cuda_tensors(case):
  g = _case(case)
  frames = torch.from_numpy(g['frames']).cuda()
  before = frames.clone()
  out = viz.paint_point_track(frames, torch.from_numpy(g['tracks']).cuda(),
                              torch.from_numpy(g['visibles']).cuda(),
                              [tuple(c) for c in g['colors'].tolist()])
  assert out.is_cuda and out.device == frames.device and out.dtype == torch.uint8
  np.testing.assert_array_equal(out.cpu().numpy(), g['out'])
  assert torch.equal(frames, before)


@pytest.mark.parametrize('shape', [(48, 256, 256, 256, np.float32), (4, 1024, 1024, 2048, np.float32),
                                   (2, 720, 1280, 300, np.float64)])
def test_random_vs_oracle(shape):
  frames, tracks, vis, colors = _random_case(7, *shape)
  ref = viz_oracle.paint_point_track(frames, tracks, vis, colors)
  out = viz.paint_point_track(torch.from_numpy(frames).cuda(), torch.from_numpy(tracks).cuda(),
                              torch.from_numpy(vis).cuda(), colors)
  np.testing.assert_array_equal(out.cpu().numpy(), ref)


@pytest.mark.parametrize('edge', [33, 34, 100, 167, 300, 500, 1024])
def test_radius_edges_vs_oracle(edge):
  """The radius rule (round half to even) at the edges where it changes or is exactly .5."""
  frames, tracks, vis, colors = _random_case(edge, 1, edge, edge + 13, 40, np.float32)
  ref = viz_oracle.paint_point_track(frames, tracks, vis, colors)
  np.testing.assert_array_equal(viz.paint_point_track(frames, tracks, vis, colors), ref)


def test_thousands_of_points_on_one_pixel():
  """5000 points over one pixel (several rounds of the CTA's hit list), distinct colours, with
  far-away points interleaved in the index order."""
  T, H, W, N = 2, 256, 256, 5000
  rng = np.random.default_rng(3)
  frames = rng.integers(0, 256, (T, H, W, 3), dtype=np.uint8)
  tracks = np.empty((N, T, 2), np.float32)
  tracks[:] = np.float32([100.3, 50.7])
  tracks[::7] = rng.uniform(0, 256, (len(tracks[::7]), T, 2)).astype(np.float32)
  tracks[1::2, 1] += rng.uniform(-1, 1, (len(tracks[1::2]), 2)).astype(np.float32)
  vis = np.ones((N, T), bool)
  vis[::11, 0] = False
  idx = np.arange(N)
  colors = np.stack([idx % 256, (idx // 256) * 13 % 256, (idx * 7) % 256], -1).astype(np.uint8)
  ref = viz_oracle.paint_point_track(frames, tracks, vis, colors)
  out = viz.paint_point_track(torch.from_numpy(frames).cuda(), torch.from_numpy(tracks).cuda(),
                              torch.from_numpy(vis).cuda(), colors)
  np.testing.assert_array_equal(out.cpu().numpy(), ref)


def test_all_points_invisible():
  frames, tracks, vis, colors = _random_case(4, 3, 200, 300, 500, np.float32)
  out = viz.paint_point_track(frames, tracks, np.zeros_like(vis), colors)
  np.testing.assert_array_equal(out, frames)


def test_end_to_end_model_tracks():
  """model(video, queries) on the device, its tracks[0] / visibles[0] painted straight from the
  device == the oracle on the same tracks copied to the host."""
  model, _, _ = get_model()
  T, N = 6, 32
  video = synth.make_video(T)
  q = synth.make_queries(N, T)
  out = model(video.cuda(), q.cuda())
  tracks = out['tracks'][0]
  # The seeded random weights leave every point occluded under the 0.5 visibility rule, so the
  # occlusion logits are cut at their median instead (about half the points paint).
  occ = out['occlusion'][0]
  visibles = occ < occ.median()
  video_u8 = ((video[0] + 1) * 127.5).round().clamp(0, 255).to(torch.uint8).cuda()
  np.random.seed(0)
  random.seed(0)
  colors = viz.get_colors(N)
  np.random.seed(0)
  random.seed(0)
  painted = viz.paint_point_track(video_u8, tracks, visibles)   # default colormap, same seeds
  ref = viz_oracle.paint_point_track(video_u8.cpu().numpy(), tracks.cpu().numpy(),
                                     visibles.cpu().numpy(), colors)
  assert tracks.dtype == torch.float32 and bool(visibles.any())
  np.testing.assert_array_equal(painted.cpu().numpy(), ref)
  assert not np.array_equal(ref, video_u8.cpu().numpy())


def test_repeatable_and_side_stream():
  frames, tracks, vis, colors = _random_case(5, 8, 512, 512, 1000, np.float32)
  args = (torch.from_numpy(frames).cuda(), torch.from_numpy(tracks).cuda(), torch.from_numpy(vis).cuda())
  a = viz.paint_point_track(*args, colors)
  b = viz.paint_point_track(*args, colors)
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    c = viz.paint_point_track(*args, colors)
  torch.cuda.current_stream().wait_stream(side)
  assert torch.equal(a, b) and torch.equal(a, c)


def test_c_abi_argument_errors():
  lib = _lib.load()
  T, H, W, N = 2, 40, 50, 4
  frames = torch.zeros(T, H, W, 3, dtype=torch.uint8, device='cuda')
  out = torch.empty_like(frames)
  tracks = torch.zeros(N, T, 2, device='cuda')
  vis = torch.ones(N, T, dtype=torch.uint8, device='cuda')
  colors = torch.zeros(N, 3, dtype=torch.uint8, device='cuda')
  need = lib.tapir_paint_point_track_workspace_bytes(T, N)
  assert need >= T * N * 24 and lib.tapir_paint_point_track_workspace_bytes(T, 0) == 0
  ws = torch.empty(need, dtype=torch.uint8, device='cuda')
  s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
  p = lambda t: t.data_ptr()  # noqa: E731

  def call(frames_p=None, T_=T, H_=H, W_=W, tracks_p=None, fp64=0, N_=N, out_p=None, ws_p=None,
           ws_bytes=need):
    return lib.tapir_paint_point_track(frames_p or p(frames), T_, H_, W_, tracks_p or p(tracks), fp64,
                                       p(vis), N_, p(colors), out_p or p(out), ws_p or p(ws), ws_bytes, s)

  bad = {'negative T': dict(T_=-1), 'negative H': dict(H_=-2), 'negative N': dict(N_=-1),
         'tracks_fp64': dict(fp64=2), 'small workspace': dict(ws_bytes=need - 1),
         'out overlaps frames': dict(out_p=p(frames) + 64), 'out is frames': dict(out_p=p(frames)),
         'misaligned workspace': dict(ws_p=p(ws) + 8, ws_bytes=need)}
  for what, kw in bad.items():
    assert call(**kw) == 1, what
    assert b'tapir_paint_point_track' in lib.tapir_last_error(), what
  assert lib.tapir_paint_point_track(None, T, H, W, p(tracks), 0, p(vis), N, p(colors), p(out), p(ws),
                                     need, s) == 1
  assert lib.tapir_paint_point_track(p(frames), T, H, W, None, 0, p(vis), N, p(colors), p(out), p(ws),
                                     need, s) == 1
  assert call() == 0
  torch.cuda.synchronize()
  assert torch.equal(out, frames)
