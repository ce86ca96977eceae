"""CPU: the numpy restatement of paint_point_track (oracle/viz_oracle.py) and viz.get_colors
against fixtures made by the reference's own functions (oracle/make_golden_viz.py), and the
argument checks of viz.paint_point_track, which run before any CUDA call."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import viz_oracle
from tapnet_b200 import _lib, viz

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'io_viz.npz')
CASES = [str(c) for c in np.load(GOLDEN)['cases']]


@pytest.fixture(scope='module')
def golden():
  return np.load(GOLDEN)


@pytest.mark.parametrize('case', CASES)
def test_oracle_matches_reference(golden, case):
  g = {k: golden[f'{case}_{k}'] for k in ('frames', 'tracks', 'visibles', 'colors', 'out')}
  out = viz_oracle.paint_point_track(g['frames'], g['tracks'], g['visibles'], g['colors'])
  np.testing.assert_array_equal(out, g['out'])


def test_fixture_covers_the_listed_cases(golden):
  assert golden['r0_out'].shape == (3, 20, 30, 3)
  np.testing.assert_array_equal(golden['r0_out'], golden['r0_frames'])   # radius 0 paints nothing
  assert golden['f64_480x500_tracks'].dtype == np.float64
  assert golden['f32_256_tracks'].dtype == np.float32
  assert golden['n0_tracks'].shape[0] == 0 and golden['t1_frames'].shape[0] == 1
  assert not golden['invisible_visibles'].any()
  tr = golden['designed_tracks']
  assert np.isinf(tr).any() and (tr < 0).any() and (tr[..., 0] > 240).any()
  colors = golden['designed_colors']
  assert (colors == 0).all(-1).any() and (colors == 255).all(-1).any()


@pytest.mark.parametrize('key', [k for k in np.load(GOLDEN).files if k.startswith('colors_')])
def test_get_colors_matches_reference(golden, key):
  n, seed = (int(v) for v in key[len('colors_'):].split('_seed'))
  np.random.seed(seed)
  random.seed(seed)
  got = viz.get_colors(n)
  assert all(isinstance(v, int) for c in got for v in c)
  np.testing.assert_array_equal(np.array(got, np.int64), golden[key])


@pytest.mark.parametrize('edge,r', [(33, 0), (34, 1), (100, 2), (167, 3), (300, 4), (500, 8),
                                    (1024, 15)])
def test_radius_rule(edge, r):
  # float64 product, round half to even: 100 * 0.015 = 1.5 -> 2, 300 * 0.015 = 4.5 -> 4
  assert viz_oracle.radius(edge, edge + 7) == r
  assert viz_oracle.radius(edge + 50, edge) == r


def _args(T=2, H=24, W=30, N=3):
  frames = np.zeros((T, H, W, 3), np.uint8)
  tracks = np.full((N, T, 2), 5.0, np.float32)
  vis = np.ones((N, T), bool)
  return frames, tracks, vis


@pytest.fixture
def no_cuda_calls(monkeypatch):
  """Fails the test if the wrapper reaches CUDA or the library."""
  def boom(*a, **k):
    raise AssertionError('CUDA reached before the arguments were checked')
  monkeypatch.setattr(torch.cuda, 'is_available', boom)
  monkeypatch.setattr(torch.cuda, 'current_device', boom)
  monkeypatch.setattr(_lib, 'load', boom)


@pytest.mark.parametrize('bad', ['frames_dtype', 'frames_rank', 'frames_channels', 'tracks_frames',
                                 'tracks_last', 'tracks_dtype', 'visibles_shape', 'colormap_short',
                                 'colormap_high', 'colormap_negative', 'colormap_fraction',
                                 'colormap_nan', 'colormap_width', 'colormap_strings'])
def test_argument_errors_before_cuda(no_cuda_calls, bad):
  frames, tracks, vis = _args()
  colormap = [(1, 2, 3)] * 3
  if bad == 'frames_dtype':
    frames = frames.astype(np.float32)
  elif bad == 'frames_rank':
    frames = frames[0]
  elif bad == 'frames_channels':
    frames = np.zeros((2, 24, 30, 4), np.uint8)
  elif bad == 'tracks_frames':
    tracks = tracks[:, :1]
  elif bad == 'tracks_last':
    tracks = np.zeros((3, 2, 3), np.float32)
  elif bad == 'tracks_dtype':
    tracks = tracks.astype(np.float16)
  elif bad == 'visibles_shape':
    vis = vis.T
  elif bad == 'colormap_short':
    colormap = colormap[:2]
  elif bad == 'colormap_high':
    colormap = [(1, 2, 256)] * 3
  elif bad == 'colormap_negative':
    colormap = [(1, -1, 3)] * 3
  elif bad == 'colormap_fraction':
    colormap = [(1, 2, 3.5)] * 3
  elif bad == 'colormap_nan':
    colormap = [(1, 2, float('nan'))] * 3
  elif bad == 'colormap_width':
    colormap = [(1, 2)] * 3
  elif bad == 'colormap_strings':
    colormap = [('a', 'b', 'c')] * 3
  with pytest.raises(ValueError):
    viz.paint_point_track(frames, tracks, vis, colormap)


def test_valid_arguments_without_cuda_raise():
  if torch.cuda.is_available():
    pytest.skip('a CUDA device is present')
  frames, tracks, vis = _args()
  with pytest.raises(RuntimeError):
    viz.paint_point_track(frames, tracks, vis)
