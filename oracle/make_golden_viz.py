"""TEST INFRASTRUCTURE - generates tests/golden/io_viz.npz by executing the reference's own
paint_point_track and get_colors (tapnet/utils/viz_utils.py:32-124).

Needs a checkout of the reference (oracle/reference_loader.py, TAPNET_REFERENCE_ROOT):
  python -m oracle.make_golden_viz

viz_utils.py imports jax, matplotlib and mediapy (absent here), so its FunctionDefs are compiled
unmodified by make_golden_io.reference_functions.  The fixture holds inputs and the reference's
outputs only.  Frames are blockwise ramps so the file compresses.
"""
import colorsys
import os
import random
from typing import List, Optional, Tuple

import numpy as np

from oracle import reference_loader
from oracle.make_golden_io import GOLDEN_DIR, reference_functions

# (name, T, H, W, N, tracks dtype)
RANDOM_CASES = [
    ('r0', 3, 20, 30, 6, np.float32),          # radius 0: the output equals the input
    ('r1', 2, 64, 96, 10, np.float32),         # radius 1
    ('half_even_100', 2, 100, 130, 12, np.float32),  # 1.5 -> 2
    ('half_even_300', 1, 300, 310, 16, np.float32),  # 4.5 -> 4
    ('f32_256', 3, 256, 256, 40, np.float32),
    ('f64_480x500', 2, 480, 500, 30, np.float64),
]


def smooth_frames(T, H, W, seed):
  """Constant over 4 x 4 pixel blocks, ramping from block to block."""
  y, x = np.mgrid[0:H, 0:W] // 4
  out = np.empty((T, H, W, 3), np.uint8)
  for t in range(T):
    for c in range(3):
      out[t, ..., c] = (x * (3 * c + 5) + y * (11 - 3 * c) + 37 * t + 80 * c + seed) % 256
  return out


def random_case(rng, T, H, W, N, dtype):
  tracks = np.stack([rng.uniform(-0.1 * W, 1.1 * W, (N, T)),
                     rng.uniform(-0.1 * H, 1.1 * H, (N, T))], -1).astype(dtype)
  visibles = rng.uniform(size=(N, T)) < 0.8
  colors = rng.integers(0, 256, (N, 3), dtype=np.uint8)
  return tracks, visibles, colors


def designed_case(rng):
  """Positions on pixel centres and corners, exactly 0 / W / H, negative, beyond, +-inf; a cluster
  of overlapping points of different colours; colours 0 and 255; some invisible points."""
  T, H, W = 2, 200, 240   # radius 3
  pts = [(10.5, 20.5), (33.0, 44.0), (0.0, 0.0), (float(W), float(H)), (0.0, float(H)),
         (float(W), 0.0), (-0.5, 50.0), (-0.5001, 60.25), (-3.0, -7.0), (W + 5.0, H + 9.0),
         (W - 0.5, H - 0.5), (np.inf, 100.0), (-np.inf, 120.0), (50.0, np.inf), (60.0, -np.inf),
         (np.inf, np.inf), (W - 0.75, 3.3), (1e9, -1e9)]
  cluster = [(120.0 + dx, 100.0 + dy) for dx, dy in rng.uniform(-2.5, 2.5, (12, 2))]
  pts += cluster
  N = len(pts)
  tracks = np.empty((N, T, 2), np.float32)
  tracks[:, 0] = np.array(pts, np.float32)
  tracks[:, 1] = np.array(pts, np.float32) + np.float32(0.25)
  visibles = np.ones((N, T), bool)
  visibles[3, 1] = visibles[7, 0] = visibles[20, 1] = False
  colors = rng.integers(1, 255, (N, 3), dtype=np.uint8)
  colors[0] = (0, 0, 0)
  colors[1] = (255, 255, 255)
  colors[len(pts) - len(cluster):] = rng.integers(0, 256, (len(cluster), 3), dtype=np.uint8)
  colors[-1] = (255, 0, 255)
  colors[-2] = (0, 255, 0)
  return smooth_frames(T, H, W, 9), tracks, visibles, colors


def main():
  scope = dict(np=np, colorsys=colorsys, random=random, List=List, Optional=Optional, Tuple=Tuple)
  get_colors, paint_point_track = reference_functions(
      'tapnet/utils/viz_utils.py', ['get_colors', 'paint_point_track'], scope)
  rng = np.random.default_rng(17)
  out = {}
  cases = []
  for k, (name, T, H, W, N, dtype) in enumerate(RANDOM_CASES):
    tracks, visibles, colors = random_case(rng, T, H, W, N, dtype)
    cases.append((name, smooth_frames(T, H, W, k), tracks, visibles, colors))
  cases.append(('designed',) + designed_case(rng))
  tracks, visibles, colors = random_case(rng, 3, 40, 50, 5, np.float32)
  cases.append(('invisible', smooth_frames(3, 40, 50, 3), tracks, np.zeros_like(visibles), colors))
  cases.append(('n0', smooth_frames(2, 40, 50, 4), np.zeros((0, 2, 2), np.float32),
                np.zeros((0, 2), bool), np.zeros((0, 3), np.uint8)))
  tracks, visibles, colors = random_case(rng, 1, 72, 80, 9, np.float64)
  cases.append(('t1', smooth_frames(1, 72, 80, 5), tracks, visibles, colors))
  names = []
  for name, frames, tracks, visibles, colors in cases:
    colormap = [tuple(int(v) for v in c) for c in colors]
    with np.errstate(divide='ignore', invalid='ignore'):
      painted = paint_point_track(frames, tracks, visibles, colormap)
    assert painted.dtype == np.uint8 and painted.shape == frames.shape
    out.update({f'{name}_frames': frames, f'{name}_tracks': tracks,
                f'{name}_visibles': visibles, f'{name}_colors': colors, f'{name}_out': painted})
    names.append(name)
  out['cases'] = np.array(names)
  # get_colors under fixed seeds; at 161 colours np.arange yields one extra hue
  for n, seed in ((1, 0), (7, 1), (20, 2), (161, 3), (256, 4)):
    np.random.seed(seed)
    random.seed(seed)
    out[f'colors_{n}_seed{seed}'] = np.array(get_colors(n), np.int64)
  np.savez_compressed(os.path.join(GOLDEN_DIR, 'io_viz.npz'), **out)
  print('io_viz.npz', names)


if __name__ == '__main__':
  reference_loader.load()
  main()
