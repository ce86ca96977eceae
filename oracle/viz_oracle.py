"""CPU oracle of the point-track painting (tapnet/utils/viz_utils.py:47-124 paint_point_track),
restated in numpy one point at a time.

The semantics the CUDA kernels reproduce bit for bit:
  * radius r = int(round(min(H, W) * 0.015)) (float64, round half to even);
  * the icon is (2r+1)^2 values 1 - clip((dy^2 + dx^2 - r^2 / 2.0) / (2r * 0.15), 0, 1) at offsets
    dy, dx in -r-1 .. r-1 (the reference's centre is one pixel off; kept).  r = 0 divides by zero:
    the icon is all zeros and nothing is painted;
  * a visible point's centre is track + 0.5 in the tracks' dtype, clamped as
    min(max(v, 0.0), size); (x1, y1) = floor of it.  Its (2r+2)^2 patch mixes four copies of the
    icon, padded on the bottom/right, top/right, bottom/left and top/left, with the weights
    (x1+1-x)(y1+1-y), (x1+1-x)(y-y1), (x-x1)(y1+1-y) and (x-x1)(y-y1), evaluated as
    ((icon * wx) * wy) summed left to right, and covers rows y1-r-1 .. y1+r and the same columns;
  * every pixel under the patch becomes uint8(trunc((1 - p) v + p c)) in float64, points in index
    order, so each blend starts from the previous truncated value.
Points with a NaN coordinate are skipped (the reference's floor(nan).astype(int32) is undefined).
"""
import math

import numpy as np

DOT_FRACTION = 0.015
SHARPNESS = 0.15


def radius(H, W):
  return int(round(min(H, W) * DOT_FRACTION))


def icon(r):
  """[2r+1, 2r+1] float64 dot; all zeros at r = 0."""
  off = np.arange(2 * r + 1) - r - 1
  q = (off[:, None] ** 2 + off[None, :] ** 2) - r * r / 2.0
  with np.errstate(divide='ignore', invalid='ignore'):
    return 1 - np.clip(q / (r * 2 * SHARPNESS), 0, 1)


def _shifted_icons(r):
  """The four (2r+2)^2 copies of the icon: padded bottom/right, top/right, bottom/left, top/left."""
  ic = icon(r)
  d = 2 * r + 2
  out = np.zeros((4, d, d))
  out[0, :-1, :-1] = ic
  out[1, 1:, :-1] = ic
  out[2, :-1, 1:] = ic
  out[3, 1:, 1:] = ic
  return out


def _clamp(v, size):
  return min(max(float(v), 0.0), float(size))


def paint_point_track(frames, point_tracks, visibles, colormap):
  """frames [T, H, W, 3] uint8, point_tracks [N, T, 2] (x, y), visibles [N, T], colormap >= N
  (r, g, b) integer triples -> painted copy of frames."""
  frames = np.asarray(frames)
  tracks = np.asarray(point_tracks)
  visibles = np.asarray(visibles)
  T, H, W = frames.shape[:3]
  N = tracks.shape[0]
  video = frames.copy()
  if N == 0 or T == 0:
    return video
  r = radius(H, W)
  i1, i2, i3, i4 = _shifted_icons(r)
  d = 2 * r + 2
  colors = np.asarray(colormap[:N], dtype=np.float64).reshape(N, 3)
  for t in range(T):
    image = video[t]
    for i in range(N):
      if not visibles[i, t]:
        continue
      xy = tracks[i, t] + 0.5           # in the tracks' dtype (float32 + 0.5 stays float32)
      x, y = _clamp(xy[0], W), _clamp(xy[1], H)
      if math.isnan(x) or math.isnan(y):
        continue
      x1, y1 = math.floor(x), math.floor(y)
      wx1, wx2 = x - x1, (x1 + 1) - x
      wy1, wy2 = y - y1, (y1 + 1) - y
      patch = i1 * wx2 * wy2 + i2 * wx2 * wy1 + i3 * wx1 * wy2 + i4 * wx1 * wy1
      # patch row a covers frame row y1 - r - 1 + a; keep the rows / columns inside the frame
      top, left = y1 - r - 1, x1 - r - 1
      ra, rb = max(0, -top), min(d, H - top)
      ca, cb = max(0, -left), min(d, W - left)
      if ra >= rb or ca >= cb:
        continue
      p = patch[ra:rb, ca:cb, None]
      window = image[top + ra:top + rb, left + ca:left + cb]
      blended = (1 - p) * window + p * colors[i]
      window[...] = np.trunc(blended).astype(np.uint8)  # blends stay in (-1, 256)
  return video

