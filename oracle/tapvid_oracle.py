"""TEST INFRASTRUCTURE - numpy restatement of the TAP-Vid evaluation front end's arithmetic.

* `lanczos_weights` / `resize`: PIL's 8-bit Lanczos resize (Image.resize(..., LANCZOS) on a uint8
  RGB image, which is what mediapy.resize_video runs per uint8 frame), in int64: per axis
  (in -> out) scale = in / out, fs = max(scale, 1), support = 3 fs, ksize = 2 ceil(support) + 1;
  output o reads xmin = max(0, (int)(c - support + 0.5)) .. min(in, (int)(c + support + 0.5)) - 1,
  c = (o + 0.5) scale, with taps lanczos((i + xmin - c + 0.5) * (1 / fs)) normalised by their
  sequential sum and rounded half away from zero to 22 fraction bits; a pass is
  clamp((2^21 + sum src * tap) >> 22, 0, 255); horizontal first (uint8 in between), each pass
  only when its size changes.  The taps are computed in float64 with np.sin, which agrees with
  libm's sin (the C ABI's `tapir_lanczos_weights`) on the arguments used here; the fixture's PIL
  outputs pin the whole restatement.
* `mean_scalars`: the dataset mean of the reference's evaluation loop
  (training/supervised_point_prediction.py:937-948): per-video scalars as float32, summed in video
  order in float32, divided by the video count.
"""
import math

import numpy as np

PRECISION_BITS = 22


def _sinc(x):
  xp = x * math.pi
  with np.errstate(invalid='ignore', divide='ignore'):
    return np.where(x == 0.0, 1.0, np.sin(xp) / xp)


def _lanczos(x):
  return np.where((-3.0 <= x) & (x < 3.0), _sinc(x) * _sinc(x / 3), 0.0)


def lanczos_weights(in_size, out_size):
  """int64 bounds [out_size, 2] (xmin, n) and taps [out_size, ksize] of one axis."""
  scale = in_size / out_size
  fs = max(scale, 1.0)
  ss = 1.0 / fs
  support = 3.0 * fs
  ksize = int(math.ceil(support)) * 2 + 1
  center = (np.arange(out_size, dtype=np.float64) + 0.5) * scale
  xmin = np.maximum(np.trunc(center - support + 0.5), 0).astype(np.int64)
  xmax = np.minimum(np.trunc(center + support + 0.5), in_size).astype(np.int64)
  n = xmax - xmin
  i = np.arange(ksize)
  x = ((i[None, :] + xmin[:, None]).astype(np.float64) - center[:, None] + 0.5) * ss
  k = np.where(i[None, :] < n[:, None], _lanczos(x), 0.0)
  ww = np.zeros(out_size)
  for j in range(ksize):  # C's left-to-right sum, not numpy's pairwise one
    ww = ww + k[:, j]
  k = np.where(ww[:, None] != 0.0, k / np.where(ww == 0.0, 1.0, ww)[:, None], k)
  scaled = k * (1 << PRECISION_BITS)
  taps = np.where(k < 0, np.trunc(-0.5 + scaled), np.trunc(0.5 + scaled)).astype(np.int64)
  return np.stack([xmin, n], -1), taps


def _pass(img, axis, out_size):
  in_size = img.shape[axis]
  bounds, taps = lanczos_weights(in_size, out_size)
  shape = [1] * img.ndim
  shape[axis] = out_size
  acc = np.full(img.shape[:axis % img.ndim] + (out_size,) + img.shape[axis % img.ndim + 1:],
                1 << (PRECISION_BITS - 1), np.int64)
  for i in range(taps.shape[1]):
    idx = np.minimum(bounds[:, 0] + i, in_size - 1)
    k = np.where(i < bounds[:, 1], taps[:, i], 0).reshape(shape)
    acc += np.take(img, idx, axis=axis).astype(np.int64) * k
  return np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)


def resize(frames, h, w):
  """uint8 [..., H, W, C] -> [..., h, w, C]."""
  out = np.asarray(frames)
  if out.shape[-2] != w:
    out = _pass(out, -2, w)
  if out.shape[-3] != h:
    out = _pass(out, -3, h)
  return out.copy() if out is frames else out


def mean_scalars(per_video):
  """float32 dataset mean of a list of per-video {name: scalar} dicts, in list order."""
  n = np.float32(len(per_video))
  return {k: np.cumsum(np.array([m[k] for m in per_video], np.float32), dtype=np.float32)[-1] / n
          for k in per_video[0]}
