"""Painting point tracks onto video frames on the GPU (the step after the path, DESIGN f5).

Same names as `tapnet/utils/viz_utils.py`, so the colab call becomes

    from tapnet_b200 import viz
    video = viz.paint_point_track(frames, tracks, visibles[, colormap])

and returns, bit for bit, what the reference's numpy function returns (two CUDA launches,
`tapir_paint_point_track`).  numpy inputs are copied to the current CUDA device and the result is
copied back; with CUDA tensor frames the result is a CUDA tensor on the frames' device, painted on
its current stream without a host sync, so the model's `tracks[0]` / `visibles[0]` go straight in.

Differences from the reference: N = 0 returns a copy of the frames (the reference's default
colormap divides by zero there); points with a NaN coordinate are not painted (undefined in the
reference); the frame count of `frames` and `point_tracks` must agree.
"""
import colorsys
import random

import numpy as np
import torch

from tapnet_b200 import _lib


def get_colors(num_colors):
  """The reference's default colormap, drawing from the same global random state: hues evenly
  spaced by np.arange(0, 360, 360 / num_colors) (which can give one hue more than asked), each
  with lightness 0.5 + 0.1 u and saturation 0.9 + 0.1 u from two np.random.rand() draws (lightness
  first), converted from HLS and truncated to int after * 255; then shuffled by `random.shuffle`.
  Returns a list of (r, g, b) int tuples."""
  hues = np.arange(0.0, 360.0, 360.0 / num_colors)
  draws = np.random.rand(len(hues), 2)   # the same stream as 2 * len(hues) scalar draws
  lightness = (50 + draws[:, 0] * 10) / 100.0
  saturation = (90 + draws[:, 1] * 10) / 100.0
  colors = []
  for h, l, s in zip(hues / 360.0, lightness, saturation):
    colors.append(tuple(int(c * 255) for c in colorsys.hls_to_rgb(float(h), float(l), float(s))))
  random.shuffle(colors)
  return colors


def _shape(x):
  return tuple(int(v) for v in x.shape)


def _check_colormap(colormap, N):
  try:
    cm = np.asarray(colormap[:N] if N else [])
  except TypeError as e:
    raise ValueError(f'paint_point_track: colormap must be a sequence of (r, g, b): {e}') from None
  if N == 0:
    return np.zeros((0, 3), np.uint8)
  if cm.ndim != 2 or cm.shape != (N, 3):
    raise ValueError(f'paint_point_track: colormap needs at least {N} (r, g, b) entries, '
                     f'got {len(colormap)} of shape {cm.shape[1:]}')
  if cm.dtype.kind not in 'biuf':
    raise ValueError(f'paint_point_track: colormap entries must be integers, got {cm.dtype}')
  if not (np.all(np.isfinite(cm)) and np.all(cm == np.round(cm)) and cm.min() >= 0 and cm.max() <= 255):
    raise ValueError('paint_point_track: colormap entries must be integers in 0..255')
  return cm.astype(np.uint8)


def _track_dtype(dtype, is_torch):
  """float32 / float64 stay (the + 0.5 is taken in that dtype); integers become float64 as numpy
  promotes them."""
  if is_torch:
    if dtype in (torch.float32, torch.float64):
      return dtype
    if not dtype.is_floating_point and not dtype.is_complex and dtype != torch.bool:
      return torch.float64
  else:
    if dtype in (np.float32, np.float64):
      return dtype
    if dtype.kind in 'iu':
      return np.float64
  raise ValueError(f'paint_point_track: point_tracks must be float32, float64 or integer, got {dtype}')


def paint_point_track(frames, point_tracks, visibles, colormap=None):
  """frames [T, H, W, 3] uint8, point_tracks [N, T, 2] (x, y in pixels), visibles [N, T] bool,
  colormap: at least N (r, g, b) integer triples in 0..255 (default get_colors(N)).

  Returns the painted video [T, H, W, 3] uint8: a numpy array for numpy frames, a CUDA tensor on
  the frames' device for CUDA frames.  The input is never modified."""
  on_device = isinstance(frames, torch.Tensor) and frames.is_cuda
  if on_device:
    if frames.dtype != torch.uint8:
      raise ValueError(f'paint_point_track: frames must be uint8, got {frames.dtype}')
    tracks = point_tracks if isinstance(point_tracks, torch.Tensor) else torch.as_tensor(np.asarray(point_tracks))
    vis = visibles if isinstance(visibles, torch.Tensor) else torch.as_tensor(np.asarray(visibles))
  else:
    frames = np.asarray(frames)
    if frames.dtype != np.uint8:
      raise ValueError(f'paint_point_track: frames must be uint8, got {frames.dtype}')
    tracks = np.asarray(point_tracks)
    vis = np.asarray(visibles)
  if frames.ndim != 4 or frames.shape[3] != 3:
    raise ValueError(f'paint_point_track: frames must be [T, H, W, 3], got {_shape(frames)}')
  T, H, W = _shape(frames)[:3]
  if tracks.ndim != 3 or tracks.shape[2] != 2 or tracks.shape[1] != T:
    raise ValueError(f'paint_point_track: point_tracks must be [N, {T}, 2], got {_shape(tracks)}')
  N = int(tracks.shape[0])
  if _shape(vis) != (N, T):
    raise ValueError(f'paint_point_track: visibles must be [{N}, {T}], got {_shape(vis)}')
  tdtype = _track_dtype(tracks.dtype, isinstance(tracks, torch.Tensor))
  if max(T, H, W, N) >= 1 << 31:
    raise ValueError('paint_point_track: sizes must fit int32')
  if colormap is None:
    colormap = get_colors(N) if N else []
  colors = _check_colormap(colormap, N)
  if not torch.cuda.is_available():
    raise RuntimeError('paint_point_track needs a CUDA device (tapnet_b200 has no CPU fallback)')

  dev = frames.device if on_device else torch.device('cuda', torch.cuda.current_device())
  frames_d = _to_device(frames, dev)
  tracks_d = _to_device(tracks, dev).to(_torch_dtype(tdtype)).contiguous()
  vis_d = (_to_device(vis, dev) != 0).contiguous()   # bool: one byte, 0 / 1
  colors_d = _to_device(colors, dev)
  out = torch.empty_like(frames_d)
  with torch.cuda.device(dev):
    ws_bytes = _lib.paint_point_track_workspace_bytes(T, N)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)[:ws_bytes]
    _lib.paint_point_track(frames_d, tracks_d, vis_d, colors_d, out, ws)
  return out if on_device else out.cpu().numpy()


def _to_device(x, dev):
  """Host data goes through pinned memory with a stream-ordered copy, so that painting CUDA frames
  with host-side tracks or colours does not wait for the device."""
  if isinstance(x, torch.Tensor) and x.is_cuda:
    return x.to(dev).contiguous()
  t = torch.as_tensor(np.ascontiguousarray(x))
  return t.pin_memory().to(dev, non_blocking=True)


def _torch_dtype(dtype):
  if isinstance(dtype, torch.dtype):
    return dtype
  return torch.float64 if np.dtype(dtype) == np.float64 else torch.float32
