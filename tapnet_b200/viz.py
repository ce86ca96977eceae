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

`get_homographies_wrt_frame` is the rainbow demo's camera-motion step (DESIGN f8): one homography
per frame into the reference frame, each track's squared distance to its canonical point per
frame, and the canonical points, in float64 on the GPU (`tapir_homographies_wrt_frame`).
`foreground_tracks` is the demo's last step: the tracks that do not follow the camera.
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


def _host(x):
  return np.asarray(x.detach().cpu() if isinstance(x, torch.Tensor) else x)


def get_homographies_wrt_frame(pts, occ, image_dimensions, reference_frame=None, thresh=0.07,
                               outlier_point_threshold=0.95, targ_inlier_frac=0.7,
                               num_refinement_passes=2, *, return_ransac_stats=False):
  """viz_utils.get_homographies_wrt_frame on the GPU: pts [N, T, 2] (x, y pixels, float32 or
  float64), occ [N, T] (bool or 0 / 1; read as occ != 0), image_dimensions (width, height).

  Returns (homogs [T, 3, 3], err [N, T], canonical_pts [N, 2]), float64: numpy arrays for numpy
  input, CUDA tensors on the input's device (computed on its current stream, no host sync) for
  CUDA tensors.  With return_ransac_stats, a fourth value [T, 2] int32 holds each frame's RANSAC
  hypotheses evaluated and best inlier count (0 / 0 for the reference frame and frames with <= 4
  usable points).  RANSAC and the re-initialisation of canonical points draw from a fixed
  generator, so the result is a function of the inputs (DESIGN f8)."""
  fn = 'get_homographies_wrt_frame'
  on_device = isinstance(pts, torch.Tensor) and pts.is_cuda
  if not on_device:
    pts = _host(pts)
    occ = _host(occ)
  if pts.ndim != 3 or pts.shape[2] != 2 or pts.shape[0] < 1 or pts.shape[1] < 1:
    raise ValueError(f'{fn}: pts must be [N, T, 2] with N, T >= 1, got {_shape(pts)}')
  N, T = _shape(pts)[:2]
  if _shape(occ) != (N, T):
    raise ValueError(f'{fn}: occ must be [{N}, {T}], got {_shape(occ)}')
  if on_device:
    if not (isinstance(occ, torch.Tensor) and occ.device == pts.device):
      raise ValueError(f'{fn}: occ must be a tensor on {pts.device}')
    if pts.dtype not in (torch.float32, torch.float64):
      raise ValueError(f'{fn}: pts must be float32 or float64, got {pts.dtype}')
    if occ.dtype.is_complex:
      raise ValueError(f'{fn}: occ must be bool or real, got {occ.dtype}')
  else:
    if pts.dtype.kind not in 'fiu':
      raise ValueError(f'{fn}: pts must be real, got {pts.dtype}')
    if pts.dtype not in (np.float32, np.float64):
      pts = pts.astype(np.float64)
    if occ.dtype.kind not in 'biuf' or not np.all((occ == 0) | (occ == 1)):
      raise ValueError(f'{fn}: occ must hold only 0 / 1 (the reference computes 1 - occ)')
  dims = [float(v) for v in image_dimensions]
  if len(dims) != 2 or not all(np.isfinite(v) and v > 0 for v in dims):
    raise ValueError(f'{fn}: image_dimensions must be (width, height) > 0, got {image_dimensions}')
  ref = T // 2 if reference_frame is None else int(reference_frame)
  if not 0 <= ref < T:
    raise ValueError(f'{fn}: reference_frame {reference_frame} outside [0, {T})')
  for name, v in (('thresh', thresh), ('outlier_point_threshold', outlier_point_threshold),
                  ('targ_inlier_frac', targ_inlier_frac)):
    if not (np.isfinite(float(v)) and float(v) > 0):
      raise ValueError(f'{fn}: {name} must be positive, got {v}')
  passes = int(num_refinement_passes)
  if passes < 0 or passes != num_refinement_passes:
    raise ValueError(f'{fn}: num_refinement_passes must be an integer >= 0, got {num_refinement_passes}')
  if max(N, T) >= 1 << 31 or N * T > 1 << 30:
    raise ValueError(f'{fn}: {N} x {T} tracks exceed one call (N T <= 2^30)')
  thr = _lib.ransac_stop_thresholds(N, targ_inlier_frac)
  if not torch.cuda.is_available():
    raise RuntimeError(f'{fn} needs a CUDA device (tapnet_b200 has no CPU fallback)')

  dev = pts.device if on_device else torch.device('cuda', torch.cuda.current_device())
  with torch.cuda.device(dev):
    tracks_d = _to_device(pts, dev).contiguous()
    occ_d = _to_device(occ, dev)
    occ_d = (occ_d != 0).contiguous()
    thr_d = _to_device(thr, dev)
    f64 = dict(dtype=torch.float64, device=dev)
    homogs = torch.empty(T, 3, 3, **f64)
    err = torch.empty(N, T, **f64)
    canonical = torch.empty(N, 2, **f64)
    stats = torch.empty(T, 2, dtype=torch.int32, device=dev) if return_ransac_stats else None
    ws = torch.empty(_lib.homographies_workspace_bytes(T, N), dtype=torch.uint8, device=dev)
    _lib.homographies_wrt_frame(tracks_d, occ_d, dims[0], dims[1], ref, thresh, outlier_point_threshold,
                                passes, thr_d, homogs, err, canonical, stats, ws)
  out = (homogs, err, canonical) + ((stats,) if return_ransac_stats else ())
  return out if on_device else tuple(t.cpu().numpy() for t in out)


def foreground_tracks(err, visibles, inlier_threshold=0.07, foreground_frac=0.6):
  """The rainbow demo's last step: track n is foreground when
  sum((err < t^2) * vis) / max(1, sum(vis)) <= foreground_frac over its frames.  err [N, T] and
  visibles [N, T] as numpy arrays or tensors; returns bool [N] of the same kind."""
  if isinstance(err, torch.Tensor):
    vis = torch.as_tensor(visibles, device=err.device).to(torch.float64)
    inl = (err < inlier_threshold ** 2).to(torch.float64) * vis
    return inl.sum(1) / vis.sum(1).clamp(min=1.0) <= foreground_frac
  vis = np.asarray(visibles).astype(np.float64)
  inl = (np.asarray(err) < inlier_threshold ** 2) * vis
  return inl.sum(1) / np.maximum(1.0, vis.sum(1)) <= foreground_frac
