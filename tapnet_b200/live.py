"""The steps either side of the hot path, on the device (SURVEY 8f rows 1 and 2).

Mirrors the helper functions of `tapnet/pytorch_live_demo.py` (same names and argument meaning),
each one a single kernel of libtapir_b200.so instead of a chain of ATen ops:

  preprocess_frames        :30-41   uint8 [0,255] -> float [-1,1]
  get_frame / crop window  :88-95   centre square crop of a camera frame
  ingest_frames            crop + preprocess + utils.bilinear (torch/utils.py:26-42) in one pass
  postprocess_occlusions   :57-59   visibility flag from the two logits
  online_model_init        :44-54
  online_model_predict     :62-85

`TAPIR.get_feature_grids` also accepts the uint8 frames directly (normalisation fused into the
stem conv), which is what `online_model_*` do here, so a live frame crosses PCIe as uint8 and is
never materialised as float.  `YUV420Frames` carries NV12 / I420 device frames (video decoders,
cameras) the same way, the colour conversion fused into the same reads; `yuv420_to_rgb`
converts alone.  CUDA only; raises without the shared library.
"""
from typing import Optional, Tuple

import torch

from tapnet_b200 import _lib


def _require_cuda(t, what):
  if t.device.type != 'cuda':
    raise RuntimeError(f'{what}: tensor on {t.device}; tapnet_b200 runs on CUDA only '
                       '(no CPU fallback)')


def center_square_window(height: int, width: int) -> Tuple[int, int, int, int]:
  """(y0, x0, h, w) of the window `get_frame` keeps (pytorch_live_demo.py:88-95): |w-h|//2
  pixels trimmed from both ends of the longer side.  The reference's `[trunc:-trunc]` slice is
  empty when the sides differ by exactly one pixel; that case raises instead."""
  trunc = abs(width - height) // 2
  if width != height and trunc == 0:
    raise ValueError('frame sides differ by one pixel: the reference crop would be empty')
  if width > height:
    return 0, trunc, height, width - 2 * trunc
  if width < height:
    return trunc, 0, height - 2 * trunc, width
  return 0, 0, height, width


_MATRICES = {'bt601': 601, 'bt709': 709}


class YUV420Frames:
  """A clip of 8-bit YUV 4:2:0 frames on a CUDA device, as video decoders and cameras deliver it.

  y: [B, T, H, W] uint8; u, v: [B, T, ceil(H/2), ceil(W/2)] uint8.  Rows may be pitched (any row
  stride); the last-dim step is 1 for luma and 1 (I420) or 2 (NV12's interleaved UV) for chroma.
  `matrix` is 'bt601' or 'bt709', `full_range` selects 0-255 instead of 16-235 luma, and
  `window` (y0, x0, h, w) is the crop the model sees (default: the whole frame).  The conversion
  is the integer one of include/tapir_b200.h (tapir_yuv420_frames); `TAPIR` results on these
  frames equal, bit for bit, its results on `yuv420_to_rgb(frames)`.
  """

  def __init__(self, y: torch.Tensor, u: torch.Tensor, v: torch.Tensor, matrix: str = 'bt601',
               full_range: bool = False, window: Optional[Tuple[int, int, int, int]] = None):
    self.window = _check_planes(y, u, v, matrix, window)
    for name, t in (('y', y), ('u', u), ('v', v)):
      if t.device.type != 'cuda':
        raise RuntimeError(f'YUV420Frames: {name} on {t.device}; YUV frames are read on CUDA '
                           'only (host YUV clips are not supported: copy them to the device)')
    if u.device != y.device or v.device != y.device:
      raise ValueError('YUV420Frames: planes on different devices')
    self.y, self.u, self.v = y, u, v
    self.matrix, self.full_range = matrix, bool(full_range)

  @classmethod
  def nv12(cls, y: torch.Tensor, uv: torch.Tensor, **kwargs) -> 'YUV420Frames':
    """y [B, T, H, W] and the interleaved chroma plane uv [B, T, ceil(H/2), ceil(W/2), 2]."""
    if not isinstance(uv, torch.Tensor) or uv.dim() != 5 or uv.shape[-1] != 2:
      raise ValueError('YUV420Frames.nv12: uv must be [B, T, ceil(H/2), ceil(W/2), 2]')
    return cls(y, uv[..., 0], uv[..., 1], **kwargs)

  @classmethod
  def i420(cls, y: torch.Tensor, u: torch.Tensor, v: torch.Tensor, **kwargs) -> 'YUV420Frames':
    """Three separate planes: y [B, T, H, W], u and v [B, T, ceil(H/2), ceil(W/2)]."""
    return cls(y, u, v, **kwargs)

  def with_window(self, window: Optional[Tuple[int, int, int, int]]) -> 'YUV420Frames':
    """The same planes with another crop window (None: the whole frame)."""
    return YUV420Frames(self.y, self.u, self.v, self.matrix, self.full_range, window)

  @property
  def frame_size(self) -> Tuple[int, int]:
    """(H, W) of the full frame."""
    return int(self.y.shape[2]), int(self.y.shape[3])

  @property
  def shape(self) -> torch.Size:
    """(B, T, h, w, 3): the shape of the RGB clip the window converts to."""
    return torch.Size((int(self.y.shape[0]), int(self.y.shape[1]), self.window[2], self.window[3], 3))

  @property
  def device(self) -> torch.device:
    return self.y.device

  def c_struct(self, frame0: int = 0) -> '_lib.Yuv420Frames':
    """The tapir_yuv420_frames descriptor of frames frame0, frame0 + 1, ... of the flattened
    [B * T] clip."""
    desc, self._keep = _descriptor(self.y, self.u, self.v, self.window, self.matrix,
                                   self.full_range, frame0)
    return desc


def _check_planes(y, u, v, matrix, window):
  """Validates the planes' dtype, shapes and layout, the matrix and the window; returns the
  window as (y0, x0, h, w)."""
  for name, t in (('y', y), ('u', u), ('v', v)):
    if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8:
      raise ValueError(f'YUV420Frames: {name} must be a uint8 tensor')
    if t.dim() != 4:
      raise ValueError(f'YUV420Frames: {name} must be [B, T, rows, cols], got {tuple(t.shape)}')
  B, T, H, W = (int(d) for d in y.shape)
  chroma = (B, T, (H + 1) // 2, (W + 1) // 2)
  if tuple(u.shape) != chroma or tuple(v.shape) != chroma:
    raise ValueError(f'YUV420Frames: chroma planes must be {list(chroma)} for luma '
                     f'{list(y.shape)}, got {list(u.shape)} and {list(v.shape)}')
  if y.stride(3) != 1 and W > 1:
    raise ValueError('YUV420Frames: luma rows must be dense (last-dim step 1)')
  if chroma[3] > 1 and (u.stride(3) != v.stride(3) or u.stride(3) not in (1, 2)):
    raise ValueError('YUV420Frames: chroma last-dim step must be 1 (I420) or 2 (NV12) and the '
                     f'same for u and v, got {u.stride(3)} and {v.stride(3)}')
  if matrix not in _MATRICES:
    raise ValueError(f'YUV420Frames: matrix must be one of {sorted(_MATRICES)}, got {matrix!r}')
  y0, x0, h, w = (0, 0, H, W) if window is None else (int(a) for a in window)
  if h <= 0 or w <= 0 or y0 < 0 or x0 < 0 or y0 + h > H or x0 + w > W:
    raise ValueError(f'YUV420Frames: window {(y0, x0, h, w)} outside the {H}x{W} frame')
  return y0, x0, h, w


def _descriptor(y, u, v, window, matrix, full_range, frame0=0):
  """(tapir_yuv420_frames, planes it points into) for frames frame0.. of the [B * T]-flattened
  planes.  Planes whose B and T axes do not merge into one frame stride are copied first; the
  caller keeps the returned planes alive until the launches that read them have run."""
  y, u, v = (t.flatten(0, 1) for t in (y, u, v))
  step = u.stride(2) if u.shape[2] > 1 else 1
  if u.shape[2] > 1 and u.stride(2) != v.stride(2):  # only one of u, v was copied
    u, v = u.contiguous(), v.contiguous()
    step = 1
  H, W = int(y.shape[1]), int(y.shape[2])
  y0, x0, h, w = window
  f = int(frame0)
  desc = _lib.Yuv420Frames(
      y[f:].data_ptr(), u[f:].data_ptr(), v[f:].data_ptr(), y.stride(0), u.stride(0), v.stride(0),
      y.stride(1), u.stride(1), v.stride(1), step, H, W, y0, x0, h, w, _MATRICES[matrix],
      int(bool(full_range)), 0)
  return desc, (y, u, v)


def yuv420_to_rgb(frames: YUV420Frames) -> torch.Tensor:
  """The crop window of YUV 4:2:0 frames as uint8 RGB [B, T, h, w, 3] (dense)."""
  if not isinstance(frames, YUV420Frames):
    raise ValueError('yuv420_to_rgb: expected YUV420Frames')
  out = torch.empty(frames.shape, dtype=torch.uint8, device=frames.device)
  n = out.shape[0] * out.shape[1]
  if n > 0:
    with torch.cuda.device(frames.device):
      _lib.yuv420_to_rgb(frames, out)
  return out


def _ingest_yuv420(frames: YUV420Frames, window, resolution) -> torch.Tensor:
  if window is not None:
    frames = frames.with_window(window)
  B, T, h, w, _ = frames.shape
  oh, ow = (h, w) if resolution is None else (int(resolution[0]), int(resolution[1]))
  out = torch.empty(B, T, oh, ow, 3, dtype=torch.float32, device=frames.device)
  if B * T > 0:
    with torch.cuda.device(frames.device):
      _lib.ingest_frames(frames, out)
  return out


def ingest_frames(frames, window: Optional[Tuple[int, int, int, int]] = None,
                  resolution: Optional[Tuple[int, int]] = None) -> torch.Tensor:
  """frames: [..., H, W, 3] uint8 on a CUDA device.  Crops to `window` (y0, x0, h, w), normalises
  to [-1, 1] and resizes to `resolution` (h, w) with the reference's bilinear; returns float32
  [..., h, w, 3].  A `YUV420Frames` clip is converted to RGB in the same pass (`window`, when
  given, replaces the clip's own window; it is in full-frame coordinates) -> [B, T, h, w, 3]."""
  if isinstance(frames, YUV420Frames):
    return _ingest_yuv420(frames, window, resolution)
  _require_cuda(frames, 'ingest_frames')
  if frames.dtype != torch.uint8 or frames.dim() < 3 or frames.shape[-1] != 3:
    raise ValueError('ingest_frames: expected uint8 frames [..., H, W, 3]')
  frames = frames.contiguous()
  H, W = int(frames.shape[-3]), int(frames.shape[-2])
  y0, x0, ch, cw = (0, 0, H, W) if window is None else (int(v) for v in window)
  oh, ow = (ch, cw) if resolution is None else (int(resolution[0]), int(resolution[1]))
  out = torch.empty(*frames.shape[:-3], oh, ow, 3, dtype=torch.float32, device=frames.device)
  if frames.shape[:-3].numel() > 0:
    _lib.ingest_frames(frames, out, (y0, x0, ch, cw))
  return out


def preprocess_frames(frames: torch.Tensor) -> torch.Tensor:
  """[num_frames, height, width, 3] uint8 -> float32 in [-1, 1] (pytorch_live_demo.py:30-41)."""
  return ingest_frames(frames)


def postprocess_occlusions(occlusions: torch.Tensor, expected_dist: torch.Tensor) -> torch.Tensor:
  """visibles = (1 - sigmoid(occlusions)) * (1 - sigmoid(expected_dist)) > 0.5, bool."""
  _require_cuda(occlusions, 'postprocess_occlusions')
  if occlusions.shape != expected_dist.shape:
    raise ValueError('postprocess_occlusions: shape mismatch')
  occ = occlusions.to(torch.float32).contiguous()
  expd = expected_dist.to(torch.float32).contiguous()
  out = torch.empty(occ.shape, dtype=torch.uint8, device=occ.device)
  if occ.numel() > 0:
    _lib.postprocess_occlusions(occ, expd, out)
  return out.view(torch.bool)


def online_model_init(model, frames: torch.Tensor, points: torch.Tensor):
  """Query features for `points` [1, N, 3] (t, y, x) on `frames` [1, T, H, W, 3] (uint8 or
  already-normalised float) - pytorch_live_demo.py:44-54."""
  feature_grids = model.get_feature_grids(frames, is_training=False)
  return model.get_query_features(frames, is_training=False, query_points=points,
                                  feature_grids=feature_grids)


def online_model_predict(model, frames: torch.Tensor, features, causal_context):
  """One online step - pytorch_live_demo.py:62-85.  Returns (tracks, visibles, causal_context)
  for the final resolution, like the reference."""
  feature_grids = model.get_feature_grids(frames, is_training=False)
  trajectories = model.estimate_trajectories(
      frames.shape[-3:-1], is_training=False, feature_grids=feature_grids,
      query_features=features, query_points_in_video=None, query_chunk_size=64,
      causal_context=causal_context, get_causal_context=True)
  causal_context = trajectories['causal_context']
  tracks = trajectories['tracks'][-1]
  visibles = postprocess_occlusions(trajectories['occlusion'][-1],
                                    trajectories['expected_dist'][-1])
  return tracks, visibles, causal_context
