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
never materialised as float.  `YUVFrames` carries device frames of video decoders and cameras
(NV12 / I420, P010 / P016, 10- and 12-bit planar 4:2:0, 4:4:4, packed YUYV / UYVY) the same way,
the colour conversion fused into the same reads; `yuv_to_rgb` converts alone.  `YUV420Frames`
(8-bit 4:2:0) and `yuv420_to_rgb` are the 4:2:0 forms of both.  CUDA only; raises without the shared library.
"""
import functools
from typing import Callable, NamedTuple, Optional, Tuple

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


_MATRICES = {'bt601': 601, 'bt709': 709, 'bt2020': 2020}
_WORDS = (torch.uint16, torch.int16)  # 16-bit samples (int16: the same bits, as decoders hand back)


class YUVFrames:
  """A clip of YUV frames on a CUDA device in any layout of include/tapir_b200.h's tapir_yuv_frames:
  8- to 16-bit samples, 4:2:0, 4:2:2 or 4:4:4 chroma, planar, semi-planar or packed.  Build it with
  the constructor of the layout the source delivers (`nv12`, `i420`, `p010`, `p016`, `yuv420p`,
  `yuv444`, `yuyv`, `uyvy`); each takes `matrix` ('bt601', 'bt709' or 'bt2020'), `full_range` and
  `window` (y0, x0, h, w: the crop the model sees, default the whole frame).  Rows may be pitched.

  The planes y [B, T, H, W], u and v [B, T, ceil(H / 2^sy), ceil(W / 2^sx)] are views into the
  constructor's `buffers`, their last-dim step the sample step.  The conversion is the integer one
  of tapir_yuv_frames; `TAPIR` results on these frames equal, bit for bit, its results on
  `yuv_to_rgb(frames)`.
  """

  def __init__(self, y: torch.Tensor, u: torch.Tensor, v: torch.Tensor, *, chroma_shift=(1, 1),
               bits: int = 8, lsb_aligned: bool = False, matrix: str = 'bt601',
               full_range: bool = False, window: Optional[Tuple[int, int, int, int]] = None,
               layout: str = 'planar', buffers=None, _make=None):
    name = type(self).__name__
    self.window = _check_layout(name, y, u, v, chroma_shift, bits, matrix, window)
    _check_devices(name, (y, u, v))
    self.y, self.u, self.v = y, u, v
    self.chroma_shift = (int(chroma_shift[0]), int(chroma_shift[1]))
    self.bits, self.lsb_aligned = int(bits), bool(lsb_aligned)
    self.matrix, self.full_range = matrix, bool(full_range)
    self.layout = layout
    self.buffers = tuple(buffers) if buffers is not None else (y, u, v)
    # how map_buffers / with_window rebuild the clip: (constructor, its layout arguments)
    self._make = _make or (lambda *b, **kw: YUVFrames(
        *b, chroma_shift=self.chroma_shift, bits=self.bits, lsb_aligned=self.lsb_aligned, **kw))

  @classmethod
  def nv12(cls, y: torch.Tensor, uv: torch.Tensor, **kw) -> 'YUVFrames':
    """8-bit 4:2:0: y [B, T, H, W] uint8 and the interleaved uv [B, T, ceil(H/2), ceil(W/2), 2]."""
    _check_uv('nv12', uv)
    return YUVFrames(y, uv[..., 0], uv[..., 1], layout='nv12', buffers=(y, uv),
                     _make=YUVFrames.nv12, **kw)

  @classmethod
  def i420(cls, y: torch.Tensor, u: torch.Tensor, v: torch.Tensor, **kw) -> 'YUVFrames':
    """8-bit 4:2:0, three planes: y [B, T, H, W], u and v [B, T, ceil(H/2), ceil(W/2)] uint8."""
    return YUVFrames(y, u, v, layout='i420', _make=YUVFrames.i420, **kw)

  @classmethod
  def p010(cls, y: torch.Tensor, uv: torch.Tensor, **kw) -> 'YUVFrames':
    """10-bit 4:2:0 in 16-bit MSB-aligned samples (NVDEC's 10-bit output): y [B, T, H, W] and
    uv [B, T, ceil(H/2), ceil(W/2), 2], torch.uint16 or torch.int16 (read as the same bits)."""
    _check_uv('p010', uv)
    return YUVFrames(y, uv[..., 0], uv[..., 1], bits=10, layout='p010', buffers=(y, uv),
                     _make=YUVFrames.p010, **kw)

  @classmethod
  def p016(cls, y: torch.Tensor, uv: torch.Tensor, **kw) -> 'YUVFrames':
    """16-bit (or 12-bit MSB-aligned) 4:2:0, laid out as p010."""
    _check_uv('p016', uv)
    return YUVFrames(y, uv[..., 0], uv[..., 1], bits=16, layout='p016', buffers=(y, uv),
                     _make=YUVFrames.p016, **kw)

  @classmethod
  def yuv420p(cls, y: torch.Tensor, u: torch.Tensor, v: torch.Tensor, bits: int,
              **kw) -> 'YUVFrames':
    """9- to 16-bit 4:2:0, three planes of LSB-aligned 16-bit samples (ffmpeg's yuv420p10le,
    yuv420p12le): y [B, T, H, W], u and v [B, T, ceil(H/2), ceil(W/2)]."""
    bits = int(bits)
    return YUVFrames(y, u, v, bits=bits, lsb_aligned=True, layout=f'yuv420p{bits}',
                     _make=lambda *b, **k: YUVFrames.yuv420p(*b, bits=bits, **k), **kw)

  @classmethod
  def yuv444(cls, y: torch.Tensor, u: torch.Tensor, v: torch.Tensor, bits: Optional[int] = None,
             **kw) -> 'YUVFrames':
    """4:4:4, three [B, T, H, W] planes: uint8, or 16-bit samples holding `bits` (default 16;
    fewer: LSB-aligned, as ffmpeg's yuv444p10le)."""
    wide = isinstance(y, torch.Tensor) and y.dtype in _WORDS
    bits = int(bits) if bits is not None else (16 if wide else 8)
    return YUVFrames(y, u, v, chroma_shift=(0, 0), bits=bits, lsb_aligned=wide and bits < 16,
                     layout=f'yuv444p{bits}' if wide else 'yuv444',
                     _make=lambda *b, **k: YUVFrames.yuv444(*b, bits=bits, **k), **kw)

  @classmethod
  def yuyv(cls, frames: torch.Tensor, **kw) -> 'YUVFrames':
    """Packed 8-bit 4:2:2 (V4L2 / UVC cameras): uint8 [B, T, H, 2W] rows Y0 U Y1 V ...; W even."""
    _check_packed('yuyv', frames)
    return YUVFrames(frames[..., 0::2], frames[..., 1::4], frames[..., 3::4], chroma_shift=(1, 0),
                     layout='yuyv', buffers=(frames,), _make=YUVFrames.yuyv, **kw)

  @classmethod
  def uyvy(cls, frames: torch.Tensor, **kw) -> 'YUVFrames':
    """Packed 8-bit 4:2:2 (HDMI / SDI capture): uint8 [B, T, H, 2W] rows U Y0 V Y1 ...; W even."""
    _check_packed('uyvy', frames)
    return YUVFrames(frames[..., 1::2], frames[..., 0::4], frames[..., 2::4], chroma_shift=(1, 0),
                     layout='uyvy', buffers=(frames,), _make=YUVFrames.uyvy, **kw)

  @staticmethod
  def zeros(layout: str, B: int, T: int, H: int, W: int, device, **kw) -> 'YUVFrames':
    """A zero clip of B x T frames of H x W in `layout` (a YUV_LAYOUTS name: 'nv12', 'i420',
    'p010', 'p016', 'yuv420p10', 'yuv444', 'yuv444p16', 'yuyv', ...), dense rows."""
    spec = YUV_LAYOUTS.get(layout) if isinstance(layout, str) else None
    if spec is None:
      raise ValueError(f'YUVFrames.zeros: unknown layout {layout!r}')
    sx, sy = spec.chroma_shift
    ch, cw = -(-H // (1 << sy)), -(-W // (1 << sx))

    def z(*shape):
      return torch.zeros(B, T, *shape, dtype=spec.dtype, device=device)
    if spec.form == 'packed':
      return spec.make(z(H, 2 * W), **kw)
    if spec.form == 'semi':
      return spec.make(z(H, W), z(ch, cw, 2), **kw)
    return spec.make(z(H, W), z(ch, cw), z(ch, cw), **kw)

  def with_buffers(self, buffers) -> 'YUVFrames':
    """A clip of the same layout, matrix, range and window over other buffers of the same frame
    size (e.g. another batch of frames, or storage of its own)."""
    return self._make(*buffers, matrix=self.matrix, full_range=self.full_range, window=self.window)

  def map_buffers(self, fn) -> 'YUVFrames':
    """with_buffers of fn(buffer) for every buffer (fn selects or repeats frames along the leading
    [B, T] axes)."""
    return self.with_buffers([fn(b) for b in self.buffers])

  def with_window(self, window: Optional[Tuple[int, int, int, int]]) -> 'YUVFrames':
    """The same planes with another crop window (None: the whole frame)."""
    return self._make(*self.buffers, matrix=self.matrix, full_range=self.full_range, window=window)

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

  @property
  def sampling(self) -> Tuple[int, Optional[int], bool, Tuple[int, int]]:
    """(sample bytes, bits of LSB-aligned samples (None otherwise: the conversion reads all 8 or
    16), LSB-aligned, chroma shift): what the conversion reads, whatever the planes'
    interleaving.  P010 and P016 frames share it."""
    return (self.y.element_size(), self.bits if self.lsb_aligned else None, self.lsb_aligned,
            self.chroma_shift)

  def yuv_struct(self, frame0: int = 0) -> '_lib.YuvFrames':
    """The tapir_yuv_frames descriptor of frames frame0, frame0 + 1, ... of the flattened
    [B * T] clip."""
    desc, self._keep = _descriptor_yuv(self.y, self.u, self.v, self.window, self.matrix,
                                       self.full_range, frame0, self.chroma_shift, self.bits,
                                       self.lsb_aligned)
    return desc


class YUVLayout(NamedTuple):
  """One named layout: its constructor (taking the buffers), the buffers' sample dtype, the sample
  bits, whether they are LSB-aligned, the chroma shift (x, y) and the buffer form ('semi': y and
  an interleaved uv [..., 2]; 'planar': y, u, v; 'packed': one [B, T, H, 2W] buffer)."""
  make: Callable[..., YUVFrames]
  dtype: torch.dtype
  bits: int
  lsb_aligned: bool
  chroma_shift: Tuple[int, int]
  form: str


def _layouts():
  t = {'nv12': YUVLayout(YUVFrames.nv12, torch.uint8, 8, False, (1, 1), 'semi'),
       'i420': YUVLayout(YUVFrames.i420, torch.uint8, 8, False, (1, 1), 'planar'),
       'p010': YUVLayout(YUVFrames.p010, torch.int16, 10, False, (1, 1), 'semi'),
       'p016': YUVLayout(YUVFrames.p016, torch.int16, 16, False, (1, 1), 'semi'),
       'yuv444': YUVLayout(YUVFrames.yuv444, torch.uint8, 8, False, (0, 0), 'planar'),
       'yuyv': YUVLayout(YUVFrames.yuyv, torch.uint8, 8, False, (1, 0), 'packed'),
       'uyvy': YUVLayout(YUVFrames.uyvy, torch.uint8, 8, False, (1, 0), 'packed')}
  for b in range(8, 17):
    t[f'yuv420p{b}'] = YUVLayout(functools.partial(YUVFrames.yuv420p, bits=b), torch.int16, b, True,
                                 (1, 1), 'planar')
    t[f'yuv444p{b}'] = YUVLayout(functools.partial(YUVFrames.yuv444, bits=b), torch.int16, b,
                                 b < 16, (0, 0), 'planar')
  return t


# layout name (YUVFrames.layout) -> YUVLayout: what YUVFrames.zeros builds and an OnlineTracker's
# yuv_layout names
YUV_LAYOUTS = _layouts()


def is_yuv_layout(name) -> bool:
  """Whether `name` is a layout YUVFrames.zeros builds (an OnlineTracker's yuv_layout)."""
  return isinstance(name, str) and name in YUV_LAYOUTS


class YUV420Frames(YUVFrames):
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
    window = _check_planes(y, u, v, matrix, window)
    super().__init__(y, u, v, matrix=matrix, full_range=full_range, window=window,
                     layout='yuv420', _make=YUV420Frames)

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

  def c_struct(self, frame0: int = 0) -> '_lib.Yuv420Frames':
    """The tapir_yuv420_frames descriptor of frames frame0, frame0 + 1, ... of the flattened
    [B * T] clip."""
    desc, self._keep = _descriptor(self.y, self.u, self.v, self.window, self.matrix,
                                   self.full_range, frame0)
    return desc


def _check_devices(who, planes):
  for pname, t in zip('yuv', planes):
    if t.device.type != 'cuda':
      raise RuntimeError(f'{who}: {pname} on {t.device}; YUV frames are read on CUDA '
                         'only (host YUV clips are not supported: copy them to the device)')
  if any(t.device != planes[0].device for t in planes):
    raise ValueError(f'{who}: planes on different devices')


def _check_uv(who, uv):
  if not isinstance(uv, torch.Tensor) or uv.dim() != 5 or uv.shape[-1] != 2:
    raise ValueError(f'YUVFrames.{who}: uv must be [B, T, ceil(H/2), ceil(W/2), 2]')


def _check_packed(who, frames):
  if (not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8 or frames.dim() != 4
      or frames.shape[3] % 4 != 0 or (frames.stride(3) != 1 and frames.shape[3] > 1)):
    got = (f'{frames.dtype} {tuple(frames.shape)}' if isinstance(frames, torch.Tensor)
           else type(frames).__name__)
    raise ValueError(f'YUVFrames.{who}: expected uint8 [B, T, H, 2W] packed rows with dense '
                     f'bytes and an even W, got {got}')


def _check_layout(who, y, u, v, chroma_shift, bits, matrix, window):
  """Validates the planes' dtype, shapes and steps, the sample bits, the matrix and the window
  against tapir_yuv_frames' rules; returns the window as (y0, x0, h, w)."""
  for name, t in (('y', y), ('u', u), ('v', v)):
    if not isinstance(t, torch.Tensor) or t.dtype not in (torch.uint8,) + _WORDS:
      raise ValueError(f'{who}: {name} must be a uint8, uint16 or int16 tensor')
    if t.dim() != 4:
      raise ValueError(f'{who}: {name} must be [B, T, rows, cols], got {tuple(t.shape)}')
  wide = y.dtype in _WORDS
  if any((t.dtype in _WORDS) != wide for t in (u, v)):
    raise ValueError(f'{who}: planes of mixed sample sizes {y.dtype}, {u.dtype}, {v.dtype}')
  if not (8 <= int(bits) <= 16) or (not wide and int(bits) != 8):
    raise ValueError(f'{who}: {bits}-bit samples in {y.dtype} planes (8 for uint8, 8..16 for '
                     '16-bit)')
  sx, sy = (int(a) for a in chroma_shift)
  if sx not in (0, 1) or sy not in (0, 1):
    raise ValueError(f'{who}: chroma_shift must be 0 or 1 per axis, got {tuple(chroma_shift)}')
  B, T, H, W = (int(d) for d in y.shape)
  chroma = (B, T, -(-H // (1 << sy)), -(-W // (1 << sx)))
  if tuple(u.shape) != chroma or tuple(v.shape) != chroma:
    raise ValueError(f'{who}: chroma planes must be {list(chroma)} for luma {list(y.shape)}, got '
                     f'{list(u.shape)} and {list(v.shape)}')
  if (W > 1 and y.stride(3) < 1) or (chroma[3] > 1 and (u.stride(3) < 1 or u.stride(3) != v.stride(3))):
    raise ValueError(f'{who}: sample steps must be >= 1 and the same for u and v, got y '
                     f'{y.stride(3)}, u {u.stride(3)}, v {v.stride(3)}')
  if matrix not in _MATRICES:
    raise ValueError(f'{who}: matrix must be one of {sorted(_MATRICES)}, got {matrix!r}')
  y0, x0, h, w = (0, 0, H, W) if window is None else (int(a) for a in window)
  if h <= 0 or w <= 0 or y0 < 0 or x0 < 0 or y0 + h > H or x0 + w > W:
    raise ValueError(f'{who}: window {(y0, x0, h, w)} outside the {H}x{W} frame')
  if W > 1 and y.stride(3) == 2 and (W % 2 or x0 % 2 or w % 2):
    raise ValueError(f'{who}: packed 4:2:2 rows need an even frame width, window column and '
                     f'window width, got W={W}, window {(y0, x0, h, w)}')
  return y0, x0, h, w


def _check_planes(y, u, v, matrix, window):
  """Validates 8-bit 4:2:0 planes (YUV420Frames): uint8, dense luma rows, chroma step 1 or 2,
  BT.601 / BT.709; returns the window as (y0, x0, h, w)."""
  for name, t in (('y', y), ('u', u), ('v', v)):
    if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8:
      raise ValueError(f'YUV420Frames: {name} must be a uint8 tensor')
  window = _check_layout('YUV420Frames', y, u, v, (1, 1), 8, matrix, window)
  if y.stride(3) != 1 and y.shape[3] > 1:
    raise ValueError('YUV420Frames: luma rows must be dense (last-dim step 1)')
  if u.shape[3] > 1 and u.stride(3) not in (1, 2):
    raise ValueError('YUV420Frames: chroma last-dim step must be 1 (I420) or 2 (NV12) and the '
                     f'same for u and v, got {u.stride(3)} and {v.stride(3)}')
  if matrix not in ('bt601', 'bt709'):
    raise ValueError(f"YUV420Frames: matrix must be one of ['bt601', 'bt709'], got {matrix!r}")
  return window


def _descriptor_yuv(y, u, v, window, matrix, full_range, frame0=0, chroma_shift=(1, 1), bits=8,
                    lsb_aligned=False):
  """(tapir_yuv_frames, planes it points into) for frames frame0.. of the [B * T]-flattened
  planes.  Planes whose B and T axes do not merge into one frame stride are copied first; the
  caller keeps the returned planes alive until the launches that read them have run."""
  y, u, v = (t.flatten(0, 1) for t in (y, u, v))
  step = u.stride(2) if u.shape[2] > 1 else 1
  if u.shape[2] > 1 and u.stride(2) != v.stride(2):  # only one of u, v was copied
    u, v = u.contiguous(), v.contiguous()
    step = 1
  H, W = int(y.shape[1]), int(y.shape[2])
  b = y.element_size()
  y0, x0, h, w = window
  f = int(frame0)
  desc = _lib.YuvFrames(
      y[f:].data_ptr(), u[f:].data_ptr(), v[f:].data_ptr(),
      y.stride(0) * b, u.stride(0) * b, v.stride(0) * b, y.stride(1) * b, u.stride(1) * b,
      v.stride(1) * b, H, W, y0, x0, h, w, _MATRICES[matrix], int(bool(full_range)), b, int(bits),
      int(bool(lsb_aligned) and b == 2), y.stride(2) if W > 1 else 1, step, int(chroma_shift[0]),
      int(chroma_shift[1]), 0)
  return desc, (y, u, v)


def _descriptor(y, u, v, window, matrix, full_range, frame0=0):
  """_descriptor_yuv of 8-bit 4:2:0 planes as a tapir_yuv420_frames."""
  d, keep = _descriptor_yuv(y, u, v, window, matrix, full_range, frame0)
  return _lib.Yuv420Frames(**{f: getattr(d, f) for f, _ in _lib.Yuv420Frames._fields_}), keep


def yuv_to_rgb(frames: YUVFrames) -> torch.Tensor:
  """The crop window of YUV frames as uint8 RGB [B, T, h, w, 3] (dense)."""
  if not isinstance(frames, YUVFrames):
    raise ValueError('yuv_to_rgb: expected YUVFrames')
  out = torch.empty(frames.shape, dtype=torch.uint8, device=frames.device)
  n = out.shape[0] * out.shape[1]
  if n > 0:
    with torch.cuda.device(frames.device):
      _lib.yuv_to_rgb(frames, out)
  return out


def yuv420_to_rgb(frames: YUV420Frames) -> torch.Tensor:
  """The crop window of YUV 4:2:0 frames as uint8 RGB [B, T, h, w, 3] (dense)."""
  if not isinstance(frames, YUV420Frames):
    raise ValueError('yuv420_to_rgb: expected YUV420Frames')
  return yuv_to_rgb(frames)


def _ingest_yuv(frames: YUVFrames, window, resolution) -> torch.Tensor:
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
  [..., h, w, 3].  A `YUVFrames` clip is converted to RGB in the same pass (`window`, when
  given, replaces the clip's own window; it is in full-frame coordinates) -> [B, T, h, w, 3]."""
  if isinstance(frames, YUVFrames):
    return _ingest_yuv(frames, window, resolution)
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
