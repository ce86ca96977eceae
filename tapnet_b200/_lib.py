"""ctypes binding of libtapir_b200.so (include/tapir_b200.h).

There is no CPU fallback: if the shared library is missing or cannot be loaded every
compute entry point raises.  `load()` never builds implicitly on import; use
`__graft_entry__.build()` / `python -m tapnet_b200.build`.

Below the structs and `SIGNATURES`, one tensor-level function per entry point the package calls:
the only place that knows the C ABI's argument layout.  Each one reads every size, stride and
byte offset off the tensors it is given and checks them on the host first (dtype, device, unit
inner stride, shapes that must agree), since the C side sees only pointers and cannot.  The checks
read tensor attributes only (no allocation, no synchronisation), so the calls can be captured in a
CUDA graph.  Outputs and workspaces are tensors the caller passes in.
"""
import ctypes
import math
import os
from ctypes import POINTER, Structure, byref, c_char_p, c_double, c_float, c_int32, c_int64, c_size_t, c_ulonglong, c_void_p

import torch

from tapnet_b200 import schema

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'libtapir_b200.so')

MAX_MIXER_BLOCKS = 12
NUM_RESNET_BLOCKS = 8
MAX_EXTRA_BLOCKS = 5
MAX_CORR_LEVELS = 5
MAX_RAGGED_CLIPS = 64
MAX_QUERY_GRIDS = 16
MAX_RESIZE_SIDE = 65535


class Linear(Structure):
  _fields_ = [('w', c_void_p), ('bias', c_void_p), ('N', c_int32), ('K', c_int32),
              ('planes', c_int32), ('k_logical', c_int32)]


class ResnetBlock(Structure):
  _fields_ = [('proj', Linear), ('conv0', Linear), ('conv1', Linear),
              ('bn0_w', c_void_p), ('bn0_b', c_void_p), ('bn1_w', c_void_p), ('bn1_b', c_void_p),
              ('cin', c_int32), ('cout', c_int32), ('stride', c_int32), ('has_proj', c_int32)]


class ExtraBlock(Structure):
  _fields_ = [('ln_w', c_void_p), ('ln_b', c_void_p), ('conv', Linear), ('conv1', Linear)]


class BackboneWeights(Structure):
  _fields_ = [('stem_w', c_void_p), ('blocks', ResnetBlock * NUM_RESNET_BLOCKS),
              ('extra', ExtraBlock * MAX_EXTRA_BLOCKS), ('num_extra', c_int32),
              ('planes', c_int32)]


class HeadWeights(Structure):
  _fields_ = [(n, c_void_p) for n in ('hid1_w', 'hid1_b', 'hid2_w', 'hid2_b', 'hid3_w', 'hid3_b',
                                      'hid4_w', 'hid4_b', 'occ_w', 'occ_b')]


class MixerBlock(Structure):
  _fields_ = [('ln_w', c_void_p), ('dw1_w', c_void_p), ('dw1_b', c_void_p), ('dw2_w', c_void_p),
              ('dw2_b', c_void_p), ('ln1_w', c_void_p), ('up', Linear), ('down', Linear)]


class MixerWeights(Structure):
  _fields_ = [('linear', Linear), ('linear_1', Linear), ('ln_w', c_void_p),
              ('blocks', MixerBlock * MAX_MIXER_BLOCKS), ('num_blocks', c_int32),
              ('planes', c_int32)]


class MixerIO(Structure):
  _fields_ = [('x_planes', c_void_p), ('x_plane_stride', c_int64), ('ldx', c_int32),
              ('num_points', c_int32), ('num_frames', c_int32), ('causal', c_int32),
              ('ctx1_in', POINTER(c_void_p)), ('ctx2_in', POINTER(c_void_p)),
              ('ctx1_out', POINTER(c_void_p)), ('ctx2_out', POINTER(c_void_p)),
              ('out', c_void_p), ('ldo', c_int32), ('reserved', c_int32)]


class CorrLevel(Structure):
  _fields_ = [('grid', c_void_p), ('h', c_int32), ('w', c_int32), ('C', c_int32),
              ('reserved', c_int32)]


class CorrArgs(Structure):
  _fields_ = [('levels', CorrLevel * MAX_CORR_LEVELS), ('num_levels', c_int32),
              ('num_points', c_int32), ('num_frames', c_int32), ('init_h', c_int32),
              ('init_w', c_int32), ('planes', c_int32),
              ('pos', c_void_p), ('occ', c_void_p), ('expd', c_void_p),
              ('feat_hi', c_void_p), ('feat_hi_stride_n', c_int64), ('feat_hi_stride_t', c_int64),
              ('feat_lo', c_void_p), ('feat_lo_stride_n', c_int64), ('feat_lo_stride_t', c_int64),
              ('out_planes', c_void_p), ('out_plane_stride', c_int64), ('ld', c_int32),
              ('reserved', c_int32)]


class QueryGrid(Structure):
  _fields_ = [('grid', c_void_p), ('clip_stride', c_int64), ('out', c_void_p), ('h', c_int32),
              ('w', c_int32), ('C', c_int32), ('reserved', c_int32)]


class UpdateArgs(Structure):
  _fields_ = [('res', c_void_p), ('ld_res', c_int32), ('num_points', c_int32),
              ('num_frames', c_int32), ('init_h', c_int32), ('init_w', c_int32),
              ('resize_h', c_int32), ('resize_w', c_int32), ('video_h', c_int32),
              ('video_w', c_int32), ('reserved', c_int32),
              ('feat_hi', c_void_p), ('feat_hi_stride_n', c_int64), ('feat_hi_stride_t', c_int64),
              ('feat_lo', c_void_p), ('feat_lo_stride_n', c_int64), ('feat_lo_stride_t', c_int64),
              ('pos', c_void_p), ('occ_in', c_void_p), ('expd_in', c_void_p),
              ('occ_out', c_void_p), ('expd_out', c_void_p), ('feat_out', c_void_p),
              ('tracks_out', c_void_p)]


class TapvidArgs(Structure):
  _fields_ = [('query_points', c_void_p), ('gt_occluded', c_void_p), ('gt_tracks', c_void_p),
              ('pred_occluded', c_void_p), ('pred_occ_logits', c_void_p),
              ('pred_expd_logits', c_void_p), ('pred_tracks', c_void_p),
              ('B', c_int32), ('N', c_int32), ('T', c_int32), ('query_mode', c_int32),
              ('counts', c_void_p)]


REDETECTION_MAX_THRESHOLDS = 16


class RedetectionArgs(Structure):
  _fields_ = [('gt_visible', c_void_p), ('pred_visible', c_void_p), ('pred_occ_logits', c_void_p),
              ('pred_expd_logits', c_void_p), ('pred_tracks', c_void_p), ('gt_tracks', c_void_p),
              ('thresholds', c_float * REDETECTION_MAX_THRESHOLDS), ('num_thresholds', c_int32),
              ('B', c_int32), ('N', c_int32), ('T', c_int32), ('capacity', c_int64),
              ('event_t', c_void_p), ('event_duration', c_void_p), ('event_values', c_void_p),
              ('event_count', c_void_p)]


class HomographyArgs(Structure):
  _fields_ = [('tracks', c_void_p), ('tracks_fp64', c_int32), ('N', c_int32), ('T', c_int32),
              ('reference_frame', c_int32), ('occluded', c_void_p), ('width', c_double),
              ('height', c_double), ('thresh', c_double), ('outlier_point_threshold', c_double),
              ('num_refinement_passes', c_int32), ('reserved', c_int32),
              ('stop_thresholds', c_void_p), ('homogs', c_void_p), ('err', c_void_p),
              ('canonical', c_void_p), ('ransac_stats', c_void_p), ('workspace', c_void_p),
              ('workspace_bytes', c_size_t)]


class Yuv420Frames(Structure):
  _fields_ = [('y', c_void_p), ('u', c_void_p), ('v', c_void_p),
              ('y_frame_stride', c_int64), ('u_frame_stride', c_int64), ('v_frame_stride', c_int64),
              ('y_pitch', c_int64), ('u_pitch', c_int64), ('v_pitch', c_int64),
              ('chroma_step', c_int32), ('H', c_int32), ('W', c_int32),
              ('y0', c_int32), ('x0', c_int32), ('h', c_int32), ('w', c_int32),
              ('matrix', c_int32), ('full_range', c_int32), ('reserved', c_int32)]


class YuvFrames(Structure):
  _fields_ = [('y', c_void_p), ('u', c_void_p), ('v', c_void_p),
              ('y_frame_stride', c_int64), ('u_frame_stride', c_int64), ('v_frame_stride', c_int64),
              ('y_pitch', c_int64), ('u_pitch', c_int64), ('v_pitch', c_int64),
              ('H', c_int32), ('W', c_int32), ('y0', c_int32), ('x0', c_int32), ('h', c_int32),
              ('w', c_int32), ('matrix', c_int32), ('full_range', c_int32),
              ('sample_bytes', c_int32), ('bits', c_int32), ('lsb_aligned', c_int32),
              ('luma_step', c_int32), ('chroma_step', c_int32), ('chroma_shift_x', c_int32),
              ('chroma_shift_y', c_int32), ('reserved', c_int32)]


class IngestDesc(Structure):
  _fields_ = [('src', c_void_p), ('pitch', c_int64), ('format', c_int32), ('H', c_int32),
              ('W', c_int32), ('y0', c_int32), ('x0', c_int32), ('h', c_int32), ('w', c_int32),
              ('reserved', c_int32), ('yuv', Yuv420Frames)]


INGEST_U8, INGEST_YUV420, INGEST_YUV = 1, 2, 3
INGEST_MAX_FRAMES = 64
TAPVID_COUNTERS = 18

# name -> (restype, argtypes); this table is also what tests/test_abi.py checks against
# include/tapir_b200.h
SIGNATURES = {
    'tapir_last_error': (c_char_p, []),
    'tapir_abi_version': (ctypes.c_int, []),
    'tapir_launch_count': (c_ulonglong, []),
    'tapir_profile_enable': (None, [c_int32]),
    'tapir_profile_report': (ctypes.c_int, [ctypes.c_char_p, c_size_t]),
    'tapir_split_planes': (ctypes.c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int64,
                                          c_int32, c_int32, c_int32, c_void_p]),
    'tapir_gemm': (ctypes.c_int, [c_void_p, c_int32, c_int64, POINTER(Linear), c_int64, c_int32,
                                  c_int32, c_int32, c_int32, c_int32, c_void_p, c_int32, c_int32,
                                  c_void_p, c_int32, c_void_p, c_int32, c_int64, c_int32, c_void_p,
                                  c_int32, c_int32, c_void_p]),
    'tapir_gemm_ex': (ctypes.c_int, [c_void_p, c_int32, c_int64, POINTER(Linear), c_int64, c_int32,
                                     c_int32, c_int32, c_int32, c_int32, c_void_p, c_int32, c_int32,
                                     c_void_p, c_int32, c_void_p, c_int32, c_int64, c_int32,
                                     c_void_p, c_int32, c_int32, c_void_p, c_size_t, c_void_p]),
    'tapir_bilinear_resize': (ctypes.c_int, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p,
                                             c_int32, c_int32, c_void_p]),
    'tapir_stem_conv': (ctypes.c_int, [c_void_p, c_int32, c_void_p, c_int32, c_int32, c_int32,
                                       c_void_p, c_void_p]),
    'tapir_instnorm_stats': (ctypes.c_int, [c_void_p, c_int32, c_int64, c_int32, c_void_p,
                                            c_void_p]),
    'tapir_instnorm_relu_split': (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int32,
                                                 c_int64, c_int32, c_void_p, c_int64, c_int32,
                                                 c_void_p, c_int32, c_void_p]),
    'tapir_im2col_s2': (ctypes.c_int, [c_void_p, c_int64, c_int32, c_int32, c_int32, c_int32,
                                       c_int32, c_void_p, c_int64, c_int32, c_void_p]),
    'tapir_layernorm_split': (ctypes.c_int, [c_void_p, c_int64, c_int32, c_void_p, c_void_p,
                                             c_void_p, c_void_p, c_int64, c_int32, c_void_p]),
    'tapir_l2_normalize': (ctypes.c_int, [c_void_p, c_int64, c_int32, c_void_p, c_void_p]),
    'tapir_backbone_workspace_bytes': (c_size_t, [c_int32, c_int32, c_int32, c_int32, c_int32]),
    'tapir_backbone_forward': (ctypes.c_int, [POINTER(BackboneWeights), c_void_p, c_int32, c_int32,
                                              c_int32, c_void_p, c_void_p, c_void_p, c_size_t,
                                              c_void_p]),
    'tapir_backbone_forward_u8': (ctypes.c_int, [POINTER(BackboneWeights), c_void_p, c_int32,
                                                 c_int32, c_int32, c_void_p, c_void_p, c_void_p,
                                                 c_size_t, c_void_p]),
    'tapir_backbone_forward_ex': (ctypes.c_int, [POINTER(BackboneWeights), c_void_p, c_int32,
                                                 c_int32, c_int32, c_int32, c_void_p, c_void_p,
                                                 c_void_p, c_size_t, c_void_p, c_void_p]),
    'tapir_backbone_stem': (ctypes.c_int, [POINTER(BackboneWeights), c_void_p, c_int32, c_int32,
                                           c_int32, c_int32, c_int32, c_int32, c_void_p, c_size_t,
                                           c_void_p]),
    'tapir_ingest_frames': (ctypes.c_int, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32,
                                           c_int32, c_int32, c_void_p, c_int32, c_int32, c_void_p]),
    'tapir_yuv420_to_rgb': (ctypes.c_int, [POINTER(Yuv420Frames), c_int32, c_void_p, c_void_p]),
    'tapir_ingest_frames_yuv420': (ctypes.c_int, [POINTER(Yuv420Frames), c_int32, c_void_p,
                                                  c_int32, c_int32, c_void_p]),
    'tapir_yuv_to_rgb': (ctypes.c_int, [POINTER(YuvFrames), c_int32, c_void_p, c_void_p]),
    'tapir_ingest_frames_yuv': (ctypes.c_int, [POINTER(YuvFrames), c_int32, c_void_p, c_int32,
                                               c_int32, c_void_p]),
    'tapir_ingest_frames_multi': (ctypes.c_int, [POINTER(IngestDesc), c_int32, c_void_p, c_int32,
                                                 c_int32, c_void_p]),
    'tapir_backbone_forward_yuv420': (ctypes.c_int, [POINTER(BackboneWeights), POINTER(Yuv420Frames),
                                                     c_int32, c_void_p, c_void_p, c_void_p,
                                                     c_size_t, c_void_p, c_void_p]),
    'tapir_backbone_forward_yuv': (ctypes.c_int, [POINTER(BackboneWeights), POINTER(YuvFrames),
                                                  c_int32, c_void_p, c_void_p, c_void_p, c_size_t,
                                                  c_void_p, c_void_p]),
    'tapir_postprocess_occlusions': (ctypes.c_int, [c_void_p, c_void_p, c_int64, c_void_p,
                                                    c_void_p]),
    'tapir_tapvid_counts': (ctypes.c_int, [POINTER(TapvidArgs), c_void_p]),
    'tapir_redetection_max_events': (c_int32, [c_int32]),
    'tapir_redetection_events': (ctypes.c_int, [POINTER(RedetectionArgs), c_void_p]),
    'tapir_sample_query_features': (ctypes.c_int, [c_void_p, c_int32, c_int32, c_int32, c_int32,
                                                   c_void_p, c_int32, c_int32, c_int32, c_int32,
                                                   c_void_p, c_void_p]),
    'tapir_sample_query_features_ex': (ctypes.c_int, [c_void_p, c_int32, c_int32, c_int32, c_int32,
                                                      c_void_p, c_int32, c_int32, c_int32, c_int32,
                                                      c_void_p, c_void_p, c_void_p]),
    'tapir_sample_query_rows': (ctypes.c_int, [POINTER(QueryGrid), c_int32, c_int32, c_int32, c_int32,
                                               c_int32, c_void_p, c_void_p, c_void_p, c_void_p,
                                               c_int32, c_void_p]),
    'tapir_cost_volume_workspace_bytes': (c_size_t, [c_int32, c_int32, c_int32, c_int32, c_int32]),
    'tapir_cost_volume_tracks': (ctypes.c_int, [POINTER(HeadWeights), c_void_p, c_void_p, c_int32,
                                                c_int32, c_int32, c_int32, c_int32, c_void_p,
                                                c_float, c_int32, c_int32, c_void_p, c_void_p,
                                                c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'tapir_cost_volume_batched_workspace_bytes': (c_size_t, [c_int32, c_int32, c_int32, c_int32,
                                                             c_int32, c_int32]),
    'tapir_cost_volume_tracks_batched': (ctypes.c_int, [POINTER(HeadWeights), c_void_p, c_void_p,
                                                        c_int32, c_int32, c_int32, c_int32, c_int32,
                                                        c_int32, c_void_p, c_float, c_int32, c_int32,
                                                        c_void_p, c_void_p, c_void_p, c_void_p,
                                                        c_void_p, c_size_t, c_void_p]),
    'tapir_cost_volume_ragged_workspace_bytes': (c_size_t, [c_int32, c_int32, c_int32, c_int32,
                                                            c_int32, c_int32]),
    'tapir_cost_volume_tracks_ragged': (ctypes.c_int, [POINTER(HeadWeights), c_void_p, c_void_p,
                                                       c_int32, POINTER(c_int32), c_int32, c_int32,
                                                       c_int32, c_int32, c_void_p, c_float, c_int32,
                                                       c_int32, c_void_p, c_void_p, c_void_p, c_void_p,
                                                       c_void_p, c_size_t, c_void_p]),
    'tapir_pool_pyramid': (ctypes.c_int, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p,
                                          c_void_p]),
    'tapir_local_corr': (ctypes.c_int, [POINTER(CorrArgs), c_void_p]),
    'tapir_local_corr_batched': (ctypes.c_int, [POINTER(CorrArgs), c_int32, c_void_p]),
    'tapir_local_corr_ragged': (ctypes.c_int, [POINTER(CorrArgs), c_int32, c_void_p, c_void_p]),
    'tapir_mixer_workspace_bytes': (c_size_t, [c_int64, c_int32]),
    'tapir_mixer_forward': (ctypes.c_int, [POINTER(MixerWeights), POINTER(MixerIO), c_void_p,
                                           c_size_t, c_void_p]),
    'tapir_mixer_dw': (ctypes.c_int, [POINTER(MixerBlock), c_void_p, c_int32, c_int32, c_int32, c_void_p,
                                      c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32,
                                      c_void_p]),
    'tapir_refine_update': (ctypes.c_int, [POINTER(UpdateArgs), c_void_p]),
    'tapir_refine_update_ex': (ctypes.c_int, [POINTER(UpdateArgs), c_void_p, c_int32, c_void_p]),
    'tapir_refine_update_ragged': (ctypes.c_int, [POINTER(UpdateArgs), c_void_p, c_void_p, c_void_p]),
    'tapir_paint_point_track_workspace_bytes': (c_size_t, [c_int32, c_int32]),
    'tapir_paint_point_track': (ctypes.c_int, [c_void_p, c_int32, c_int32, c_int32, c_void_p, c_int32,
                                               c_void_p, c_int32, c_void_p, c_void_p, c_void_p, c_size_t,
                                               c_void_p]),
    'tapir_ransac_stop_thresholds': (ctypes.c_int, [c_int32, c_double, c_void_p]),
    'tapir_homographies_workspace_bytes': (c_size_t, [c_int32, c_int32]),
    'tapir_homographies_wrt_frame': (ctypes.c_int, [POINTER(HomographyArgs), c_void_p]),
    'tapir_lanczos_weights': (c_int32, [c_int32, c_int32, c_void_p, c_void_p]),
    'tapir_resize_lanczos_u8_workspace_bytes': (c_size_t, [c_int32, c_int32, c_int32, c_int32, c_int32]),
    'tapir_resize_lanczos_u8': (ctypes.c_int, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32,
                                               c_int32, c_void_p, c_void_p, c_int32, c_void_p, c_void_p,
                                               c_int32, c_void_p, c_size_t, c_void_p]),
}

_lib = None


class TapirB200Error(RuntimeError):
  pass


def load():
  """Loads the shared library (once).  Raises if it has not been built."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise TapirB200Error(
        f'{LIB_PATH} not found: build it first (python -m tapnet_b200.build or '
        '__graft_entry__.build()).  tapnet_b200 has no CPU / PyTorch fallback.')
  lib = ctypes.CDLL(LIB_PATH)
  for name, (restype, argtypes) in SIGNATURES.items():
    fn = getattr(lib, name)  # AttributeError if a declared symbol is missing
    fn.restype = restype
    fn.argtypes = argtypes
  _lib = lib
  return lib


def check(status, what=''):
  if status != 0:
    msg = load().tapir_last_error()
    raise TapirB200Error(f'{what} failed (status {status}): {msg.decode() if msg else "?"}')


# ------------------------------------------------------------------------------ host checks
def ptr(t):
  """The tensor's data pointer as a c_void_p (None stays None)."""
  return None if t is None else c_void_p(t.data_ptr())


def stream(device=None):
  """The current CUDA stream of `device` (default: the current device) as a c_void_p."""
  return c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _need(ok, fn, msg):
  if not ok:
    raise ValueError(f'{fn}: {msg}')


def _bad(fn, name, t, want):
  raise ValueError(f'{fn}: {name} must be {want}, got {t.dtype} {tuple(t.shape)} with strides '
                   f'{t.stride()} on {t.device}')


def _check(fn, name, t, dtype, shape=None, dense=True, device=None):
  """t has `dtype`, and `shape` and `device` when given, and is contiguous (dense) or at least
  unit-stride in its last dim."""
  if (t.dtype != dtype or (shape is not None and t.shape != shape)
      or (device is not None and t.device != device)
      or not (t.is_contiguous() if dense else t.stride(-1) == 1)):
    _bad(fn, name, t, f'{"contiguous" if dense else "unit-stride"} {dtype} '
         f'{"[...]" if shape is None else list(shape)} on {device or "its device"}')


def _rows(fn, name, t, Q, T, width):
  """t is contiguous fp32 [..., T] (width 0) or [..., T, width] holding Q x T rows; its leading
  dims may be [clips, queries]."""
  if (t.dtype is not torch.float32 or t.numel() != Q * T * (width or 1)
      or t.shape[-1] != (width or T) or not t.is_contiguous()):
    _bad(fn, name, t, f'contiguous float32 [..., {T}{f", {width}" if width else ""}] of {Q} x {T} rows')


def _feat(fn, name, f, Q, T, C):
  """(pointer, stride_n, stride_t) of a [Q, T, C] feature view: per-(query, frame) rows, or
  per-query vectors with stride 0 over T."""
  _check(fn, name, f, torch.float32, (Q, T, C), False)
  return f.data_ptr(), f.stride(0), f.stride(1)


def _nbytes(t):
  return t.numel() * t.element_size()


def _is_yuv(x):
  return hasattr(x, 'yuv_struct')  # live.YUVFrames (live imports this module)


def _frames(fn, frames, dtypes=(torch.uint8, torch.float32)):
  """[..., H, W, 3] contiguous frames of one of `dtypes` (a YUV clip checks its own planes)."""
  if not _is_yuv(frames) and (frames.dtype not in dtypes or frames.dim() < 3
                              or frames.shape[-1] != 3 or not frames.is_contiguous()):
    _bad(fn, 'frames', frames, f'contiguous [..., H, W, 3] {" or ".join(map(str, dtypes))}')


# ------------------------------------------------------------------------------ weights
def split_planes(src, dst):
  """fp32 src [rows, cols] -> bf16 planes dst [P, rows, kpad >= cols] (padding zeroed)."""
  fn = 'tapir_split_planes'
  P, rows, kpad = dst.shape
  _check(fn, 'dst', dst, torch.bfloat16)
  _check(fn, 'src', src, torch.float32, dense=False, device=dst.device)
  _need(src.dim() == 2 and src.shape[0] == rows and src.shape[1] <= kpad, fn,
        f'src {tuple(src.shape)} does not fit planes {tuple(dst.shape)}')
  check(load().tapir_split_planes(ptr(src), src.stride(0), ptr(dst), kpad, rows * kpad, rows,
                                  src.shape[1], kpad, P, stream()), fn)


def padded_k(k):
  """A GEMM operand's K rounded up to whole 64-wide k-blocks: the width its bf16 planes have."""
  return (k + 63) // 64 * 64


def pack_weights(sd, planes, extra_convs, device):
  """The backbone, head and mixer weight structs of state dict `sd` with `planes` bf16 planes:
  dict(backbone, head, mixer, keep, mixer_in, num_blocks), `keep` holding what they point into."""
  keep = []

  def f32(t):
    keep.append(t.to(device=device, dtype=torch.float32).contiguous().clone())
    return keep[-1].data_ptr()

  def linear(w2d, bias=None):
    n, k = w2d.shape
    kp = padded_k(k)
    keep.append(torch.empty(planes, n, kp, dtype=torch.bfloat16, device=device))
    split_planes(w2d.to(device=device, dtype=torch.float32).contiguous(), keep[-1])
    return Linear(w=keep[-1].data_ptr(), bias=f32(bias) if bias is not None else None, N=n, K=kp,
                  planes=planes, k_logical=k)

  def conv(key, bias=False):
    w = sd[key + '.weight']
    return linear(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1),  # K order (ky, kx, cin)
                  sd[key + '.bias'] if bias else None)

  def lin(key):
    return linear(sd[key + '.weight'], sd[key + '.bias'])

  bw = BackboneWeights(stem_w=f32(sd['resnet_torch.initial_conv.weight'].permute(2, 3, 1, 0)),
                       planes=planes)  # [7, 7, 3, 64]
  cin = 64
  for g, (cout, stride) in enumerate(zip(schema.GROUP_CHANNELS, schema.GROUP_STRIDES)):
    for b in range(2):
      p = f'resnet_torch.block_groups.{g}.blocks.{b}.'
      blk = bw.blocks[2 * g + b]
      blk.cin, blk.cout = (cin if b == 0 else cout), cout
      blk.stride, blk.has_proj = (stride, 1) if b == 0 else (1, 0)
      if b == 0:
        blk.proj = conv(p + 'proj_conv')
      blk.conv0, blk.conv1 = conv(p + 'conv_0'), conv(p + 'conv_1')
      blk.bn0_w, blk.bn0_b = f32(sd[p + 'bn_0.weight']), f32(sd[p + 'bn_0.bias'])
      blk.bn1_w, blk.bn1_b = f32(sd[p + 'bn_1.weight']), f32(sd[p + 'bn_1.bias'])
    cin = cout
  bw.num_extra = schema.NUM_EXTRA_CONV_BLOCKS if extra_convs else 0
  for i in range(bw.num_extra):
    p = f'extra_convs.blocks.{i}.'
    eb = bw.extra[i]
    eb.ln_w, eb.ln_b = f32(sd[p + 'layer_norm.weight']), f32(sd[p + 'layer_norm.bias'])
    eb.conv, eb.conv1 = conv(p + 'conv', True), conv(p + 'conv_1', True)

  m = 'torch_cost_volume_track_mods.'
  hw = HeadWeights(**{f'{name}_{wb}': f32(sd[f'{m}{key}.{full}'])
                      for name, key in (('hid1', 'hid1'), ('hid2', 'hid2'), ('hid3', 'hid3'),
                                        ('hid4', 'hid4'), ('occ', 'occ_out'))
                      for wb, full in (('w', 'weight'), ('b', 'bias'))})

  x = 'torch_pips_mixer.'
  nb = len([k for k in sd if k.startswith(x + 'blocks.') and k.endswith('.layer_norm.weight')])
  mw = MixerWeights(linear=lin(x + 'linear'), linear_1=lin(x + 'linear_1'),
                    ln_w=f32(sd[x + 'layer_norm.weight']), num_blocks=nb, planes=planes)
  for i in range(nb):
    p = f'{x}blocks.{i}.'
    blk = mw.blocks[i]
    blk.ln_w, blk.ln1_w = f32(sd[p + 'layer_norm.weight']), f32(sd[p + 'layer_norm_1.weight'])
    blk.dw1_w, blk.dw1_b = f32(sd[p + 'mlp1_up.weight']), f32(sd[p + 'mlp1_up.bias'])
    blk.dw2_w, blk.dw2_b = f32(sd[p + 'mlp1_up_1.weight']), f32(sd[p + 'mlp1_up_1.bias'])
    blk.up = lin(p + 'conv_channels_mixer.mlp2_up')
    blk.down = lin(p + 'conv_channels_mixer.mlp2_down')
  return dict(backbone=bw, head=hw, mixer=mw, keep=keep, mixer_in=int(mw.linear.K), num_blocks=nb)


# ------------------------------------------------------------------------------ frames
def ingest_frames(frames, out, window=None):
  """uint8 frames [..., H, W, 3] cropped to `window` (y0, x0, h, w), or a YUV clip (cropped to its
  own window) -> float32 [-1, 1] out [..., oh, ow, 3] with the reference's bilinear resize."""
  fn = 'ingest_frames'
  _frames(fn, frames, (torch.uint8,))
  _check(fn, 'out', out, torch.float32, device=frames.device)
  _need(out.shape[:-3] == frames.shape[:-3] and out.shape[-1] == 3, fn,
        f'out {tuple(out.shape)} does not match frames {tuple(frames.shape)}')
  nf, (oh, ow), (H, W) = math.prod(out.shape[:-3]), out.shape[-3:-1], frames.shape[-3:-1]
  if _is_yuv(frames):
    _need(window is None, fn, 'a YUV clip carries its own window')
    desc = frames.yuv_struct()
    return check(load().tapir_ingest_frames_yuv(byref(desc), nf, ptr(out), oh, ow, stream()),
                 'tapir_ingest_frames_yuv')
  y0, x0, h, w = (0, 0, H, W) if window is None else window
  check(load().tapir_ingest_frames(ptr(frames), nf, H, W, y0, x0, h, w, ptr(out), oh, ow,
                                   stream()), 'tapir_ingest_frames')


def resample_frames(video, out):
  """video [..., H, W, 3] (float32, uint8 or a YUV clip) resized into float32 out [..., h, w, 3]."""
  if _is_yuv(video) or video.dtype == torch.uint8:
    return ingest_frames(video, out)
  fn = 'tapir_bilinear_resize'
  _frames(fn, video, (torch.float32,))
  _check(fn, 'out', out, torch.float32, video.shape[:-3] + out.shape[-3:-1] + (3,), device=video.device)
  check(load().tapir_bilinear_resize(ptr(video), math.prod(out.shape[:-3]), video.shape[-3],
                                     video.shape[-2], 3, ptr(out), out.shape[-3], out.shape[-2],
                                     stream()), fn)


def ingest_desc(frame):
  """The tapir_ingest_desc of one frame: a uint8 [H, W, 3] tensor whose rows may be pitched (dense
  pixels), or a YUV clip of one frame (read inside its own window).  Returns (desc, what the
  descriptor points into)."""
  fn = 'ingest_desc'
  if _is_yuv(frame):
    _need(math.prod(frame.shape[:-3]) == 1, fn, f'a YUV clip of one frame, got {tuple(frame.shape)}')
    yuv = frame.yuv_struct()
    return IngestDesc(src=ctypes.addressof(yuv), format=INGEST_YUV), (yuv, frame._keep)
  if (frame.dtype != torch.uint8 or frame.dim() != 3 or frame.shape[-1] != 3
      or frame.stride(2) != 1 or frame.stride(1) != 3):
    _bad(fn, 'frame', frame, 'uint8 [H, W, 3] with dense pixels')
  H, W = frame.shape[:2]
  return IngestDesc(src=frame.data_ptr(), pitch=frame.stride(0), format=INGEST_U8, H=H, W=W, y0=0,
                    x0=0, h=H, w=W), frame


def ingest_frames_multi(frames, out):
  """Frames of their own sizes and formats (a list of ingest_desc's inputs: uint8 or YUV) -> float32
  [-1, 1] out [len(frames), oh, ow, 3]: frame i resized as resample_frames resizes it alone."""
  fn = 'tapir_ingest_frames_multi'
  _check(fn, 'out', out, torch.float32)
  _need(out.dim() == 4 and out.shape[0] == len(frames) and out.shape[-1] == 3, fn,
        f'out {tuple(out.shape)} for {len(frames)} frames')
  descs = (IngestDesc * len(frames))()
  keep = []
  for i, f in enumerate(frames):
    _need(f.device == out.device, fn, f'frame {i} on {f.device}, out on {out.device}')
    descs[i], k = ingest_desc(f)
    keep.append(k)
  check(load().tapir_ingest_frames_multi(descs, len(frames), ptr(out), out.shape[1], out.shape[2],
                                         stream()), fn)


def yuv_to_rgb(frames, out):
  """A YUV clip's window -> uint8 RGB out [B, T, h, w, 3]."""
  _check('tapir_yuv_to_rgb', 'out', out, torch.uint8, frames.shape, device=frames.device)
  desc = frames.yuv_struct()
  check(load().tapir_yuv_to_rgb(byref(desc), math.prod(out.shape[:-3]), ptr(out), stream()),
        'tapir_yuv_to_rgb')


# ------------------------------------------------------------------------------ backbone
def backbone_workspace_bytes(frames, h, w, extra_convs, planes):
  return load().tapir_backbone_workspace_bytes(frames, h, w, int(extra_convs), planes)


def backbone_stem(weights, frames, pass_frames, pass_frame0, workspace):
  """Stem convolution of frames [n, h, w, 3], frames pass_frame0 .. pass_frame0 + n - 1 of a pass
  of `pass_frames` that backbone_forward(..., stem_done=True) finishes."""
  fn = 'tapir_backbone_stem'
  _frames(fn, frames)
  n, h, w, _ = frames.shape
  _need(0 <= pass_frame0 and pass_frame0 + n <= pass_frames, fn, 'frames outside the pass')
  check(load().tapir_backbone_stem(byref(weights), ptr(frames), int(frames.dtype == torch.uint8),
                                   pass_frames, h, w, pass_frame0, n, ptr(workspace),
                                   _nbytes(workspace), stream()), fn)


def backbone_forward(weights, frames, lowres, hires, workspace, ready_event=None, frame0=0,
                     stem_done=False):
  """Backbone over frames frame0 .. frame0 + n - 1 of `frames` ([F, h, w, 3] or a YUV clip) into
  lowres [n, h/8, w/8, 256] and hires [n, h/4, w/4, 128].  `ready_event` is recorded once hires
  is final; with `stem_done`, backbone_stem has run and frames only give the size and dtype."""
  fn = 'tapir_backbone_forward'
  _frames(fn, frames)
  n, (h, w), dev = lowres.shape[0], frames.shape[-3:-1], frames.device
  _need(0 <= frame0 and frame0 + n <= math.prod(frames.shape[:-3]), fn, 'frames outside the clip')
  _check(fn, 'lowres', lowres, torch.float32, (n, h // 8, w // 8, schema.LOWRES_DIM), device=dev)
  _check(fn, 'hires', hires, torch.float32, (n, h // 4, w // 4, schema.HIRES_DIM), device=dev)
  ready = c_void_p(ready_event.cuda_event) if ready_event is not None else None
  if _is_yuv(frames):
    desc = frames.yuv_struct(frame0)
    return check(load().tapir_backbone_forward_yuv(
        byref(weights), byref(desc), n, ptr(lowres), ptr(hires), ptr(workspace), _nbytes(workspace),
        ready, stream()), 'tapir_backbone_forward_yuv')
  check(load().tapir_backbone_forward_ex(
      byref(weights), None if stem_done else ptr(frames[frame0:]), int(frames.dtype == torch.uint8),
      n, h, w, ptr(lowres), ptr(hires), ptr(workspace), _nbytes(workspace), ready, stream()), fn)


# ------------------------------------------------------------------------------ stage A
def sample_query_features(grid, query_tyx, video_shape, out, frame_slot=None):
  """Samples of grid [T, gh, gw, C] at query_tyx [N, 3] (coordinates of a video_shape = (T, H, W)
  clip) into out [N, C].  frame_slot: None (the grid holds the whole clip), or int32 [video T]
  mapping each clip frame to its slot among the grid's T frames, or -1; a query with a tap of
  nonzero weight on a frame without a slot gets a NaN row."""
  fn = 'tapir_sample_query_features' if frame_slot is None else 'tapir_sample_query_features_ex'
  _check(fn, 'grid', grid, torch.float32)
  (T, gh, gw, C), N = grid.shape, query_tyx.shape[0]
  _check(fn, 'query_tyx', query_tyx, torch.float32, (N, 3), device=grid.device)
  _check(fn, 'out', out, torch.float32, (N, C), device=grid.device)
  video_shape = tuple(int(v) for v in video_shape)
  if frame_slot is None:
    return check(load().tapir_sample_query_features(ptr(grid), T, gh, gw, C, ptr(query_tyx), N,
                                                    *video_shape, ptr(out), stream()), fn)
  _check(fn, 'frame_slot', frame_slot, torch.int32, (video_shape[0],), device=grid.device)
  check(load().tapir_sample_query_features_ex(ptr(grid), T, gh, gw, C, ptr(query_tyx), N,
                                              *video_shape, ptr(frame_slot), ptr(out), stream()), fn)


REQUEST_WORDS = 5  # tapir_query_request: row, clip and the float32 bits of t, y, x


def query_request_table(capacity, device, pin_memory=False):
  """An empty request table of sample_query_rows: int32 [1 + 5 capacity], the count first, then
  one (row, clip, t, y, x) request per 5 words."""
  return torch.zeros(1 + REQUEST_WORDS * capacity, dtype=torch.int32, device=device,
                     pin_memory=pin_memory)


def write_query_requests(table, requests):
  """Writes `requests`, a sequence of (row, clip, t, y, x), and their count into a host table of
  query_request_table."""
  n = len(requests)
  _need(table.device.type == 'cpu' and 1 + REQUEST_WORDS * n <= table.numel(), 'write_query_requests',
        f'{n} requests do not fit a host table of {table.numel()} words')
  a = table.numpy()
  a[0] = n
  if n:
    body = a[1:1 + REQUEST_WORDS * n].reshape(n, REQUEST_WORDS)
    body[:, :2] = [(r[0], r[1]) for r in requests]
    body[:, 2:].view('float32')[:] = [tuple(r[2:5]) for r in requests]


def state_pointer_table(state, rows):
  """The device pointer table of sample_query_rows over a causal state (a list of dicts of
  block_{i}_causal_1 [.., rows, 2, 512] and block_{i}_causal_2 [.., rows, 2, 2048] tensors),
  ctx1 and ctx2 of each block in turn."""
  fn = 'state_pointer_table'
  ptrs = []
  for d in state:
    for i in range(len(d) // 2):
      for k, width in ((f'block_{i}_causal_1', 512), (f'block_{i}_causal_2', 2048)):
        _need(k in d, fn, f'state entry without {k}')
        _check(fn, k, d[k], torch.float32, device=state[0][k].device)
        _need(d[k].numel() == rows * 2 * width and d[k].shape[-2:] == (2, width), fn,
              f'{k} {tuple(d[k].shape)} is not [.., {rows}, 2, {width}]')
        ptrs.append(d[k].data_ptr())
  dev = state[0]['block_0_causal_1'].device if state else 'cpu'
  return torch.tensor(ptrs, dtype=torch.int64).to(dev)


def sample_query_rows(grids, outs, video_hw, requests, state_table=None):
  """Applies the request table `requests` (query_request_table on the device) to a group of G
  one-frame clips whose queries are packed along R rows: each request's row of every outs[i]
  ([R, C] or [1, R, C]) is sampled from grids[i] ([G, 1, h, w, C] or [G, h, w, C]; each clip's
  grid dense) of its clip, and that row of every state tensor of state_table (state_pointer_table
  of R rows, or None) is zeroed.  video_hw: one (h, w) for every clip, or an int32 [G, 2] device
  table."""
  fn = 'tapir_sample_query_rows'
  _need(1 <= len(grids) == len(outs) <= MAX_QUERY_GRIDS, fn,
        f'{len(grids)} grids and {len(outs)} outputs (1..{MAX_QUERY_GRIDS}, one per grid)')
  dev = grids[0].device
  G = grids[0].shape[0]
  R = outs[0].shape[-2]
  table = (QueryGrid * len(grids))()
  for i, (g, o) in enumerate(zip(grids, outs)):
    _need(g.dim() in (4, 5) and (g.dim() == 4 or g.shape[1] == 1) and g.shape[0] == G, fn,
          f'grid {i} {tuple(g.shape)} is not [{G}, 1, h, w, C]')
    h, w, C = g.shape[-3:]
    _need(g.dtype == torch.float32 and g.device == dev and g[0].is_contiguous()
          and g.stride(0) >= h * w * C, fn, f'grid {i} must be float32 on {dev}, each clip dense')
    _check(fn, f'outs[{i}]', o, torch.float32, device=dev)
    _need(o.shape[-2:] == (R, C) and o.numel() == R * C, fn,
          f'outs[{i}] {tuple(o.shape)} is not [{R}, {C}]')
    table[i] = QueryGrid(grid=g.data_ptr(), clip_stride=g.stride(0), out=o.data_ptr(), h=h, w=w, C=C)
  _check(fn, 'requests', requests, torch.int32, (1 + REQUEST_WORDS * R,), device=dev)
  vh = vw = 0
  if isinstance(video_hw, torch.Tensor):
    _check(fn, 'video_hw', video_hw, torch.int32, (G, 2), device=dev)
  else:
    vh, vw = (int(v) for v in video_hw)
  K = 0
  if state_table is not None:
    _check(fn, 'state_table', state_table, torch.int64, device=dev)
    K = state_table.numel()
  words = ptr(requests).value
  check(load().tapir_sample_query_rows(
      table, len(grids), G, R, vh, vw, ptr(video_hw) if isinstance(video_hw, torch.Tensor) else None,
      c_void_p(words), c_void_p(words + 4), ptr(state_table), K, stream()), fn)


def pool_pyramid(grid, out):
  """2 x 2 average of grid [..., h, w, C] into out [..., h/2, w/2, C]."""
  fn = 'tapir_pool_pyramid'
  _check(fn, 'grid', grid, torch.float32)
  h, w, C = grid.shape[-3:]
  _check(fn, 'out', out, torch.float32, grid.shape[:-3] + (h // 2, w // 2, C), device=grid.device)
  check(load().tapir_pool_pyramid(ptr(grid), math.prod(grid.shape[:-3]), h, w, C, ptr(out),
                                  stream()), fn)


def cost_volume_workspace_bytes(qfeat, grid):
  """cost_volume_tracks' workspace for qfeat [G, n, C], grid [G, T, gh, gw, C] (or their shapes)."""
  G, n = getattr(qfeat, 'shape', qfeat)[:2]
  return load().tapir_cost_volume_batched_workspace_bytes(G, n, *getattr(grid, 'shape', grid)[1:])


def cost_volume_tracks(head, qfeat, grid, query_tyx, temperature, init_hw, points, occ, expd,
                       argmax, workspace):
  """Stage A of G clips: qfeat [G, n, C] against grid [G, T, gh, gw, C] -> points [G, n, T, 2]
  (initial-resolution pixels), occ, expd and (unless None) the arg-max cells argmax [G, n, T].
  query_tyx: [G, n, 3] in initial-resolution coordinates, or None."""
  fn = 'tapir_cost_volume_tracks_batched'
  _check(fn, 'qfeat', qfeat, torch.float32)
  (G, n, C), dev = qfeat.shape, qfeat.device
  _check(fn, 'grid', grid, torch.float32, device=dev)
  _need(grid.dim() == 5 and grid.shape[0] == G and grid.shape[-1] == C, fn, 'grid does not match qfeat')
  _, T, gh, gw, _ = grid.shape
  for name, t, dtype, shape in (('query_tyx', query_tyx, torch.float32, (G, n, 3)),
                                ('points', points, torch.float32, (G, n, T, 2)),
                                ('occ', occ, torch.float32, (G, n, T)),
                                ('expd', expd, torch.float32, (G, n, T)),
                                ('argmax', argmax, torch.int32, (G, n, T))):
    if t is not None or name in ('points', 'occ', 'expd'):
      _check(fn, name, t, dtype, shape, device=dev)
  check(load().tapir_cost_volume_tracks_batched(
      byref(head), ptr(qfeat), ptr(grid), G, n, T, gh, gw, C, ptr(query_tyx), float(temperature),
      init_hw[0], init_hw[1], ptr(points), ptr(occ), ptr(expd), ptr(argmax), ptr(workspace),
      _nbytes(workspace), stream()), fn)


def _counts(fn, counts):
  """The per-clip query counts of a ragged call as a list of ints (1..MAX_RAGGED_CLIPS of them,
  each >= 1)."""
  counts = [int(c) for c in counts]
  _need(1 <= len(counts) <= MAX_RAGGED_CLIPS, fn, f'{len(counts)} clips, 1..{MAX_RAGGED_CLIPS} supported')
  _need(min(counts) >= 1, fn, f'every clip needs at least one query, got {counts}')
  return counts


def cost_volume_ragged_workspace_bytes(num_clips, total_points, grid_shape):
  """cost_volume_tracks_ragged's workspace for num_clips clips with total_points queries in all
  against grids of shape [num_clips, T, gh, gw, C]."""
  return load().tapir_cost_volume_ragged_workspace_bytes(num_clips, total_points, *grid_shape[1:])


def cost_volume_tracks_ragged(head, qfeat, counts, grid, query_tyx, temperature, init_hw, points,
                              occ, expd, argmax, workspace):
  """Stage A of B = len(counts) clips with counts[b] queries each: qfeat [Q, C] (the clips' queries
  one after the other, Q = sum(counts)) against grid [B, T, gh, gw, C] -> points [Q, T, 2]
  (initial-resolution pixels), occ, expd and (unless None) argmax [Q, T].  query_tyx: [Q, 3] in
  initial-resolution coordinates, or None."""
  fn = 'tapir_cost_volume_tracks_ragged'
  counts = _counts(fn, counts)
  B, Q = len(counts), sum(counts)
  _check(fn, 'qfeat', qfeat, torch.float32)
  _need(qfeat.dim() == 2 and qfeat.shape[0] == Q, fn, f'qfeat {tuple(qfeat.shape)} for {Q} queries')
  C, dev = qfeat.shape[1], qfeat.device
  _check(fn, 'grid', grid, torch.float32, device=dev)
  _need(grid.dim() == 5 and grid.shape[0] == B and grid.shape[-1] == C, fn,
        f'grid {tuple(grid.shape)} does not match {B} clips of {C}-channel queries')
  _, T, gh, gw, _ = grid.shape
  for name, t, dtype, shape in (('query_tyx', query_tyx, torch.float32, (Q, 3)),
                                ('points', points, torch.float32, (Q, T, 2)),
                                ('occ', occ, torch.float32, (Q, T)),
                                ('expd', expd, torch.float32, (Q, T)),
                                ('argmax', argmax, torch.int32, (Q, T))):
    if t is not None or name in ('points', 'occ', 'expd'):
      _check(fn, name, t, dtype, shape, device=dev)
  check(load().tapir_cost_volume_tracks_ragged(
      byref(head), ptr(qfeat), ptr(grid), B, (c_int32 * B)(*counts), T, gh, gw, C, ptr(query_tyx),
      float(temperature), init_hw[0], init_hw[1], ptr(points), ptr(occ), ptr(expd), ptr(argmax),
      ptr(workspace), _nbytes(workspace), stream()), fn)


# ------------------------------------------------------------------------------ refinement
# corr_args, mixer_io and update_args run once per refinement iteration on the host-bound online
# step: one fused test per tensor (dtype, extent, contiguity), the device once per call.
def corr_args(levels, pos, occ, expd, feat_hi, feat_lo, out_planes, init_hw, ragged=False):
  """CorrArgs of the local correlation of G clips.  levels: grids [G, T, h, w, C], hires first;
  pos [..., T, 2], occ / expd [..., T] over Q = G x n queries (ragged: Q queries of the G clips in
  all, num_points = Q); feat_hi / feat_lo [Q, T, 128 | 256] views (stride 0 over T for per-query
  features); out_planes bf16 [P, Q * T, ld]."""
  fn, L = 'corr_args', len(levels)
  _need(1 <= L <= MAX_CORR_LEVELS, fn, f'{L} levels')
  (G, T), dev = levels[0].shape[:2], pos.device
  for g in levels:
    if (g.dtype != torch.float32 or g.dim() != 5 or g.shape[:2] != (G, T)
        or not g.is_contiguous()):
      _bad(fn, 'levels', g, f'contiguous float32 [{G}, {T}, h, w, C]')
  _need(levels[0].device == dev, fn, 'levels and pos on different devices')
  Q = pos.numel() // (2 * T) if T else 0
  _need(ragged or Q % G == 0, fn, f'{Q} queries over {G} clips')
  _rows(fn, 'pos', pos, Q, T, 2)
  _rows(fn, 'occ', occ, Q, T, 0)
  _rows(fn, 'expd', expd, Q, T, 0)
  P, _, ld = out_planes.shape
  _check(fn, 'out_planes', out_planes, torch.bfloat16, (P, Q * T, ld), False)
  _need(out_planes.stride(1) == ld and ld >= 388 + 49 * L, fn,
        f'out_planes rows must be dense and hold the {388 + 49 * L} mixer inputs')
  ca = CorrArgs(num_levels=L, num_points=Q if ragged else Q // G, num_frames=T, init_h=int(init_hw[0]),
                init_w=int(init_hw[1]), planes=P, pos=pos.data_ptr(), occ=occ.data_ptr(),
                expd=expd.data_ptr(), out_planes=out_planes.data_ptr(),
                out_plane_stride=out_planes.stride(0), ld=ld)
  for i, g in enumerate(levels):
    ca.levels[i] = CorrLevel(g.data_ptr(), g.shape[2], g.shape[3], g.shape[4], 0)
  ca.feat_hi, ca.feat_hi_stride_n, ca.feat_hi_stride_t = _feat(fn, 'feat_hi', feat_hi, Q, T, schema.HIRES_DIM)
  ca.feat_lo, ca.feat_lo_stride_n, ca.feat_lo_stride_t = _feat(fn, 'feat_lo', feat_lo, Q, T, schema.LOWRES_DIM)
  return ca


def local_corr(*args, query_clip=None):
  """Local correlation of the G = levels[0].shape[0] clips of corr_args(*args) in one launch.
  query_clip: None (clips of equal query counts), or int32 [Q] giving each query's clip."""
  G = args[0][0].shape[0]
  if query_clip is None:
    ca = corr_args(*args)
    return check(load().tapir_local_corr_batched(byref(ca), G, stream()), 'tapir_local_corr_batched')
  fn = 'tapir_local_corr_ragged'
  ca = corr_args(*args, ragged=True)
  _check(fn, 'query_clip', query_clip, torch.int32, (ca.num_points,), device=args[1].device)
  check(load().tapir_local_corr_ragged(byref(ca), G, ptr(query_clip), stream()), fn)


def mixer_workspace_bytes(x_planes):
  """mixer_forward's workspace for x_planes [P, rows, ldx] (or its shape)."""
  P, rows = getattr(x_planes, 'shape', x_planes)[:2]
  return load().tapir_mixer_workspace_bytes(rows, P)


def _ctx_array(fn, name, ctx, nb, n, width, dev):
  if ctx is None:
    return None
  # 48 tensors per call: only what bounds the memory the kernels touch (dtype, extent,
  # contiguity); the list's first tensor also has its layout and device checked
  _need(len(ctx) == nb, fn, f'{name} needs {nb} entries')
  if ctx[0].shape[-1] != width or ctx[0].device != dev:
    _bad(fn, name, ctx[0], f'[..., 2, {width}] on {dev}')
  want, f32 = n * 2 * width, torch.float32
  for t in ctx:
    if t.dtype is not f32 or t.numel() != want or not t.is_contiguous():
      _bad(fn, name, t, f'contiguous float32 [..., 2, {width}] of {n} queries')
  return (c_void_p * nb)(*[t.data_ptr() for t in ctx])


def mixer_io(weights, x_planes, out, causal, ctx1_in=None, ctx2_in=None, ctx1_out=None,
             ctx2_out=None):
  """MixerIO of the `weights` mixer over x_planes bf16 [P, n * T, ldx] into out [n, T, ldo].  The
  causal contexts are lists of one [..., 2, 512] (ctx1) / [..., 2, 2048] (ctx2) tensor per block
  holding n queries each, or None."""
  fn = 'mixer_io'
  (n, T, ldo), dev = out.shape, out.device
  P, rows, ldx = x_planes.shape
  _check(fn, 'out', out, torch.float32)
  _check(fn, 'x_planes', x_planes, torch.bfloat16, dense=False, device=dev)
  _need(rows == n * T and x_planes.stride(1) == ldx and ldx >= weights.linear.K
        and P >= weights.planes and ldo >= 388, fn,
        f'x_planes {tuple(x_planes.shape)} and out {tuple(out.shape)} do not fit the mixer '
        f'(dense rows, {weights.planes} planes of {weights.linear.K} inputs, 388 outputs)')
  nb = weights.num_blocks
  return MixerIO(x_planes=x_planes.data_ptr(), x_plane_stride=x_planes.stride(0), ldx=ldx,
                 num_points=n, num_frames=T, causal=int(causal),
                 ctx1_in=_ctx_array(fn, 'ctx1_in', ctx1_in, nb, n, 512, dev),
                 ctx2_in=_ctx_array(fn, 'ctx2_in', ctx2_in, nb, n, 2048, dev),
                 ctx1_out=_ctx_array(fn, 'ctx1_out', ctx1_out, nb, n, 512, dev),
                 ctx2_out=_ctx_array(fn, 'ctx2_out', ctx2_out, nb, n, 2048, dev),
                 out=out.data_ptr(), ldo=ldo)


def mixer_forward(weights, x_planes, out, causal, ctx1_in, ctx2_in, ctx1_out, ctx2_out, workspace):
  """The PIPs mixer (arguments as mixer_io)."""
  io = mixer_io(weights, x_planes, out, causal, ctx1_in, ctx2_in, ctx1_out, ctx2_out)
  check(load().tapir_mixer_forward(byref(weights), byref(io), ptr(workspace), _nbytes(workspace),
                                   stream()), 'tapir_mixer_forward')


def update_args(res, pos, occ_in, expd_in, feat_hi, feat_lo, occ_out, expd_out, feat_out,
                tracks_out, init_hw, resize_hw, video_hw):
  """UpdateArgs of the track update: mixer output res [Q, T, ld >= 388] moves pos [..., T, 2] (in
  place) and writes occ_out / expd_out [..., T], feat_out [Q, T, 384] (the corr_args feature
  views plus the update) and, unless None, tracks_out [..., T, 2] in video pixels."""
  fn = 'update_args'
  (Q, T, ld), dev = res.shape, res.device
  _check(fn, 'res', res, torch.float32)
  _need(ld >= 388 and pos.device == dev, fn, f'res rows hold {ld} < 388 values or res and pos are on '
        'different devices')
  for name, t, width in (('pos', pos, 2), ('occ_in', occ_in, 0), ('expd_in', expd_in, 0),
                         ('occ_out', occ_out, 0), ('expd_out', expd_out, 0),
                         ('feat_out', feat_out, schema.HIRES_DIM + schema.LOWRES_DIM),
                         ('tracks_out', tracks_out, 2)):
    if t is not None or name != 'tracks_out':
      _rows(fn, name, t, Q, T, width)
  ua = UpdateArgs(res=res.data_ptr(), ld_res=ld, num_points=Q, num_frames=T,
                  pos=pos.data_ptr(), occ_in=occ_in.data_ptr(), expd_in=expd_in.data_ptr(),
                  occ_out=occ_out.data_ptr(), expd_out=expd_out.data_ptr(),
                  feat_out=feat_out.data_ptr(), tracks_out=ptr(tracks_out))
  ua.init_h, ua.init_w, ua.resize_h, ua.resize_w, ua.video_h, ua.video_w = (
      int(v) for v in (*init_hw, *resize_hw, *video_hw))
  ua.feat_hi, ua.feat_hi_stride_n, ua.feat_hi_stride_t = _feat(fn, 'feat_hi', feat_hi, Q, T, schema.HIRES_DIM)
  ua.feat_lo, ua.feat_lo_stride_n, ua.feat_lo_stride_t = _feat(fn, 'feat_lo', feat_lo, Q, T, schema.LOWRES_DIM)
  return ua


def refine_update(*args, video_table=None, query_clip=None):
  """The track update of update_args(*args).  video_table: None, or int32 [G, 2] per-clip (h, w)
  of the G clips the rows run over (the tracks of each clip scaled to its own size; video_hw is
  then not used).  query_clip: None (clips of equal query counts), or int32 [Q] giving each
  query's clip in video_table."""
  ua = update_args(*args)
  if video_table is None:
    _need(query_clip is None, 'tapir_refine_update_ragged', 'query_clip needs a video_table')
    return check(load().tapir_refine_update(byref(ua), stream()), 'tapir_refine_update')
  fn = 'tapir_refine_update_ex' if query_clip is None else 'tapir_refine_update_ragged'
  G = video_table.shape[0]
  _check(fn, 'video_table', video_table, torch.int32, (G, 2), device=args[0].device)
  if query_clip is not None:
    _check(fn, 'query_clip', query_clip, torch.int32, (ua.num_points,), device=args[0].device)
    return check(load().tapir_refine_update_ragged(byref(ua), ptr(video_table), ptr(query_clip),
                                                   stream()), fn)
  rows = ua.num_points * ua.num_frames
  _need(G >= 1 and rows % G == 0, fn, f'{rows} rows over {G} clips')
  check(load().tapir_refine_update_ex(byref(ua), ptr(video_table), rows // G, stream()), fn)


# ------------------------------------------------------------------------------ outputs
def postprocess_occlusions(occ, expd, out):
  """out (uint8 0 / 1) = (1 - sigmoid(occ)) * (1 - sigmoid(expd)) > 0.5, all the same shape."""
  fn = 'tapir_postprocess_occlusions'
  _check(fn, 'occ', occ, torch.float32)
  _check(fn, 'expd', expd, torch.float32, occ.shape, device=occ.device)
  _check(fn, 'out', out, torch.uint8, occ.shape, device=occ.device)
  check(load().tapir_postprocess_occlusions(ptr(occ), ptr(expd), occ.numel(), ptr(out), stream()), fn)


def tapvid_counts(query_points, gt_occluded, gt_tracks, pred_occluded, pred_tracks, query_mode,
                  counts, pred_logits=None):
  """int32 counts [B, N, TAPVID_COUNTERS] of pred_tracks [B, N, T, 2] against gt_tracks (float32)
  and gt_occluded (uint8); pred_occluded (uint8) or pred_logits (occlusion, expected_dist float32
  logits); query_points [B, N, 3]; query_mode 0 (first) or 1 (strided)."""
  fn = 'tapvid_counts'
  (B, N, T), dev = pred_tracks.shape[:3], pred_tracks.device
  logits = tuple(pred_logits) if pred_logits is not None else (None, None)
  checks = [('pred_tracks', pred_tracks, torch.float32, (B, N, T, 2)),
            ('query_points', query_points, torch.float32, (B, N, 3)),
            ('gt_occluded', gt_occluded, torch.uint8, (B, N, T)),
            ('gt_tracks', gt_tracks, torch.float32, (B, N, T, 2)),
            ('counts', counts, torch.int32, (B, N, TAPVID_COUNTERS))]
  if pred_logits is None:
    checks.append(('pred_occluded', pred_occluded, torch.uint8, (B, N, T)))
  else:
    pred_occluded = None
    checks += [(name, t, torch.float32, (B, N, T)) for name, t in zip(('occlusion', 'expected_dist'), logits)]
  for name, t, dtype, shape in checks:
    _check(fn, name, t, dtype, shape, device=dev)
  args = TapvidArgs(ptr(query_points), ptr(gt_occluded), ptr(gt_tracks), ptr(pred_occluded),
                    ptr(logits[0]), ptr(logits[1]), ptr(pred_tracks), B, N, T, query_mode, ptr(counts))
  check(load().tapir_tapvid_counts(byref(args), stream()), 'tapir_tapvid_counts')


def redetection_max_events(T):
  """Host only: K(T), the most eligible reappearance events a track of T frames can have."""
  return int(load().tapir_redetection_max_events(int(T)))


def redetection_events(gt_visible, pred_visible, pred_tracks, gt_tracks, thresholds, event_t,
                       event_duration, event_values, event_count, pred_logits=None):
  """The eligible reappearance events of every track of gt_visible [B, N, T] (uint8) and their
  AJ_RD values: pred_tracks / gt_tracks float32 [B, N, T, 2], pred_visible uint8 [B, N, T] or
  pred_logits (occlusion, expected_dist float32 logits), `thresholds` a sequence of 1 ..
  REDETECTION_MAX_THRESHOLDS distances.  Outputs: event_t / event_duration int32 [B, N, K(T)],
  event_values float32 [B, N, K(T), D], event_count int32 [B, N]."""
  fn = 'tapir_redetection_events'
  thresholds = [float(d) for d in thresholds]
  nd = len(thresholds)
  _need(1 <= nd <= REDETECTION_MAX_THRESHOLDS, fn,
        f'{nd} distance thresholds, 1 .. {REDETECTION_MAX_THRESHOLDS} supported')
  (B, N, T), dev = gt_visible.shape, gt_visible.device
  K = redetection_max_events(T)
  logits = tuple(pred_logits) if pred_logits is not None else (None, None)
  checks = [('gt_visible', gt_visible, torch.uint8, (B, N, T)),
            ('pred_tracks', pred_tracks, torch.float32, (B, N, T, 2)),
            ('gt_tracks', gt_tracks, torch.float32, (B, N, T, 2)),
            ('event_t', event_t, torch.int32, (B, N, K)),
            ('event_duration', event_duration, torch.int32, (B, N, K)),
            ('event_values', event_values, torch.float32, (B, N, K, nd)),
            ('event_count', event_count, torch.int32, (B, N))]
  if pred_logits is None:
    checks.append(('pred_visible', pred_visible, torch.uint8, (B, N, T)))
  else:
    pred_visible = None
    checks += [(name, t, torch.float32, (B, N, T)) for name, t in zip(('occlusion', 'expected_dist'), logits)]
  for name, t, dtype, shape in checks:
    _need(t is not None, fn, f'{name} is missing')
    _check(fn, name, t, dtype, shape, device=dev)
  args = RedetectionArgs(ptr(gt_visible), ptr(pred_visible), ptr(logits[0]), ptr(logits[1]),
                         ptr(pred_tracks), ptr(gt_tracks), (c_float * REDETECTION_MAX_THRESHOLDS)(*thresholds),
                         nd, B, N, T, B * N * K, ptr(event_t), ptr(event_duration), ptr(event_values),
                         ptr(event_count))
  check(load().tapir_redetection_events(byref(args), stream()), fn)


def paint_point_track_workspace_bytes(T, N):
  return int(load().tapir_paint_point_track_workspace_bytes(T, N))


def paint_point_track(frames, tracks, visibles, colors, out, workspace):
  """Paints tracks [N, T, 2] (x, y; float32 or float64) where visibles [N, T] (bool) onto uint8
  frames [T, H, W, 3] -> out, with colors uint8 [N, 3].  workspace: uint8, at least
  paint_point_track_workspace_bytes(T, N) bytes."""
  fn = 'tapir_paint_point_track'
  _check(fn, 'frames', frames, torch.uint8)
  (T, H, W, _), N, dev = frames.shape, tracks.shape[0], frames.device
  fp64 = tracks.dtype == torch.float64
  _check(fn, 'tracks', tracks, torch.float64 if fp64 else torch.float32, (N, T, 2), device=dev)
  _check(fn, 'visibles', visibles, torch.bool, (N, T), device=dev)
  _check(fn, 'colors', colors, torch.uint8, (N, 3), device=dev)
  _check(fn, 'out', out, torch.uint8, frames.shape, device=dev)
  check(load().tapir_paint_point_track(
      ptr(frames), T, H, W, ptr(tracks), int(fp64), ptr(visibles), N, ptr(colors), ptr(out),
      ptr(workspace), _nbytes(workspace), stream()), fn)


def ransac_stop_thresholds(N, targ_inlier_frac):
  """Host only: the RANSAC stop table thr [N] float64 (numpy)."""
  import numpy as np  # pylint: disable=g-import-not-at-top
  out = np.empty(max(int(N), 1), np.float64)
  check(load().tapir_ransac_stop_thresholds(int(N), float(targ_inlier_frac), out.ctypes.data),
        'tapir_ransac_stop_thresholds')
  return out


def homographies_workspace_bytes(T, N):
  return int(load().tapir_homographies_workspace_bytes(int(T), int(N)))


def homographies_wrt_frame(tracks, occluded, width, height, reference_frame, thresh,
                           outlier_point_threshold, num_refinement_passes, stop_thresholds, homogs,
                           err, canonical, ransac_stats, workspace):
  """Camera homographies of tracks [N, T, 2] (x, y pixels; float32 or float64) with occluded
  [N, T] (bool / uint8): homogs float64 [T, 3, 3], err float64 [N, T], canonical float64 [N, 2],
  ransac_stats int32 [T, 2] or None.  stop_thresholds: float64 [N] on the device
  (ransac_stop_thresholds); workspace: uint8, at least homographies_workspace_bytes(T, N)."""
  fn = 'tapir_homographies_wrt_frame'
  (N, T, _), dev = tracks.shape, tracks.device
  fp64 = tracks.dtype == torch.float64
  _check(fn, 'tracks', tracks, torch.float64 if fp64 else torch.float32, (N, T, 2))
  _need(occluded.dtype in (torch.bool, torch.uint8), fn, f'occluded must be bool or uint8, got {occluded.dtype}')
  _check(fn, 'occluded', occluded, occluded.dtype, (N, T), device=dev)
  _check(fn, 'stop_thresholds', stop_thresholds, torch.float64, (N,), device=dev)
  _check(fn, 'homogs', homogs, torch.float64, (T, 3, 3), device=dev)
  _check(fn, 'err', err, torch.float64, (N, T), device=dev)
  _check(fn, 'canonical', canonical, torch.float64, (N, 2), device=dev)
  if ransac_stats is not None:
    _check(fn, 'ransac_stats', ransac_stats, torch.int32, (T, 2), device=dev)
  _check(fn, 'workspace', workspace, torch.uint8, device=dev)
  args = HomographyArgs(ptr(tracks), int(fp64), N, T, int(reference_frame), ptr(occluded), float(width),
                        float(height), float(thresh), float(outlier_point_threshold),
                        int(num_refinement_passes), 0, ptr(stop_thresholds), ptr(homogs), ptr(err),
                        ptr(canonical), ptr(ransac_stats), ptr(workspace), _nbytes(workspace))
  check(load().tapir_homographies_wrt_frame(byref(args), stream(dev)), fn)


# ------------------------------------------------------------------------------ evaluation
def lanczos_weights(in_size, out_size):
  """Host only: PIL's 8-bit Lanczos tables of one axis in_size -> out_size, as numpy int32
  bounds [out_size, 2] (xmin, n) and taps [out_size, ksize]."""
  import numpy as np  # pylint: disable=g-import-not-at-top
  lib = load()
  ksize = lib.tapir_lanczos_weights(int(in_size), int(out_size), None, None)
  if ksize < 0:
    raise ValueError(lib.tapir_last_error().decode())
  bounds = np.empty((out_size, 2), np.int32)
  taps = np.empty((out_size, ksize), np.int32)
  lib.tapir_lanczos_weights(int(in_size), int(out_size), bounds.ctypes.data, taps.ctypes.data)
  return bounds, taps


def resize_lanczos_u8_workspace_bytes(T, H, W, h, w):
  return int(load().tapir_resize_lanczos_u8_workspace_bytes(T, H, W, h, w))


def resize_lanczos_u8(src, dst, x_tables, y_tables, workspace):
  """uint8 src [..., H, W, 3] -> dst [..., h, w, 3] with PIL's Lanczos.  x_tables / y_tables:
  (bounds, taps) int32 device tensors of lanczos_weights(W, w) / (H, h), or None for an axis that
  keeps its size; workspace: uint8, at least resize_lanczos_u8_workspace_bytes."""
  fn = 'tapir_resize_lanczos_u8'
  _frames(fn, src, (torch.uint8,))
  _check(fn, 'dst', dst, torch.uint8, device=src.device)
  _need(dst.dim() == src.dim() and dst.shape[:-3] == src.shape[:-3] and dst.shape[-1] == 3, fn,
        f'dst {tuple(dst.shape)} does not match src {tuple(src.shape)}')
  (H, W), (h, w), nf = src.shape[-3:-1], dst.shape[-3:-1], math.prod(src.shape[:-3])
  tables = []
  for name, t, n_out in (('x_tables', x_tables, w), ('y_tables', y_tables, h)):
    if t is None:
      tables += [None, None, 0]
      continue
    bounds, taps = t
    _check(fn, name, bounds, torch.int32, (n_out, 2), device=src.device)
    _check(fn, name, taps, torch.int32, device=src.device)
    _need(taps.dim() == 2 and taps.shape[0] == n_out, fn, f'{name} taps {tuple(taps.shape)} for {n_out} outputs')
    tables += [ptr(bounds), ptr(taps), taps.shape[1]]
  check(load().tapir_resize_lanczos_u8(ptr(src), ptr(dst), nf, H, W, h, w, *tables, ptr(workspace),
                                       _nbytes(workspace) if workspace is not None else 0, stream()), fn)
