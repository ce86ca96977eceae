"""ctypes binding of libtapir_b200.so (include/tapir_b200.h).

There is no CPU fallback: if the shared library is missing or cannot be loaded every
compute entry point raises.  `load()` never builds implicitly on import; use
`__graft_entry__.build()` / `python -m tapnet_b200.build`.
"""
import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_float, c_int32, c_int64, c_size_t, c_ulonglong, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'libtapir_b200.so')

MAX_MIXER_BLOCKS = 12
NUM_RESNET_BLOCKS = 8
MAX_EXTRA_BLOCKS = 5
MAX_CORR_LEVELS = 5


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


class Yuv420Frames(Structure):
  _fields_ = [('y', c_void_p), ('u', c_void_p), ('v', c_void_p),
              ('y_frame_stride', c_int64), ('u_frame_stride', c_int64), ('v_frame_stride', c_int64),
              ('y_pitch', c_int64), ('u_pitch', c_int64), ('v_pitch', c_int64),
              ('chroma_step', c_int32), ('H', c_int32), ('W', c_int32),
              ('y0', c_int32), ('x0', c_int32), ('h', c_int32), ('w', c_int32),
              ('matrix', c_int32), ('full_range', c_int32), ('reserved', c_int32)]


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
    'tapir_backbone_forward_yuv420': (ctypes.c_int, [POINTER(BackboneWeights), POINTER(Yuv420Frames),
                                                     c_int32, c_void_p, c_void_p, c_void_p,
                                                     c_size_t, c_void_p, c_void_p]),
    'tapir_postprocess_occlusions': (ctypes.c_int, [c_void_p, c_void_p, c_int64, c_void_p,
                                                    c_void_p]),
    'tapir_tapvid_counts': (ctypes.c_int, [POINTER(TapvidArgs), c_void_p]),
    'tapir_sample_query_features': (ctypes.c_int, [c_void_p, c_int32, c_int32, c_int32, c_int32,
                                                   c_void_p, c_int32, c_int32, c_int32, c_int32,
                                                   c_void_p, c_void_p]),
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
    'tapir_pool_pyramid': (ctypes.c_int, [c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p,
                                          c_void_p]),
    'tapir_local_corr': (ctypes.c_int, [POINTER(CorrArgs), c_void_p]),
    'tapir_local_corr_batched': (ctypes.c_int, [POINTER(CorrArgs), c_int32, c_void_p]),
    'tapir_mixer_workspace_bytes': (c_size_t, [c_int64, c_int32]),
    'tapir_mixer_forward': (ctypes.c_int, [POINTER(MixerWeights), POINTER(MixerIO), c_void_p,
                                           c_size_t, c_void_p]),
    'tapir_mixer_dw': (ctypes.c_int, [POINTER(MixerBlock), c_void_p, c_int32, c_int32, c_int32, c_void_p,
                                      c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32,
                                      c_void_p]),
    'tapir_refine_update': (ctypes.c_int, [POINTER(UpdateArgs), c_void_p]),
    'tapir_paint_point_track_workspace_bytes': (c_size_t, [c_int32, c_int32]),
    'tapir_paint_point_track': (ctypes.c_int, [c_void_p, c_int32, c_int32, c_int32, c_void_p, c_int32,
                                               c_void_p, c_int32, c_void_p, c_void_p, c_void_p, c_size_t,
                                               c_void_p]),
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
