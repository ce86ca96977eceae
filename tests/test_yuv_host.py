"""YUV 4:2:0 input without a GPU: the integer conversion oracle against the BT.601 / BT.709
formulas, the tapir_yuv420_frames ABI mirror, the descriptor arithmetic of live.YUV420Frames
and its argument errors."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tapnet_b200 import _lib, live

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (k, luma offset, cr, gu, gv, bu) of include/tapir_b200.h
COEFFS = {('bt601', False): (298, 16, 409, 100, 208, 516),
          ('bt709', False): (298, 16, 459, 55, 136, 541),
          ('bt601', True): (256, 0, 359, 88, 183, 454),
          ('bt709', True): (256, 0, 403, 48, 120, 475)}
KR_KB = {'bt601': (0.299, 0.114), 'bt709': (0.2126, 0.0722)}


def yuv_to_rgb_oracle(Y, U, V, matrix='bt601', full_range=False):
  """int64 reference of the conversion contract: uint8 RGB [..., 3] from Y, U, V arrays."""
  k, off, cr, gu, gv, bu = COEFFS[(matrix, bool(full_range))]
  L = k * (np.asarray(Y, np.int64) - off) + 128
  D = np.asarray(U, np.int64) - 128
  E = np.asarray(V, np.int64) - 128
  rgb = np.stack([(L + cr * E) >> 8, (L - gu * D - gv * E) >> 8, (L + bu * D) >> 8], -1)
  return np.clip(rgb, 0, 255).astype(np.uint8)


def frames_oracle(y, u, v, window, matrix, full_range):
  """[B, T, H, W] / [B, T, ceil(H/2), ceil(W/2)] planes -> uint8 RGB [B, T, h, w, 3] of the
  window, chroma sample (r >> 1, c >> 1) for frame pixel (r, c)."""
  y0, x0, h, w = window
  rows = np.arange(y0, y0 + h)
  cols = np.arange(x0, x0 + w)
  Y = y[:, :, rows][:, :, :, cols]
  U = u[:, :, rows >> 1][:, :, :, cols >> 1]
  V = v[:, :, rows >> 1][:, :, :, cols >> 1]
  return yuv_to_rgb_oracle(Y, U, V, matrix, full_range)


@pytest.mark.parametrize('matrix', ['bt601', 'bt709'])
@pytest.mark.parametrize('full_range', [False, True])
def test_oracle_within_one_of_the_float_formulas(matrix, full_range):
  """All 2^24 (Y, U, V) triples: the integer matrices stay within 1 of the exact formulas (a
  mistyped coefficient moves some channel by more)."""
  kr, kb = KR_KB[matrix]
  kg = 1.0 - kr - kb
  ys, cs = (1.0, 1.0) if full_range else (255.0 / 219.0, 255.0 / 224.0)
  off = 0 if full_range else 16
  U, V = np.meshgrid(np.arange(256), np.arange(256), indexing='ij')
  D, E = (U - 128.0) * cs, (V - 128.0) * cs
  worst = 0.0
  for Y in range(256):
    got = yuv_to_rgb_oracle(np.full(U.shape, Y), U, V, matrix, full_range).astype(np.float64)
    L = (Y - off) * ys
    ref = np.stack([L + 2 * (1 - kr) * E,
                    L - 2 * (1 - kb) * kb / kg * D - 2 * (1 - kr) * kr / kg * E,
                    L + 2 * (1 - kb) * D], -1)
    worst = max(worst, float(np.abs(got - np.clip(ref, 0, 255)).max()))
  assert worst <= 1.0, worst


def test_oracle_known_values():
  # limited-range black / white / mid grey, and full-range identity on grey
  assert yuv_to_rgb_oracle(16, 128, 128).tolist() == [0, 0, 0]
  assert yuv_to_rgb_oracle(235, 128, 128).tolist() == [255, 255, 255]
  assert yuv_to_rgb_oracle(np.arange(256), 128, 128, 'bt709', True)[:, 0].tolist() == list(range(256))


def test_yuv420_struct_matches_the_compiler(tmp_path):
  gcc = shutil.which('gcc')
  if gcc is None:
    pytest.skip('no gcc')
  cls = _lib.Yuv420Frames
  lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "tapir_b200.h"', 'int main(void) {',
           '  printf("%zu", sizeof(tapir_yuv420_frames));']
  lines += [f'  printf(" %zu", offsetof(tapir_yuv420_frames, {f}));' for f, _ in cls._fields_]
  lines += ['  printf("\\n");', '  return 0;', '}']
  src = tmp_path / 'yuv_probe.c'
  src.write_text('\n'.join(lines))
  exe = tmp_path / 'yuv_probe'
  subprocess.run([gcc, '-std=c99', '-Wall', '-Werror', '-pedantic', '-I', os.path.join(ROOT, 'include'),
                  str(src), '-o', str(exe)], check=True)
  size, *offs = (int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True,
                                                text=True).stdout.split())
  assert size == ctypes.sizeof(cls) == 112
  assert offs == [getattr(cls, f).offset for f, _ in cls._fields_]


def _nv12(B, T, H, W, pitch):
  """NV12 planes with rows `pitch` bytes apart (pitch >= W), as decoders allocate them."""
  ch, cw = (H + 1) // 2, (W + 1) // 2
  y = torch.zeros(B, T, H, pitch, dtype=torch.uint8)[..., :W]
  uv = torch.zeros(B, T, ch, pitch // 2, 2, dtype=torch.uint8)[:, :, :, :cw]
  return y, uv[..., 0], uv[..., 1]


def test_descriptor_nv12_pitched_odd_window():
  B, T, H, W, pitch = 2, 3, 37, 51, 64
  y, u, v = _nv12(B, T, H, W, pitch)
  window = (3, 5, 30, 40)
  assert live._check_planes(y, u, v, 'bt709', window) == window
  d, _ = live._descriptor(y, u, v, window, 'bt709', True, frame0=4)
  assert (d.H, d.W, d.y0, d.x0, d.h, d.w) == (H, W, 3, 5, 30, 40)
  assert (d.y_pitch, d.u_pitch, d.v_pitch, d.chroma_step) == (pitch, pitch, pitch, 2)
  assert (d.y_frame_stride, d.u_frame_stride) == (H * pitch, 19 * pitch)
  assert d.y == y.data_ptr() + 4 * H * pitch
  assert d.u == u.data_ptr() + 4 * 19 * pitch and d.v == d.u + 1
  assert (d.matrix, d.full_range) == (709, 1)


def test_descriptor_i420_pitched():
  B, T, H, W = 1, 2, 16, 24
  y = torch.zeros(B, T, H, 32, dtype=torch.uint8)[..., :W]
  u = torch.zeros(B, T, 8, 16, dtype=torch.uint8)[..., :12]
  v = torch.zeros(B, T, 8, 12, dtype=torch.uint8)
  assert live._check_planes(y, u, v, 'bt601', None) == (0, 0, H, W)
  d, _ = live._descriptor(y, u, v, (0, 0, H, W), 'bt601', False)
  assert (d.chroma_step, d.y_pitch, d.u_pitch, d.v_pitch) == (1, 32, 16, 12)
  assert (d.y_frame_stride, d.u_frame_stride, d.v_frame_stride) == (H * 32, 8 * 16, 8 * 12)
  assert (d.matrix, d.full_range) == (601, 0)


def test_descriptor_unmergeable_batch_axes_are_copied():
  # T sliced out of a longer clip: B and T no longer share one frame stride
  y = torch.arange(2 * 4 * 4 * 4, dtype=torch.int32).to(torch.uint8).reshape(2, 4, 4, 4)[:, :2]
  u = torch.zeros(2, 4, 2, 2, 2, dtype=torch.uint8)[:, :2, ..., 0]
  v = torch.zeros(2, 4, 2, 2, 2, dtype=torch.uint8)[:, :2, ..., 1]
  d, (yf, uf, vf) = live._descriptor(y, u, v, (0, 0, 4, 4), 'bt601', False, frame0=3)
  assert yf.is_contiguous() and torch.equal(yf, y.flatten(0, 1))
  assert d.y == yf.data_ptr() + 3 * 16 and d.y_frame_stride == 16
  assert d.chroma_step == uf.stride(2) == vf.stride(2)


@pytest.mark.parametrize('case', ['dtype', 'dims', 'chroma_shape', 'luma_step', 'chroma_step',
                                  'matrix', 'window', 'window_zero', 'host'])
def test_argument_errors_raise_before_any_library_call(case, monkeypatch):
  def no_library():
    raise AssertionError('library called')
  monkeypatch.setattr(_lib, 'load', no_library)
  y, u, v = _nv12(1, 2, 8, 8, 8)
  kw = {}
  err = ValueError
  if case == 'dtype':
    y = y.to(torch.int16)
  elif case == 'dims':
    y = y[0]
  elif case == 'chroma_shape':
    u = u[:, :, :3]
  elif case == 'luma_step':
    y = torch.zeros(1, 2, 8, 16, dtype=torch.uint8)[..., ::2]
  elif case == 'chroma_step':
    u = torch.zeros(1, 2, 4, 12, dtype=torch.uint8)[..., ::3]
    v = torch.zeros(1, 2, 4, 12, dtype=torch.uint8)[..., ::3]
  elif case == 'matrix':
    kw['matrix'] = 'bt2020'
  elif case == 'window':
    kw['window'] = (1, 0, 8, 8)
  elif case == 'window_zero':
    kw['window'] = (0, 0, 0, 8)
  else:
    err = RuntimeError  # valid planes, but on the host
  with pytest.raises(err):
    live.YUV420Frames(y, u, v, **kw)


def test_nv12_constructor_checks_the_uv_plane():
  with pytest.raises(ValueError):
    live.YUV420Frames.nv12(torch.zeros(1, 1, 8, 8, dtype=torch.uint8),
                           torch.zeros(1, 1, 4, 4, dtype=torch.uint8))


def test_yuv420_to_rgb_rejects_other_types():
  with pytest.raises(ValueError):
    live.yuv420_to_rgb(torch.zeros(1, 1, 8, 8, 3, dtype=torch.uint8))
