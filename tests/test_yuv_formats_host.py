"""YUV frames of every layout without a GPU: the int64 oracle of the 16-bit conversion contract
(tapir_yuv_frames) against the 8-bit oracle and the float BT.601 / 709 / 2020 formulas, the
coefficient table's rounding rule, the tapir_yuv_frames ABI mirror, the descriptors
live.YUVFrames' constructors build and their argument errors, and the C ABI's checks."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tapnet_b200 import _lib, live
from tests.test_yuv_host import yuv_to_rgb_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (cr, gu, gv, bu) of include/tapir_b200.h by (matrix, full_range)
CHROMA = {('bt601', False): (409, 100, 208, 516), ('bt601', True): (359, 88, 183, 454),
          ('bt709', False): (459, 55, 136, 541), ('bt709', True): (403, 48, 120, 475),
          ('bt2020', False): (430, 48, 167, 548), ('bt2020', True): (377, 42, 146, 482)}
KR_KB = {'bt601': (0.299, 0.114), 'bt709': (0.2126, 0.0722), 'bt2020': (0.2627, 0.0593)}
MATRICES = [(m, f) for m in ('bt601', 'bt709', 'bt2020') for f in (False, True)]


def to16(s, sample_bytes=2, bits=16, lsb_aligned=False):
  """Samples normalised to 16 bits, as the contract states (int64)."""
  s = np.asarray(s, np.int64)
  if sample_bytes == 1:
    return s << 8
  if lsb_aligned:
    return (s & ((1 << bits) - 1)) << (16 - bits)
  return s


def yuv16_oracle(Y16, U16, V16, matrix='bt601', full_range=False):
  """int64 reference of the 16-bit conversion contract: uint8 RGB [..., 3] from 16-bit Y, U, V."""
  cr, gu, gv, bu = CHROMA[(matrix, bool(full_range))]
  k, off = (256, 0) if full_range else (298, 4096)
  L = k * (np.asarray(Y16, np.int64) - off) + 32768
  D = np.asarray(U16, np.int64) - 32768
  E = np.asarray(V16, np.int64) - 32768
  rgb = np.stack([(L + cr * E) >> 16, (L - gu * D - gv * E) >> 16, (L + bu * D) >> 16], -1)
  return np.clip(rgb, 0, 255).astype(np.uint8)


def float_rgb(Y16, U16, V16, matrix, full_range):
  """The exact (float) BT.601 / 709 / 2020 formulas on 16-bit samples, in 8-bit RGB units,
  clipped to [0, 255]."""
  kr, kb = KR_KB[matrix]
  kg = 1.0 - kr - kb
  ys, cs = (1.0, 1.0) if full_range else (255.0 / 219.0, 255.0 / 224.0)
  L = (np.asarray(Y16, np.float64) / 256 - (0 if full_range else 16)) * ys
  D = (np.asarray(U16, np.float64) / 256 - 128) * cs
  E = (np.asarray(V16, np.float64) / 256 - 128) * cs
  ref = np.stack([L + 2 * (1 - kr) * E, L - 2 * (1 - kb) * kb / kg * D - 2 * (1 - kr) * kr / kg * E,
                  L + 2 * (1 - kb) * D], -1)
  return np.clip(ref, 0, 255)


@pytest.mark.parametrize('matrix', ['bt601', 'bt709'])
@pytest.mark.parametrize('full_range', [False, True])
def test_16bit_oracle_equals_the_8bit_oracle_on_every_triple(matrix, full_range):
  """All 2^24 8-bit triples, shifted into the high byte: the 16-bit contract gives the 8-bit bytes."""
  U, V = np.meshgrid(np.arange(256), np.arange(256), indexing='ij')
  for Y in range(256):
    Ys = np.full(U.shape, Y)
    np.testing.assert_array_equal(
        yuv16_oracle(to16(Ys, 1), to16(U, 1), to16(V, 1), matrix, full_range),
        yuv_to_rgb_oracle(Ys, U, V, matrix, full_range))


@pytest.mark.parametrize('matrix,full_range', MATRICES)
def test_10bit_oracle_within_one_of_the_float_formulas(matrix, full_range):
  """Every third 10-bit value of Y, U and V (342^3, about 4e7 triples)."""
  grid = np.arange(0, 1024, 3)
  U, V = np.meshgrid(grid, grid, indexing='ij')
  U16, V16 = U << 6, V << 6
  worst = 0.0
  for Y in grid:
    Y16 = np.full(U.shape, Y << 6)
    got = yuv16_oracle(Y16, U16, V16, matrix, full_range).astype(np.float64)
    worst = max(worst, float(np.abs(got - float_rgb(Y16, U16, V16, matrix, full_range)).max()))
  assert worst <= 1.0, worst


def test_coefficient_table_follows_the_rounding_rule():
  """(k, cr, gu, gv, bu) = round(256 x coefficient): the BT.601 and BT.709 rows the 8-bit contract
  had, and BT.2020 from the same rule."""
  for (matrix, full), row in CHROMA.items():
    kr, kb = KR_KB[matrix]
    kg = 1.0 - kr - kb
    cs = 1.0 if full else 255.0 / 224.0
    want = [2 * (1 - kr) * cs, 2 * (1 - kb) * kb / kg * cs, 2 * (1 - kr) * kr / kg * cs,
            2 * (1 - kb) * cs]
    assert list(row) == [int(np.floor(256 * c + 0.5)) for c in want], (matrix, full)
  assert int(np.floor(256 * 255 / 219 + 0.5)) == 298
  from tests.test_yuv_host import COEFFS
  for (matrix, full), row in COEFFS.items():
    assert row[2:] == CHROMA[(matrix, full)]


def test_lsb_and_msb_normalisation():
  assert to16(0x3ff, 2, 10, True) == 0xffc0 and to16(0xfc00 | 0x155, 2, 10, True) == 0x155 << 6
  assert to16(0xabc, 2, 12, True) == 0xabc0 and to16(0xabcd) == 0xabcd and to16(0xab, 1) == 0xab00
  # a 16-bit sample holding an 8-bit value in its high byte converts as the 8-bit sample
  assert (yuv16_oracle(0xeb00, 0x8000, 0x8000) == yuv_to_rgb_oracle(235, 128, 128)).all()


def test_yuv_struct_matches_the_compiler(tmp_path):
  gcc = shutil.which('gcc')
  if gcc is None:
    pytest.skip('no gcc')
  cls = _lib.YuvFrames
  lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "tapir_b200.h"', 'int main(void) {',
           '  printf("%zu", sizeof(tapir_yuv_frames));']
  lines += [f'  printf(" %zu", offsetof(tapir_yuv_frames, {f}));' for f, _ in cls._fields_]
  lines += ['  printf(" %d\\n", TAPIR_INGEST_YUV);', '  return 0;', '}']
  src = tmp_path / 'yuv_probe.c'
  src.write_text('\n'.join(lines))
  exe = tmp_path / 'yuv_probe'
  subprocess.run([gcc, '-std=c99', '-Wall', '-Werror', '-pedantic', '-I', os.path.join(ROOT, 'include'),
                  str(src), '-o', str(exe)], check=True)
  size, *rest = (int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True,
                                                text=True).stdout.split())
  assert size == ctypes.sizeof(cls) == 136
  assert rest[:-1] == [getattr(cls, f).offset for f, _ in cls._fields_]
  assert rest[-1] == _lib.INGEST_YUV


# ------------------------------------------------------------------ constructors and descriptors
@pytest.fixture
def host_planes(monkeypatch):
  """Lets the constructors take host tensors (their descriptors are only inspected here) and fails
  any library call."""
  monkeypatch.setattr(live, '_check_devices', lambda who, planes: None)

  def no_library():
    raise AssertionError('library called')
  monkeypatch.setattr(_lib, 'load', no_library)


def _pitched(shape, pitch, dtype=torch.uint8):
  """[..., rows, cols] with rows `pitch` elements apart."""
  return torch.zeros(*shape[:-1], pitch, dtype=dtype)[..., :shape[-1]]


def _check_desc(d, H, W, window, ptrs, frame_strides, pitches, steps, b, bits, lsb, shift,
                matrix=601, full=0):
  assert (d.H, d.W, (d.y0, d.x0, d.h, d.w)) == (H, W, window)
  assert (d.y, d.u, d.v) == ptrs
  assert (d.y_frame_stride, d.u_frame_stride, d.v_frame_stride) == frame_strides
  assert (d.y_pitch, d.u_pitch, d.v_pitch) == pitches
  assert (d.luma_step, d.chroma_step) == steps
  assert (d.sample_bytes, d.bits, d.lsb_aligned) == (b, bits, lsb)
  assert (d.chroma_shift_x, d.chroma_shift_y) == shift
  assert (d.matrix, d.full_range) == (matrix, full)


def test_p010_pitched_odd_window(host_planes):
  B, T, H, W, pitch = 2, 3, 37, 51, 64  # pitch in samples
  y = _pitched((B, T, H, W), pitch, torch.int16)
  uv = torch.zeros(B, T, 19, pitch // 2, 2, dtype=torch.int16)[:, :, :, :26]
  f = live.YUVFrames.p010(y, uv, matrix='bt2020', full_range=True, window=(3, 5, 30, 40))
  assert f.layout == 'p010' and f.shape == (B, T, 30, 40, 3) and f.frame_size == (H, W)
  d = f.yuv_struct(4)
  _check_desc(d, H, W, (3, 5, 30, 40),
              (y.data_ptr() + 4 * H * pitch * 2, uv.data_ptr() + 4 * 19 * pitch * 2,
               uv.data_ptr() + 4 * 19 * pitch * 2 + 2),
              (H * pitch * 2, 19 * pitch * 2, 19 * pitch * 2), (pitch * 2,) * 3, (1, 2), 2, 10, 0,
              (1, 1), 2020, 1)
  assert live.YUVFrames.p016(y, uv).yuv_struct().bits == 16


def test_yuv420p_and_yuv444_planes(host_planes):
  B, T, H, W = 1, 2, 15, 21
  y = _pitched((B, T, H, W), 24, torch.uint16 if hasattr(torch, 'uint16') else torch.int16)
  u = _pitched((B, T, 8, 11), 16, y.dtype)
  v = _pitched((B, T, 8, 11), 12, y.dtype)
  d = live.YUVFrames.yuv420p(y, u, v, bits=12, matrix='bt709').yuv_struct()
  _check_desc(d, H, W, (0, 0, H, W), (y.data_ptr(), u.data_ptr(), v.data_ptr()),
              (H * 48, 8 * 32, 8 * 24), (48, 32, 24), (1, 1), 2, 12, 1, (1, 1), 709)
  y8, u8, v8 = (_pitched((B, T, H, W), p) for p in (32, 24, 21))
  f = live.YUVFrames.yuv444(y8, u8, v8, window=(1, 2, 10, 11))
  assert f.layout == 'yuv444'
  _check_desc(f.yuv_struct(1), H, W, (1, 2, 10, 11),
              (y8.data_ptr() + H * 32, u8.data_ptr() + H * 24, v8.data_ptr() + H * 21),
              (H * 32, H * 24, H * 21), (32, 24, 21), (1, 1), 1, 8, 0, (0, 0))
  y16, u16, v16 = (_pitched((B, T, H, W), 32, torch.int16) for _ in range(3))
  assert live.YUVFrames.yuv444(y16, u16, v16).layout == 'yuv444p16'
  d = live.YUVFrames.yuv444(y16, u16, v16, bits=10).yuv_struct()
  assert (d.sample_bytes, d.bits, d.lsb_aligned, d.y_pitch) == (2, 10, 1, 64)


@pytest.mark.parametrize('layout', ['yuyv', 'uyvy'])
def test_packed_422(host_planes, layout):
  B, T, H, W, pitch = 1, 3, 17, 30, 72  # pitch in bytes >= 2W
  p = _pitched((B, T, H, 2 * W), pitch)
  f = getattr(live.YUVFrames, layout)(p, window=(1, 4, 12, 20))
  assert f.shape == (B, T, 12, 20, 3) and f.buffers == (p,)
  base = p.data_ptr() + 2 * H * pitch
  yo, uo, vo = (0, 1, 3) if layout == 'yuyv' else (1, 0, 2)
  _check_desc(f.yuv_struct(2), H, W, (1, 4, 12, 20), (base + yo, base + uo, base + vo),
              (H * pitch,) * 3, (pitch,) * 3, (2, 4), 1, 8, 0, (1, 0))


def test_nv12_i420_and_yuv420frames_agree(host_planes):
  B, T, H, W = 1, 2, 9, 13
  y = _pitched((B, T, H, W), 16)
  uv = torch.zeros(B, T, 5, 8, 2, dtype=torch.uint8)[:, :, :, :7]
  a = live.YUVFrames.nv12(y, uv).yuv_struct()
  b = live.YUV420Frames.nv12(y, uv).yuv_struct()
  assert all(getattr(a, f) == getattr(b, f) for f, _ in _lib.YuvFrames._fields_)
  c = live.YUV420Frames.nv12(y, uv).c_struct()
  assert all(getattr(a, f) == getattr(c, f) for f, _ in _lib.Yuv420Frames._fields_)
  assert live.YUVFrames.i420(y, uv[..., 0], uv[..., 1]).yuv_struct().chroma_step == 2


def test_map_buffers_and_windows_keep_the_layout(host_planes):
  p = torch.zeros(2, 4, 6, 16, dtype=torch.uint8)
  f = live.YUVFrames.uyvy(p, matrix='bt709', window=(0, 2, 4, 4))
  g = f.map_buffers(lambda t: t[1:, 2:3])
  assert (g.layout, g.matrix, g.window, tuple(g.y.shape)) == ('uyvy', 'bt709', (0, 2, 4, 4), (1, 1, 6, 8))
  assert g.yuv_struct().y == p[1, 2].data_ptr() + 1
  assert f.with_window(None).window == (0, 0, 6, 8)
  y = torch.zeros(1, 2, 8, 8, dtype=torch.int16)
  h = live.YUVFrames.yuv420p(y, y[..., :4, :4], y[..., :4, :4], bits=10).map_buffers(lambda t: t[:, :1])
  assert (h.layout, h.bits, h.lsb_aligned) == ('yuv420p10', 10, True)
  assert h.sampling == (2, 10, True, (1, 1))


def test_unmergeable_packed_frames_are_copied(host_planes):
  p = torch.arange(2 * 4 * 2 * 8, dtype=torch.int32).to(torch.uint8).reshape(2, 4, 2, 8)[:, :2]
  f = live.YUVFrames.yuyv(p)
  d = f.yuv_struct(3)
  yf, uf, vf = f._keep
  assert torch.equal(yf, p[..., 0::2].flatten(0, 1)) and torch.equal(uf, p[..., 1::4].flatten(0, 1))
  assert d.y == yf.data_ptr() + 3 * yf.stride(0) and d.luma_step == yf.stride(2)
  assert d.chroma_step == uf.stride(2) == vf.stride(2)


def test_zeros_builds_every_layout(host_planes):
  for layout, b, shift in [('nv12', 1, (1, 1)), ('i420', 1, (1, 1)), ('p010', 2, (1, 1)),
                           ('p016', 2, (1, 1)), ('yuv420p10', 2, (1, 1)), ('yuv420p12', 2, (1, 1)),
                           ('yuv444', 1, (0, 0)), ('yuv444p16', 2, (0, 0)), ('yuyv', 1, (1, 0)),
                           ('uyvy', 1, (1, 0))]:
    assert live.is_yuv_layout(layout)
    f = live.YUVFrames.zeros(layout, 2, 1, 10, 14, 'cpu', window=(2, 2, 6, 8))
    assert f.layout == layout and f.sampling[0] == b and f.chroma_shift == shift, layout
    assert f.frame_size == (10, 14) and f.window == (2, 2, 6, 8)
  for bad in ('nv21', 'yuv420p7', 'yuv420p', 'yuv444p17', 7):
    assert not live.is_yuv_layout(bad)
  with pytest.raises(ValueError):
    live.YUVFrames.zeros('nv21', 1, 1, 8, 8, 'cpu')


def _bad_cases():
  u8 = lambda *s: torch.zeros(*s, dtype=torch.uint8)  # noqa: E731
  i16 = lambda *s: torch.zeros(*s, dtype=torch.int16)  # noqa: E731
  P = live.YUVFrames
  return {
      'p010_uint8': lambda: P.p010(u8(1, 1, 8, 8), u8(1, 1, 4, 4, 2)),
      'p010_mixed': lambda: P.p010(i16(1, 1, 8, 8), u8(1, 1, 4, 4, 2)),
      'p010_uv_dims': lambda: P.p010(i16(1, 1, 8, 8), i16(1, 1, 4, 8)),
      'p010_uv_shape': lambda: P.p010(i16(1, 1, 8, 8), i16(1, 1, 4, 3, 2)),
      'yuv420p_bits_7': lambda: P.yuv420p(i16(1, 1, 8, 8), i16(1, 1, 4, 4), i16(1, 1, 4, 4), bits=7),
      'yuv420p_bits_17': lambda: P.yuv420p(i16(1, 1, 8, 8), i16(1, 1, 4, 4), i16(1, 1, 4, 4), bits=17),
      'yuv420p_uint8_10bit': lambda: P.yuv420p(u8(1, 1, 8, 8), u8(1, 1, 4, 4), u8(1, 1, 4, 4), bits=10),
      'yuv444_chroma_shape': lambda: P.yuv444(u8(1, 1, 8, 8), u8(1, 1, 4, 4), u8(1, 1, 4, 4)),
      'yuv444_uint8_bits': lambda: P.yuv444(u8(1, 1, 8, 8), u8(1, 1, 8, 8), u8(1, 1, 8, 8), bits=10),
      'yuv444_float': lambda: P.yuv444(*(torch.zeros(1, 1, 8, 8),) * 3),
      'yuyv_odd_width': lambda: P.yuyv(u8(1, 1, 8, 14)),
      'yuyv_int16': lambda: P.yuyv(i16(1, 1, 8, 16)),
      'yuyv_dims': lambda: P.yuyv(u8(1, 8, 16)),
      'yuyv_strided_bytes': lambda: P.yuyv(u8(1, 1, 8, 32)[..., ::2]),
      'yuyv_odd_window_x0': lambda: P.yuyv(u8(1, 1, 8, 16), window=(0, 1, 4, 4)),
      'uyvy_odd_window_w': lambda: P.uyvy(u8(1, 1, 8, 16), window=(0, 2, 4, 5)),
      'nv12_matrix': lambda: P.nv12(u8(1, 1, 8, 8), u8(1, 1, 4, 4, 2), matrix='bt2021'),
      'nv12_window': lambda: P.nv12(u8(1, 1, 8, 8), u8(1, 1, 4, 4, 2), window=(1, 0, 8, 8)),
      'i420_steps_differ': lambda: P.i420(u8(1, 1, 8, 8), u8(1, 1, 4, 4), u8(1, 1, 4, 8)[..., ::2]),
      'planar_shift': lambda: P(u8(1, 1, 8, 8), u8(1, 1, 2, 8), u8(1, 1, 2, 8), chroma_shift=(0, 2)),
      'yuv420frames_bt2020': lambda: live.YUV420Frames(u8(1, 1, 8, 8), u8(1, 1, 4, 4), u8(1, 1, 4, 4),
                                                       matrix='bt2020'),
  }


@pytest.mark.parametrize('case', sorted(_bad_cases()))
def test_argument_errors_raise_before_any_library_call(host_planes, case):
  with pytest.raises(ValueError):
    _bad_cases()[case]()


def test_host_planes_are_refused(monkeypatch):
  def no_library():
    raise AssertionError('library called')
  monkeypatch.setattr(_lib, 'load', no_library)
  with pytest.raises(RuntimeError, match='CUDA only'):
    live.YUVFrames.p010(torch.zeros(1, 1, 8, 8, dtype=torch.int16),
                        torch.zeros(1, 1, 4, 4, 2, dtype=torch.int16))
  with pytest.raises(ValueError):
    live.yuv_to_rgb(torch.zeros(1, 1, 8, 8, 3, dtype=torch.uint8))


# ------------------------------------------------------------------ the C ABI's descriptor checks
def _good():
  """A valid P010 descriptor of one 48 x 64 frame at fake (never dereferenced) addresses."""
  return dict(y=0x10000, u=0x40000, v=0x40002, y_frame_stride=0, u_frame_stride=0,
              v_frame_stride=0, y_pitch=128, u_pitch=128, v_pitch=128, H=48, W=64, y0=0, x0=0,
              h=48, w=64, matrix=601, full_range=0, sample_bytes=2, bits=10, lsb_aligned=0,
              luma_step=1, chroma_step=2, chroma_shift_x=1, chroma_shift_y=1)


BAD_DESCRIPTORS = [
    ('null y', dict(y=None)), ('zero window', dict(h=0)), ('window outside', dict(x0=1)),
    ('sample_bytes 3', dict(sample_bytes=3)), ('bits 7', dict(bits=7)), ('bits 17', dict(bits=17)),
    ('bits 10 in bytes', dict(sample_bytes=1, bits=10, u=0x40000, v=0x40001, y_pitch=64,
                              u_pitch=64, v_pitch=64)),
    ('lsb_aligned 2', dict(lsb_aligned=2)), ('shift 2', dict(chroma_shift_y=2)),
    ('shift -1', dict(chroma_shift_x=-1)), ('luma_step 0', dict(luma_step=0)),
    ('chroma_step 0', dict(chroma_step=0)),
    ('packed odd W', dict(luma_step=2, W=63, w=63, y_pitch=256, u_pitch=256, v_pitch=256)),
    ('packed odd x0', dict(luma_step=2, x0=1, w=62, y_pitch=256, u_pitch=256, v_pitch=256)),
    ('packed odd w', dict(luma_step=2, w=61, y_pitch=256, u_pitch=256, v_pitch=256)),
    ('odd 16-bit plane', dict(v=0x40003)), ('odd 16-bit pitch', dict(y_pitch=129)),
    ('odd 16-bit frame stride', dict(u_frame_stride=4097)), ('short luma pitch', dict(y_pitch=126)),
    ('short chroma pitch', dict(u_pitch=124)), ('matrix 2021', dict(matrix=2021)),
    ('full_range 2', dict(full_range=2)), ('negative frame stride', dict(y_frame_stride=-128)),
]


@pytest.mark.parametrize('what,change', BAD_DESCRIPTORS, ids=[b[0] for b in BAD_DESCRIPTORS])
def test_c_abi_rejects_malformed_descriptors(what, change):
  lib = _lib.load()
  d = _lib.YuvFrames(**{**_good(), **change})
  n0 = lib.tapir_launch_count()
  buf = ctypes.c_void_p(0x80000)
  assert lib.tapir_yuv_to_rgb(ctypes.byref(d), 1, buf, None) == 1, what
  assert lib.tapir_last_error()
  assert lib.tapir_ingest_frames_yuv(ctypes.byref(d), 1, buf, 32, 32, None) == 1, what
  assert lib.tapir_backbone_forward_yuv(None, ctypes.byref(d), 1, buf, buf, buf, 1 << 20, None,
                                        None) == 1, what
  desc = _lib.IngestDesc(src=ctypes.addressof(d), format=_lib.INGEST_YUV)
  assert lib.tapir_ingest_frames_multi(ctypes.byref(desc), 1, buf, 32, 32, None) == 1, what
  assert lib.tapir_launch_count() == n0


def test_c_abi_ingest_yuv_descriptor_fields():
  """TAPIR_INGEST_YUV takes everything from *src: the uint8 fields must be 0, src non-null."""
  lib = _lib.load()
  buf = ctypes.c_void_p(0x80000)
  for kw, what in ((dict(src=None), 'src null'), (dict(src=0x10000, H=48), 'must be 0')):
    desc = _lib.IngestDesc(format=_lib.INGEST_YUV, **kw)
    assert lib.tapir_ingest_frames_multi(ctypes.byref(desc), 1, buf, 32, 32, None) == 1
    assert what in lib.tapir_last_error().decode()


def test_msb_aligned_layouts_share_their_sampling(host_planes):
  """P010 and P016 convert alike (all 16 bits of an MSB-aligned sample are read), so one tracker
  takes both; LSB-aligned layouts of different bits do not."""
  y = torch.zeros(1, 1, 8, 8, dtype=torch.int16)
  uv = torch.zeros(1, 1, 4, 4, 2, dtype=torch.int16)
  u, v = uv[..., 0], uv[..., 1]
  assert live.YUVFrames.p010(y, uv).sampling == live.YUVFrames.p016(y, uv).sampling
  assert live.YUVFrames.yuv420p(y, u, v, bits=10).sampling != live.YUVFrames.yuv420p(y, u, v, bits=12).sampling
  assert live.YUVFrames.p010(y, uv).sampling != live.YUVFrames.yuv420p(y, u, v, bits=16).sampling
  assert live.YUVFrames.nv12(y.to(torch.uint8), uv.to(torch.uint8)).sampling == \
      live.YUVFrames.i420(y.to(torch.uint8), u.to(torch.uint8), v.to(torch.uint8)).sampling


def test_layout_table_matches_the_constructors(host_planes):
  """Every YUV_LAYOUTS entry builds clips whose layout name, samples and chroma shift are its own."""
  for name, spec in live.YUV_LAYOUTS.items():
    f = live.YUVFrames.zeros(name, 1, 2, 6, 8, 'cpu')
    assert f.layout == name and f.y.dtype == spec.dtype, name
    assert (f.bits, f.lsb_aligned, f.chroma_shift) == (spec.bits, spec.lsb_aligned, spec.chroma_shift)
    assert f.map_buffers(lambda b: b[:, 1:]).layout == name
