"""Streams of different frame sizes, without a GPU: the backbone pass plan against the reference's
get_feature_grids decisions, the grouping of streams by plan, the tracker's argument errors (raised
before the library is touched) and the C layout of tapir_ingest_desc."""
import ctypes
import os
import shutil
import subprocess
import sys

import pytest
import torch

from oracle import tapir_oracle as O
from tapnet_b200 import _lib, streaming, tapir_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SIZES = [(64, 64), (200, 200), (240, 240), (240, 320), (250, 250), (255, 257), (256, 256),
         (256, 320), (260, 260), (263, 301), (300, 200), (320, 256), (480, 480), (480, 640),
         (512, 512), (720, 1280), (100, 700), (1024, 768), (999, 333)]
# explicit refinement resolutions, including the reference's quirk (a pass that follows a level at
# the video's own size reads the video itself whatever its resolution)
EXPLICIT = [((256, 256), [(256, 256), (512, 512)]), ((512, 512), [(512, 512), (256, 256)]),
            ((480, 640), [(256, 256), (480, 640), (720, 960)]), ((300, 300), [(304, 304)])]


def _reference_module():
  """The unmodified reference's tapir_model as build() installed it under oracle/_ref, or None."""
  root = os.path.join(ROOT, 'oracle', '_ref')
  if not os.path.isfile(os.path.join(root, 'tapnet', 'torch', 'tapir_model.py')):
    return None
  for p in (root, os.path.join(ROOT, 'oracle', 'shims')):
    if p not in sys.path:
      sys.path.insert(0, p)
  from tapnet.torch import tapir_model as ref  # pylint: disable=g-import-not-at-top
  return ref


def _reference_passes(hw, refinement, monkeypatch):
  """(passes as (h, w, reads the video itself), per-level sizes) of a get_feature_grids call on
  an hw video, with the backbone and resize stubbed out: the reference's own code if installed,
  else the oracle's restatement."""
  video = torch.zeros(1, 1, *hw, 3)
  passes = []

  def record(x):
    # a resize to the video's own size (align_corners=False) is the identity: get_feature_grids
    # reads the video then, as it does on the reference's quirk path
    h, w = int(x.shape[2]), int(x.shape[3])
    passes.append((h, w, x.data_ptr() == video.data_ptr() or (h, w) == tuple(hw)))
    return torch.zeros(x.shape[0], 4, 1, 1)

  def resize(v, res):
    return torch.zeros(*v.shape[:2], int(res[0]), int(res[1]), v.shape[-1])

  ref = _reference_module()
  if ref is not None:
    monkeypatch.setattr(ref.utils, 'bilinear', resize)

    class Stub:
      initial_resolution = (256, 256)
      feature_extractor_chunk_size = 0
      extra_convs = False

      def resnet_torch(self, x):
        z = record(x)
        return {'resnet_unit_3': z, 'resnet_unit_1': z}

    grids = ref.TAPIR.get_feature_grids(Stub(), video, False, refinement)
  else:
    monkeypatch.setattr(O, 'resize_video', resize)
    monkeypatch.setattr(O, 'resnet', lambda sd, x, ctx: (record(x), torch.zeros(x.shape[0], 4, 1, 1)))
    cfg = O.Config(extra_convs=False, feature_extractor_chunk_size=0)
    grids = O.get_feature_grids({}, cfg, video, refinement)
  return passes, [tuple(int(v) for v in r) for r in grids.resolutions]


@pytest.mark.parametrize('hw,refinement', [(hw, None) for hw in SIZES] + EXPLICIT)
def test_pass_plan_matches_reference_get_feature_grids(hw, refinement, monkeypatch):
  passes, levels = _reference_passes(hw, refinement, monkeypatch)
  plan = tapir_model._pass_plan(hw, (256, 256), refinement)
  assert [(p.h, p.w, p.direct) for p in plan if p.new] == passes
  assert [(p.h, p.w) for p in plan] == levels
  assert plan[0].new


def test_pass_plan_rejects_resolutions_off_the_8_grid():
  with pytest.raises(ValueError, match='multiple of 8'):
    tapir_model._pass_plan((300, 300), (256, 256), [(300, 300)])


def _specs(*hws):
  return [streaming.StreamSpec(hw, None, hw) for hw in hws]


def test_grouping_by_plan():
  # 256^2 reads its frame directly; 200^2, 240^2 and 250x200 all resample to one 256^2 pass;
  # 240x320 (wider than 256) and 480^2 add a direct pass at their own size
  groups = streaming.group_streams(_specs((256, 256), (240, 320), (200, 200), (240, 240), (480, 480),
                                          (250, 200)))
  assert [g[1] for g in groups] == [[0], [1], [2, 3, 5], [4]]
  plans = [[tuple(p) for p in g[0]] for g in groups]
  assert plans[0] == [(256, 256, True, True), (256, 256, True, False)]
  assert plans[1] == [(256, 256, False, True), (256, 256, False, False), (240, 320, True, True)]
  assert plans[2] == [(256, 256, False, True), (256, 256, False, False)]
  assert plans[3] == [(256, 256, False, True), (256, 256, False, False), (480, 480, True, True)]


def test_grouping_direct_pass_needs_one_size():
  groups = streaming.group_streams(_specs((480, 480), (200, 200), (480, 480), (480, 472), (256, 256),
                                          (256, 256)))
  assert [g[1] for g in groups] == [[0, 2], [1], [3], [4, 5]]
  # 260^2 has three levels over one resampled pass: not the plan of 200^2
  groups = streaming.group_streams(_specs((260, 260), (200, 200), (248, 256)))
  assert [g[1] for g in groups] == [[0], [1, 2]]


def test_grouping_cropped_streams():
  # a direct pass over a window: only streams of the same frame and window share it
  w480 = (0, 80, 480, 480)
  specs = [streaming.StreamSpec((480, 640), w480, (480, 480)),
           streaming.StreamSpec((480, 720), (0, 120, 480, 480), (480, 480)),
           streaming.StreamSpec((480, 640), w480, (480, 480)),
           streaming.StreamSpec((240, 320), (0, 40, 240, 240), (240, 240)),  # resampled to 256^2
           streaming.StreamSpec((200, 200), None, (200, 200))]
  assert [g[1] for g in streaming.group_streams(specs)] == [[0, 2], [1], [3, 4]]


def test_stream_specs():
  specs = streaming.stream_specs([256, 240, 480], [256, 320, 640], 3, yuv420=True,
                                 window=[None, (0, 40, 240, 240), (0, 80, 480, 480)])
  assert [s.hw for s in specs] == [(256, 256), (240, 240), (480, 480)]
  assert specs[0].window is None and specs[2].window == (0, 80, 480, 480)
  specs = streaming.stream_specs(480, [640, 720], 2, yuv420=True, window=(0, 0, 480, 480))
  assert [s.frame_hw for s in specs] == [(480, 640), (480, 720)] and specs[1].hw == (480, 480)


@pytest.fixture
def no_library(monkeypatch):
  def refuse():
    raise AssertionError('the library was touched')
  monkeypatch.setattr(_lib, 'load', refuse)


@pytest.mark.parametrize('kwargs,match', [
    (dict(height=[256, 240], width=[256, 320, 200]), 'height has 2 entries'),
    (dict(height=[256, 240, 200], width=[256, 320]), 'width has 2 entries'),
    (dict(height=[256, 240, 200], width=256, yuv420=True, window=[None, None]), 'window has 2'),
    (dict(height=[256, 240, 200], width=256, window=[None, None, None]), 'only supported with yuv420'),
    (dict(height=[256, 240, 200], width=256, yuv420=True, window=[None, (0, 0, 300, 10), None]),
     'outside'),
])
def test_constructor_errors_before_any_cuda_call(kwargs, match, no_library):
  model = tapir_model.TAPIR(use_casual_conv=True)  # on the CPU: reaching the device check fails
  with pytest.raises(ValueError, match=match):
    streaming.OnlineTracker(model, num_points=8, num_streams=3, **kwargs)
  with pytest.raises(RuntimeError, match='CUDA only'):  # good arguments get as far as the device
    streaming.OnlineTracker(model, [256, 240, 200], [256, 320, 200], 8, num_streams=3)


def _bare_tracker(*hws):
  trk = streaming.OnlineTracker.__new__(streaming.OnlineTracker)
  trk.specs, trk._yuv = _specs(*hws), None
  return trk


def test_frame_errors_before_any_cuda_call(no_library):
  trk = _bare_tracker((256, 256), (240, 320), (480, 480))
  f = [torch.zeros(256, 256, 3), torch.zeros(240, 320, 3), torch.zeros(480, 480, 3)]
  assert [tuple(x.shape) for x in trk._stream_frames(f, range(3))] == [
      (1, 1, 256, 256, 3), (1, 1, 240, 320, 3), (1, 1, 480, 480, 3)]
  with pytest.raises(ValueError, match='list of 3 frames'):
    trk._stream_frames(f[:2], range(3))
  with pytest.raises(ValueError, match='list of 3 frames'):
    trk._stream_frames(torch.zeros(3, 256, 256, 3), range(3))
  with pytest.raises(ValueError, match=r'stream 1: frame \(320, 240, 3\)'):
    trk._stream_frames([f[0], torch.zeros(320, 240, 3), f[2]], range(3))
  with pytest.raises(ValueError, match='mixed formats'):
    trk._stream_frames([f[0], f[1].to(torch.uint8), f[2]], range(3))
  with pytest.raises(ValueError, match='tensor frame'):
    trk._stream_frames([f[0], f[1].numpy(), f[2]], range(3))
  # update_query: one frame, that stream's size
  assert tuple(trk._stream_frames([f[1][None]], [1])[0].shape) == (1, 1, 240, 320, 3)
  with pytest.raises(ValueError, match='stream 2'):
    trk._stream_frames([f[1]], [2])


def test_ingest_desc_layout_matches_the_compiler(tmp_path):
  gcc = shutil.which('gcc')
  if gcc is None:
    pytest.skip('no gcc')
  cls = _lib.IngestDesc
  lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "tapir_b200.h"', 'int main(void) {',
           '  printf("%zu", sizeof(tapir_ingest_desc));']
  lines += [f'  printf(" %zu", offsetof(tapir_ingest_desc, {f}));' for f, _ in cls._fields_]
  lines += ['  printf(" %d %d %d\\n", TAPIR_INGEST_U8, TAPIR_INGEST_YUV420, TAPIR_INGEST_MAX_FRAMES);',
            '  return 0;', '}']
  src = tmp_path / 'probe.c'
  src.write_text('\n'.join(lines))
  exe = tmp_path / 'probe'
  subprocess.run([gcc, '-std=c99', '-Wall', '-Werror', '-pedantic', '-I', os.path.join(ROOT, 'include'),
                  str(src), '-o', str(exe)], check=True)
  size, *rest = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True,
                                                text=True).stdout.split()]
  offs, consts = rest[:len(cls._fields_)], rest[len(cls._fields_):]
  assert size == ctypes.sizeof(cls)
  assert offs == [getattr(cls, f).offset for f, _ in cls._fields_]
  assert consts == [_lib.INGEST_U8, _lib.INGEST_YUV420, _lib.INGEST_MAX_FRAMES]


def test_new_entry_points_reject_bad_arguments():
  """rc 1 and a message, before any CUDA call (the pointers are never dereferenced)."""
  lib = _lib.load()
  buf = ctypes.c_void_p(0x10000)

  def desc(**kw):
    d = dict(src=0x10000, pitch=3 * 64, format=_lib.INGEST_U8, H=48, W=64, y0=0, x0=0, h=48, w=64)
    d.update(kw)
    return _lib.IngestDesc(**d)

  def ingest(descs, frames=None, dst=buf, oh=32, ow=32):
    arr = (_lib.IngestDesc * max(1, len(descs)))(*descs)
    rc = lib.tapir_ingest_frames_multi(arr if descs else None, len(descs) if frames is None else frames,
                                       dst, oh, ow, None)
    return rc, lib.tapir_last_error().decode()

  yuv = _lib.Yuv420Frames(0x10000, 0x20000, 0x20001, 0, 0, 0, 64, 64, 64, 2, 48, 64, 0, 0, 48, 64,
                          601, 0, 0)
  for args, kw, what in (
      ([], {}, 'bad arguments'), ([desc()], dict(frames=0), 'bad arguments'),
      ([desc()], dict(dst=None), 'bad arguments'), ([desc()], dict(oh=0), 'bad arguments'),
      ([desc(format=3)], {}, 'format 3'), ([desc(src=None)], {}, 'frame 0'),
      ([desc(), desc(pitch=3 * 64 - 1)], {}, 'frame 1'), ([desc(y0=1)], {}, 'outside'),
      ([desc(x0=60, w=5)], {}, 'outside'), ([desc(format=0)], {}, 'format 0'),
      ([desc(format=_lib.INGEST_YUV420, yuv=_lib.Yuv420Frames(**{
          f: getattr(yuv, f) for f, _ in _lib.Yuv420Frames._fields_ if f != 'chroma_step'}, chroma_step=3))],
       {}, 'chroma_step')):
    rc, msg = ingest(args, **kw)
    assert rc == 1 and what in msg, (what, rc, msg)
  ua = _lib.UpdateArgs(res=0x10000, ld_res=388, num_points=6, num_frames=2, init_h=256, init_w=256,
                       resize_h=256, resize_w=256, pos=0x10000, occ_in=0x10000, expd_in=0x10000,
                       occ_out=0x10000, expd_out=0x10000, feat_out=0x10000, tracks_out=0x10000,
                       feat_hi=0x10000, feat_lo=0x10000)
  for table, rows, what in ((buf, 5, 'rows_per_clip'), (buf, 3, 'rows_per_clip'),
                            (buf, 0, 'rows_per_clip'), (ctypes.c_void_p(0x10002), 4, 'aligned')):
    rc = lib.tapir_refine_update_ex(ctypes.byref(ua), table, rows, None)
    msg = lib.tapir_last_error().decode()
    assert rc == 1 and what in msg, (what, rc, msg)
  ua.tracks_out = None
  assert lib.tapir_refine_update_ex(ctypes.byref(ua), buf, 4, None) == 1
  assert 'tracks_out' in lib.tapir_last_error().decode()
