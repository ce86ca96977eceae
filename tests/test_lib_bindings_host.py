"""The tensor-level bindings of tapnet_b200._lib on CPU tensors: the structs they build carry the
sizes, strides and byte offsets of the tensors passed in (both feature layouts of the refinement
loop), and operands that disagree raise ValueError before the library is reached."""
import pytest
import torch

from tapnet_b200 import _lib

G, N, T, P = 2, 3, 4, 3
Q = G * N
KIN = 388 + 49 * 3
z = torch.zeros


def _corr_inputs(per_row):
  levels = [z(G, T, 16, 16, 128), z(G, T, 8, 8, 256), z(G, T, 4, 4, 256)]
  if per_row:
    f = z(Q, T, 384)
    feat = (f[..., :128], f[..., 128:])
  else:
    feat = tuple(z(G, N, c).view(Q, 1, c).expand(Q, T, c) for c in (128, 256))
  return [levels, z(G, N, T, 2), z(G, N, T), z(G, N, T), *feat, z(P, Q * T, KIN, dtype=torch.bfloat16),
          (256, 320)]


def _update_inputs(per_row, **bad):
  _, pos, occ, expd, fh, fl, _, _ = _corr_inputs(per_row)
  a = dict(res=z(Q, T, 388), pos=pos, occ_in=occ, expd_in=expd, feat_hi=fh, feat_lo=fl,
           occ_out=z(G, N, T), expd_out=z(G, N, T), feat_out=z(Q, T, 384), tracks_out=z(G, N, T, 2),
           init_hw=(256, 256), resize_hw=(320, 384), video_hw=(480, 640))
  a.update(bad)
  return list(a.values())


def _mixer():
  w = _lib.MixerWeights(num_blocks=12, planes=P)
  w.linear.K = KIN
  return w


@pytest.mark.parametrize('per_row', [True, False], ids=['rows', 'query'])
def test_struct_fields(per_row):
  args = _corr_inputs(per_row)
  levels, pos, occ, expd, fh, fl, out, _ = args
  ca = _lib.corr_args(*args)
  assert (ca.num_levels, ca.num_points, ca.num_frames, ca.init_h, ca.init_w, ca.planes) == (3, N, T, 256, 320, P)
  assert [(lv.grid, lv.h, lv.w, lv.C) for lv in ca.levels[:3]] == [(g.data_ptr(), *g.shape[2:]) for g in levels]
  assert (ca.pos, ca.occ, ca.expd) == (pos.data_ptr(), occ.data_ptr(), expd.data_ptr())
  assert (ca.out_planes, ca.out_plane_stride, ca.ld) == (out.data_ptr(), Q * T * KIN, KIN)
  res, _, _, _, _, _, occ_o, expd_o, feat_o, trk = _update_inputs(per_row)[:10]
  ua = _lib.update_args(res, pos, occ, expd, fh, fl, occ_o, expd_o, feat_o, trk, (256, 256), (320, 384), (480, 640))
  # per-row: [Q, T, 384] rows, the low half 128 floats in; per-query: vectors with stride_t 0
  for s in (ca, ua):
    assert (s.feat_hi_stride_n, s.feat_hi_stride_t, s.feat_lo_stride_n, s.feat_lo_stride_t) == (
        (T * 384, 384, T * 384, 384) if per_row else (128, 0, 256, 0))
    assert (s.feat_hi, s.feat_lo) == (fh.data_ptr(), fl.data_ptr())
  assert not per_row or fl.data_ptr() == fh.data_ptr() + 512
  assert (ua.res, ua.ld_res, ua.num_points, ua.num_frames) == (res.data_ptr(), 388, Q, T)
  assert (ua.init_h, ua.init_w, ua.resize_h, ua.resize_w, ua.video_h, ua.video_w) == (256, 256, 320, 384, 480, 640)
  assert (ua.pos, ua.occ_in, ua.expd_in, ua.occ_out, ua.expd_out, ua.feat_out, ua.tracks_out) == tuple(
      t.data_ptr() for t in (pos, occ, expd, occ_o, expd_o, feat_o, trk))
  assert _lib.update_args(*_update_inputs(per_row, tracks_out=None)).tracks_out is None


def test_mixer_io_fields():
  x, out = z(P, Q * T, KIN, dtype=torch.bfloat16), z(Q, T, 388)
  c1, c2 = [z(G, N, 2, 512) for _ in range(12)], [z(Q, 2, 2048) for _ in range(12)]
  io = _lib.mixer_io(_mixer(), x, out, True, c1, c2)
  assert (io.x_planes, io.x_plane_stride, io.ldx) == (x.data_ptr(), Q * T * KIN, KIN)
  assert (io.num_points, io.num_frames, io.causal, io.out, io.ldo) == (Q, T, 1, out.data_ptr(), 388)
  assert [io.ctx1_in[i] for i in range(12)] == [t.data_ptr() for t in c1]
  assert [io.ctx2_in[i] for i in range(12)] == [t.data_ptr() for t in c2]
  assert not io.ctx1_out and not io.ctx2_out


BAD_CORR = {  # argument index -> replacement
    'pos_frames': (1, lambda a: z(G, N, T + 1, 2)), 'occ_shape': (2, lambda a: z(G, N + 1, T)),
    'expd_dtype': (3, lambda a: a[3].double()), 'pos_not_dense': (1, lambda a: z(G, N, T, 4)[..., :2]),
    'feat_inner_stride': (4, lambda a: z(Q, T, 256)[..., ::2]), 'feat_width': (5, lambda a: z(Q, T, 128)),
    'level_frames': (0, lambda a: [z(G, T + 1, 16, 16, 128)] + a[0][1:]),
    'clips_do_not_divide': (0, lambda a: [z(4, T, *g.shape[2:]) for g in a[0]]),
    'out_rows': (6, lambda a: z(P, Q * T - 1, KIN, dtype=torch.bfloat16)),
    'out_too_narrow': (6, lambda a: z(P, Q * T, KIN - 1, dtype=torch.bfloat16)),
    'out_dtype': (6, lambda a: a[6].float()), 'too_many_levels': (0, lambda a: a[0] * 2),
}
BAD_UPDATE = {
    'res_frames': dict(res=z(Q, T + 1, 388)), 'res_narrow': dict(res=z(Q, T, 387)),
    'feat_out_width': dict(feat_out=z(Q, T, 383)), 'tracks_fp64': dict(tracks_out=z(G, N, T, 2).double()),
}
BAD_MIXER = {
    'rows': lambda x, o, c: (x, z(Q, T + 1, 388), c), 'context_queries': lambda x, o, c: (x, o, [z(Q + 1, 2, 512)] * 12),
    'context_blocks': lambda x, o, c: (x, o, c[:11]), 'x_fp32': lambda x, o, c: (x.float(), o, c),
    'x_narrow': lambda x, o, c: (x[..., :KIN - 1], o, c), 'x_planes': lambda x, o, c: (x[:P - 1], o, c),
}


@pytest.fixture
def no_library(monkeypatch):
  monkeypatch.setattr(_lib, 'load', lambda: pytest.fail('the library was reached'))


@pytest.mark.parametrize('name', list(BAD_CORR) + [f'update_{k}' for k in BAD_UPDATE] +
                         [f'mixer_{k}' for k in BAD_MIXER])
def test_bad_arguments_raise_before_the_library(no_library, name):
  if name.startswith('update_'):
    with pytest.raises(ValueError):
      _lib.refine_update(*_update_inputs(True, **BAD_UPDATE[name[7:]]))
  elif name.startswith('mixer_'):
    x, o, c = BAD_MIXER[name[6:]](z(P, Q * T, KIN, dtype=torch.bfloat16), z(Q, T, 388), [z(Q, 2, 512)] * 12)
    with pytest.raises(ValueError):
      _lib.mixer_forward(_mixer(), x, o, True, c, None, None, None, None)
  else:
    args = _corr_inputs(True)
    index, bad = BAD_CORR[name]
    args[index] = bad(args)
    with pytest.raises(ValueError):
      _lib.local_corr(*args)


def test_stage_a_and_frame_calls_reject_mismatches(no_library):
  qf, grid = z(G, N, 256), z(G, T, 8, 8, 256)
  outs = [z(G, N, T, 2), z(G, N, T), z(G, N, T), None, z(16, dtype=torch.uint8)]
  for call in (lambda: _lib.cost_volume_tracks(None, qf, z(G + 1, T, 8, 8, 256), None, 20.0, (64, 64), *outs),
               lambda: _lib.cost_volume_tracks(None, qf, grid, None, 20.0, (64, 64), z(G, N, T + 1, 2), *outs[1:]),
               lambda: _lib.cost_volume_tracks(None, qf, grid, z(G, N, 2), 20.0, (64, 64), *outs),
               lambda: _lib.pool_pyramid(z(T, 8, 8, 256), z(T, 4, 3, 256)),
               lambda: _lib.ingest_frames(z(T, 8, 8, 3), z(T, 8, 8, 3)),
               lambda: _lib.resample_frames(z(1, T, 8, 8, 3), z(1, T + 1, 16, 16, 3)),
               lambda: _lib.backbone_forward(None, z(T, 16, 16, 3), z(T, 2, 2, 256), z(T, 8, 8, 128), outs[-1]),
               lambda: _lib.split_planes(z(5, 70), z(P, 5, 64, dtype=torch.bfloat16))):
    with pytest.raises(ValueError):
      call()
