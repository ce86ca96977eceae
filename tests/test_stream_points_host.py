"""Per-stream point counts without a GPU: the work groups, the grouped GEMM's m-tile tables,
and the argument checks of the tracker, estimate_trajectories and the new C-ABI calls."""
import ctypes
import random

import pytest
import torch

from tapnet_b200 import _lib, streaming, tapir_model

kBlockM = 128  # the wgmma GEMM's m-tile (gemm_tc.cu)


# ------------------------------------------------------------------------- work groups
def _uniform_groups(B, N, T):
  """The work groups of B clips of N queries each as (b0, b1, query slice): whole clips while the
  group's rows fit _MAX_ROWS_PER_CHUNK and its queries 65535, else query chunks of one clip."""
  if N * T <= tapir_model._MAX_ROWS_PER_CHUNK and N <= 65535:
    g = max(1, min(B, tapir_model._MAX_ROWS_PER_CHUNK // (N * T), 65535 // N))
    return [(b0, min(b0 + g, B), slice(0, N)) for b0 in range(0, B, g)]
  chunk_q = max(1, min(N, tapir_model._MAX_ROWS_PER_CHUNK // T, 65535))
  return [(bi, bi + 1, slice(q0, min(q0 + chunk_q, N)))
          for bi in range(B) for q0 in range(0, N, chunk_q)]


def _flat(groups, N):
  """(b0, b1, query slice) groups as flattened (b0, b1, q0, q1)."""
  return [(b0, b1, b0 * N + sl.start, (b1 - 1) * N + sl.stop) for b0, b1, sl in groups]


@pytest.mark.parametrize('B,N,T', [(1, 1, 1), (8, 64, 1), (5, 1024, 1), (3, 7, 48), (200, 1, 1),
                                   (4, 65535, 1), (2, 70000, 1), (3, 5000, 24), (2, 98304, 2),
                                   (70, 1500, 1)])
def test_equal_counts_work_groups_are_the_uniform_groups(B, N, T):
  assert tapir_model._work_groups([N] * B, T) == _flat(_uniform_groups(B, N, T), N)


def _check_cover(counts, T):
  groups = tapir_model._work_groups(counts, T)
  offs = [sum(counts[:b]) for b in range(len(counts) + 1)]
  q = 0
  for b0, b1, q0, q1 in groups:
    assert q0 == q and q1 > q0, (counts, T, groups)  # every query once, in order
    q = q1
    if b1 - b0 > 1 or (q0, q1) == (offs[b0], offs[b1]):  # whole clips
      assert (q0, q1) == (offs[b0], offs[b1])
      if b1 - b0 > 1:  # several clips share a group only within both bounds
        assert (q1 - q0) * T <= tapir_model._MAX_ROWS_PER_CHUNK and q1 - q0 <= 65535
    else:  # a query chunk of one clip too large on its own
      assert offs[b0] <= q0 and q1 <= offs[b0 + 1]
      assert counts[b0] * T > tapir_model._MAX_ROWS_PER_CHUNK or counts[b0] > 65535
    assert (q1 - q0) * T <= max(tapir_model._MAX_ROWS_PER_CHUNK, T) and q1 - q0 <= 65535
  assert q == offs[-1]


def test_work_groups_cover_every_query_once_within_the_bounds():
  rng = random.Random(7)
  for _ in range(300):
    counts = [rng.choice([1, 2, 63, 64, 65, 200, 1024, 5000, 65535, 70000])
              for _ in range(rng.randint(1, 12))]
    _check_cover(counts, rng.choice([1, 2, 3, 24, 48]))
  _check_cover([1], 1)
  _check_cover([65535], 1)
  _check_cover([65535, 1, 65535], 1)
  _check_cover([1] * 70000, 1)


# ------------------------------------------------------------------------- grouped GEMM tiles
def _tile_tables(counts):
  """What common_params builds for a grouped GEMM: group_row0, group_tile0."""
  row0, tile0 = [0], [0]
  for n in counts:
    row0.append(row0[-1] + n)
    tile0.append(tile0[-1] + -(-n // kBlockM))
  return row0, tile0


def _tile_group(tile0, m_tile):
  """gemm_tc.cu tile_group: the last g with tile0[g] <= m_tile, by the same binary search."""
  lo, hi = 0, len(tile0) - 2
  while lo < hi:
    mid = (lo + hi + 1) >> 1
    if tile0[mid] <= m_tile:
      lo = mid
    else:
      hi = mid - 1
  return lo


@pytest.mark.parametrize('counts', [[1], [63], [64], [65], [127], [128], [129], [200],
                                    [1, 63, 64, 65, 127, 128, 129, 200], [200, 1, 129, 128, 1],
                                    [1] * 64, [129] * 64])
def test_grouped_m_tiles_cover_each_clip_exactly(counts):
  row0, tile0 = _tile_tables(counts)
  stored = []
  for m_tile in range(tile0[-1]):
    g = _tile_group(tile0, m_tile)
    local = m_tile - tile0[g]
    rows = row0[g + 1] - row0[g]
    first = local * kBlockM
    assert 0 <= first < rows  # the tile starts inside its clip ...
    # ... and stores only rows of that clip (the rest of its 128 are loaded, never stored)
    stored += [row0[g] + r for r in range(first, min(first + kBlockM, rows))]
  assert stored == list(range(row0[-1]))


# ------------------------------------------------------------------------- argument checks
class _Model:
  use_casual_conv = True
  initial_resolution = (256, 256)

  def parameters(self):
    return iter([torch.zeros(1)])


def test_tracker_rejects_bad_counts():
  m = _Model()
  with pytest.raises(ValueError, match='2 counts for 3 streams'):
    streaming.OnlineTracker(m, 256, 256, [4, 5], num_streams=3)
  with pytest.raises(ValueError, match='at least one point'):
    streaming.OnlineTracker(m, 256, 256, [4, 0], num_streams=2)


def _cpu_tracker(counts, num_streams=None):
  """A tracker's argument handling without a device: construction stops at the CUDA check, so the
  checks under test are run on a bare instance.  counts: one int (num_streams streams) or a list."""
  trk = object.__new__(streaming.OnlineTracker)
  trk.num_streams = num_streams if isinstance(counts, int) else len(counts)
  trk._counts = [counts] * trk.num_streams if isinstance(counts, int) else counts
  trk.num_points, trk.dev = counts, torch.device('cpu')
  return trk


def test_tracker_query_points_are_checked():
  """The list form of a tracker of per-stream counts, and the tensor forms of one count."""
  trk = _cpu_tracker([3, 1])
  with pytest.raises(ValueError, match='list of 2 query point tensors'):
    trk._query_points(torch.zeros(2, 3, 3))
  with pytest.raises(ValueError, match='list of 2 query point tensors'):
    trk._query_points([torch.zeros(3, 3)])
  with pytest.raises(ValueError, match=r'stream 1: query points must be \[1, 3\]'):
    trk._query_points([torch.zeros(3, 3), torch.zeros(2, 3)])
  assert [tuple(q.shape) for q in trk._query_points([torch.zeros(3, 3), torch.zeros(1, 3)])] == [
      (3, 3), (1, 3)]
  trk = _cpu_tracker(4, num_streams=2)
  assert [tuple(q.shape) for q in trk._query_points(torch.zeros(2, 4, 3))] == [(4, 3), (4, 3)]
  with pytest.raises(ValueError, match=r'query_points must be \[2, N, 3\], got \(1, 4, 3\)'):
    trk._query_points(torch.zeros(4, 3))
  with pytest.raises(ValueError, match=r'query_points must be \[2, N, 3\]'):
    trk._query_points(torch.zeros(2, 4, 2))
  with pytest.raises(ValueError, match='expected 4 query points, got 5'):
    trk._query_points(torch.zeros(2, 5, 3))
  one = _cpu_tracker(4, num_streams=1)
  assert [tuple(q.shape) for q in one._query_points(torch.zeros(4, 3))] == [(4, 3)]
  assert [tuple(q.shape) for q in one._query_points(torch.zeros(1, 4, 3))] == [(4, 3)]
  with pytest.raises(ValueError, match='expected 4 query points, got 3'):
    one._query_points(torch.zeros(3, 3))


def test_update_query_checks_the_streams_own_count():
  trk = _cpu_tracker([3, 1])
  trk.query_features = object()
  with pytest.raises(ValueError, match=r'point 1 out of range \[0, 1\) of stream 1'):
    trk.update_query(torch.zeros(8, 8, 3), torch.zeros(3), 1, stream=1)
  with pytest.raises(ValueError, match=r'point 3 out of range \[0, 3\) of stream 0'):
    trk.update_query(torch.zeros(8, 8, 3), torch.zeros(3), 3, stream=0)


def test_estimate_trajectories_checks_points_per_clip():
  fg = tapir_model.FeatureGrids((torch.zeros(2, 1, 32, 32, 256),), (torch.zeros(2, 1, 64, 64, 128),),
                                ((256, 256),))
  qf = tapir_model.QueryFeatures((torch.zeros(1, 5, 256),), (torch.zeros(1, 5, 128),), ((256, 256),))
  chk = tapir_model.TAPIR._check_points_per_clip
  assert chk([2, 3], fg, qf, None) == [2, 3]
  with pytest.raises(ValueError, match='3 counts for 2 clips'):
    chk([1, 2, 2], fg, qf, None)
  with pytest.raises(ValueError, match='at least one point'):
    chk([5, 0], fg, qf, None)
  with pytest.raises(ValueError, match=r'needs \[1, 4'):
    chk([1, 3], fg, qf, None)
  with pytest.raises(ValueError, match='query_points_in_video'):
    chk([2, 3], fg, qf, torch.zeros(1, 4, 3))


# ------------------------------------------------------------------------- C ABI
def test_ragged_entry_points_reject_bad_arguments_without_a_gpu():
  lib = _lib.load()
  head = _lib.HeadWeights()
  buf = ctypes.create_string_buffer(4096)
  p = ctypes.c_void_p(ctypes.addressof(buf) + (-ctypes.addressof(buf) % 256))
  counts = (ctypes.c_int32 * 3)(4, 1, 7)

  def cv(head_p=ctypes.byref(head), q=p, B=3, c=counts, T=2, ws=p):
    return lib.tapir_cost_volume_tracks_ragged(head_p, q, p, B, c, T, 32, 32, 256, None, 20.0, 256, 256,
                                               p, p, p, None, ws, 1 << 40, None)

  assert cv(head_p=None) == 1
  assert cv(q=None) == 1
  assert cv(c=None) == 1
  assert cv(ws=None) == 1
  assert cv(B=0) == 1
  assert cv(B=_lib.MAX_RAGGED_CLIPS + 1) == 1
  assert cv(c=(ctypes.c_int32 * 3)(4, 0, 7)) == 1
  assert cv(T=0) == 1
  assert b'tapir_cost_volume_tracks_ragged' in lib.tapir_last_error()
  assert lib.tapir_cost_volume_ragged_workspace_bytes(3, 12, 2, 32, 32, 256) > 12 * 2 * 1024 * 4
  assert lib.tapir_cost_volume_ragged_workspace_bytes(0, 12, 2, 32, 32, 256) == 0

  ca = _lib.CorrArgs(num_levels=2, num_points=5, num_frames=1, init_h=256, init_w=256, planes=2,
                     pos=p.value, occ=p.value, expd=p.value, feat_hi=p.value, feat_lo=p.value,
                     out_planes=p.value, out_plane_stride=5 * 512, ld=512)
  for i in range(2):
    ca.levels[i] = _lib.CorrLevel(p.value, 8, 8, 128 if i == 0 else 256, 0)
  assert lib.tapir_local_corr_ragged(None, 2, p, None) == 1
  assert lib.tapir_local_corr_ragged(ctypes.byref(ca), 2, None, None) == 1
  assert lib.tapir_local_corr_ragged(ctypes.byref(ca), 0, p, None) == 1
  ca.num_points = 0
  assert lib.tapir_local_corr_ragged(ctypes.byref(ca), 2, p, None) == 1

  ua = _lib.UpdateArgs(res=p.value, ld_res=400, num_points=5, num_frames=1, init_h=256, init_w=256,
                       resize_h=256, resize_w=256, feat_hi=p.value, feat_lo=p.value, pos=p.value,
                       occ_in=p.value, expd_in=p.value, occ_out=p.value, expd_out=p.value,
                       feat_out=p.value, tracks_out=p.value)
  assert lib.tapir_refine_update_ragged(None, p, p, None) == 1
  assert lib.tapir_refine_update_ragged(ctypes.byref(ua), None, p, None) == 1
  assert lib.tapir_refine_update_ragged(ctypes.byref(ua), p, None, None) == 1
  ua.num_points = 0
  assert lib.tapir_refine_update_ragged(ctypes.byref(ua), p, p, None) == 1
  ua.num_points, ua.tracks_out = 5, None
  assert lib.tapir_refine_update_ragged(ctypes.byref(ua), p, p, None) == 1


def test_ragged_bindings_check_tensors_before_the_library():
  z = torch.zeros
  with pytest.raises(ValueError, match='at least one query'):
    _lib.cost_volume_tracks_ragged(None, z(5, 256), [5, 0], z(2, 1, 8, 8, 256), None, 20.0, (64, 64),
                                   z(5, 1, 2), z(5, 1), z(5, 1), None, None)
  with pytest.raises(ValueError, match='clips'):
    _lib.cost_volume_tracks_ragged(None, z(65, 256), [1] * 65, z(65, 1, 8, 8, 256), None, 20.0,
                                   (64, 64), z(65, 1, 2), z(65, 1), z(65, 1), None, None)
  with pytest.raises(ValueError, match='for 6 queries'):
    _lib.cost_volume_tracks_ragged(None, z(5, 256), [5, 1], z(2, 1, 8, 8, 256), None, 20.0, (64, 64),
                                   z(6, 1, 2), z(6, 1), z(6, 1), None, None)
  with pytest.raises(ValueError, match='points'):
    _lib.cost_volume_tracks_ragged(None, z(6, 256), [5, 1], z(2, 1, 8, 8, 256), None, 20.0, (64, 64),
                                   z(6, 2, 2), z(6, 1), z(6, 1), None, None)
