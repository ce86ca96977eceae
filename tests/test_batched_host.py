"""Host-side argument checks of the batched entry points and the multi-stream tracker, and the
clip grouping of estimate_trajectories (no GPU)."""
import ctypes

import pytest

from tapnet_b200 import _lib, streaming, tapir_model

DUMMY = ctypes.c_void_p(256)  # never dereferenced: every call below fails its argument check


def _error(lib):
  return lib.tapir_last_error().decode()


def test_cost_volume_batched_rejects_bad_arguments():
  lib = _lib.load()
  hw = _lib.HeadWeights()

  def call(B, qfeat=DUMMY, grid=DUMMY, N=16, points=DUMMY):
    return lib.tapir_cost_volume_tracks_batched(ctypes.byref(hw), qfeat, grid, B, N, 2, 32, 32, 256,
                                                None, 20.0, 256, 256, points, DUMMY, DUMMY, None,
                                                DUMMY, 1 << 30, None)

  assert call(0) == 1 and 'clip count' in _error(lib)
  assert call(-3) == 1 and 'clip count' in _error(lib)
  assert call(2, qfeat=None) == 1 and 'null pointer' in _error(lib)
  assert call(2, grid=None) == 1 and 'null pointer' in _error(lib)
  assert call(2, points=None) == 1 and 'null pointer' in _error(lib)
  assert call(1000, N=100) == 1 and '65535' in _error(lib)
  assert lib.tapir_cost_volume_tracks_batched(None, DUMMY, DUMMY, 2, 16, 2, 32, 32, 256, None, 20.0,
                                              256, 256, DUMMY, DUMMY, DUMMY, None, DUMMY, 1 << 30,
                                              None) == 1


def test_cost_volume_batched_workspace():
  lib = _lib.load()
  one = lib.tapir_cost_volume_workspace_bytes(40, 6, 32, 32, 256)
  assert lib.tapir_cost_volume_batched_workspace_bytes(1, 40, 6, 32, 32, 256) == one
  assert lib.tapir_cost_volume_batched_workspace_bytes(3, 40, 6, 32, 32, 256) > 2 * one
  assert lib.tapir_cost_volume_batched_workspace_bytes(0, 40, 6, 32, 32, 256) == 0


def test_local_corr_batched_rejects_bad_arguments():
  lib = _lib.load()
  assert lib.tapir_local_corr_batched(None, 2, None) == 1 and 'level count' in _error(lib)
  ca = _lib.CorrArgs()
  for i in range(3):
    ca.levels[i].grid = 256
    ca.levels[i].h, ca.levels[i].w, ca.levels[i].C = 32, 32, 128 if i == 0 else 256
  ca.num_levels, ca.num_points, ca.num_frames, ca.planes, ca.ld = 3, 16, 2, 2, 576
  for name in ('pos', 'occ', 'expd', 'feat_hi', 'feat_lo', 'out_planes'):
    setattr(ca, name, 256)
  assert lib.tapir_local_corr_batched(ctypes.byref(ca), 0, None) == 1 and 'clip count' in _error(lib)
  assert lib.tapir_local_corr_batched(ctypes.byref(ca), -1, None) == 1 and 'clip count' in _error(lib)
  ca.pos = None
  assert lib.tapir_local_corr_batched(ctypes.byref(ca), 2, None) == 1 and 'null pointer' in _error(lib)
  assert lib.tapir_local_corr(ctypes.byref(ca), None) == 1 and 'null pointer' in _error(lib)


def test_tracker_rejects_a_stream_count_below_one():
  model = tapir_model.TAPIR(use_casual_conv=True)
  for s in (0, -2):
    with pytest.raises(ValueError, match='num_streams'):
      streaming.OnlineTracker(model, 256, 256, 8, num_streams=s)


@pytest.mark.parametrize('B,N,T,bound', [(1, 16, 24, 98304), (8, 64, 24, 98304), (3, 21, 4, 168),
                                         (3, 21, 4, 32), (2, 5000, 48, 98304), (40, 4000, 1, 98304),
                                         (5, 70000, 1, 10 ** 9)])
def test_work_groups_of_equal_counts_cover_every_clip_and_query_within_bounds(B, N, T, bound, monkeypatch):
  monkeypatch.setattr(tapir_model, '_MAX_ROWS_PER_CHUNK', bound)
  groups = tapir_model._work_groups([N] * B, T)
  seen = [[0] * N for _ in range(B)]
  for b0, b1, q0, q1 in groups:  # queries q0..q1-1 of the flattened [B * N] point axis
    assert b1 > b0 and q1 > q0 and q1 - q0 <= 65535
    if b1 - b0 > 1:  # several clips: whole clips within the row bound
      assert (q0, q1) == (b0 * N, b1 * N) and (b1 - b0) * N * T <= bound
    for q in range(q0, q1):
      assert b0 <= q // N < b1
      seen[q // N][q % N] += 1
  assert all(c == 1 for row in seen for c in row)
  if N * T <= bound and N <= 65535:
    assert all((q0, q1) == (b0 * N, b1 * N) for b0, b1, q0, q1 in groups)
  if B == 1 and N * T <= bound:
    assert groups == [(0, 1, 0, N)]
