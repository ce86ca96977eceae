"""The point-edit bookkeeping of OnlineTracker (retarget / add_points / remove_points) as pure
functions, and the tracker's argument checks, which all run before anything is queued (no GPU)."""
import numpy as np
import pytest
import torch

from tapnet_b200 import _lib, streaming


def test_retarget_last_edit_wins():
  p = streaming.retarget_requests({}, 5, [1, 3], [[0, 1, 2], [0, 3, 4]])
  assert p == {1: (0.0, 1.0, 2.0), 3: (0.0, 3.0, 4.0)}
  p = streaming.retarget_requests(p, 5, torch.tensor([3, 3]), torch.tensor([[0, 5, 5], [1, 6, 7.5]]))
  assert p == {1: (0.0, 1.0, 2.0), 3: (1.0, 6.0, 7.5)}
  assert streaming.retarget_requests(p, 5, 4, [0, 8, 9])[4] == (0.0, 8.0, 9.0)
  assert 2 in streaming.retarget_requests(p, 5, np.array([2]), np.zeros((1, 3), np.float32))


def test_add_appends_and_remove_shifts_and_cancels():
  p, n, new = streaming.add_requests({2: (0.0, 1.0, 1.0)}, 4, [[0, 5, 5], [0, 6, 6]])
  assert (n, new) == (6, [4, 5])
  assert p == {2: (0.0, 1.0, 1.0), 4: (0.0, 5.0, 5.0), 5: (0.0, 6.0, 6.0)}
  # removing 2 (pending) drops its request; 4 and 5 shift down to 2 and 3
  p, keep = streaming.remove_requests(p, n, [0, 2])
  assert keep == [1, 3, 4, 5]
  assert p == {2: (0.0, 5.0, 5.0), 3: (0.0, 6.0, 6.0)}
  # indices refer to the current points: a second removal sees the shifted ones
  p, keep = streaming.remove_requests(p, 4, [2])
  assert keep == [0, 1, 3] and p == {2: (0.0, 6.0, 6.0)}


def test_packed_offsets():
  assert streaming.packed_offsets([3, 1, 4]) == [0, 3, 4]
  assert streaming.packed_offsets([]) == []


@pytest.mark.parametrize('idx', [5, -1, [0, 7], 1.0, [True], torch.tensor([0.5]),
                                 torch.zeros(2, 2, dtype=torch.int64), np.array([0.0])])
def test_bad_indices_raise(idx):
  with pytest.raises(ValueError):
    streaming.retarget_requests({}, 5, idx, [[0, 1, 1]] * (2 if isinstance(idx, list) else 1))


def test_bad_points_and_removals_raise():
  with pytest.raises(ValueError):  # one point for two indices
    streaming.retarget_requests({}, 5, [0, 1], [[0, 1, 1]])
  with pytest.raises(ValueError):
    streaming.add_requests({}, 5, torch.zeros(2, 2))
  with pytest.raises(ValueError):  # repeated
    streaming.remove_requests({}, 5, [1, 1])
  with pytest.raises(ValueError):  # a stream keeps at least one point
    streaming.remove_requests({}, 3, [0, 1, 2])
  assert streaming.remove_requests({}, 3, [0, 2])[1] == [1]


def test_request_table_layout():
  t = _lib.query_request_table(3, 'cpu')
  assert t.shape == (16,) and t.dtype == torch.int32
  _lib.write_query_requests(t, [(2, 1, 0.0, 1.5, 2.5), (0, 0, 3.0, 4.0, 5.0)])
  assert t[0] == 2
  body = t[1:11].view(2, 5)
  assert body[:, :2].tolist() == [[2, 1], [0, 0]]
  assert body[:, 2:].contiguous().view(torch.float32).tolist() == [[0.0, 1.5, 2.5], [3.0, 4.0, 5.0]]
  _lib.write_query_requests(t, [])
  assert t[0] == 0
  with pytest.raises(ValueError):
    _lib.write_query_requests(t, [(0, 0, 0.0, 0.0, 0.0)] * 4)


def _stub(num_points, S, initialised=True):
  """An OnlineTracker with only what the edit checks read (the constructor needs a GPU)."""
  trk = streaming.OnlineTracker.__new__(streaming.OnlineTracker)
  trk.num_streams = S
  trk.num_points = num_points
  trk._counts = [num_points] * S if isinstance(num_points, int) else list(num_points)
  trk._pending = [{} for _ in range(S)]
  trk.query_features = object() if initialised else None
  return trk


def test_tracker_edit_checks():
  with pytest.raises(RuntimeError):
    _stub(4, 1, initialised=False).retarget(torch.zeros(1, 3), [0])
  with pytest.raises(RuntimeError):
    _stub([4, 2], 2, initialised=False).add_points(torch.zeros(1, 3))
  with pytest.raises(RuntimeError):
    _stub([4, 2], 2, initialised=False).remove_points([0])
  # one int count for several streams: counts stay fixed
  for call in (lambda t: t.add_points(torch.zeros(1, 3), stream=1),
               lambda t: t.remove_points([0], stream=1)):
    with pytest.raises(ValueError, match='num_points'):
      call(_stub(4, 2))
  with pytest.raises(ValueError):
    _stub([4, 2], 2).retarget(torch.zeros(1, 3), [0], stream=2)
  with pytest.raises(ValueError):
    _stub([4, 2], 2).retarget(torch.zeros(1, 3), [2], stream=1)
  trk = _stub([4, 1], 2)
  with pytest.raises(ValueError):  # stream 1 keeps its one point
    trk.remove_points([0], stream=1)
  assert trk._pending == [{}, {}] and trk._counts == [4, 1]  # nothing queued by a failed edit
