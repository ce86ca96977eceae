"""-m gpu: AJ_RD on the device (tapir_redetection_events + metrics.compute_redetection_metrics)
bit for bit against the reference's outputs in tests/golden/io_redetection.npz and against the
numpy oracle on large clips; repeatability, side streams and graph replay; `evaluate` with
redetection=True and with window_frames."""
import pickle

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import redetection_oracle as R  # noqa: E402
from tapnet_b200 import _lib, metrics, tapvid  # noqa: E402
from tests.test_redetection_host import check_raw, check_scalars, fixture_cases, same_float  # noqa: E402
from tests.test_stages_gpu import get_model  # noqa: E402


def _cuda(x):
  return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in x.items()}


def _raw_numpy(m, dist):
  return (tuple(i.cpu().numpy() for i in m['raw_stats/indices']), m['raw_stats/durations'].cpu().numpy(),
          {d: {'aj_rd': m['raw_stats/metrics_per_dist'][d]['aj_rd'].cpu().numpy()} for d in dist})


def _check_device_raw(m, dist):
  assert all(i.is_cuda and i.dtype == torch.int64 for i in m['raw_stats/indices'])
  assert m['raw_stats/durations'].is_cuda and m['raw_stats/durations'].dtype == torch.int32
  assert list(m['raw_stats/metrics_per_dist']) == list(dist)
  for v in m['raw_stats/metrics_per_dist'].values():
    assert list(v) == ['aj_rd'] and v['aj_rd'].is_cuda and v['aj_rd'].dtype == torch.float32


def test_fixture_bit_for_bit():
  for i, case, x, g in fixture_cases():
    d = _cuda(x)
    m = metrics.compute_redetection_metrics(d['pred_tracks'], d['pred_visible'], d['gt_tracks'],
                                            d['gt_visible'], case['dist_thresholds'], case['d_min_thresholds'])
    assert list(m) == case['keys'], case['name']
    check_scalars(case, m)
    for k, _, typ in case['scalars']:
      assert type(m[k]).__name__ == typ, (case['name'], k, type(m[k]))
    if case['events']:
      dist = case['dist_thresholds'] or metrics.DIST_THRESHOLDS
      _check_device_raw(m, dist)
      check_raw(g, i, case, *_raw_numpy(m, dist))
    # visibility as 0 / 1 floats goes through .bool() as in the reference
    m2 = metrics.compute_redetection_metrics(d['pred_tracks'], d['pred_visible'].float(), d['gt_tracks'],
                                             d['gt_visible'].to(torch.uint8), case['dist_thresholds'],
                                             case['d_min_thresholds'])
    check_scalars(case, m2)


def _logits(rng, shape):
  occ = torch.from_numpy(rng.normal(0, 2, shape).astype(np.float32)).cuda()
  expd = torch.from_numpy(rng.normal(-1, 2, shape).astype(np.float32)).cuda()
  vis = torch.empty(shape, dtype=torch.uint8, device='cuda')
  _lib.postprocess_occlusions(occ, expd, vis)
  return occ, expd, vis


def _same_metrics(a, b):
  assert list(a) == list(b)
  for k in a:
    if k.startswith('raw_stats/'):
      continue
    assert same_float(float(a[k]), float(b[k])), (k, a[k], b[k])
  if 'raw_stats/indices' in a:
    for x, y in zip(a['raw_stats/indices'], b['raw_stats/indices']):
      assert torch.equal(x, y)
    assert torch.equal(a['raw_stats/durations'], b['raw_stats/durations'])
    for d in a['raw_stats/metrics_per_dist']:
      x, y = a['raw_stats/metrics_per_dist'][d]['aj_rd'], b['raw_stats/metrics_per_dist'][d]['aj_rd']
      assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def test_fixture_logits_path_equals_postprocess_occlusions():
  rng = np.random.default_rng(4)
  for _, case, x, _ in fixture_cases():
    d = _cuda(x)
    tm = {k: d[k].transpose(1, 2).contiguous() for k in d}
    occ, expd, vis = _logits(rng, tuple(tm['gt_visible'].shape))
    a = metrics.redetection_metrics_tracks(tm['pred_tracks'], vis, tm['gt_tracks'], tm['gt_visible'],
                                           case['dist_thresholds'], case['d_min_thresholds'])
    b = metrics.redetection_metrics_tracks(tm['pred_tracks'], None, tm['gt_tracks'], tm['gt_visible'],
                                           case['dist_thresholds'], case['d_min_thresholds'],
                                           pred_logits=(occ, expd))
    _same_metrics(a, b)


def _markov_clip(seed, B, T, N, stay_visible=0.97, stay_hidden=0.9, noise=2.0):
  rng = np.random.default_rng(seed)
  gv = np.zeros((B, T, N), bool)
  gv[:, 0] = rng.uniform(size=(B, N)) < 0.7
  for t in range(1, T):
    stay = np.where(gv[:, t - 1], stay_visible, stay_hidden)
    gv[:, t] = np.where(rng.uniform(size=(B, N)) < stay, gv[:, t - 1], ~gv[:, t - 1])
  gt = rng.uniform(0, 256, (B, T, N, 2)).astype(np.float32)
  pred = (gt + rng.normal(0, noise, gt.shape)).astype(np.float32)
  pv = np.where(rng.uniform(size=(B, T, N)) < 0.85, gv, ~gv)
  return dict(pred_tracks=pred, pred_visible=pv, gt_tracks=gt, gt_visible=gv)


def _check_against_oracle(x, dist=None, dmin=None):
  want, raw = R.metrics(x['pred_tracks'], x['pred_visible'], x['gt_tracks'], x['gt_visible'], dist, dmin)
  d = _cuda(x)
  got = metrics.compute_redetection_metrics(d['pred_tracks'], d['pred_visible'], d['gt_tracks'],
                                            d['gt_visible'], dist, dmin)
  for k, v in want.items():
    assert same_float(float(got[k]), v), (k, got[k], v)
  if raw is None:
    assert 'raw_stats/durations' not in got
    return got
  dist = dist or R.DIST_THRESHOLDS
  idx, dur, per = _raw_numpy(got, dist)
  for a, b in zip(idx, raw['indices']):
    np.testing.assert_array_equal(a, b)
  np.testing.assert_array_equal(dur, raw['durations'])
  for dd in dist:
    a, b = per[dd]['aj_rd'], raw['metrics_per_dist'][dd]['aj_rd']
    np.testing.assert_array_equal(np.isnan(a), np.isnan(b))
    np.testing.assert_array_equal(a[~np.isnan(a)].view(np.int32), b[~np.isnan(b)].view(np.int32))
  return got


@pytest.mark.parametrize('shape', [(1, 1, 5), (2, 2, 7), (1, 31, 33), (2, 300, 64), (1, 1500, 256),
                                   (2, 1500, 2048)], ids=lambda s: 'x'.join(map(str, s)))
def test_random_clips_equal_oracle(shape):
  B, T, N = shape
  x = _markov_clip(sum(shape), B, T, N)
  got = _check_against_oracle(x)
  if T >= 300:
    assert len(got['raw_stats/durations']) > B * N // 4


def test_thresholds_and_d_min_equal_oracle():
  x = _markov_clip(9, 2, 200, 96, noise=0.3)
  _check_against_oracle(x, [0.1, 0.25, 2.5, 3, 100, 1e-30], [0, 2, 7, 1000])
  _check_against_oracle(x, list(range(1, 17)), [1])


def test_maximal_event_track_long_clip():
  T = 65536
  K = _lib.redetection_max_events(T)
  vis = np.ones(T, bool)
  t = 0
  for d in range(1, K + 1):
    vis[t:t + d] = False
    t += d + 1
  rng = np.random.default_rng(2)
  gv = np.stack([vis, np.roll(vis, 5)], 1)[None]   # [1, T, 2]
  gt = rng.uniform(0, 64, (1, T, 2, 2)).astype(np.float32)
  x = dict(pred_tracks=(gt + rng.normal(0, 3, gt.shape)).astype(np.float32),
           pred_visible=rng.uniform(size=gv.shape) < 0.9, gt_tracks=gt, gt_visible=gv)
  got = _check_against_oracle(x)
  durations = got['raw_stats/durations'].cpu().numpy()
  n = got['raw_stats/indices'][2].cpu().numpy()
  assert np.array_equal(durations[n == 0], np.arange(1, K + 1))


def test_track_major_equals_reference_layout():
  x = _markov_clip(12, 2, 120, 40)
  d = _cuda(x)
  a = metrics.compute_redetection_metrics(d['pred_tracks'], d['pred_visible'], d['gt_tracks'], d['gt_visible'])
  tm = {k: d[k].transpose(1, 2).contiguous() for k in d}
  b = metrics.redetection_metrics_tracks(tm['pred_tracks'], tm['pred_visible'], tm['gt_tracks'], tm['gt_visible'])
  _same_metrics(a, b)


def _track_major_inputs(seed=3, B=2, T=400, N=300):
  x = _markov_clip(seed, B, T, N)
  d = _cuda(x)
  return {k: d[k].transpose(1, 2).contiguous() for k in d}


def _events(tm):
  return metrics.redetection_events(tm['pred_tracks'], tm['pred_visible'], tm['gt_tracks'], tm['gt_visible'],
                                    metrics.DIST_THRESHOLDS)


def test_repeat_side_stream_and_graph_replay():
  tm = _track_major_inputs()
  first = _events(tm)
  for _ in range(3):
    assert torch.equal(_events(tm), first)
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    outs = [_events(tm) for _ in range(3)]
  torch.cuda.current_stream().wait_stream(side)
  for o in outs:
    assert torch.equal(o, first)
  # capture: the kernel, the sort and the packing are stream-ordered with no host sync
  warm = torch.cuda.Stream()
  warm.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(warm):
    _events(tm)
  torch.cuda.current_stream().wait_stream(warm)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    captured = _events(tm)
  for _ in range(2):
    captured.zero_()
    graph.replay()
    assert torch.equal(captured, first)
  # new inputs copied into the captured buffers give their own result
  tm2 = _track_major_inputs(seed=8)
  for k in tm:
    tm[k].copy_(tm2[k])
  graph.replay()
  assert torch.equal(captured, _events(tm2))


# ------------------------------------------------------------------------------ evaluate
def _davis_pickle(path, seed=17):
  rng = np.random.default_rng(seed)
  data = {}
  for name, (T, H, W, N) in (('long', (40, 36, 48, 10)), ('short', (23, 30, 40, 8))):
    occ = np.zeros((N, T), bool)
    for t in range(1, T):
      occ[:, t] = np.where(rng.uniform(size=N) < np.where(occ[:, t - 1], 0.8, 0.9), occ[:, t - 1], ~occ[:, t - 1])
    occ[0, :] = False
    data[name] = {'video': rng.integers(0, 256, (T, H, W, 3), dtype=np.uint8),
                  'points': rng.uniform(0, 1, (N, T, 2)).astype(np.float32), 'occluded': occ}
  with open(path, 'wb') as f:
    pickle.dump(data, f)
  return path


def _same_dicts(a, b):
  assert len(a) == len(b)
  for x, y in zip(a, b):
    assert list(x) == list(y)
    for k in x:
      assert same_float(x[k], y[k]), (k, x[k], y[k])


def test_evaluate_redetection(tmp_path):
  path = _davis_pickle(str(tmp_path / 'davis.pkl'))
  model = get_model()[0]
  mean0, per0 = tapvid.evaluate(model, tapvid.create_davis_dataset(path, 'strided'), 'strided')
  mean1, per1 = tapvid.evaluate(model, tapvid.create_davis_dataset(path, 'strided'), 'strided', redetection=True)
  for m0, m1 in zip(per0, per1):
    assert list(m1)[:len(m0)] == list(m0)
    assert all(same_float(m1[k], v) for k, v in m0.items())
    assert all(k.startswith('AJ_RD') for k in list(m1)[len(m0):])
  assert all(mean1[k] == v or (np.isnan(v) and np.isnan(mean1[k])) for k, v in mean0.items())
  # the AJ_RD keys against the oracle on the same model outputs
  for m1, sample in zip(per1, tapvid.create_davis_dataset(path, 'strided')):
    ex = sample['davis']
    qp = torch.from_numpy(ex['query_points'].astype(np.float32)).cuda()
    with torch.no_grad():
      out = model(ex['video'], qp)
    vis = torch.empty(out['occlusion'].shape, dtype=torch.uint8, device='cuda')
    _lib.postprocess_occlusions(out['occlusion'], out['expected_dist'], vis)
    want, raw = R.metrics(out['tracks'].cpu().numpy().transpose(0, 2, 1, 3), vis.cpu().numpy().transpose(0, 2, 1),
                          ex['target_points'].astype(np.float32).transpose(0, 2, 1, 3),
                          ~ex['occluded'].transpose(0, 2, 1))
    assert raw is not None
    for k, v in want.items():
      assert same_float(m1[k], v), (k, m1[k], v)
  for k in [k for k in per1[0] if k.startswith('AJ_RD')]:
    vals = [m[k] for m in per1 if not np.isnan(m[k])]
    assert mean1[f'{k}/videos'] == len(vals)
    if vals:
      assert mean1[k] == tapvid.dataset_mean([{k: v} for v in vals])[k]


@pytest.mark.parametrize('window_frames', [16, 'auto'])
def test_evaluate_windowed_equals_whole_clip(tmp_path, window_frames):
  path = _davis_pickle(str(tmp_path / 'davis.pkl'), seed=5)
  model = get_model()[0]
  mean0, per0 = tapvid.evaluate(model, tapvid.create_davis_dataset(path, 'first'), 'first', redetection=True)
  mean1, per1 = tapvid.evaluate(model, tapvid.create_davis_dataset(path, 'first'), 'first', redetection=True,
                                window_frames=window_frames)
  _same_dicts(per0, per1)
  assert list(mean0) == list(mean1)
  assert all(same_float(mean0[k], mean1[k]) for k in mean0)


def test_robotap_evaluate(tmp_path):
  d = tmp_path / 'robotap'
  d.mkdir()
  _davis_pickle(str(d / 'a.pkl'), seed=1)
  _davis_pickle(str(d / 'b.pkl'), seed=2)
  model = get_model()[0]
  _, per = tapvid.evaluate(model, tapvid.create_robotap_dataset(str(d)), 'strided', redetection=True)
  _, per_a = tapvid.evaluate(model, tapvid.create_davis_dataset(str(d / 'a.pkl')), 'strided', redetection=True)
  _, per_b = tapvid.evaluate(model, tapvid.create_davis_dataset(str(d / 'b.pkl')), 'strided', redetection=True)
  _same_dicts(per, per_a + per_b)
