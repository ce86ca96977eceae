"""AJ_RD without a GPU: the numpy oracle against the reference's outputs in
tests/golden/io_redetection.npz, the oracle's distance against torch.linalg.norm, K(T) from the C
ABI against a brute force, the C layout of tapir_redetection_args, argument errors before any CUDA
call, and the RoboTAP reader against the DAVIS reader."""
import ctypes
import math
import os
import pickle
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import redetection_oracle as R
from oracle import tapvid_oracle
from tapnet_b200 import _lib, metrics, tapvid
from tests.test_tapvid_host import check_converted

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'io_redetection.npz')


def golden():
  import json  # pylint: disable=g-import-not-at-top
  g = dict(np.load(GOLDEN))
  g['meta'] = json.loads(bytes(g['meta']).decode())
  return g


def fixture_cases():
  """(index, case meta, inputs dict [B, T, N] layout) of every fixture case."""
  g = golden()
  for i, c in enumerate(g['meta']['cases']):
    yield i, c, {k: g[f'c{i}_{k}'] for k in ('pred_tracks', 'pred_visible', 'gt_tracks', 'gt_visible')}, g


def same_float(a, b):
  return (np.isnan(a) and np.isnan(b)) or a == b


def check_raw(g, i, case, indices, durations, per_dist):
  """Raw stats (numpy) equal the fixture's case i: order, dtypes, values bitwise, NaN for NaN."""
  assert len(durations) == case['events']
  for name, idx in zip(('b', 't', 'n'), indices):
    assert idx.dtype == np.int64
    np.testing.assert_array_equal(idx, g[f'c{i}_idx_{name}'])
  assert durations.dtype == np.int32
  np.testing.assert_array_equal(durations, g[f'c{i}_durations'])
  dist = case['dist_thresholds'] or R.DIST_THRESHOLDS
  assert list(per_dist) == list(dist)
  for j, d in enumerate(dist):
    v = per_dist[d]['aj_rd']
    assert v.dtype == np.float32
    want = g[f'c{i}_aj_rd'][j]
    np.testing.assert_array_equal(np.isnan(v), np.isnan(want))
    np.testing.assert_array_equal(v[~np.isnan(v)].view(np.int32), want[~np.isnan(want)].view(np.int32))


def check_scalars(case, got):
  """Metric dict `got` has the fixture's scalar keys in order and its values, NaN for NaN."""
  want = case['scalars']
  assert [k for k in got if not k.startswith('raw_stats/')] == [k for k, _, _ in want]
  for k, v, _ in want:
    assert same_float(float(got[k]), v), (case['name'], k, got[k], v)


def test_oracle_equals_fixture():
  names = []
  for i, case, x, g in fixture_cases():
    names.append(case['name'])
    got, raw = R.metrics(x['pred_tracks'], x['pred_visible'], x['gt_tracks'], x['gt_visible'],
                         case['dist_thresholds'], case['d_min_thresholds'])
    check_scalars(case, got)
    if case['events'] == 0:
      assert raw is None
      continue
    check_raw(g, i, case, raw['indices'], raw['durations'], raw['metrics_per_dist'])
  assert 'markov' in names and 'maximal_events' in names


def test_fixture_covers_the_designed_cases():
  cases = {c['name']: c for c in golden()['meta']['cases']}
  assert cases['durations_3_1_5_5_7']['events'] == 4          # 3, 5, 7 on one track + one
  assert cases['maximal_events']['events'] == 18              # K(64) = 9 on each of two tracks
  assert cases['t1']['events'] == cases['all_visible']['events'] == cases['all_invisible']['events'] == 0
  assert all(math.isnan(v) for _, v, _ in cases['t1']['scalars'])
  assert 'AJ_RD_D0.1_dmin0' in cases['thresholds']['keys'] and 'AJ_RD_D2.5_dmin1000' in cases['thresholds']['keys']
  assert all(math.isnan(v) for k, v, _ in cases['thresholds']['scalars'] if k.endswith('dmin1000'))
  assert cases['markov']['events'] > 100


def test_oracle_norm_equals_torch():
  rng = np.random.default_rng(11)
  for _ in range(5):
    a = rng.uniform(-32, 32, (2_000_000, 2)).astype(np.float32)
    b = rng.uniform(-32, 32, (2_000_000, 2)).astype(np.float32)
    d = a - b
    want = torch.linalg.norm(torch.from_numpy(a) - torch.from_numpy(b), dim=-1).numpy()
    np.testing.assert_array_equal(R.norm(d[:, 0], d[:, 1]).view(np.int32), want.view(np.int32))
  # the fixture's near-threshold pairs (exact D, one ulp either side, FMA vs plain sum at D)
  for i, case, x, _ in fixture_cases():
    if case['name'].startswith('near_'):
      d = x['pred_tracks'][0, 1] - x['gt_tracks'][0, 1]
      want = torch.linalg.norm(torch.from_numpy(d), dim=-1).numpy()
      np.testing.assert_array_equal(R.norm(d[:, 0], d[:, 1]).view(np.int32), want.view(np.int32))
      plain = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1])
      assert np.any(plain != want)   # the cases that tell the two forms apart


def test_max_events_equals_brute_force():
  k = 0
  for T in range(1, 5001):
    while (k + 1) * (k + 4) // 2 <= T:
      k += 1
    assert _lib.redetection_max_events(T) == k, T
  assert _lib.redetection_max_events(64) == 9 and _lib.redetection_max_events(1024) == 43
  assert _lib.redetection_max_events(1) == 0 and _lib.redetection_max_events(2) == 1
  assert _lib.redetection_max_events(0) == 0 and _lib.redetection_max_events(-5) == 0


def test_redetection_args_layout_matches_the_compiler(tmp_path):
  gcc = shutil.which('gcc')
  if gcc is None:
    pytest.skip('no gcc')
  cls = _lib.RedetectionArgs
  lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "tapir_b200.h"', 'int main(void) {',
           '  printf("%zu", sizeof(tapir_redetection_args));']
  lines += [f'  printf(" %zu", offsetof(tapir_redetection_args, {f}));' for f, _ in cls._fields_]
  lines += ['  printf(" %d\\n", TAPIR_REDETECTION_MAX_THRESHOLDS);', '  return 0;', '}']
  src = tmp_path / 'probe.c'
  src.write_text('\n'.join(lines))
  exe = tmp_path / 'probe'
  subprocess.run([gcc, '-std=c99', '-Wall', '-Werror', '-pedantic', '-I', os.path.join(ROOT, 'include'),
                  str(src), '-o', str(exe)], check=True)
  size, *rest = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True,
                                                text=True).stdout.split()]
  assert size == ctypes.sizeof(cls)
  assert rest[:-1] == [getattr(cls, f).offset for f, _ in cls._fields_]
  assert rest[-1] == _lib.REDETECTION_MAX_THRESHOLDS


def test_c_abi_rejects_bad_arguments():
  """rc 1 and a message, before any CUDA call (the pointers are never dereferenced)."""
  lib = _lib.load()
  p = 0x10000
  B, N, T = 2, 3, 64   # K(64) = 9

  def args(**kw):
    a = dict(gt_visible=p, pred_visible=p, pred_tracks=p, gt_tracks=p, num_thresholds=5, B=B, N=N, T=T,
             capacity=B * N * 9, event_t=p, event_duration=p, event_values=p, event_count=p)
    a.update(kw)
    return _lib.RedetectionArgs(**a)

  for kw, what in ((dict(B=0), 'bad shape'), (dict(N=-1), 'bad shape'), (dict(T=0), 'bad shape'),
                   (dict(num_thresholds=0), 'num_thresholds'), (dict(num_thresholds=17), 'num_thresholds'),
                   (dict(gt_visible=None), 'null pointer'), (dict(pred_tracks=None), 'null pointer'),
                   (dict(gt_tracks=None), 'null pointer'), (dict(event_count=None), 'null pointer'),
                   (dict(pred_visible=None), 'logit'), (dict(pred_visible=None, pred_occ_logits=p), 'logit'),
                   (dict(event_t=None), 'event array'), (dict(event_values=None), 'event array'),
                   (dict(event_duration=None), 'event array'), (dict(capacity=B * N * 9 - 1), 'capacity')):
    a = args(**kw)
    assert lib.tapir_redetection_events(ctypes.byref(a), None) == 1, kw
    assert what in lib.tapir_last_error().decode(), (kw, lib.tapir_last_error())
  assert lib.tapir_redetection_events(None, None) == 1


@pytest.fixture
def no_library(monkeypatch):
  def refuse():
    raise AssertionError('the library was touched')
  monkeypatch.setattr(_lib, 'load', refuse)
  monkeypatch.setattr(_lib, 'redetection_max_events', lambda T: 9)


def test_binding_raises_before_any_cuda_call(no_library):
  B, N, T, K = 1, 2, 64, 9
  u8 = torch.zeros(B, N, T, dtype=torch.uint8)
  tr = torch.zeros(B, N, T, 2)
  outs = dict(event_t=torch.zeros(B, N, K, dtype=torch.int32), event_duration=torch.zeros(B, N, K, dtype=torch.int32),
              event_values=torch.zeros(B, N, K, 5), event_count=torch.zeros(B, N, dtype=torch.int32))

  def call(thresholds=(1, 2, 4, 8, 16), **kw):
    a = dict(gt_visible=u8, pred_visible=u8, pred_tracks=tr, gt_tracks=tr, **outs)
    a.update(kw)
    _lib.redetection_events(a['gt_visible'], a['pred_visible'], a['pred_tracks'], a['gt_tracks'], thresholds,
                            a['event_t'], a['event_duration'], a['event_values'], a['event_count'],
                            a.get('pred_logits'))

  for kw, match in ((dict(thresholds=[]), 'thresholds'), (dict(thresholds=list(range(17))), 'thresholds'),
                    (dict(pred_visible=u8.bool()), 'pred_visible'), (dict(gt_tracks=tr.double()), 'gt_tracks'),
                    (dict(pred_tracks=tr[..., :1]), 'pred_tracks'), (dict(event_t=outs['event_t'][..., :8]), 'event_t'),
                    (dict(event_values=torch.zeros(B, N, K, 4)), 'event_values'),
                    (dict(event_count=outs['event_count'].float()), 'event_count'),
                    (dict(pred_tracks=tr.transpose(1, 2).contiguous().transpose(1, 2)), 'pred_tracks'),
                    (dict(pred_logits=(tr[..., 0].contiguous(), None)), 'expected_dist')):
    with pytest.raises(ValueError, match=match):
      call(**kw)
  with pytest.raises(RuntimeError, match='CUDA'):
    metrics.compute_redetection_metrics(torch.zeros(1, T, N, 2), torch.zeros(1, T, N), torch.zeros(1, T, N, 2),
                                        torch.zeros(1, T, N))


def test_evaluate_rejects_bad_window_frames():
  for bad in (0, -3, 2.5, '16', True):
    with pytest.raises(ValueError, match='window_frames'):
      tapvid.evaluate(None, [], 'strided', window_frames=bad)
  assert tapvid._window_frames('auto') == 'auto' and tapvid._window_frames('16') == 16


def _davis_format_pickle(rng, videos):
  data = {}
  for name, (T, H, W, N) in videos.items():
    occluded = rng.uniform(size=(N, T)) < 0.3
    occluded[0, ::5] = True
    data[name] = {'video': rng.integers(0, 256, (T, H, W, 3), dtype=np.uint8),
                  'points': rng.uniform(0, 1, (N, T, 2)).astype(np.float32), 'occluded': occluded}
  return data


def test_robotap_reader_equals_davis_reader(tmp_path, monkeypatch):
  """A directory of two RoboTAP pickles reads, video for video and in sorted file order, as the
  DAVIS reader reads each file; one pickle path reads as that file."""
  def host_clip(frames, resolution, staging):
    frames = np.asarray(frames)
    if resolution is not None and tuple(resolution) != frames.shape[1:3]:
      frames = tapvid_oracle.resize(frames, *resolution)
    return frames

  monkeypatch.setattr(tapvid, '_clip', host_clip)
  rng = np.random.default_rng(41)
  files = {'b_robotap.pkl': _davis_format_pickle(rng, {'grasp': (9, 20, 28, 5), 'stack': (6, 16, 16, 4)}),
           'a_robotap.pkl': _davis_format_pickle(rng, {'push': (12, 24, 20, 6)})}
  d = tmp_path / 'robotap'
  d.mkdir()
  for name, data in files.items():
    (d / name).write_bytes(pickle.dumps(data))
  (d / 'notes.txt').write_text('not a pickle')
  for mode in ('strided', 'first'):
    want = []
    for name in sorted(files):
      want += [s['davis'] for s in tapvid.create_davis_dataset(str(d / name), mode, resolution=(16, 24))]
    got = list(tapvid.create_robotap_dataset(str(d), mode, resolution=(16, 24)))
    assert len(got) == len(want) == 3
    for g_s, w in zip(got, want):
      assert list(g_s) == ['robotap']
      ref = {f'x_{k}': v for k, v in w.items()}
      check_converted(ref, 'x', g_s['robotap'], video=lambda v: v)
    one = list(tapvid.create_robotap_dataset(str(d / 'a_robotap.pkl'), mode, resolution=(16, 24)))
    assert len(one) == 1 and set(one[0]['robotap']) == set(want[0])
  with pytest.raises(ValueError, match='query mode'):
    next(tapvid.create_robotap_dataset(str(d), 'middle'))
