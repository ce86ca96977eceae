"""TEST INFRASTRUCTURE - generates tests/golden/io_redetection.npz from the reference's own AJ_RD
functions (tapnet/tapnextpp/metrics/aj_rd.py), run unmodified on the CPU.

Run in the build container only (needs /root/reference):
    python -m oracle.make_golden_redetection

The module needs only numpy and torch; its FunctionDefs are compiled into a scope that provides
them, as make_golden_tapvid does with its module.  Each case stores its inputs ([B, T, N, 2]
float32 tracks, [B, T, N] bool visibility), its thresholds, the reference's raw stats (indices,
durations, per-threshold values) and its metric dict (keys in order, values as the reference
returns them, NaN included).
"""
import json
import os
from typing import Any

import numpy as np
import torch

from oracle import redetection_oracle as R
from oracle.make_golden_io import GOLDEN_DIR, reference_functions

FUNCTIONS = ['calculate_jaccard_for_segment', 'count_consecutive_invisibility',
             'compute_raw_redetection_stats', 'compute_redetection_metrics']


def reference_scope():
  scope = dict(np=np, torch=torch, Any=Any)
  return dict(zip(FUNCTIONS, reference_functions('tapnet/tapnextpp/metrics/aj_rd.py', FUNCTIONS, scope)))


def _vis_runs(T, runs, start_visible=True):
  """A [T] bool track from alternating run lengths, the rest visible."""
  v = np.ones(T, bool)
  t, vis = 0, start_visible
  for r in runs:
    v[t:t + r] = vis
    t += r
    vis = not vis
  return v


def _case(rng, B, T, N, gt_visible=None, noise=0.5):
  gt = rng.uniform(0, 64, (B, T, N, 2)).astype(np.float32)
  pred = (gt + rng.normal(0, noise * 4, gt.shape)).astype(np.float32)
  gv = rng.uniform(size=(B, T, N)) < 0.7 if gt_visible is None else gt_visible
  pv = np.where(rng.uniform(size=(B, T, N)) < 0.8, gv, ~gv)
  return dict(pred_tracks=pred, pred_visible=pv, gt_tracks=gt, gt_visible=gv)


def _near_threshold_pairs(rng, thresholds, per_threshold=12):
  """(dx, dy) float32 pairs whose distance is exactly D, one ulp either side, and pairs where
  sqrt(fma(dy, dy, dx * dx)) and sqrt(dx * dx + dy * dy) (float32) fall on opposite sides of D."""
  pairs = []
  for D in np.asarray(thresholds, np.float32):
    for x in (D, np.nextafter(D, np.float32(np.inf)), np.nextafter(D, np.float32(0))):
      pairs += [(x, np.float32(0)), (np.float32(0), x)]
    found = 0
    while found < per_threshold:
      dx = rng.uniform(0, D, 4096).astype(np.float32)
      dy0 = np.sqrt(np.float32(D) * np.float32(D) - dx * dx).astype(np.float32)
      for step in range(-3, 4):
        dy = dy0
        for _ in range(abs(step)):
          dy = np.nextafter(dy, np.float32(np.inf) if step > 0 else np.float32(0))
        fma = R.norm(dx, dy) <= D
        plain = np.sqrt(dx * dx + dy * dy) <= D
        for i in np.nonzero(fma != plain)[0][:per_threshold - found]:
          pairs.append((dx[i], dy[i]))
          found += 1
        if found >= per_threshold:
          break
  return np.array(pairs, np.float32)


def cases():
  rng = np.random.default_rng(31)
  out = []

  def add(name, c, dist=None, dmin=None):
    out.append((name, c, dist, dmin))

  add('all_visible', _case(rng, 1, 20, 3, np.ones((1, 20, 3), bool)))
  add('all_invisible', _case(rng, 1, 20, 3, np.zeros((1, 20, 3), bool)))
  add('t1', _case(rng, 2, 1, 4))
  # durations 3, 1, 5, 5, 7: eligible, not, eligible, not (equal), eligible
  T = 40
  gv = np.ones((1, T, 2), bool)
  gv[0, :, 0] = _vis_runs(T, [2, 3, 2, 1, 3, 5, 1, 5, 2, 7, 1])
  gv[0, :, 1] = _vis_runs(T, [1, 2, 4, 2])
  add('durations_3_1_5_5_7', _case(rng, 1, T, 2, gv, noise=0.3))
  # invisible from frame 0; reappearing on the last frame; both
  T = 16
  gv = np.ones((1, T, 3), bool)
  gv[0, :, 0] = _vis_runs(T, [5, 3, 4], start_visible=False)
  gv[0, :, 1] = _vis_runs(T, [6, 9, 1])
  gv[0, :, 2] = _vis_runs(T, [15, 1], start_visible=False)
  add('frame0_and_last_frame', _case(rng, 1, T, 3, gv))
  # the maximal-event track: durations 1 .. K(64) = 9, from frame 0
  T = 64
  runs = []
  for d in range(1, 10):
    runs += [d, 1]
  gv = np.ones((1, T, 2), bool)
  gv[0, :, 0] = _vis_runs(T, runs, start_visible=False)
  gv[0, :, 1] = _vis_runs(T, [1] + runs, start_visible=True)
  add('maximal_events', _case(rng, 1, T, 2, gv, noise=0.2))
  # distances at the thresholds: one track per pair, frame 0 invisible, frame 1 visible
  for name, dist in (('near_default_thresholds', [1, 2, 4, 8, 16]), ('near_fraction_thresholds', [0.1, 2.5])):
    pairs = _near_threshold_pairs(rng, dist)
    N = len(pairs)
    gt = rng.uniform(0, 4, (1, 2, N, 2)).astype(np.float32)
    gt[0, 1] = 0   # the differences are the pairs exactly
    pred = gt.copy()
    pred[0, 1] = pairs
    assert np.array_equal(pred[0, 1] - gt[0, 1], pairs)
    gv = np.ones((1, 2, N), bool)
    gv[0, 0] = False
    c = dict(pred_tracks=pred.astype(np.float32), pred_visible=np.ones((1, 2, N), bool),
             gt_tracks=gt.astype(np.float32), gt_visible=gv)
    add(name, c, dist, [1] if name.endswith('default_thresholds') else [0, 1000])
  # NaN and infinite predictions, predicted visible where the ground truth is not
  c = _case(rng, 1, 12, 8, _vis_runs(12, [1, 2, 9])[None, :, None].repeat(8, 2))
  specials = [np.nan, np.inf, -np.inf]
  for n in range(6):
    c['pred_tracks'][0, 3 + n % 3:, n, n % 2] = specials[n % 3]
  c['gt_tracks'][0, 5:, 6, 0] = np.inf
  c['pred_tracks'][0, 5:, 6, 0] = np.inf
  c['pred_tracks'][0, 4:, 7, :] = c['gt_tracks'][0, 4:, 7, :]
  c['pred_visible'][0, :, 7] = True    # visible where the ground truth is not (frames 0 and 1..2)
  add('nan_inf_false_positives', c)
  # order: two clips with events on the same frames in several tracks
  gv = np.ones((2, 10, 5), bool)
  gv[:, 2:4, :] = False
  gv[:, 5:8, 1:4] = False
  gv[1, 1, 2] = False
  add('order_same_frame', _case(rng, 2, 10, 5, gv))
  # non-default thresholds: D = 0.1 and 2.5, d_min = 0 and one above every duration
  add('thresholds', _case(rng, 1, 30, 16, noise=0.05), [0.1, 2.5], [0, 1000])
  # a seeded Markov-visibility clip
  B, T, N = 2, 300, 64
  gv = np.zeros((B, T, N), bool)
  gv[:, 0] = rng.uniform(size=(B, N)) < 0.8
  for t in range(1, T):
    stay = np.where(gv[:, t - 1], 0.95, 0.9)
    gv[:, t] = np.where(rng.uniform(size=(B, N)) < stay, gv[:, t - 1], ~gv[:, t - 1])
  add('markov', _case(rng, B, T, N, gv, noise=1.0))
  return out


def make():
  ref = reference_scope()
  out, meta = {}, {'cases': [], 'torch': torch.__version__}
  for i, (name, c, dist, dmin) in enumerate(cases()):
    for k, v in c.items():
      out[f'c{i}_{k}'] = v
    t = {k: torch.from_numpy(v) for k, v in c.items()}
    raw = ref['compute_raw_redetection_stats'](t['pred_tracks'], t['pred_visible'], t['gt_tracks'],
                                               t['gt_visible'], dist)
    m = ref['compute_redetection_metrics'](t['pred_tracks'], t['pred_visible'], t['gt_tracks'],
                                           t['gt_visible'], dist, dmin)
    scalars = [[k, float(v), type(v).__name__] for k, v in m.items() if not k.startswith('raw_stats/')]
    events = 0
    if raw is not None:
      for name_i, idx in zip(('b', 't', 'n'), raw['indices']):
        out[f'c{i}_idx_{name_i}'] = idx.numpy()
      out[f'c{i}_durations'] = raw['durations'].numpy()
      out[f'c{i}_aj_rd'] = np.stack([v['aj_rd'].numpy() for v in raw['metrics_per_dist'].values()])
      events = len(raw['durations'])
      assert [k for k in m if k.startswith('raw_stats/')] == ['raw_stats/indices', 'raw_stats/durations',
                                                             'raw_stats/metrics_per_dist']
    meta['cases'].append(dict(name=name, dist_thresholds=dist, d_min_thresholds=dmin, events=events,
                              keys=list(m), scalars=scalars))
    print(f'{name}: {tuple(c["gt_visible"].shape)} {events} events')
  out['meta'] = np.frombuffer(json.dumps(meta).encode(), np.uint8)
  dst = os.path.join(GOLDEN_DIR, 'io_redetection.npz')
  np.savez_compressed(dst, **out)
  print(dst, os.path.getsize(dst), 'bytes,', len(out), 'arrays')


if __name__ == '__main__':
  make()
