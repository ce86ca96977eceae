"""TEST INFRASTRUCTURE - a numpy restatement of AJ_RD (tapnet/tapnextpp/metrics/aj_rd.py), read
the way the reference reads: every reappearance in (b, t_r, n) order, its duration from the
invisible run before it, eligibility per track in t order, then one event at a time over the rest
of the clip.  Used to pin the device kernel on inputs larger than the reference can score in
reasonable time, and pinned itself to the reference by tests/golden/io_redetection.npz.

The distance is what torch's CPU `torch.linalg.norm(., dim=-1)` gives for float32 pairs:
sqrt(fma(dy, dy, dx * dx)) with dx * dx rounded to float32 and the sum rounded once.  `norm`
forms the sum in float64 and corrects the one case where rounding that to float32 would round
twice (a float64 sum on a float32 tie), with the sum's exact error from TwoSum.
"""
import numpy as np

DIST_THRESHOLDS = [1, 2, 4, 8, 16]
D_MIN_THRESHOLDS = [1, 4, 16, 64, 256]


def _round_once(hi, lo):
  """float32 nearest to the exact hi + lo (float64 arrays, |lo| <= ulp(hi) / 2)."""
  r = hi.astype(np.float32)
  with np.errstate(invalid='ignore', over='ignore'):
    r64 = r.astype(np.float64)
    other = np.nextafter(r, np.where(hi > r64, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    tie = np.isfinite(hi) & (hi != r64) & (hi == (r64 + other.astype(np.float64)) / 2) & (lo != 0)
  # on a tie the exact sum lies on lo's side of it
  toward_other = np.where(other.astype(np.float64) > r64, lo > 0, lo < 0)
  return np.where(tie & toward_other, other, r)


def norm(dx, dy):
  """float32 dx, dy -> float32 sqrt(fma(dy, dy, dx * dx)), each step rounded as the CPU does."""
  dx = np.asarray(dx, np.float32)
  dy = np.asarray(dy, np.float32)
  with np.errstate(over='ignore', invalid='ignore'):
    p = (dx * dx).astype(np.float64)                 # float32 product, rounded
    q = dy.astype(np.float64) * dy.astype(np.float64)  # exact: 48 significant bits
    s = p + q
    bp = s - q                                       # TwoSum: s + err == p + q exactly
    err = (p - bp) + (q - (s - bp))
    err = np.where(np.isfinite(err), err, 0.0)
    return np.sqrt(_round_once(s, err))


def _reappearances(gt_visible):
  """[B, T, N] bool -> (b, t, n) index arrays of t >= 1 with vis[t] & ~vis[t-1], in (b, t, n)
  order, and their durations (count_consecutive_invisibility at t)."""
  B, T, N = gt_visible.shape
  d = np.zeros((B, T, N), np.int64)
  for t in range(1, T):
    d[:, t] = np.where(~gt_visible[:, t - 1], d[:, t - 1] + 1, 0)
  mask = np.zeros_like(gt_visible)
  mask[:, 1:] = gt_visible[:, 1:] & ~gt_visible[:, :-1]
  b, t, n = np.nonzero(mask)
  return b, t, n, d[b, t, n].astype(np.int32)


def raw_stats(pred_tracks, pred_visible, gt_tracks, gt_visible, dist_thresholds=None):
  """compute_raw_redetection_stats: None, or dict(indices=(b, t_r, n) int64, durations int32,
  metrics_per_dist={D: {'aj_rd': float32 [events]}})."""
  dist_thresholds = DIST_THRESHOLDS if dist_thresholds is None else dist_thresholds
  pred_tracks = np.asarray(pred_tracks, np.float32)
  gt_tracks = np.asarray(gt_tracks, np.float32)
  pv, gv = np.asarray(pred_visible).astype(bool), np.asarray(gt_visible).astype(bool)
  T = gv.shape[1]
  b, t, n, dur = _reappearances(gv)
  if len(b) == 0:
    return None
  eligible = np.zeros(len(b), bool)
  best = {}
  for i in np.lexsort((t, n, b)):   # per track in t order
    key = (b[i], n[i])
    if dur[i] > best.get(key, -1):
      eligible[i] = True
      best[key] = dur[i]
  b, t, n, dur = b[eligible], t[eligible], n[eligible], dur[eligible]
  thr = np.asarray(dist_thresholds, np.float32)
  values = np.full((len(thr), len(b)), np.nan, np.float32)
  for i in range(len(b)):
    seg = slice(t[i], T)
    with np.errstate(invalid='ignore'):   # inf - inf
      diff = pred_tracks[b[i], seg, n[i]] - gt_tracks[b[i], seg, n[i]]
    dist = norm(diff[:, 0], diff[:, 1])
    g, p = gv[b[i], seg, n[i]], pv[b[i], seg, n[i]]
    within = dist[None] <= thr[:, None]
    tp = np.sum(within & g & p, axis=1)
    fp = np.sum(p & (~g | ~within), axis=1)
    den = np.sum(g) + fp
    with np.errstate(invalid='ignore'):
      values[:, i] = np.where(den == 0, np.nan, tp.astype(np.float32) / den.astype(np.float32))
  return {'indices': (b.astype(np.int64), t.astype(np.int64), n.astype(np.int64)),
          'durations': dur,
          'metrics_per_dist': {d: {'aj_rd': values[j]} for j, d in enumerate(dist_thresholds)}}


def metrics(pred_tracks, pred_visible, gt_tracks, gt_visible, dist_thresholds=None,
            d_min_thresholds=None):
  """compute_redetection_metrics' scalar keys (float, or nan) and the raw stats (or None).  Each
  (d_min, D) mean is torch's CPU mean of the float32 values, as the reference takes it there."""
  import torch  # pylint: disable=g-import-not-at-top
  dist_thresholds = DIST_THRESHOLDS if dist_thresholds is None else dist_thresholds
  d_min_thresholds = D_MIN_THRESHOLDS if d_min_thresholds is None else d_min_thresholds
  raw = raw_stats(pred_tracks, pred_visible, gt_tracks, gt_visible, dist_thresholds)
  out = {}
  for d_min in d_min_thresholds:
    mask = raw['durations'] >= d_min if raw is not None else np.zeros(0, bool)
    if not mask.any():
      for d_thresh in dist_thresholds:
        out[f'AJ_RD_D{d_thresh}_dmin{d_min}'] = float('nan')
      out[f'AJ_RD_dmin{d_min}'] = float('nan')
      continue
    per_d = []
    for d_thresh in dist_thresholds:
      v = raw['metrics_per_dist'][d_thresh]['aj_rd'][mask]
      v = v[~np.isnan(v)]
      per_d.append(torch.mean(torch.from_numpy(v)).item() if len(v) else float('nan'))
      out[f'AJ_RD_D{d_thresh}_dmin{d_min}'] = per_d[-1]
    out[f'AJ_RD_dmin{d_min}'] = float(np.nanmean(per_d)) if not np.all(np.isnan(per_d)) else float('nan')
  final = [out[f'AJ_RD_dmin{d}'] for d in d_min_thresholds]
  out['AJ_RD'] = float(np.nanmean(final)) if not np.all(np.isnan(final)) else float('nan')
  return out, raw
