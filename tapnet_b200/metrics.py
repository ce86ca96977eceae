"""TAP-Vid metrics on the device (SURVEY 8f row 2).

`compute_tapvid_metrics` has the signature and result keys of
`tapnet/tapvid/evaluation_datasets.py:48-192` (numpy in the reference).  Here the per-track
integer counters come from one kernel (`tapir_tapvid_counts`) over tensors that are already on
the GPU - typically the model's own outputs - and only the [B, N, 18] counters are reduced and
divided (float64, 0/0 -> nan as in numpy).  The visibility threshold of
`postprocess_occlusions` can be fused in by passing the two logit tensors instead of
`pred_occluded`.

`compute_redetection_metrics` has the signature, defaults, key names and result types of
`tapnet/tapnextpp/metrics/aj_rd.py:209-308` (AJ_RD, the re-detection Average Jaccard).  One kernel
(`tapir_redetection_events`) finds every track's eligible reappearance events and their AJ_RD
values in one pass over the track; the events are put in the reference's (b, t_r, n) order on the
device and copied to the host once, where each mean is torch's own CPU mean over the same float32
values in the same order, so every result is bit for bit the reference's on the CPU.
"""
from typing import Mapping, Optional

import numpy as np
import torch

from tapnet_b200 import _lib

THRESHOLDS = (1, 2, 4, 8, 16)
_MODES = {'first': 0, 'strided': 1}


def _dev_tensor(x, dtype, dev):
  t = torch.as_tensor(x)
  if t.dtype == torch.bool and dtype == torch.uint8:
    t = t.to(torch.uint8)
  return t.to(device=dev, dtype=dtype).contiguous()


def tapvid_counts(query_points, gt_occluded, gt_tracks, pred_occluded, pred_tracks, query_mode,
                  pred_logits=None) -> torch.Tensor:
  """int32 [B, N, 18] counters (layout: include/tapir_b200.h).  `pred_logits` = (occlusion,
  expected_dist) logits replaces `pred_occluded` (pass None for it)."""
  if query_mode not in _MODES:
    raise ValueError('Unknown query mode ' + str(query_mode))
  pt = torch.as_tensor(pred_tracks)
  if pt.device.type != 'cuda':
    raise RuntimeError('tapvid_counts: pred_tracks must be on a CUDA device (no CPU fallback)')
  dev = pt.device
  pt = pt.to(torch.float32).contiguous()
  B, N, T = (int(v) for v in pt.shape[:3])
  qp = _dev_tensor(query_points, torch.float32, dev)
  go = _dev_tensor(gt_occluded, torch.uint8, dev)
  gt = _dev_tensor(gt_tracks, torch.float32, dev)
  po = logits = None
  if pred_logits is not None:
    logits = tuple(_dev_tensor(x, torch.float32, dev) for x in pred_logits[:2])
  else:
    po = _dev_tensor(pred_occluded, torch.uint8, dev)
  counts = torch.empty(B, N, _lib.TAPVID_COUNTERS, dtype=torch.int32, device=dev)
  with torch.cuda.device(dev):
    _lib.tapvid_counts(qp, go, gt, po, pt, _MODES[query_mode], counts, logits)
  return counts


def metrics_from_counts(counts: torch.Tensor, get_trackwise_metrics: bool = False
                        ) -> Mapping[str, torch.Tensor]:
  c = counts.to(torch.int64)
  if not get_trackwise_metrics:
    c = c.sum(dim=1)
  c = c.to(torch.float64)
  out = {'occlusion_accuracy': c[..., 1] / c[..., 0]}
  within, jac = [], []
  for i, thresh in enumerate(THRESHOLDS):
    w = c[..., 3 + i] / c[..., 2]
    j = c[..., 8 + i] / (c[..., 2] + c[..., 13 + i])
    out[f'pts_within_{thresh}'] = w
    out[f'jaccard_{thresh}'] = j
    within.append(w)
    jac.append(j)
  # numpy's mean over 5 values is a left-to-right sum divided by 5; same order here.  The
  # divisor is a tensor: torch's CUDA division by a Python scalar multiplies by the reciprocal
  # (1 ulp off the IEEE quotient numpy returns).
  five = torch.full_like(jac[0], 5.0)
  out['average_jaccard'] = ((((jac[0] + jac[1]) + jac[2]) + jac[3]) + jac[4]) / five
  out['average_pts_within_thresh'] = ((((within[0] + within[1]) + within[2]) + within[3])
                                      + within[4]) / five
  return out


def compute_tapvid_metrics(query_points, gt_occluded, gt_tracks, pred_occluded, pred_tracks,
                           query_mode: str, get_trackwise_metrics: bool = False,
                           pred_logits: Optional[tuple] = None) -> Mapping[str, torch.Tensor]:
  """Reference signature (evaluation_datasets.py:48-56) + optional fused `pred_logits`.
  Returns float64 CUDA tensors of shape [B] (or [B, N] trackwise)."""
  counts = tapvid_counts(query_points, gt_occluded, gt_tracks, pred_occluded, pred_tracks,
                         query_mode, pred_logits)
  return metrics_from_counts(counts, get_trackwise_metrics)


# ------------------------------------------------------------------------------ AJ_RD
DIST_THRESHOLDS = [1, 2, 4, 8, 16]
D_MIN_THRESHOLDS = [1, 4, 16, 64, 256]
_PACK_COLS = 4   # int32 columns of a packed event row: b, t_r, n, duration, then the values' bits


def redetection_events(pred_tracks, pred_visible, gt_tracks, gt_visible, dist_thresholds,
                       pred_logits=None) -> torch.Tensor:
  """Track-major inputs ([B, N, T, 2] tracks, [B, N, T] visibility, or `pred_logits` =
  (occlusion, expected_dist) logits in place of `pred_visible`) -> int32 [B N K(T), 4 + D] on the
  device: one row per event slot, (b, t_r, n, duration, the D float32 values' bits), the eligible
  events first in the reference's (b, t_r, n) order, then the unused slots (b = B, t_r = 0, zero
  duration and values).  Stream-ordered, no host sync."""
  pt = torch.as_tensor(pred_tracks)
  if pt.device.type != 'cuda':
    raise RuntimeError('redetection_events: pred_tracks must be on a CUDA device (no CPU fallback)')
  dev = pt.device
  pt = pt.to(torch.float32).contiguous()
  if pt.dim() != 4 or pt.shape[-1] != 2:
    raise ValueError(f'redetection_events: pred_tracks must be [B, N, T, 2], got {tuple(pt.shape)}')
  B, N, T = (int(v) for v in pt.shape[:3])
  gv = _dev_tensor(torch.as_tensor(gt_visible).bool(), torch.uint8, dev)
  gt = _dev_tensor(gt_tracks, torch.float32, dev)
  pv = logits = None
  if pred_logits is not None:
    logits = tuple(_dev_tensor(x, torch.float32, dev) for x in pred_logits[:2])
  else:
    pv = _dev_tensor(torch.as_tensor(pred_visible).bool(), torch.uint8, dev)
  K, nd = _lib.redetection_max_events(T), len(dist_thresholds)
  with torch.cuda.device(dev):
    ev_t = torch.empty(B, N, K, dtype=torch.int32, device=dev)
    ev_d = torch.empty(B, N, K, dtype=torch.int32, device=dev)
    ev_v = torch.empty(B, N, K, nd, dtype=torch.float32, device=dev)
    count = torch.empty(B, N, dtype=torch.int32, device=dev)
    _lib.redetection_events(gv, pv, pt, gt, dist_thresholds, ev_t, ev_d, ev_v, count, logits)
    # slots are in (b, n, k) order; a stable sort on b T + t_r gives torch.where's (b, t_r, n)
    used = torch.arange(K, device=dev) < count[..., None]
    b = torch.arange(B, device=dev, dtype=torch.int64)[:, None, None]
    key = torch.where(used, b * T + ev_t, B * T).reshape(-1)
    key, order = torch.sort(key, stable=True)
    n = torch.div(order, K, rounding_mode='floor') % N
    event = key < B * T   # the kernel leaves the unused slots unwritten: zero them
    rows = [torch.div(key, T, rounding_mode='floor'), key % T, n,
            torch.where(event, ev_d.reshape(-1)[order], 0)]
    values = torch.where(event[:, None], ev_v.reshape(-1, nd)[order], 0.0)
    return torch.cat([torch.stack(rows, 1).to(torch.int32), values.view(torch.int32)], 1)


def redetection_metrics_from_events(events, B, dist_thresholds=None, d_min_thresholds=None,
                                    events_device=None):
  """compute_redetection_metrics' dict from the host copy (numpy) of `redetection_events`' rows
  of B clips.  With `events_device` (the device rows themselves) the raw_stats/* entries are added
  as device tensors, as the reference returns them; without, only the scalars."""
  dist_thresholds = DIST_THRESHOLDS if dist_thresholds is None else dist_thresholds
  d_min_thresholds = D_MIN_THRESHOLDS if d_min_thresholds is None else d_min_thresholds
  events = np.asarray(events)
  E = int(np.searchsorted(events[:, 0], B))   # sorted by b; unused slots carry b = B
  metrics = {}
  if E == 0:
    for d_min in d_min_thresholds:
      for d_thresh in dist_thresholds:
        metrics[f'AJ_RD_D{d_thresh}_dmin{d_min}'] = float('nan')
      metrics[f'AJ_RD_dmin{d_min}'] = float('nan')
    metrics['AJ_RD'] = float('nan')
    return metrics
  durations = torch.from_numpy(np.ascontiguousarray(events[:E, 3]))
  values = [torch.from_numpy(np.ascontiguousarray(events[:E, _PACK_COLS + j]).view(np.float32))
            for j in range(len(dist_thresholds))]
  # aj_rd.py:258-292, on the CPU as the reference computes it there
  for d_min in d_min_thresholds:
    d_min_mask = durations >= d_min
    if torch.sum(d_min_mask).item() == 0:
      for d_thresh in dist_thresholds:
        metrics[f'AJ_RD_D{d_thresh}_dmin{d_min}'] = float('nan')
      metrics[f'AJ_RD_dmin{d_min}'] = float('nan')
      continue
    for d_thresh, aj_rd_d in zip(dist_thresholds, values):
      d_min_aj_rd_d = aj_rd_d[d_min_mask]
      valid = d_min_aj_rd_d[~torch.isnan(d_min_aj_rd_d)]
      metrics[f'AJ_RD_D{d_thresh}_dmin{d_min}'] = (torch.mean(valid).item() if len(valid) > 0
                                                   else float('nan'))
    per_d = [metrics[f'AJ_RD_D{d_thresh}_dmin{d_min}'] for d_thresh in dist_thresholds]
    metrics[f'AJ_RD_dmin{d_min}'] = (np.nanmean(per_d) if any(~np.isnan(v) for v in per_d)
                                     else float('nan'))
  if events_device is not None:
    rows = events_device[:E]
    metrics['raw_stats/indices'] = tuple(rows[:, c].to(torch.int64) for c in range(3))
    metrics['raw_stats/durations'] = rows[:, 3].contiguous()
    metrics['raw_stats/metrics_per_dist'] = {
        d_thresh: {'aj_rd': rows[:, _PACK_COLS + j].contiguous().view(torch.float32)}
        for j, d_thresh in enumerate(dist_thresholds)}
  final = [metrics[f'AJ_RD_dmin{d}'] for d in d_min_thresholds if f'AJ_RD_dmin{d}' in metrics]
  metrics['AJ_RD'] = np.nanmean(final) if any(~np.isnan(v) for v in final) else float('nan')
  return metrics


def redetection_metrics_tracks(pred_tracks, pred_visible, gt_tracks, gt_visible,
                               dist_thresholds=None, d_min_thresholds=None, pred_logits=None):
  """compute_redetection_metrics on track-major inputs: tracks [B, N, T, 2], visibility
  [B, N, T] (the model's own output layout), `pred_logits` = (occlusion, expected_dist) logits
  in place of `pred_visible` (thresholded as postprocess_occlusions does).  One host sync."""
  dist_thresholds = DIST_THRESHOLDS if dist_thresholds is None else dist_thresholds
  ev = redetection_events(pred_tracks, pred_visible, gt_tracks, gt_visible, dist_thresholds, pred_logits)
  return redetection_metrics_from_events(ev.cpu().numpy(), int(torch.as_tensor(pred_tracks).shape[0]),
                                         dist_thresholds, d_min_thresholds, events_device=ev)


def compute_redetection_metrics(pred_tracks, pred_visible, gt_tracks, gt_visible,
                                dist_thresholds=None, d_min_thresholds=None):
  """aj_rd.py:209-308 compute_redetection_metrics: tracks [B, T, N, 2] and visibility [B, T, N]
  (taken through .bool()), pred_tracks on a CUDA device, the tracks compared in float32.  Keys
  AJ_RD_D{D}_dmin{d}, AJ_RD_dmin{d} and AJ_RD (Python / numpy floats), and, when there is an
  event, raw_stats/indices ((b, t_r, n) int64), raw_stats/durations (int32) and
  raw_stats/metrics_per_dist ({D: {'aj_rd': float32}}) on the device.  Up to
  REDETECTION_MAX_THRESHOLDS (16) distance thresholds."""
  def track_major(x):
    return torch.as_tensor(x).transpose(1, 2)

  return redetection_metrics_tracks(track_major(pred_tracks), track_major(pred_visible).bool(),
                                    track_major(gt_tracks), track_major(gt_visible).bool(),
                                    dist_thresholds, d_min_thresholds)
