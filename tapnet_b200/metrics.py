"""TAP-Vid metrics on the device (SURVEY 8f row 2).

`compute_tapvid_metrics` has the signature and result keys of
`tapnet/tapvid/evaluation_datasets.py:48-192` (numpy in the reference).  Here the per-track
integer counters come from one kernel (`tapir_tapvid_counts`) over tensors that are already on
the GPU - typically the model's own outputs - and only the [B, N, 18] counters are reduced and
divided (float64, 0/0 -> nan as in numpy).  The visibility threshold of
`postprocess_occlusions` can be fused in by passing the two logit tensors instead of
`pred_occluded`.
"""
from typing import Mapping, Optional

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
