"""AJ_RD on the device: the tapir_redetection_events kernel (CUDA events over many launches), the
whole compute_redetection_metrics call (host clock around a call that ends in its copy to the
host) and the event count, for seeded Markov-visibility clips; the repository's numpy oracle on
the host at the smaller sizes.  Prints one JSON line per size, with the card's name and power
limit read in the same run.

    python scripts/redetection_bench.py [--sizes 1x300x256 1x1024x1024 1x2048x4096]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import redetection_oracle as R  # noqa: E402
from tapnet_b200 import _lib, metrics  # noqa: E402


def card():
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                     capture_output=True, text=True, check=False).stdout.strip().splitlines()
  return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def clip(B, T, N, seed=0):
  """[B, T, N] Markov visibility (stay visible 0.97, stay hidden 0.9), tracks with 2 px noise."""
  rng = np.random.default_rng(seed)
  gv = np.zeros((B, T, N), bool)
  gv[:, 0] = rng.uniform(size=(B, N)) < 0.7
  for t in range(1, T):
    stay = np.where(gv[:, t - 1], 0.97, 0.9)
    gv[:, t] = np.where(rng.uniform(size=(B, N)) < stay, gv[:, t - 1], ~gv[:, t - 1])
  gt = rng.uniform(0, 256, (B, T, N, 2)).astype(np.float32)
  pred = (gt + rng.normal(0, 2, gt.shape)).astype(np.float32)
  pv = np.where(rng.uniform(size=(B, T, N)) < 0.85, gv, ~gv)
  return pred, pv, gt, gv


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--sizes', nargs='*', default=['1x300x256', '1x1024x1024', '1x2048x4096'])
  p.add_argument('--launches', type=int, default=200)
  p.add_argument('--oracle-max-tracks-frames', type=int, default=1024 * 1024)
  a = p.parse_args()
  info = card()
  for size in a.sizes:
    B, T, N = (int(v) for v in size.split('x'))
    pred, pv, gt, gv = clip(B, T, N)
    d = [torch.from_numpy(x).cuda() for x in (pred, pv, gt, gv)]
    tm = [x.transpose(1, 2).contiguous() for x in d]   # track-major, as the model outputs them
    K, nd = _lib.redetection_max_events(T), len(metrics.DIST_THRESHOLDS)
    outs = [torch.empty(B, N, K, dtype=torch.int32, device='cuda'), torch.empty(B, N, K, dtype=torch.int32, device='cuda'),
            torch.empty(B, N, K, nd, device='cuda'), torch.empty(B, N, dtype=torch.int32, device='cuda')]
    gvu, pvu = tm[3].to(torch.uint8), tm[1].to(torch.uint8)

    def launch():
      _lib.redetection_events(gvu, pvu, tm[0], tm[2], metrics.DIST_THRESHOLDS, *outs)

    for _ in range(10):
      launch()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(a.launches):
      launch()
    stop.record()
    stop.synchronize()
    kernel_ms = start.elapsed_time(stop) / a.launches
    in_bytes = B * N * T * (1 + 1 + 8 + 8)

    for _ in range(3):
      m = metrics.compute_redetection_metrics(*d)
    torch.cuda.synchronize()
    reps = 10
    t0 = time.perf_counter()
    for _ in range(reps):
      m = metrics.compute_redetection_metrics(*d)
    call_ms = (time.perf_counter() - t0) / reps * 1e3
    events = len(m['raw_stats/durations']) if 'raw_stats/durations' in m else 0
    row = dict(B=B, T=T, N=N, card=info, events=events, kernel_ms=round(kernel_ms, 4),
               kernel_input_GBps=round(in_bytes / kernel_ms / 1e6, 1), metrics_call_ms=round(call_ms, 3),
               AJ_RD=float(m['AJ_RD']))
    if B * N * T <= a.oracle_max_tracks_frames:
      t0 = time.perf_counter()
      want, _ = R.metrics(pred, pv, gt, gv)
      row['oracle_host_s'] = round(time.perf_counter() - t0, 3)
      row['oracle_equal'] = all((np.isnan(v) and np.isnan(float(m[k]))) or v == float(m[k]) for k, v in want.items())
    print(json.dumps(row), flush=True)


if __name__ == '__main__':
  main()
