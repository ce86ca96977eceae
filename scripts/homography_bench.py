"""viz.get_homographies_wrt_frame on the GPU, one JSON line per item; the first line names the
card, its power limit and max SM clock.

Workloads: panning clips (oracle/make_golden_homography.panning_clip: planar background, 20 %
independent foreground tracks, 10 % occlusion) of (T, N) = (50, 1024) (the rainbow demo's clip at
stride 8), (200, 4096) and (1000, 4096); and the demo end to end: the model on 50 x 256^2 with a
stride-8 query grid (1024 points), then the homographies, then foreground_tracks.
  * gpu_ms: the whole call on CUDA tensors (CUDA events), median of 5 calls after 1 warm-up;
  * launches: kernels per call (tapir_launch_count);
  * oracle_s: oracle/homography_oracle.py (numpy float64, one process) on the same input, one run
    (skipped above T = 200, where it takes minutes).
Usage: python scripts/homography_bench.py"""
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import homography_oracle as H  # noqa: E402
from oracle import synth  # noqa: E402
from oracle.make_golden_homography import panning_clip  # noqa: E402
from tapnet_b200 import _lib, tapir_model, viz  # noqa: E402

CALLS, WARM = 5, 1


def median_gpu_ms(fn):
  for _ in range(WARM):
    fn()
  times = []
  for _ in range(CALLS):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    times.append(a.elapsed_time(b))
  return statistics.median(times)


def main():
  if not torch.cuda.is_available():
    raise SystemExit('homography_bench.py needs a CUDA device')
  card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                         '--format=csv,noheader', '-i', '0'], capture_output=True, text=True).stdout
  print(json.dumps(dict(item='device', nvidia_smi=card.strip())), flush=True)
  lib = _lib.load()
  for T, N in ((50, 1024), (200, 4096), (1000, 4096)):
    pts, occ = panning_clip(np.random.default_rng(T + N), T, N, W=256, H_=256)
    p, o = torch.from_numpy(pts).cuda(), torch.from_numpy(occ).cuda()
    n0 = lib.tapir_launch_count()
    viz.get_homographies_wrt_frame(p, o, (256, 256))
    launches = lib.tapir_launch_count() - n0
    ms = median_gpu_ms(lambda: viz.get_homographies_wrt_frame(p, o, (256, 256)))
    oracle_s = None
    if T <= 200:
      t0 = time.perf_counter()
      with np.errstate(divide='ignore', invalid='ignore'):
        H.homographies_wrt_frame(pts, occ, (256, 256))
      oracle_s = round(time.perf_counter() - t0, 3)
    print(json.dumps(dict(item=f'homographies T={T} N={N}', gpu_ms=round(ms, 3), launches=int(launches),
                          oracle_s=oracle_s)), flush=True)
  # the rainbow demo end to end: model, homographies, foreground
  sd = synth.make_state_dict(0)
  model = tapir_model.TAPIR(pyramid_level=1)
  model.load_state_dict(sd)
  model = model.cuda().eval()
  T = 50
  video = synth.make_video(T).cuda()
  g = (np.arange(32) * 8 + 4).astype(np.float32)
  yy, xx = np.meshgrid(g, g, indexing='ij')
  q = torch.from_numpy(np.stack([np.zeros(1024, np.float32), yy.ravel(), xx.ravel()], -1))[None].cuda()

  def demo():
    with torch.no_grad():
      out = model(video, q)
    tracks, occ = out['tracks'][0], out['occlusion'][0]
    vis = occ < occ.median()   # seeded random weights: cut the occlusion logits at their median
    _, err, _ = viz.get_homographies_wrt_frame(tracks, ~vis, (256, 256))
    return viz.foreground_tracks(err, vis)

  def model_only():
    with torch.no_grad():
      model(video, q)

  print(json.dumps(dict(item='demo 50x256^2 stride-8 grid (1024 points): model + homographies + foreground',
                        gpu_ms=round(median_gpu_ms(demo), 3), model_only_ms=round(median_gpu_ms(model_only), 3))),
        flush=True)


if __name__ == '__main__':
  main()
