"""viz.paint_point_track on the GPU, one JSON line per item; the first line names the card, its
power limit and max SM clock.

For each workload (c2's output 48 x 256^2 with 256 points; a colab-sized clip 48 x 480 x 854 with
64 float64 tracks; 64 x 1024^2 with 8192 points; random tracks, 80 % visible):
  * kernels_ms: the two launches of tapir_paint_point_track on preallocated device buffers;
  * device_call_ms: viz.paint_point_track on CUDA tensors (what a caller holding the model's
    outputs pays: the call's allocations and the colour upload included);
  * numpy_call_ms: numpy in, numpy out (host-to-device and device-to-host copies included);
  * GB/s: frame bytes read + written over kernels_ms;
  * oracle_s: the numpy oracle (oracle/viz_oracle.py, one thread) on the first frames, scaled to
    the clip by the frame count (the reference's own function is slower still: it recopies the
    whole frame after every point).
GPU times are medians over 25 calls after 3 warm-up calls (CUDA events; the numpy path uses a host
clock around a call that ends in a device-to-host copy).
Usage: python scripts/viz_bench.py"""
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import viz_oracle  # noqa: E402
from tapnet_b200 import _lib, viz  # noqa: E402

WORKLOADS = [('c2 output 48x256^2, 256 points, fp32', 48, 256, 256, 256, np.float32),
             ('colab clip 48x480x854, 64 points, fp64', 48, 480, 854, 64, np.float64),
             ('64x1024^2, 8192 points, fp32', 64, 1024, 1024, 8192, np.float32)]
CALLS, WARM = 25, 3


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


def median_host_ms(fn, calls=CALLS):
  for _ in range(WARM):
    fn()
  times = []
  for _ in range(calls):
    t0 = time.perf_counter()
    fn()
    times.append((time.perf_counter() - t0) * 1e3)
  return statistics.median(times)


def workload(seed, T, H, W, N, dtype):
  rng = np.random.default_rng(seed)
  frames = rng.integers(0, 256, (T, H, W, 3), dtype=np.uint8)
  tracks = np.stack([rng.uniform(0, W, (N, T)), rng.uniform(0, H, (N, T))], -1).astype(dtype)
  vis = rng.uniform(size=(N, T)) < 0.8
  colors = rng.integers(0, 256, (N, 3), dtype=np.uint8)
  return frames, tracks, vis, colors


def main():
  if not torch.cuda.is_available():
    raise SystemExit('viz_bench.py needs a CUDA device')
  card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                         '--format=csv,noheader', '-i', '0'], capture_output=True, text=True).stdout
  print(json.dumps(dict(item='device', nvidia_smi=card.strip())), flush=True)
  dev = torch.device('cuda')
  lib = _lib.load()
  for k, (name, T, H, W, N, dtype) in enumerate(WORKLOADS):
    frames, tracks, vis, colors = workload(k, T, H, W, N, dtype)
    colormap = [tuple(c) for c in colors.tolist()]
    f_d = torch.from_numpy(frames).to(dev)
    t_d = torch.from_numpy(tracks).to(dev)
    v_d = torch.from_numpy(vis).to(dev)
    c_d = torch.from_numpy(colors).to(dev)
    out = torch.empty_like(f_d)
    ws_bytes = int(lib.tapir_paint_point_track_workspace_bytes(T, N))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    fp64 = int(dtype == np.float64)

    def kernels():
      _lib.check(lib.tapir_paint_point_track(f_d.data_ptr(), T, H, W, t_d.data_ptr(), fp64,
                                             v_d.data_ptr(), N, c_d.data_ptr(), out.data_ptr(),
                                             ws.data_ptr(), ws_bytes, stream), 'paint')

    kernels_ms = median_gpu_ms(kernels)
    device_ms = median_gpu_ms(lambda: viz.paint_point_track(f_d, t_d, v_d, colormap))
    numpy_ms = median_host_ms(lambda: viz.paint_point_track(frames, tracks, vis, colormap))
    painted = viz.paint_point_track(f_d, t_d, v_d, colormap)
    sample = 1 if N * T > 4096 else 4
    t0 = time.perf_counter()
    ref = viz_oracle.paint_point_track(frames[:sample], tracks[:, :sample], vis[:, :sample], colors)
    oracle_s = (time.perf_counter() - t0) * T / sample
    same = bool(np.array_equal(painted[:sample].cpu().numpy(), ref))
    frame_bytes = 2 * T * H * W * 3
    print(json.dumps(dict(item=name, kernels_ms=round(kernels_ms, 4), device_call_ms=round(device_ms, 4),
                          numpy_call_ms=round(numpy_ms, 2),
                          kernels_GBps=round(frame_bytes / kernels_ms / 1e6, 1),
                          oracle_s=round(oracle_s, 2), oracle_frames_timed=sample,
                          oracle_over_kernels=round(oracle_s * 1e3 / kernels_ms),
                          equal_to_oracle_on_timed_frames=same, radius=viz_oracle.radius(H, W))),
          flush=True)
    del f_d, t_d, v_d, c_d, out, ws, painted


if __name__ == '__main__':
  main()
