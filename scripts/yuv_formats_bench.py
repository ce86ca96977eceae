"""Every YUV layout against uint8 RGB input, one JSON line per item; the first line names the card,
its power limit and its SM clocks.

  * get_feature_grids on 48 frames of 256^2, per layout: the layout's frames (conversion inside the
    stem conv's loads), the uint8 RGB frames, and yuv_to_rgb + the uint8 pass;
  * OnlineTracker step at 1280x720, centre-square crop, 256 points: P010 against NV12.
The variants alternate inside each round; each item reports the median and range over the rounds.
Usage: python scripts/yuv_formats_bench.py [--rounds R]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tapnet_b200 import synth  # noqa: E402  (seeded weights)
from tapnet_b200 import live, streaming, tapir_model  # noqa: E402

LAYOUTS = ['nv12', 'i420', 'p010', 'p016', 'yuv420p10', 'yuv420p12', 'yuv444', 'yuv444p16',
           'yuyv', 'uyvy']


def timeit(fn, n):
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(n):
    fn()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b) / n


def clip(layout, B, T, H, W, dev, **kw):
  """Random frames of `layout` (a zero clip whose buffers are filled with random bytes)."""
  f = live.YUVFrames.zeros(layout, B, T, H, W, dev, **kw)
  for b in f.buffers:
    b.view(torch.uint8).random_(0, 256)
  return f


def summary(ms):
  return dict(median=round(statistics.median(ms), 4), min=round(min(ms), 4), max=round(max(ms), 4))


def card():
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                      '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                     capture_output=True, text=True).stdout.strip()
  return dict(item='device', name_power_limit_sm_clock_max_sm_clock=q)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--rounds', type=int, default=5)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('yuv_formats_bench.py needs a CUDA device')
  print(json.dumps(card()))
  dev = torch.device('cuda')
  torch.manual_seed(0)

  model = tapir_model.TAPIR(pyramid_level=1)
  model.load_state_dict(synth.make_state_dict(0))
  model = model.to(dev).eval()
  for layout in LAYOUTS:
    frames = clip(layout, 1, 48, 256, 256, dev)
    rgb = live.yuv_to_rgb(frames)
    variants = {'fused': lambda: model.get_feature_grids(frames, False),
                'uint8_rgb': lambda: model.get_feature_grids(rgb, False),
                'convert_then_uint8': lambda: model.get_feature_grids(live.yuv_to_rgb(frames), False),
                'convert_kernel_alone': lambda: live.yuv_to_rgb(frames)}
    for fn in variants.values():  # warm-up: workspaces, packed weights
      fn()
    ms = {k: [] for k in variants}
    for _ in range(args.rounds):  # alternate the variants so drift hits all of them alike
      for k, fn in variants.items():
        ms[k].append(timeit(fn, 50 if k == 'convert_kernel_alone' else 5))
    print(json.dumps(dict(item=f'get_feature_grids 48x256^2 {layout}',
                          **{f'ms_{k}': summary(v) for k, v in ms.items()})))
    del frames, rgb
  del model

  causal = tapir_model.TAPIR(pyramid_level=1, use_casual_conv=True)
  causal.load_state_dict(synth.make_state_dict(0))
  causal = causal.to(dev).eval()
  H, W, N = 720, 1280, 256
  window = live.center_square_window(H, W)
  qp = torch.cat([torch.zeros(1, N, 1), torch.rand(1, N, 2) * window[2]], -1).to(dev)
  trackers = {}
  for layout in ('p010', 'nv12'):
    frames = clip(layout, 1, 1, H, W, dev, window=window)
    trk = streaming.OnlineTracker(causal, H, W, N, yuv_layout=layout, window=window)
    trk.init(frames, qp)
    trk.step(frames)
    trackers[layout] = (trk, frames)
  ms = {k: [] for k in trackers}
  for _ in range(args.rounds):
    for k, (trk, frames) in trackers.items():
      ms[k].append(timeit(lambda: trk.step(frames), 50))
  print(json.dumps(dict(item=f'OnlineTracker step 1280x720 centre crop, S=1, {N} points',
                        **{f'ms_{k}': summary(v) for k, v in ms.items()})))
  for trk, _ in trackers.values():
    trk.close()
  print(json.dumps(card()))


if __name__ == '__main__':
  main()
