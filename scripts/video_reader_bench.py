"""windowed.track_video against windowed_forward: one JSON line per configuration.

  1024      a 1024 x 1024 uint8 clip of --frames-1024 frames in pinned host memory: track_video
            reading it window by window against windowed_forward on the same clip, at the same
            core length; ms per frame (medians of --reps alternated runs), peak allocated device
            bytes, the host-to-device bytes each one copies (counted from the calls), and whether
            the outputs are torch.equal.
  1080p     a 1920 x 1080 NV12 video of --frames-1080p frames on the device, --points-1080p points,
            automatic core length: ms per frame and peak allocated bytes; whether windowed_forward
            would fit at all (from its byte model: its full-length outputs next to its sweep).

Every line carries the card's name, power limit and max SM clock, read in the same run.  Random
weights (tapnet_b200.synth), random query points.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tapnet_b200 import live, synth, tapir_model, windowed  # noqa: E402
from scripts.long_video_bench import gpu_info, make_video, queries  # noqa: E402


def peak_run(fn):
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  base = torch.cuda.memory_allocated()
  t0 = time.perf_counter()
  out = fn()
  torch.cuda.synchronize()
  return out, (time.perf_counter() - t0) * 1e3, torch.cuda.max_memory_allocated() - base


def reader_run(model, read, T, q, **kw):
  """track_video's windows concatenated on the host, as a caller keeping the tracks would."""
  parts = [{k: v.cpu() for k, v in out.items()}
           for _, _, out in windowed.track_video(model, read, T, q, **kw)]
  return {k: torch.cat([p[k] for p in parts], dim=2) for k in parts[0]}


def config_1024(model, args, info):
  T, H, W, C = args.frames_1024, 1024, 1024, args.core_1024
  host = make_video(T, H, W, 'cuda', out=torch.empty(1, T, H, W, 3, dtype=torch.uint8).pin_memory())
  q = queries(args.points, T, H, W, 'cuda')
  copied = {'reader': 0, 'windowed': 0}

  def read(a, z):
    copied['reader'] += (z - a) * H * W * 3
    return host[0, a:z]

  run_pass = windowed._run_pass

  def counting_pass(model_, pk, video, step, a, z, out, dev):
    if video.device.type == 'cpu':
      copied['windowed'] += (z - a) * H * W * 3
    return run_pass(model_, pk, video, step, a, z, out, dev)
  windowed._run_pass = counting_pass
  runs = {'reader': lambda: reader_run(model, read, T, q, window_frames=C),
          'windowed': lambda: {k: v.cpu() for k, v in windowed.windowed_forward(
              model, host, q.cpu(), window_frames=C).items() if not k.startswith('unrefined')}}
  ms = {k: [] for k in runs}
  peak, outs = {}, {}
  for rep in range(args.reps + 1):  # the first round warms up
    for k, fn in runs.items():
      copied[k] = 0
      outs[k], t, peak[k] = peak_run(fn)
      if rep:
        ms[k].append(t)
  windowed._run_pass = run_pass
  med = {k: statistics.median(v) for k, v in ms.items()}
  print(json.dumps(dict(
      config='1024', frames=T, size=[H, W], points=args.points, window_frames=C,
      reader='pinned host uint8', **info,
      ms_per_frame={k: round(v / T, 3) for k, v in med.items()},
      peak_allocated_bytes=peak, h2d_bytes=dict(copied), clip_bytes=T * H * W * 3,
      torch_equal=all(torch.equal(outs['reader'][k], outs['windowed'][k]) for k in outs['reader']))),
      flush=True)


def config_1080p(model, args, info):
  T, H, W, N = args.frames_1080p, 1080, 1920, args.points_1080p
  g = torch.Generator(device='cuda').manual_seed(3)
  frame_y = torch.randint(0, 256, (1, 16, H, W), generator=g, device='cuda', dtype=torch.uint8)
  frame_uv = torch.randint(0, 256, (1, 16, H // 2, W // 2, 2), generator=g, device='cuda',
                           dtype=torch.uint8)

  def read(a, z):  # a decoder's NV12 surfaces: 16 distinct frames, cycled
    idx = torch.arange(a, z, device='cuda') % 16
    return live.YUV420Frames.nv12(frame_y[:, idx], frame_uv[:, idx], matrix='bt709')
  q = queries(N, T, H, W, 'cuda')
  free = windowed._free_device_bytes(torch.device('cuda'))
  shape = (1, T, H, W)
  try:
    windowed.choose_window_frames(model, shape, N, free)
    fits = True
  except ValueError:
    fits = False
  C = windowed.choose_reader_window_frames(model, shape, N, free, frame_bytes=H * W * 3 // 2)

  def run():
    for _ in windowed.track_video(model, read, T, q):
      pass
  _, ms, peak = peak_run(run)
  print(json.dumps(dict(
      config='1080p', frames=T, size=[H, W], points=N, reader='device NV12', **info,
      window_frames=C, ms_per_frame=round(ms / T, 3), peak_allocated_bytes=peak,
      windowed_forward_output_bytes=windowed.output_bytes(model, shape, N),
      windowed_forward_fits=fits)), flush=True)


def main():
  p = argparse.ArgumentParser(description=__doc__.split('\n')[0])
  p.add_argument('--configs', default='1024,1080p')
  p.add_argument('--frames-1024', type=int, default=256)
  p.add_argument('--core-1024', type=int, default=128)
  p.add_argument('--points', type=int, default=256)
  p.add_argument('--frames-1080p', type=int, default=8000)
  p.add_argument('--points-1080p', type=int, default=8192)
  p.add_argument('--reps', type=int, default=2)
  args = p.parse_args()
  info = gpu_info()
  model = tapir_model.TAPIR()
  model.load_state_dict(synth.make_state_dict(0, 1, True))
  model = model.cuda().eval()
  with torch.no_grad():
    for c in args.configs.split(','):
      {'1024': config_1024, '1080p': config_1080p}[c](model, args, info)


if __name__ == '__main__':
  main()
