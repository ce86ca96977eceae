"""Windowed offline tracking (tapnet_b200.windowed) on long clips: one JSON line per configuration.

  fits      a clip whole-clip tracking can hold: model(video, queries) against windowed_forward at
            two core lengths, alternated, median of `--reps`; peak allocated bytes of each and
            whether every output is torch.equal to the whole-clip call's.
  long      a pinned uint8 host clip whose grids do not fit the card whole (the whole-clip call is
            not run): windowed with the automatic core length; ms per frame, peak allocated bytes,
            the chosen core, the query pre-pass time on its own, and the refinement work the halos
            add per level, sum over windows of the level's frame range over the core frames.

Every line carries the card's name, power limit and max SM clock, read in the same run.
Random weights (tapnet_b200.synth), random query points.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tapnet_b200 import synth, tapir_model, windowed  # noqa: E402


def gpu_info():
  out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                        '--format=csv,noheader', '-i', '0'], capture_output=True, text=True,
                       check=True).stdout.strip().split(', ')
  return dict(gpu=out[0], power_limit=out[1], max_sm_clock=out[2])


def make_video(T, H, W, dev, out=None, seed=0):
  """uint8 [1, T, H, W, 3]: a smooth texture drifting across the frame plus noise, made on the GPU
  64 frames at a time and written into `out` (which may be a pinned host tensor)."""
  g = torch.Generator(device=dev).manual_seed(seed)
  base = torch.rand(1, 3, H // 8 + 10, W // 8 + 10, generator=g, device=dev) * 255
  base = torch.nn.functional.interpolate(base, scale_factor=8, mode='bilinear', align_corners=False)
  base = base[0].permute(1, 2, 0)
  if out is None:
    out = torch.empty(1, T, H, W, 3, dtype=torch.uint8, device=dev)
  for t0 in range(0, T, 64):
    frames = torch.stack([base[(t * 2) % 71:(t * 2) % 71 + H, (t * 3) % 73:(t * 3) % 73 + W]
                          for t in range(t0, min(T, t0 + 64))])
    noise = torch.rand(frames.shape, generator=g, device=dev) * 24
    out[0, t0:t0 + frames.shape[0]].copy_((frames * 0.9 + noise).clamp(0, 255).to(torch.uint8))
  return out


def queries(N, T, H, W, dev, seed=1):
  g = torch.Generator().manual_seed(seed)
  t = torch.randint(0, T, (1, N, 1), generator=g).float()
  yx = torch.rand(1, N, 2, generator=g) * torch.tensor([H - 1.0, W - 1.0])
  return torch.cat([t, yx], -1).to(dev)


def timed(fn):
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  base = torch.cuda.memory_allocated()
  t0 = time.perf_counter()
  out = fn()
  torch.cuda.synchronize()
  return out, (time.perf_counter() - t0) * 1e3, torch.cuda.max_memory_allocated() - base


def all_equal(a, b):
  return all(torch.equal(x, y) for k in b
             for x, y in (zip(a[k], b[k]) if isinstance(b[k], list) else [(a[k], b[k])]))


def halo_work(model, T, hw, C):
  """Per refinement level: frames refined over frames output, sum over windows."""
  plan = tapir_model._pass_plan(hw, model.initial_resolution)
  wins = windowed.window_plan(T, C, windowed.halo_frames(model, hw), plan)
  return [round(sum(w.levels[l][1] - w.levels[l][0] for w in wins) / T, 3)
          for l in range(len(plan) - 1)]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--size', type=int, default=1024)
  ap.add_argument('--fit-frames', type=int, default=200)
  ap.add_argument('--cores', type=int, nargs=2, default=(64, 128))
  ap.add_argument('--long-frames', type=int, default=2000)
  ap.add_argument('--points', type=int, default=256)
  ap.add_argument('--reps', type=int, default=3)
  args = ap.parse_args()
  dev = torch.device('cuda:0')
  torch.cuda.set_device(dev)
  info = gpu_info()
  model = tapir_model.TAPIR(pyramid_level=1)
  model.load_state_dict(synth.make_state_dict(0))
  model = model.to(dev).eval()
  S, N = args.size, args.points

  # ---- a clip that fits whole
  T = args.fit_frames
  video, q = make_video(T, S, S, dev), queries(N, T, S, S, dev)
  runs = {'whole': lambda: model(video, q)}
  for c in args.cores:
    runs[f'windowed_C{c}'] = lambda c=c: windowed.windowed_forward(model, video, q, window_frames=c)
  with torch.no_grad():
    ref = model(video, q)  # warm-up (and the reference outputs)
    for fn in runs.values():
      fn()
    ms = {k: [] for k in runs}
    peak, equal = {}, {}
    for _ in range(args.reps):
      for k, fn in runs.items():
        out, t, p = timed(fn)
        ms[k].append(t)
        peak[k] = p
        equal[k] = all_equal(out, ref)
        del out
  print(json.dumps(dict(config='fits', frames=T, size=[S, S], points=N, **info,
                        ms={k: round(statistics.median(v), 1) for k, v in ms.items()},
                        ms_per_frame={k: round(statistics.median(v) / T, 3) for k, v in ms.items()},
                        peak_allocated_bytes=peak, torch_equal=equal,
                        halo_work={f'C{c}': halo_work(model, T, (S, S), c) for c in args.cores})),
        flush=True)
  del video, q, ref

  # ---- a clip whose grids do not fit whole: a pinned uint8 host clip
  T = args.long_frames
  host = torch.empty(1, T, S, S, 3, dtype=torch.uint8, pin_memory=True)
  make_video(T, S, S, dev, out=host, seed=3)
  q = queries(N, T, S, S, dev, seed=4)
  shape = (1, T, S, S)
  C = windowed.choose_window_frames(model, shape, N, windowed._free_device_bytes(dev), None, True, 1)
  plan = tapir_model._pass_plan((S, S), model.initial_resolution)
  grids_whole = sum(st.h * st.w * 48 for st in plan if st.new) * T
  with torch.no_grad():
    _, pre_ms, _ = timed(lambda: windowed._query_features(model, model._pack(), host, 0, 1, q[0], plan, 64, dev))
    out, total_ms, p = timed(lambda: windowed.windowed_forward(model, host, q, window_frames=C))
  finite = bool(torch.isfinite(out['tracks']).all())
  print(json.dumps(dict(config='long', frames=T, size=[S, S], points=N, host_pinned_uint8=True,
                        **info, window_frames=C, whole_clip_grid_bytes=grids_whole,
                        ms=round(total_ms, 1), ms_per_frame=round(total_ms / T, 3),
                        prepass_ms=round(pre_ms, 1), peak_allocated_bytes=p,
                        halo_work=halo_work(model, T, (S, S), C), tracks_finite=finite)), flush=True)


if __name__ == '__main__':
  main()
