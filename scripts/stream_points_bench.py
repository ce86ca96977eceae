"""Camera streams with different point counts: one ragged OnlineTracker (each stream its own count)
against one tracker with every stream padded to the largest count and against one tracker per
stream stepped in turn.  256^2 float frames, counts (1024, 64 x 7) by default.  Reports ms per
frame-set (one frame of every stream) and point-frames/s of the useful points, rounds alternating
between the three in this process, with the card's name, power limit and SM clock read in the same
run.  Prints one JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from tapnet_b200 import streaming, synth, tapir_model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--counts', type=str, default='1024,64,64,64,64,64,64,64')
ap.add_argument('--size', type=int, default=256)
ap.add_argument('--steps', type=int, default=50)
ap.add_argument('--rounds', type=int, default=5)
a = ap.parse_args()


def gpu_info():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                          '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, limit, sm, sm_max = [x.strip() for x in out.split(',')]
  except Exception:  # pylint: disable=broad-except
    name, limit, sm, sm_max = torch.cuda.get_device_name(), 'unknown', 'unknown', 'unknown'
  return dict(gpu=name, power_limit=limit, sm_clock=sm, sm_clock_max=sm_max)


def time_steps(step, n):
  ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
  ev[0].record()
  for _ in range(n):
    step()
  ev[1].record()
  torch.cuda.synchronize()
  return ev[0].elapsed_time(ev[1]) / n


def main():
  sd = synth.make_state_dict(0)
  model = tapir_model.TAPIR(pyramid_level=1, use_casual_conv=True)
  model.load_state_dict(sd)
  model = model.cuda().eval()
  counts = [int(c) for c in a.counts.split(',')]
  S, H, top = len(counts), a.size, max(counts)
  frames = torch.stack([synth.make_video(1, H, H, seed=3 + s)[0, 0] for s in range(S)]).cuda()
  full = [synth.make_queries(top, 1, H, H, seed=5 + s, frame0_only=True)[0].cuda() for s in range(S)]
  ragged = streaming.OnlineTracker(model, H, H, counts, num_streams=S)
  ragged.init(frames, [q[:n] for q, n in zip(full, counts)])
  padded = streaming.OnlineTracker(model, H, H, top, num_streams=S)
  padded.init(frames, torch.stack(full))
  singles = [streaming.OnlineTracker(model, H, H, n) for n in counts]
  for s, t in enumerate(singles):
    t.init(frames[s], full[s][:counts[s]])

  def step_singles():
    for s, t in enumerate(singles):
      t.step(frames[s])

  runs = {'ragged': lambda: ragged.step(frames), 'padded': lambda: padded.step(frames),
          'per_stream': step_singles}
  for f in runs.values():  # capture + warm-up
    for _ in range(3):
      f()
  torch.cuda.synchronize()
  ms = {k: [] for k in runs}
  for _ in range(a.rounds):
    for k, f in runs.items():
      ms[k].append(time_steps(f, a.steps))
  useful = sum(counts)
  out = dict(size=H, counts=counts, useful_points=useful, padded_points=top * S)
  for k, v in ms.items():
    med = statistics.median(v)
    out[f'{k}_ms'] = round(med, 3)
    out[f'{k}_ms_range'] = [round(min(v), 3), round(max(v), 3)]
    out[f'{k}_point_frames_per_s'] = round(useful / med * 1e3)
  out['speedup_vs_padded'] = round(statistics.median(ms['padded']) / statistics.median(ms['ragged']), 3)
  out['speedup_vs_per_stream'] = round(statistics.median(ms['per_stream']) / statistics.median(ms['ragged']), 3)
  print(json.dumps(dict(**out, **gpu_info())))
  for t in [ragged, padded] + singles:
    t.close()


if __name__ == '__main__':
  main()
