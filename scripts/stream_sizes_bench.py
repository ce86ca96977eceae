"""Streams of different frame sizes: one mixed-size OnlineTracker against one tracker per stream
stepped in turn, in ms per frame-set (one frame of every stream), rounds alternating between the
two in this process.  Prints one JSON line per mix, with the card's name and power limit read in
the same run.

Mixes: {240x320, 256^2, 256^2, the 480x480 centre window of a 480x640 camera} and an 8-stream
mix, float frames, --points points per stream.
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

MIXES = {
    'four': [(240, 320), (256, 256), (256, 256), (480, 480)],
    'eight': [(240, 320), (256, 256), (256, 256), (480, 480), (200, 200), (240, 240), (480, 480),
              (256, 256)],
}

ap = argparse.ArgumentParser()
ap.add_argument('--points', type=int, default=256)
ap.add_argument('--steps', type=int, default=50)
ap.add_argument('--rounds', type=int, default=5)
ap.add_argument('--mixes', type=str, default='four,eight')
a = ap.parse_args()


def gpu_info():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader',
                          '-i', str(torch.cuda.current_device())],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, limit = [x.strip() for x in out.split(',')]
  except Exception:  # pylint: disable=broad-except
    name, limit = torch.cuda.get_device_name(), 'unknown'
  return dict(gpu=name, power_limit=limit)


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
  info = gpu_info()
  N = a.points
  for name in a.mixes.split(','):
    sizes = MIXES[name]
    S = len(sizes)
    frames = [synth.make_video(1, h, w, seed=3 + s)[0, 0].cuda() for s, (h, w) in enumerate(sizes)]
    q = torch.stack([synth.make_queries(N, 1, h, w, seed=5 + s, frame0_only=True)[0]
                     for s, (h, w) in enumerate(sizes)]).cuda()
    mixed = streaming.OnlineTracker(model, [h for h, _ in sizes], [w for _, w in sizes], N,
                                    num_streams=S)
    mixed.init(frames, q)
    singles = [streaming.OnlineTracker(model, h, w, N) for h, w in sizes]
    for s, t in enumerate(singles):
      t.init(frames[s], q[s])

    def step_mixed():
      mixed.step(frames)

    def step_singles():
      for s, t in enumerate(singles):
        t.step(frames[s])

    for f in (step_mixed, step_singles):  # capture + warm-up
      for _ in range(3):
        f()
    torch.cuda.synchronize()
    ms_m, ms_s = [], []
    for _ in range(a.rounds):
      ms_m.append(time_steps(step_mixed, a.steps))
      ms_s.append(time_steps(step_singles, a.steps))
    groups = [[sizes[s] for s in g.streams] for g in mixed._groups]
    print(json.dumps(dict(
        mix=name, sizes=sizes, groups=groups, points=N,
        mixed_ms=round(statistics.median(ms_m), 3), mixed_ms_range=[round(min(ms_m), 3), round(max(ms_m), 3)],
        per_stream_ms=round(statistics.median(ms_s), 3),
        per_stream_ms_range=[round(min(ms_s), 3), round(max(ms_s), 3)],
        speedup=round(statistics.median(ms_s) / statistics.median(ms_m), 3), **info)))
    mixed.close()
    for t in singles:
      t.close()


if __name__ == '__main__':
  main()
