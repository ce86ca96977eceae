"""Batched offline tracking: one model(video[B], queries[B]) call against the same B clips called
one at a time.  Default: 8 clips of 256x256x24, 64 queries each (non-causal TAPIR, pyramid level
1).  Rounds alternate between the two in this process; prints ms per call (median and every
round), launches per call, the largest output difference, and the GPU's name and power limit.
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

from tapnet_b200 import _lib  # noqa: E402
from tapnet_b200 import synth  # noqa: E402
from tapnet_b200 import tapir_model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--clips', type=int, default=8)
ap.add_argument('--frames', type=int, default=24)
ap.add_argument('--res', type=int, default=256)
ap.add_argument('--queries', type=int, default=64)
ap.add_argument('--rounds', type=int, default=7)
ap.add_argument('--warm', type=int, default=2)
a = ap.parse_args()

out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                      str(torch.cuda.current_device())], capture_output=True, text=True,
                     timeout=30).stdout.strip()
gpu, power_limit = [x.strip() for x in out.split(',')] if ',' in out else (torch.cuda.get_device_name(), 'unknown')

model = tapir_model.TAPIR(pyramid_level=1)
model.load_state_dict(synth.make_state_dict(0))
model = model.cuda().eval()
lib = _lib.load()
B, T, R, N = a.clips, a.frames, a.res, a.queries
video = torch.cat([synth.make_video(T, R, R, seed=1 + b) for b in range(B)]).cuda()
q = torch.cat([synth.make_queries(N, T, R, R, seed=2 + b) for b in range(B)]).cuda()


def batched():
  return model(video, q)


def one_at_a_time():
  return [model(video[b:b + 1], q[b:b + 1]) for b in range(B)]


def timed(fn):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  e0.record()
  fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1)


def launches(fn):
  torch.cuda.synchronize()
  l0 = lib.tapir_launch_count()
  fn()
  torch.cuda.synchronize()
  return int(lib.tapir_launch_count() - l0)


for _ in range(a.warm):
  batched()
  one_at_a_time()
ms_b, ms_s = [], []
for _ in range(a.rounds):
  ms_b.append(timed(batched))
  ms_s.append(timed(one_at_a_time))
both, ones = batched(), one_at_a_time()
diff = max(max((both[k][b] - ones[b][k][0]).abs().max().item() for b in range(B))
           for k in ('tracks', 'occlusion', 'expected_dist'))
mb, ms = statistics.median(ms_b), statistics.median(ms_s)
print(json.dumps(dict(
    workload=f'{B} clips of {R}x{R}x{T}, {N} queries each, TAPIR pyramid_level=1 bf16x3',
    ms_batched=round(mb, 3), ms_one_at_a_time=round(ms, 3), speedup=round(ms / mb, 3),
    ms_batched_rounds=[round(x, 3) for x in ms_b], ms_one_at_a_time_rounds=[round(x, 3) for x in ms_s],
    launches_batched=launches(batched), launches_one_at_a_time=launches(one_at_a_time),
    max_abs_diff=diff, gpu=gpu, power_limit=power_limit)))
