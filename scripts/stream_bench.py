"""BASELINE config 3: causal/online BootsTAPIR, 256x256 streaming, N query points (live_demo path).

Per frame: get_feature_grids(1 frame) + estimate_trajectories(T=1, causal state in/out), exactly
the call pattern of tapnet/pytorch_live_demo.py:62-85.  Reports frames/s and point-frames/s.

--streams 1,2,4,8 instead compares, for each stream count S and each --stream-points value, one
S-stream OnlineTracker against S single-stream trackers stepped in turn (rounds alternate between
the two in this process): ms per frame-set (one frame of every stream), aggregate point-frames/s
and kernel launches per step.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from tapnet_b200 import synth  # noqa: E402
from tapnet_b200 import tapir_model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--frames', type=int, default=250)
ap.add_argument('--warm', type=int, default=10)
ap.add_argument('--queries', type=int, default=1024)
ap.add_argument('--streams', type=str, default='',
                help='comma-separated stream counts: multi-stream vs single-stream trackers')
ap.add_argument('--stream-points', type=str, default='8,256', help='points per stream')
ap.add_argument('--rounds', type=int, default=5, help='alternating timing rounds (--streams)')
a = ap.parse_args()
sd = synth.make_state_dict(0)
model = tapir_model.TAPIR(pyramid_level=1, use_casual_conv=True)
model.load_state_dict(sd)
model = model.cuda().eval()


def gpu_info():
  """Name and power limit of the GPU, read in the same run as the numbers."""
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader',
                          '-i', str(torch.cuda.current_device())],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, limit = [x.strip() for x in out.split(',')]
  except Exception:  # pylint: disable=broad-except
    name, limit = torch.cuda.get_device_name(), 'unknown'
  return dict(gpu=name, power_limit=limit)


def multi_stream_bench():
  from tapnet_b200 import _lib, streaming  # pylint: disable=g-import-not-at-top
  lib = _lib.load()
  info = gpu_info()
  print(json.dumps(dict(mode='gpu', **info)))
  streams = [int(x) for x in a.streams.split(',')]
  smax = max(streams)
  clips = torch.cat([synth.make_video(16, seed=1 + s) for s in range(smax)]).cuda()  # [S, 16, H, W, 3]
  for n in [int(x) for x in a.stream_points.split(',')]:
    q = torch.cat([synth.make_queries(n, 1, seed=2 + s, frame0_only=True) for s in range(smax)]).cuda()
    for S in streams:
      multi = streaming.OnlineTracker(model, 256, 256, n, num_streams=S)
      multi.init(clips[:S, 0], q[:S])
      singles = [streaming.OnlineTracker(model, 256, 256, n) for _ in range(S)]
      for s, trk in enumerate(singles):
        trk.init(clips[s, 0], q[s])

      def step_multi(t):
        multi.step(clips[:S, t % 16])

      def step_singles(t):
        for s, trk in enumerate(singles):
          trk.step(clips[s, t % 16])

      for _ in range(2):  # captures; a second pass re-captures any graph a later capture outdated
        for t in range(a.warm):
          step_multi(t)
          step_singles(t)

      def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for t in range(a.frames):
          fn(t)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.frames

      ms_multi, ms_single = [], []
      for _ in range(a.rounds):
        ms_multi.append(timed(step_multi))
        ms_single.append(timed(step_singles))

      def launches(trk):  # one eager step (a graph replay does not pass through the counter)
        trk._frame.copy_(clips[:trk.num_streams, :1])
        torch.cuda.synchronize()
        l0 = lib.tapir_launch_count()
        trk._step_eager()
        torch.cuda.synchronize()
        return int(lib.tapir_launch_count() - l0)

      l_multi, l_single = launches(multi), launches(singles[0]) * S
      for trk in [multi] + singles:
        trk.close()
      mm, ms = statistics.median(ms_multi), statistics.median(ms_single)
      print(json.dumps(dict(
          mode='multi-stream', streams=S, points_per_stream=n, frames=a.frames, rounds=a.rounds,
          ms_per_frame_set_multi=round(mm, 3), ms_per_frame_set_singles=round(ms, 3),
          ms_multi_rounds=[round(x, 3) for x in ms_multi],
          ms_singles_rounds=[round(x, 3) for x in ms_single],
          point_frames_per_s_multi=round(S * n * 1e3 / mm, 1),
          point_frames_per_s_singles=round(S * n * 1e3 / ms, 1),
          speedup=round(ms / mm, 3), launches_per_step_multi=l_multi,
          launches_per_step_singles=l_single, **info)), flush=True)


if a.streams:
  multi_stream_bench()
  sys.exit(0)
clip = synth.make_video(16).cuda()  # frames are cycled; content does not affect timing
q = synth.make_queries(a.queries, 1, frame0_only=True).cuda()
g0 = model.get_feature_grids(clip[:, :1], False)
qf = model.get_query_features(clip[:, :1], False, q, g0)
state = model.construct_initial_causal_state(a.queries, len(qf.resolutions) - 1)
state = [{k: v.cuda() for k, v in d.items()} for d in state]


def step(t, state):
  frame = clip[:, t % 16:t % 16 + 1]
  grids = model.get_feature_grids(frame, False)
  r = model.estimate_trajectories((256, 256), False, grids, qf, None, 64, causal_context=state,
                                  get_causal_context=True)
  vis = (1 - torch.sigmoid(r['occlusion'][-1])) * (1 - torch.sigmoid(r['expected_dist'][-1])) > 0.5
  return r['tracks'][-1], vis, r['causal_context']


for t in range(a.warm):
  _, _, state = step(t, state)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
t0 = time.perf_counter()
e0.record()
for t in range(a.frames):
  tracks, vis, state = step(a.warm + t, state)
e1.record()
torch.cuda.synchronize()
wall = time.perf_counter() - t0
ms = e0.elapsed_time(e1)
eager = dict(config='causal BootsTAPIR streaming 256x256', frames=a.frames, queries=a.queries,
                      ms_per_frame_device=round(ms / a.frames, 3), ms_per_frame_wall=round(wall * 1e3 / a.frames, 3),
                      frames_per_s=round(a.frames / wall, 1),
                      point_frames_per_s=round(a.frames * a.queries / wall, 1),
                      finite=bool(torch.isfinite(tracks).all()))
print(json.dumps(dict(mode='eager', **eager)))

# per-kernel-class device time of the eager step (CUDA events around every launch)
import ctypes  # noqa: E402
from tapnet_b200 import _lib  # noqa: E402
lib = _lib.load()
lib.tapir_profile_enable(1)
for t in range(4):
  _, _, state = step(t, state)
buf = ctypes.create_string_buffer(1 << 16)
if lib.tapir_profile_report(buf, len(buf)) == 0:
  prof = json.loads(buf.value.decode())
  tot = sum(v['ms'] for v in prof.values())
  print('per-frame kernel time by class (ms), total %.3f:' % (tot / 4))
  for k, v in sorted(prof.items(), key=lambda kv: -kv[1]['ms']):
    print('  %-26s %7.3f ms  %4d launches  avg %6.1f us' % (k, v['ms'] / 4, v['launches'] // 4, v['ms'] / v['launches'] * 1e3))
lib.tapir_profile_enable(0)

# CUDA-graph replay of the same per-frame step
from tapnet_b200 import streaming  # noqa: E402

trk = streaming.OnlineTracker(model, 256, 256, a.queries)
trk.init(clip[0, 0], q)
for t in range(a.warm):
  trk.step(clip[0, t % 16])
torch.cuda.synchronize()
t0 = time.perf_counter()
e0.record()
for t in range(a.frames):
  tracks, vis = trk.step(clip[0, (a.warm + t) % 16])
e1.record()
torch.cuda.synchronize()
wall = time.perf_counter() - t0
ms = e0.elapsed_time(e1)
print(json.dumps(dict(mode='cuda-graph', config='causal BootsTAPIR streaming 256x256', frames=a.frames,
                      queries=a.queries, ms_per_frame_device=round(ms / a.frames, 3),
                      ms_per_frame_wall=round(wall * 1e3 / a.frames, 3), frames_per_s=round(a.frames / wall, 1),
                      point_frames_per_s=round(a.frames * a.queries / wall, 1),
                      finite=bool(torch.isfinite(tracks).all()))))

