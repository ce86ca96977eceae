"""Point edits of an OnlineTracker inside its graph-replayed step.  For each configuration:

- click step: `retarget` + `step` against `update_query(frame)` + `step` on the same frame (the
  reference live demo's click path: a one-frame backbone pass for the new point, then the step);
- plain step: a tracker that has been edited (one extra launch per group, with no request) against
  one that never was;
- re-capture: the first step after `add_points` of one point (re-pack, capture, replay).

Configurations: one 256^2 uint8 stream of 1024 points; one 1280x720 NV12 stream tracked in its
centre 720^2 window, 1024 points; eight 256^2 float streams of (1024, 64 x 7) points, the click on
the 1024-point stream.  Rounds alternate between the arms in this process; each arm reports the
median and range of its rounds.  Prints one JSON line per configuration with the card's name,
power limit and SM clocks read in the same run.
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

from tapnet_b200 import live, streaming, synth, tapir_model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--steps', type=int, default=30)
ap.add_argument('--rounds', type=int, default=5)
ap.add_argument('--configs', type=str, default='s1_uint8,nv12_720p,rig8')
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
  torch.cuda.synchronize()
  ev[0].record()
  for i in range(n):
    step(i)
  ev[1].record()
  torch.cuda.synchronize()
  return ev[0].elapsed_time(ev[1]) / n


def config(name):
  """(tracker kwargs, frames, query points, stream clicked, its (h, w), its point count)."""
  if name == 's1_uint8':
    f = synth.make_video(1, 256, 256, seed=3)[0, 0]
    frames = ((f + 1) * 127.5).round().clamp(0, 255).to(torch.uint8).cuda()
    q = synth.make_queries(1024, 1, 256, 256, seed=5, frame0_only=True)[0].cuda()
    return dict(height=256, width=256, num_points=1024, uint8_frames=True), frames, q, 0, (256, 256), 1024
  if name == 'nv12_720p':
    H, W = 720, 1280
    g = torch.Generator().manual_seed(7)
    y = torch.randint(16, 236, (1, 1, H, W), generator=g, dtype=torch.uint8).cuda()
    uv = torch.randint(16, 241, (1, 1, H // 2, W // 2, 2), generator=g, dtype=torch.uint8).cuda()
    win = live.center_square_window(H, W)
    frames = live.YUV420Frames.nv12(y, uv, window=win)
    q = synth.make_queries(1024, 1, win[2], win[3], seed=5, frame0_only=True)[0].cuda()
    return (dict(height=H, width=W, num_points=1024, yuv420=True, window=win), frames, q, 0,
            (win[2], win[3]), 1024)
  if name == 'rig8':
    counts = [1024] + [64] * 7
    frames = torch.stack([synth.make_video(1, 256, 256, seed=3 + s)[0, 0] for s in range(8)]).cuda()
    q = [synth.make_queries(n, 1, 256, 256, seed=5 + s, frame0_only=True)[0].cuda()
         for s, n in enumerate(counts)]
    return dict(height=256, width=256, num_points=counts, num_streams=8), frames, q, 0, (256, 256), 1024
  raise ValueError(name)


def run(name, model):
  kw, frames, q, stream, (h, w), n = config(name)
  one = (frames if isinstance(frames, live.YUV420Frames) or frames.dim() == 3 else frames[stream])
  trk = {k: streaming.OnlineTracker(model, **kw) for k in ('retarget', 'update_query', 'never_edited')}
  for t in trk.values():
    t.init(frames, q)
  g = torch.Generator().manual_seed(11)
  pts = torch.cat([torch.zeros(64, 1), torch.rand(64, 1, generator=g) * h,
                   torch.rand(64, 1, generator=g) * w], 1)

  def click_retarget(i):
    trk['retarget'].retarget(pts[i % 64][None], [i % n], stream=stream)
    trk['retarget'].step(frames)

  def click_update_query(i):
    trk['update_query'].update_query(one, pts[i % 64].cuda(), i % n, stream=stream)
    trk['update_query'].step(frames)

  arms = {'click_retarget': click_retarget, 'click_update_query': click_update_query,
          'plain_edited': lambda i: trk['retarget'].step(frames),
          'plain_never_edited': lambda i: trk['never_edited'].step(frames)}
  for f in arms.values():  # capture + warm-up
    for i in range(3):
      f(i)
  ms = {k: [] for k in arms}
  for _ in range(a.rounds):
    for k, f in arms.items():
      ms[k].append(time_steps(f, a.steps))
  # re-capture: add one point, then the first step (re-pack, capture, replay), host clock
  rec = trk['never_edited']
  recapture = []
  for i in range(3):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rec.add_points(pts[i][None], stream=stream)
    rec.step(frames)
    torch.cuda.synchronize()
    recapture.append((time.perf_counter() - t0) * 1e3)
  out = dict(config=name, clicked_stream_points=n, steps=a.steps, rounds=a.rounds)
  for k, v in ms.items():
    out[f'{k}_ms'] = round(statistics.median(v), 3)
    out[f'{k}_ms_range'] = [round(min(v), 3), round(max(v), 3)]
  out['click_saving_ms'] = round(out['click_update_query_ms'] - out['click_retarget_ms'], 3)
  out['edited_plain_step_extra_ms'] = round(out['plain_edited_ms'] - out['plain_never_edited_ms'], 3)
  out['recapture_step_ms'] = round(statistics.median(recapture), 1)
  out['recapture_step_ms_range'] = [round(min(recapture), 1), round(max(recapture), 1)]
  print(json.dumps(dict(**out, **gpu_info())), flush=True)
  for t in trk.values():
    t.close()


def main():
  sd = synth.make_state_dict(0)
  model = tapir_model.TAPIR(pyramid_level=1, use_casual_conv=True)
  model.load_state_dict(sd)
  model = model.cuda().eval()
  for name in a.configs.split(','):
    run(name, model)


if __name__ == '__main__':
  main()
