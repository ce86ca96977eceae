"""TAP-Vid evaluation front end on the GPU against the reference's host path, one JSON line per
item; the first line names the card and its power limit (read in the same run).

  * resize: tapir_resize_lanczos_u8 on preallocated device buffers, DAVIS shape (50 x 480 x 854)
    and Kinetics shape (250 x 360 x 640) -> 256^2: kernel time per frame (CUDA events over 20
    calls after 3 warm-up calls), and bytes moved (source read, uint8 intermediate written and
    read, output written) over kernel time against the H100 SXM's 3.35 TB/s;
  * pil: PIL's Lanczos resize of one frame on this host (the reference's path), per frame;
  * evaluate: wall time of tapvid.evaluate over seeded datasets (2 DAVIS-shape videos of 50
    frames, 1 Kinetics-shape video of 250 JPEG frames; 20 tracks; a seeded random-weight TAPIR),
    with the GPU resize, and with the frames resized on the host by PIL and then uploaded.
Usage: python scripts/tapvid_bench.py"""
import io
import json
import os
import pickle
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tapnet_b200 import _lib, synth, tapir_model, tapvid  # noqa: E402

CALLS, WARM = 20, 3
HBM_BYTES_PER_S = 3.35e12


def card():
  q = 'name,power.limit'
  try:
    return subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), f'--query-gpu={q}',
                           '--format=csv,noheader'], capture_output=True, text=True, check=True).stdout.strip()
  except (OSError, subprocess.CalledProcessError):
    return f'{torch.cuda.get_device_name()} (nvidia-smi unavailable)'


def bench_resize(T, H, W, h=256, w=256):
  src = torch.randint(0, 256, (T, H, W, 3), dtype=torch.uint8, device='cuda')
  dst = torch.empty(T, h, w, 3, dtype=torch.uint8, device='cuda')
  xt, yt = tapvid._tables(W, w, src.device), tapvid._tables(H, h, src.device)  # pylint: disable=protected-access
  need = _lib.load().tapir_resize_lanczos_u8_workspace_bytes(T, H, W, h, w)
  ws = torch.empty(need, dtype=torch.uint8, device='cuda')
  for _ in range(WARM):
    _lib.resize_lanczos_u8(src, dst, xt, yt, ws)
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(CALLS):
    _lib.resize_lanczos_u8(src, dst, xt, yt, ws)
  e1.record()
  e1.synchronize()
  ms = e0.elapsed_time(e1) / CALLS
  moved = src.numel() + 2 * need + dst.numel()
  return dict(item='resize', shape=f'{T}x{H}x{W} -> {h}x{w}', kernel_ms=round(ms, 4),
              us_per_frame=round(ms * 1e3 / T, 3), bytes_moved=moved,
              GBps=round(moved / (ms * 1e-3) / 1e9, 1), share_of_hbm=round(moved / (ms * 1e-3) / HBM_BYTES_PER_S, 3))


def bench_pil(H, W, frames=20):
  img = np.random.default_rng(0).integers(0, 256, (H, W, 3), dtype=np.uint8)
  Image.fromarray(img).resize((256, 256), resample=Image.Resampling.LANCZOS)
  t = time.perf_counter()
  for _ in range(frames):
    Image.fromarray(img).resize((256, 256), resample=Image.Resampling.LANCZOS)
  return dict(item='pil', shape=f'{H}x{W} -> 256x256', ms_per_frame=round((time.perf_counter() - t) / frames * 1e3, 3),
              host_cpus=os.cpu_count())


def make_datasets(d):
  rng = np.random.default_rng(1)

  def tracks(T):
    return rng.uniform(0, 1, (20, T, 2)).astype(np.float32), rng.uniform(size=(20, T)) < 0.2

  def frames(T, H, W):
    y, x = np.mgrid[0:H, 0:W]
    base = np.stack([(x + y) % 256, (2 * x) % 256, (3 * y) % 256], -1)
    return ((base[None] + rng.integers(0, 30, (T, H, W, 3))) % 256).astype(np.uint8)

  davis = {}
  for name in ('a', 'b'):
    p, o = tracks(50)
    davis[name] = {'video': frames(50, 480, 854), 'points': p, 'occluded': o}
  with open(os.path.join(d, 'davis.pkl'), 'wb') as f:
    pickle.dump(davis, f)
  jpegs = []
  for fr in frames(250, 360, 640):
    b = io.BytesIO()
    Image.fromarray(fr).save(b, format='JPEG', quality=90)
    jpegs.append(b.getvalue())
  p, o = tracks(250)
  os.makedirs(os.path.join(d, 'kinetics'))
  with open(os.path.join(d, 'kinetics', '0000_of_0010.pkl'), 'wb') as f:
    pickle.dump([{'video': jpegs, 'points': p, 'occluded': o}], f)


def host_clip(frames, resolution, staging):
  """The reference's path: PIL Lanczos per frame on the host, then the upload."""
  frames = np.stack([np.asarray(Image.fromarray(f).resize((resolution[1], resolution[0]),
                                                           resample=Image.Resampling.LANCZOS)) for f in frames])
  return staging.to_device(frames)


def bench_evaluate(model, d):
  out = []
  gpu_clip = tapvid._clip  # pylint: disable=protected-access
  readers = {'davis': lambda: tapvid.create_davis_dataset(os.path.join(d, 'davis.pkl')),
             'kinetics': lambda: tapvid.create_kinetics_dataset(os.path.join(d, 'kinetics'))}
  for name, make in readers.items():
    tapvid.evaluate(model, make(), 'strided')   # warm-up (tables, workspaces, model)
    row = dict(item='evaluate', dataset=name)
    for arm, clip in (('gpu_resize_s', gpu_clip), ('host_pil_resize_s', host_clip)):
      tapvid._clip = clip  # pylint: disable=protected-access
      torch.cuda.synchronize()
      t = time.perf_counter()
      mean, _ = tapvid.evaluate(model, make(), 'strided')
      row[arm] = round(time.perf_counter() - t, 3)
      row[arm.replace('_s', '_aj')] = float(mean['average_jaccard'])
    tapvid._clip = gpu_clip  # pylint: disable=protected-access
    out.append(row)
  return out


def main():
  assert torch.cuda.is_available(), 'tapvid_bench measures the GPU path: no CUDA device'
  print(json.dumps(dict(item='card', card=card(), torch=torch.__version__)), flush=True)
  for shape in ((50, 480, 854), (250, 360, 640), (1, 2160, 3840)):
    print(json.dumps(bench_resize(*shape)), flush=True)
  for H, W in ((480, 854), (360, 640)):
    print(json.dumps(bench_pil(H, W)), flush=True)
  model = tapir_model.TAPIR()
  model.load_state_dict(synth.make_state_dict(0))
  model = model.cuda().eval()
  with tempfile.TemporaryDirectory() as d:
    make_datasets(d)
    for row in bench_evaluate(model, d):
      print(json.dumps(row), flush=True)


if __name__ == '__main__':
  main()
