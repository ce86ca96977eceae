"""YUV 4:2:0 input against uint8 RGB input, one JSON line per item; the first line names the card,
its power limit and max SM clock.

  * backbone pass (get_feature_grids) on 48 frames of 256^2: NV12 frames (conversion inside the
    stem conv's loads), uint8 RGB frames, and a separate conversion kernel + the uint8 pass;
  * OnlineTracker step at 1280x720 NV12, centre-square crop, S = 1 and 8 streams, 256 points:
    the yuv420 tracker against a uint8 tracker fed by a conversion done outside it.
Usage: python scripts/yuv_bench.py"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tapnet_b200 import synth  # noqa: E402  (seeded weights)
from tapnet_b200 import live, streaming, tapir_model  # noqa: E402


def timeit(fn, n=20, warm=3):
  for _ in range(warm):
    fn()
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(n):
    fn()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b) / n


def nv12(B, T, H, W, g, dev):
  y = torch.randint(16, 236, (B, T, H, W), generator=g, dtype=torch.uint8).to(dev)
  uv = torch.randint(16, 241, (B, T, H // 2, W // 2, 2), generator=g, dtype=torch.uint8).to(dev)
  return y, uv


def main():
  if not torch.cuda.is_available():
    raise SystemExit('yuv_bench.py needs a CUDA device')
  card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                         '--format=csv,noheader', '-i', '0'], capture_output=True, text=True).stdout
  print(json.dumps(dict(item='device', nvidia_smi=card.strip())))
  dev = torch.device('cuda')
  g = torch.Generator().manual_seed(0)

  model = tapir_model.TAPIR(pyramid_level=1)
  model.load_state_dict(synth.make_state_dict(0))
  model = model.to(dev).eval()
  y, uv = nv12(1, 48, 256, 256, g, dev)
  frames = live.YUV420Frames.nv12(y, uv)
  rgb = live.yuv420_to_rgb(frames)
  for _ in range(3):  # alternate the variants so drift hits all of them alike
    ms_yuv = timeit(lambda: model.get_feature_grids(frames, False), n=5)
    ms_u8 = timeit(lambda: model.get_feature_grids(rgb, False), n=5)
    ms_conv = timeit(lambda: model.get_feature_grids(live.yuv420_to_rgb(frames), False), n=5)
    ms_kernel = timeit(lambda: live.yuv420_to_rgb(frames), n=50)
    print(json.dumps(dict(item='get_feature_grids 48x256^2', ms_nv12_fused=round(ms_yuv, 3),
                          ms_uint8_rgb=round(ms_u8, 3), ms_convert_then_uint8=round(ms_conv, 3),
                          ms_convert_kernel_alone=round(ms_kernel, 4))))
  del model, frames, rgb, y, uv

  causal = tapir_model.TAPIR(pyramid_level=1, use_casual_conv=True)
  causal.load_state_dict(synth.make_state_dict(0))
  causal = causal.to(dev).eval()
  H, W, N = 720, 1280, 256
  window = live.center_square_window(H, W)
  for S in (1, 8):
    y, uv = nv12(S, 1, H, W, g, dev)
    frames = live.YUV420Frames.nv12(y, uv, window=window)
    qp = torch.cat([torch.zeros(S, N, 1), torch.rand(S, N, 2, generator=g) * window[2]], -1).to(dev)
    a = streaming.OnlineTracker(causal, H, W, N, num_streams=S, yuv420=True, window=window)
    b = streaming.OnlineTracker(causal, window[2], window[3], N, uint8_frames=True, num_streams=S)
    a.init(frames, qp)
    b.init(live.yuv420_to_rgb(frames), qp)
    for _ in range(2):
      ms_a = timeit(lambda: a.step(frames), n=50)
      ms_b = timeit(lambda: b.step(live.yuv420_to_rgb(frames)), n=50)
      print(json.dumps(dict(item=f'OnlineTracker step 1280x720 NV12 centre crop, S={S}, {N} points',
                            ms_yuv420_tracker=round(ms_a, 4),
                            ms_convert_then_uint8_tracker=round(ms_b, 4))))
    a.close()
    b.close()


if __name__ == '__main__':
  main()
