"""Every `backbone.conv` launch of the c2 backbone (48 frames of 256 x 256, split-bf16 P = 2), one
line each, as backbone_forward issues it: the C = 64 halo convolution of the first ResNet group,
the generic implicit-GEMM convolution, or the plain GEMM over the im2col columns of a stride-2
`conv0`; fused InstanceNorm statistics with the frame's rows, and the residual on `conv1`.

  python scripts/backbone_conv_bench.py [--reps 20] [--rounds 3]

Per launch: the median of all launches (CUDA events, L2 flushed before each), the MMA-bound time
(three bf16 MMAs per product at the data-sheet 989 TFLOP/s) and the HBM-bound time (A planes, fp32
output and residual at the data-sheet 3.35 TB/s).  Variants, alternated `rounds` times in one
process: the dispatcher's choice, statistics off, and each schedule forced through
TAPIR_B200_GEMM_SCHEDULE.  The card's name, power limit and SM clocks are read in the same run.
"""
import argparse
import ctypes
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from tapnet_b200 import _lib, schema  # noqa: E402
from tests import gpu_util as U  # noqa: E402

P = 2
FRAMES, H0 = 48, 128  # stem output of 48 frames of 256 x 256
MMA_TFLOPS, HBM_TBS = 989.0, 3.35
VARIANTS = [('auto', {}, True), ('no stats', {}, False),
            ('coop', {'TAPIR_B200_GEMM_SCHEDULE': 'coop'}, True),
            ('pingpong', {'TAPIR_B200_GEMM_SCHEDULE': 'pingpong'}, True)]


def launches():
  """(name, kind, M, N, K, (frames, h, w, cin) or None, residual, stats) per backbone.conv launch."""
  out, h = [], H0
  cin = schema.GROUP_CHANNELS[0]
  n_blocks = sum(schema.BLOCKS_PER_GROUP)
  bi = 0
  for g, (cout, stride) in enumerate(zip(schema.GROUP_CHANNELS, schema.GROUP_STRIDES)):
    for b in range(schema.BLOCKS_PER_GROUP[g]):
      s = stride if b == 0 else 1
      c_in = cin if b == 0 else cout
      oh = h // s
      m = FRAMES * oh * oh
      fuse = s == 1 or (oh * oh) % 128 == 0
      if s == 1:
        kind = 'halo' if c_in == 64 and cout == 64 else 'conv'
        out.append((f'g{g}.b{b}.conv0', kind, m, cout, 9 * c_in, (FRAMES, oh, oh, c_in), False, fuse))
      else:
        out.append((f'g{g}.b{b}.conv0', 'im2col', m, cout, 9 * c_in, None, False, fuse))
      kind = 'halo' if cout == 64 else 'conv'
      out.append((f'g{g}.b{b}.conv1', kind, m, cout, 9 * cout, (FRAMES, oh, oh, cout), True,
                  bi + 1 < n_blocks))
      h, bi = oh, bi + 1
    cin = cout
  return out


def make(M, N, K, conv, resid, stats):
  """The launch's operands; returns call(with_stats)."""
  lib = _lib.load()
  g = torch.Generator(device='cuda').manual_seed(0)
  if conv is None:
    a = torch.randn(P, M, K, generator=g, device='cuda').to(torch.bfloat16)
  else:
    f, h, w, c = conv
    a = torch.randn(P, f, h, w, c, generator=g, device='cuda').to(torch.bfloat16)
  wt = (torch.randn(P, N, K, generator=g, device='cuda') / K ** 0.5).to(torch.bfloat16)
  r = torch.randn(M, N, generator=g, device='cuda') if resid else None
  o = torch.empty(M, N, device='cuda')
  st = torch.zeros(FRAMES, N, 2, dtype=torch.float64, device='cuda') if stats else None
  lin = U.make_linear(wt, None)
  rpf = M // FRAMES

  def call(with_stats):
    keep = (a, wt, r, o, st, lin)  # noqa: F841  the buffers live as long as the closure
    sp = U.ptr(st) if with_stats else None
    if conv is None:
      rc = lib.tapir_gemm(U.ptr(a), K, M * K, ctypes.byref(lin), M, 0, 0, 0, 0, 0, U.ptr(r), N, 0,
                          U.ptr(o), N, None, N, M * N, 0, sp, rpf if with_stats else 0, 0, U.stream())
    else:
      f, h, w, c = conv
      rc = lib.tapir_gemm(U.ptr(a), 0, M * c, ctypes.byref(lin), M, 1, f, h, w, c, U.ptr(r), N, 0,
                          U.ptr(o), N, None, N, M * N, 0, sp, 0, 0, U.stream())
    _lib.check(rc, 'tapir_gemm')
  return call


def time_us(call, reps, flush):
  for _ in range(3):
    call()
  torch.cuda.synchronize()
  evs = []
  for _ in range(reps):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    call()
    e1.record()
    evs.append((e0, e1))
  torch.cuda.synchronize()
  return [a.elapsed_time(b) * 1e3 for a, b in evs]


def card():
  q = 'name,power.limit,clocks.max.sm,clocks.sm'
  try:
    return subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), f'--query-gpu={q}',
                           '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    return f'{torch.cuda.get_device_name()} (nvidia-smi unavailable)'


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=3)
  a = ap.parse_args()
  assert torch.cuda.is_available(), 'needs a CUDA device'
  print(f'card (name, power limit, max SM clock, SM clock): {card()}')
  flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
  rows = launches()
  calls = [make(M, N, K, conv, resid, stats) for _, _, M, N, K, conv, resid, stats in rows]
  ts = {(i, v): [] for i in range(len(rows)) for v, _, _ in VARIANTS}
  for _ in range(a.rounds):
    for i, call in enumerate(calls):
      for v, env, st in VARIANTS:
        with_stats = st and rows[i][7]
        with U.switches(**env):
          ts[(i, v)] += time_us(lambda: call(with_stats), a.reps, flush)
  names = [v for v, _, _ in VARIANTS]
  print(f'{"launch":12s} {"path":6s} {"M":>7s} {"N":>4s} {"K":>5s} {"res":>3s} {"st":>2s} '
        + ' '.join(f'{n + " us":>12s}' for n in names) + f' {"MMA us":>8s} {"HBM us":>8s}')
  tot = {n: 0.0 for n in names}
  tot_mma = tot_hbm = 0.0
  for i, (name, kind, M, N, K, conv, resid, stats) in enumerate(rows):
    med = {n: statistics.median(ts[(i, n)]) for n in names}
    mma = 2.0 * M * N * K * 3 / (MMA_TFLOPS * 1e12) * 1e6
    a_bytes = P * 2 * (M * conv[3] if conv else M * K)
    hbm = (a_bytes + 4 * M * N * (2 if resid else 1)) / (HBM_TBS * 1e12) * 1e6
    for n in names:
      tot[n] += med[n]
    tot_mma += mma
    tot_hbm += hbm
    print(f'{name:12s} {kind:6s} {M:7d} {N:4d} {K:5d} {int(resid):3d} {int(stats):2d} '
          + ' '.join(f'{med[n]:12.1f}' for n in names) + f' {mma:8.1f} {hbm:8.1f}', flush=True)
  print(f'{"total":12s} {"":6s} {"":>7s} {"":>4s} {"":>5s} {"":>3s} {"":>2s} '
        + ' '.join(f'{tot[n]:12.1f}' for n in names) + f' {tot_mma:8.1f} {tot_hbm:8.1f}')
  print(f'card after: {card()}')


if __name__ == '__main__':
  main()
