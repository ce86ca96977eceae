"""Micro-benchmark of tapir_gemm shapes/epilogues (CUDA events, L2 flushed between launches).

  python scripts/gemm_bench.py               every shape under the dispatcher's own choice
  python scripts/gemm_bench.py --schedules   the offline clip's GEMM shapes under both wgmma
                                             schedules (TAPIR_B200_GEMM_SCHEDULE), alternated
  python scripts/gemm_bench.py --tile-cost   time per launch against tile count at constant MMA
                                             work, both schedules and BLOCK_N = 64 / 128
"""
import argparse
import ctypes
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from tapnet_b200 import _lib  # noqa: E402
from tests import gpu_util as U  # noqa: E402

lib = _lib.load()
dev = 'cuda'
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def _peak():
  path = os.path.join(ROOT, 'MEASURED_PEAKS.json')
  if os.path.exists(path):
    with open(path) as fh:
      return json.load(fh)['bf16_tflops'], 'measured (MEASURED_PEAKS.json)'
  return 989.0, 'H100 SXM data sheet, dense bf16, not measured'


PEAK, PEAK_SOURCE = _peak()


def make(M, N, K, P=2, bias=True, gelu=False, resid=False, planes_out=0, f32_out=True, conv=None):
  """Operands and outputs of one GEMM; returns (call, M, K)."""
  g = torch.Generator().manual_seed(0)
  if conv is None:
    a = torch.randn(P, M, K, generator=g).to(dev).to(torch.bfloat16)
  else:
    f, h, w, c = conv
    a = torch.randn(P, f, h, w, c, generator=g).to(dev).to(torch.bfloat16)
    M, K = f * h * w, 9 * c
  wt = torch.randn(P, N, K, generator=g).to(dev).to(torch.bfloat16)
  b = torch.randn(N, device=dev) if bias else None
  r = torch.randn(M, N, device=dev) if resid else None
  o32 = torch.empty(M, N, device=dev) if f32_out else None
  opl = torch.empty(planes_out, M, N, dtype=torch.bfloat16, device=dev) if planes_out else None
  lin = U.make_linear(wt, b)

  def call():
    keep = (a, wt, b, r, o32, opl, lin)  # noqa: F841  the buffers live as long as the closure
    if conv is None:
      st = lib.tapir_gemm(U.ptr(a), K, M * K, ctypes.byref(lin), M, 0, 0, 0, 0, 0, U.ptr(r), N, int(gelu),
                          U.ptr(o32), N, U.ptr(opl), N, M * N, planes_out, None, 0, 0, U.stream())
    else:
      f, h, w, c = conv
      st = lib.tapir_gemm(U.ptr(a), 0, M * c, ctypes.byref(lin), M, 1, f, h, w, c, U.ptr(r), N, int(gelu),
                          U.ptr(o32), N, U.ptr(opl), N, M * N, planes_out, None, 0, 0, U.stream())
    _lib.check(st, 'tapir_gemm')
  return call, M, K


def time_ms(call, reps, flush_l2):
  """Per-launch times (ms) of `reps` launches after 3 warm-up launches."""
  for _ in range(3):
    call()
  torch.cuda.synchronize()
  evs = []
  for _ in range(reps):
    if flush_l2:
      flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); call(); e1.record()
    evs.append((e0, e1))
  torch.cuda.synchronize()
  return [a_.elapsed_time(b_) for a_, b_ in evs]


def run(name, M, N, K, P=2, reps=10, flush_l2=False, **kw):
  call, M, K = make(M, N, K, P, **kw)
  ms = sorted(time_ms(call, reps, flush_l2))[reps // 2]
  fl = 2.0 * M * N * K
  npairs = P * (P + 1) // 2
  print(f'{name:34s} M={M:6d} N={N:5d} K={K:5d} P={P} {ms * 1e3:8.1f} us  alg {fl / ms / 1e9:7.1f} TF/s  '
        f'mma {fl * npairs / ms / 1e9:7.1f} TF/s ({fl * npairs / ms / 1e9 / PEAK:5.1%} of {PEAK:g})', flush=True)


# the GEMM classes of the offline clip step (48 frames of 256 x 256, 256 queries)
CLIP = [
    ('mixer.up: gelu+planes', dict(M=12288, N=2048, K=512, gelu=True, planes_out=2, f32_out=False)),
    ('mixer.up: f32 out, no bias', dict(M=12288, N=2048, K=512, bias=False)),
    ('mixer.down: bias+resid f32', dict(M=12288, N=512, K=2048, resid=True)),
    ('mixer.linear_in', dict(M=12288, N=512, K=576)),
    ('mixer.linear_out', dict(M=12288, N=388, K=512)),
    ('extra conv 256->1024 gelu+planes', dict(M=0, N=1024, K=0, gelu=True, planes_out=2, f32_out=False,
                                              conv=(48, 32, 32, 256))),
    ('extra conv 1024->256 resid', dict(M=0, N=256, K=0, resid=True, conv=(48, 32, 32, 1024))),
    ('resnet conv 128->128 @64', dict(M=0, N=128, K=0, bias=False, conv=(48, 64, 64, 128))),
    ('resnet conv 256->256 @32', dict(M=0, N=256, K=0, bias=False, conv=(48, 32, 32, 256))),
]


def compare_schedules(rounds, reps):
  """Each clip shape under both schedules, alternating coop / pingpong `rounds` times in this
  process (L2 flushed before every launch); median and min / max of all launches per schedule."""
  print(f'{"shape":34s} {"coop us (min-max)":>24s} {"pingpong us (min-max)":>24s} {"gain":>6s}')
  for name, kw in CLIP:
    call, _, _ = make(**kw)
    ts = {'coop': [], 'pingpong': []}
    for _ in range(rounds):
      for s in ts:
        with U.switches(TAPIR_B200_GEMM_SCHEDULE=s):
          ts[s] += time_ms(call, reps, True)
    med = {s: statistics.median(v) * 1e3 for s, v in ts.items()}
    cells = [f'{med[s]:8.1f} ({min(v) * 1e3:.1f}-{max(v) * 1e3:.1f})' for s, v in ts.items()]
    print(f'{name:34s} {cells[0]:>24s} {cells[1]:>24s} {1 - med["pingpong"] / med["coop"]:6.1%}', flush=True)


# GEMMs of mixer `up`'s MMA work (12288 x 2048 x 512) with fewer, longer tiles: same k-blocks per
# CTA, 4x fewer tiles from the first shape to the last two
TILE_COST_SHAPES = [(12288, 2048, 512), (12288, 1024, 1024), (12288, 512, 2048), (3072, 2048, 2048)]
TILE_COST_EPILOGUES = [('f32', dict(bias=False), 4),
                       ('gelu+plane', dict(gelu=True, planes_out=1, f32_out=False), 2),
                       ('gelu+planes', dict(gelu=True, planes_out=2, f32_out=False), 4)]


def _card():
  """Card name, power limit and max SM clock, read now (nvidia-smi queries only)."""
  import subprocess  # pylint: disable=g-import-not-at-top
  q = 'name,power.limit,clocks.max.sm,clocks.sm'
  try:
    out = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), f'--query-gpu={q}',
                          '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout
    return out.strip()
  except (OSError, subprocess.SubprocessError):
    return f'{torch.cuda.get_device_name()} (nvidia-smi unavailable)'


def tile_cost(rounds, reps):
  """Time per launch against tile count at constant MMA work: every shape x epilogue x schedule x
  BLOCK_N, alternated `rounds` times in this process (L2 flushed before every launch), median of
  all launches.  Per tile and per k-block figures divide by the busiest CTA's share."""
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  print(f'card: {_card()}')
  calls = {}
  for M, N, K in TILE_COST_SHAPES:
    for epi, kw, _ in TILE_COST_EPILOGUES:
      calls[(M, N, K, epi)] = make(M, N, K, **kw)[0]
  out_bytes = {epi: b for epi, _, b in TILE_COST_EPILOGUES}
  configs = [(shape_epi, sched, bn) for shape_epi in calls for sched in ('coop', 'pingpong') for bn in (128, 64)]
  ts = {c: [] for c in configs}
  for _ in range(rounds):
    for c in configs:
      shape_epi, sched, bn = c
      with U.switches(TAPIR_B200_GEMM_SCHEDULE=sched, TAPIR_B200_BLOCK_N=bn):
        ts[c] += time_ms(calls[shape_epi], reps, True)
  print(f'{"M x N x K":>18s} {"epilogue":>12s} {"sched":>8s} {"BN":>3s} {"tiles":>5s} {"t/CTA":>5s} '
        f'{"kb/t":>4s} {"us/launch (min-max)":>22s} {"us/tile":>8s} {"us/kblk":>8s} {"TF/s":>6s} {"out MB":>7s}')
  for c in configs:
    (M, N, K, epi), sched, bn = c
    tiles = -(-M // 128) * -(-N // bn)
    per_cta = -(-tiles // sms)
    kb = K // 64
    med = statistics.median(ts[c]) * 1e3
    tf = 2.0 * M * N * K * 3 / (med * 1e-6) / 1e12  # P = 2: three bf16 MMAs per product
    out_mb = M * N * out_bytes[epi] / 1e6
    rng = f'{med:8.1f} ({min(ts[c]) * 1e3:.1f}-{max(ts[c]) * 1e3:.1f})'
    print(f'{f"{M} x {N} x {K}":>18s} {epi:>12s} {sched:>8s} {bn:3d} {tiles:5d} {per_cta:5d} {kb:4d} '
          f'{rng:>22s} {med / per_cta:8.2f} {med / (per_cta * kb) * (128 / bn):8.3f} {tf:6.1f} {out_mb:7.1f}',
          flush=True)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--schedules', action='store_true', help='compare the two wgmma schedules')
  ap.add_argument('--tile-cost', action='store_true',
                  help='time per launch against tile count at constant MMA work')
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--reps', type=int, default=10)
  a = ap.parse_args()
  print(f'peak {PEAK:g} TFLOP/s bf16 ({PEAK_SOURCE}); {torch.cuda.get_device_name()}')
  if a.schedules:
    compare_schedules(a.rounds, a.reps)
    return
  if a.tile_cost:
    tile_cost(a.rounds, a.reps)
    return
  print('BLOCK_N override:', os.environ.get('TAPIR_B200_BLOCK_N', 'auto'))
  print('schedule override:', os.environ.get('TAPIR_B200_GEMM_SCHEDULE', 'auto'))
  run('up: gelu+planes', 12288, 2048, 512, gelu=True, planes_out=2, f32_out=False)
  run('up: planes only (no gelu)', 12288, 2048, 512, gelu=False, planes_out=2, f32_out=False)
  run('up: gelu + f32 out', 12288, 2048, 512, gelu=True)
  run('up: f32 out, no bias', 12288, 2048, 512, bias=False)
  run('up x4 rows: gelu+planes', 49152, 2048, 512, gelu=True, planes_out=2, f32_out=False)
  run('down: bias+resid f32', 12288, 512, 2048, resid=True)
  run('down: f32 only', 12288, 512, 2048, bias=False)
  run('down x4 rows', 49152, 512, 2048, resid=True)
  run('extra conv 256->1024 gelu+planes', 0, 1024, 0, gelu=True, planes_out=2, f32_out=False, conv=(48, 32, 32, 256))
  run('extra conv 1024->256 resid', 0, 256, 0, resid=True, conv=(48, 32, 32, 1024))
  run('resnet conv 64->64 @128', 0, 64, 0, bias=False, conv=(48, 128, 128, 64))
  run('resnet conv 128->128 @64', 0, 128, 0, bias=False, conv=(48, 64, 64, 128))
  run('resnet conv 256->256 @32', 0, 256, 0, bias=False, conv=(48, 32, 32, 256))
  run('linear_in 576->512', 12288, 512, 576)
  run('cost volume c2 (256 q x 48 f)', 256, 49152, 256, P=3, bias=False)
  run('cost volume c4/GPU (512 q x 96 f)', 512, 98304, 256, P=3, bias=False)
  run('cost volume 4096 q x 96 f', 4096, 98304, 256, P=3, bias=False, reps=5)
  run('P=1 up: gelu+planes(1)', 12288, 2048, 512, P=1, gelu=True, planes_out=1, f32_out=False)
  run('P=1 big square', 8192, 8192, 8192, P=1, bias=False, reps=5)
  run('P=2 big square', 8192, 8192, 4096, P=2, bias=False, reps=5)


if __name__ == '__main__':
  main()
