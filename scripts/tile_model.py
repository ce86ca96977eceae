"""Wave model of the GEMM launches of one inference step (no GPU needed).

For every GEMM of the step it replays the tile choice of csrc/gemm_tc.cu (persistent wgmma
kernel, 128 x {64,128} tiles over 132 CTAs; 64-wide for N = 64 and for problems too small to fill
the GPU) and reports tiles, rounds, the wave-quantisation efficiency tiles / (rounds * workers),
and the time the issued bf16 MMA work would take at the given peak (default: the H100 SXM data
sheet's dense bf16 figure, not a measured rate).

  python scripts/tile_model.py [--frames 48 --queries 256] [--peak 989]
"""
import argparse
import math

SMS = 132


def choice(m_rows, n, planes):
  """Replays gemm_tc.cu's dispatch (plain GEMMs, no split-K).  Returns (kernel, tiles, workers,
  rounds)."""
  del planes  # the tile choice does not depend on the number of planes
  m_tiles = math.ceil(m_rows / 128)
  small = m_tiles * math.ceil(n / 128) * 10 < SMS * 6
  bn = 64 if (n <= 64 or (small and m_tiles * math.ceil(n / 128) * 2 <= SMS)) else 128
  tiles = m_tiles * math.ceil(n / bn)
  return f'128x{bn}', tiles, SMS, math.ceil(tiles / SMS)


def step_gemms(frames, queries):
  g = []
  hw = {0: 128 * 128, 1: 64 * 64, 2: 32 * 32, 3: 32 * 32}
  ch = (64, 128, 256, 256)
  cin = 64
  for grp in range(4):
    rows, c = frames * hw[grp], ch[grp]
    g.append((f'resnet g{grp} proj 1x1', rows, c, max(cin, 64), 2, 1))
    g.append((f'resnet g{grp} conv_0', rows, c, 9 * cin, 2, 1))
    g.append((f'resnet g{grp} conv 3x3 x3', rows, c, 9 * c, 2, 3))
    cin = c
  rows = frames * 32 * 32
  g.append(('extra_convs 256->1024', rows, 1024, 9 * 256, 2, 5))
  g.append(('extra_convs 1024->256', rows, 256, 9 * 1024, 2, 5))
  g.append(('cost volume (6 MMAs)', queries, frames * 1024, 256, 3, 1))  # M = queries, N = cells
  r = queries * frames
  g.append(('mixer linear_in', r, 512, 576, 2, 4))
  g.append(('mixer up', r, 2048, 512, 2, 48))
  g.append(('mixer down', r, 512, 2048, 2, 48))
  g.append(('mixer linear_out', r, 388, 512, 2, 4))
  return g


# wave-model row -> key of bench.py's kernel_breakdown
_CLASS = {'proj': 'backbone.proj', 'resnet': 'backbone.conv', 'extra_convs': 'backbone.extra_conv',
          'cost volume': 'cost_volume.gemm', 'linear_in': 'mixer.linear_in', 'mixer up': 'mixer.up',
          'mixer down': 'mixer.down', 'linear_out': 'mixer.linear_out'}


def _class_of(name):
  for k in ('proj', 'extra_convs', 'cost volume', 'linear_in', 'mixer up', 'mixer down', 'linear_out',
            'resnet'):
    if k in name:
      return _CLASS[k]
  return None


def compare(bench_json, frames, queries, peak, chunks=1):
  """Per GEMM class: measured ms (bench.py kernel_breakdown) against the MMA-bound time at the
  given peak and against that time divided by the wave-quantisation efficiency."""
  import json
  with open(bench_json) as fh:
    line = [l for l in fh if l.startswith('{')][-1]
  kb = json.loads(line)['kernel_breakdown']
  agg = {}
  for name, m, n, k, planes, count in step_gemms(frames, queries):
    kind, tiles, workers, rounds = choice(m, n, planes)
    eff = tiles / (rounds * workers)
    terms = planes * (planes + 1) // 2
    ms = 2.0 * m * n * k * terms / (peak * 1e12) * 1e3 * count
    c = _class_of(name)
    if c.startswith('mixer') or c.startswith('cost_volume'):
      ms *= chunks  # the host runs the query-dependent stages once per chunk of queries
    a = agg.setdefault(c, [0.0, 0.0])
    a[0] += ms
    a[1] += ms / eff
  print('| class | measured ms | MMA-bound ms | quantisation-bound ms | measured / quantisation-bound |')
  print('|---|---|---|---|---|')
  tm = tb = tq = 0.0
  for c, (ms, msq) in agg.items():
    meas = kb[c]['ms_per_step']
    tm, tb, tq = tm + meas, tb + ms, tq + msq
    print(f'| {c} | {meas:.3f} | {ms:.3f} | {msq:.3f} | {meas / msq:.2f} |')
  print(f'| all GEMMs | {tm:.2f} | {tb:.2f} | {tq:.2f} | {tm / tq:.2f} |')


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--bench', help='bench.py JSON line to compare the model with')
  ap.add_argument('--chunks', type=int, default=1,
                  help='query chunks per step (--queries is then the chunk size)')
  ap.add_argument('--frames', type=int, default=48)
  ap.add_argument('--queries', type=int, default=256)
  ap.add_argument('--peak', type=float, default=989.0, help='bf16 TFLOP/s (H100 SXM data sheet, dense)')
  a = ap.parse_args()
  if a.bench:
    compare(a.bench, a.frames, a.queries, a.peak, a.chunks)
    return
  print(f'| GEMM | M x N x K | tile | tiles | rounds | quantisation | launches | MMA-bound ms/step |')
  print('|---|---|---|---|---|---|---|---|')
  total = 0.0
  for name, m, n, k, planes, count in step_gemms(a.frames, a.queries):
    kind, tiles, workers, rounds = choice(m, n, planes)
    eff = tiles / (rounds * workers)
    terms = planes * (planes + 1) // 2
    ms = 2.0 * m * n * k * terms / (a.peak * 1e12) * 1e3 * count
    total += ms
    print(f'| {name} | {m} x {n} x {k} | {kind} | {tiles} | {rounds:.3g} | {eff:.0%} | {count} | {ms:.3f} |')
  print(f'| total | | | | | | | {total:.2f} |')


if __name__ == '__main__':
  main()
