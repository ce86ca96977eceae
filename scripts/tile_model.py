"""Wave model of the GEMM launches of one inference step (no GPU needed).

For every GEMM of the step it replays the tile and schedule choice of csrc/gemm_tc.cu (persistent
wgmma kernel, 128 x {64,128} tiles over 132 CTAs; 64-wide for N = 64 and for problems too small to
fill the GPU; the ping-pong schedule for P <= 2 with at least two tiles per CTA and either four
tiles per CTA or 16 k-blocks per tile, else the cooperative one) and reports tiles, rounds, the wave-quantisation efficiency tiles / (rounds *
workers), and the time the issued bf16 MMA work would take at the given peak (default: the H100 SXM
data sheet's dense bf16 figure, not a measured rate).

--bench adds the epilogue: its HBM traffic (outputs stored, residual read) at the given bandwidth.
The cooperative schedule runs it after each tile's mainloop, so its bound is MMA + epilogue; the
ping-pong schedule runs it under the other warpgroup's mainloop, so its bound is the larger of the
two plus the exposed epilogue of each CTA's last tile.

  python scripts/tile_model.py [--frames 48 --queries 256] [--peak 989] [--hbm 3350]
  python scripts/tile_model.py --bench <bench.py JSON output>
"""
import argparse
import math

SMS = 132


def choice(m_rows, n, planes, halo=False, k=None):
  """Replays gemm_tc.cu's dispatch (no split-K; halo: a C = 64 -> 64 3x3 convolution, which runs
  conv3x3_halo_kernel).  Returns (kernel, tiles, workers, rounds); kernel is '<tile> <schedule>'."""
  if halo:
    tiles = math.ceil(m_rows / 128)
    return '128x64 halo', tiles, SMS, math.ceil(tiles / SMS)
  m_tiles = math.ceil(m_rows / 128)
  small = m_tiles * math.ceil(n / 128) * 10 < SMS * 6
  bn = 64 if (n <= 64 or (small and m_tiles * math.ceil(n / 128) * 2 <= SMS)) else 128
  tiles = m_tiles * math.ceil(n / bn)
  long_k = k is not None and k // 64 >= 16
  schedule = 'pingpong' if planes <= 2 and tiles >= 2 * SMS and (tiles >= 4 * SMS or long_k) else 'coop'
  return f'128x{bn} {schedule}', tiles, SMS, math.ceil(tiles / SMS)


def step_gemms(frames, queries):
  """(name, M, N, K, planes, launches, epilogue bytes per output element)."""
  g = []
  hw = {0: 128 * 128, 1: 64 * 64, 2: 32 * 32, 3: 32 * 32}
  ch = (64, 128, 256, 256)
  cin = 64
  for grp in range(4):
    rows, c = frames * hw[grp], ch[grp]
    g.append((f'resnet g{grp} proj 1x1', rows, c, max(cin, 64), 2, 1, 4))
    g.append((f'resnet g{grp} conv_0', rows, c, 9 * cin, 2, 1, 4))
    g.append((f'resnet g{grp} conv 3x3 x3', rows, c, 9 * c, 2, 3, 4))
    cin = c
  rows = frames * 32 * 32
  g.append(('extra_convs 256->1024', rows, 1024, 9 * 256, 2, 5, 4))  # two bf16 planes
  g.append(('extra_convs 1024->256', rows, 256, 9 * 1024, 2, 5, 8))  # fp32 + residual
  g.append(('cost volume (6 MMAs)', queries, frames * 1024, 256, 3, 1, 4))  # M = queries, N = cells
  r = queries * frames
  g.append(('mixer linear_in', r, 512, 576, 2, 4, 4))
  g.append(('mixer up', r, 2048, 512, 2, 48, 4))
  g.append(('mixer down', r, 512, 2048, 2, 48, 8))
  g.append(('mixer linear_out', r, 388, 512, 2, 4, 4))
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


def compare(bench_json, frames, queries, peak, hbm, chunks=1):
  """Per GEMM class: measured ms (bench.py kernel_breakdown) against the MMA-bound time at the
  given peak, that time divided by the wave-quantisation efficiency, and the schedule's bound with
  the epilogue's HBM time added (cooperative) or overlapped (ping-pong)."""
  import json
  with open(bench_json) as fh:
    line = [l for l in fh if l.startswith('{')][-1]
  kb = json.loads(line)['kernel_breakdown']
  agg = {}
  for name, m, n, k, planes, count, out_bytes in step_gemms(frames, queries):
    kind, tiles, workers, rounds = choice(m, n, planes, halo=name.startswith('resnet g0 conv'), k=k)
    eff = tiles / (rounds * workers)
    terms = planes * (planes + 1) // 2
    ms = 2.0 * m * n * k * terms / (peak * 1e12) * 1e3 * count
    epi = m * n * out_bytes / (hbm * 1e9) * 1e3 * count
    msq = ms / eff
    if kind.endswith('pingpong'):
      bound = max(msq, epi) + epi / rounds  # the last tile's epilogue of each CTA is exposed
    else:
      bound = msq + epi
    c = _class_of(name)
    scale = chunks if (c.startswith('mixer') or c.startswith('cost_volume')) else 1
    a = agg.setdefault(c, [0.0, 0.0, 0.0, set()])
    a[0] += ms * scale  # the host runs the query-dependent stages once per chunk of queries
    a[1] += msq * scale
    a[2] += bound * scale
    a[3].add(kind.split()[1])
  print('| class | schedule | measured ms | MMA-bound ms | quantisation-bound ms | with epilogue ms '
        '| measured / with epilogue |')
  print('|---|---|---|---|---|---|---|')
  tm = tb = tq = te = 0.0
  for c, (ms, msq, bound, kinds) in agg.items():
    meas = kb[c]['ms_per_step']
    tm, tb, tq, te = tm + meas, tb + ms, tq + msq, te + bound
    print(f'| {c} | {"/".join(sorted(kinds))} | {meas:.3f} | {ms:.3f} | {msq:.3f} | {bound:.3f} '
          f'| {meas / bound:.2f} |')
  print(f'| all GEMMs | | {tm:.2f} | {tb:.2f} | {tq:.2f} | {te:.2f} | {tm / te:.2f} |')


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--bench', help='bench.py JSON line to compare the model with')
  ap.add_argument('--chunks', type=int, default=1,
                  help='query chunks per step (--queries is then the chunk size)')
  ap.add_argument('--frames', type=int, default=48)
  ap.add_argument('--queries', type=int, default=256)
  ap.add_argument('--peak', type=float, default=989.0, help='bf16 TFLOP/s (H100 SXM data sheet, dense)')
  ap.add_argument('--hbm', type=float, default=3350.0, help='HBM GB/s (H100 SXM data sheet)')
  a = ap.parse_args()
  if a.bench:
    compare(a.bench, a.frames, a.queries, a.peak, a.hbm, a.chunks)
    return
  print(f'| GEMM | M x N x K | tile | tiles | rounds | quantisation | launches | MMA-bound ms/step |')
  print('|---|---|---|---|---|---|---|---|')
  total = 0.0
  for name, m, n, k, planes, count, _ in step_gemms(a.frames, a.queries):
    kind, tiles, workers, rounds = choice(m, n, planes, halo=name.startswith('resnet g0 conv'), k=k)
    eff = tiles / (rounds * workers)
    terms = planes * (planes + 1) // 2
    ms = 2.0 * m * n * k * terms / (a.peak * 1e12) * 1e3 * count
    total += ms
    print(f'| {name} | {m} x {n} x {k} | {kind} | {tiles} | {rounds:.3g} | {eff:.0%} | {count} | {ms:.3f} |')
  print(f'| total | | | | | | | {total:.2f} |')


if __name__ == '__main__':
  main()
