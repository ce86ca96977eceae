"""Designed cost maps for the stage-A track heads, and the float64 pieces their tests compare with.

A designed map reaches a head through the public cost-volume entry point: query n's feature is the
one-hot e_{n mod 256} and the map is channel n mod 256 of the feature grid, so the cost volume is
the map itself.  Map values are multiples of 1/8 in [-32, 32].  They are exact in bf16, so the
three split planes of a grid value are (v, 0, 0), the one-hot query is (1, 0, 0), and every
split-bf16 GEMM variant returns v exactly.

Two head weight sets run the designs: the synthetic head the model runs, and an identity head
whose heat map is exactly temperature * map, so that the designed geometry (ties, corners, the
radius-5 window) is the geometry the soft-argmax sees.

tests/test_stage_a_cases.py checks on the CPU that each family can catch the bug it targets;
tests/test_stage_a_gpu.py runs the families through the two heads.
"""
from typing import NamedTuple, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle import synth

C = 256
TEMPERATURES = (20.0, 1.0, 0.05)
HEAD_KINDS = ('synth', 'identity')
POINT_TOL = 1e-3  # px: the project's track budget
LOGIT_TOL = 1e-4
# exp(x) rounds to 0 in fp32 below about -103.97 (half the smallest denormal).  A map whose fp64
# heat gap between its two largest cells exceeds this bound has probability exactly 1 at its peak
# in every head, and every other cell contributes exactly 0.  Only the identity head reaches it
# (the designed gap is 120 at temperature 20); the synthetic head's gaps stay below 30.
SATURATED_GAP = 110.0
# argmax is compared where the fp64 top-two heat gap exceeds this fraction of the heat's
# magnitude bound (see heat_fp64): the kernels' fp32 heat cannot reorder such a pair
MARGIN = 1e-4
HEAD_PREFIX = 'torch_cost_volume_track_mods.'
HEAD_KEYS = ('hid1', 'hid2', 'hid3', 'hid4', 'occ_out')

# 32 x 32 heads and their pixel-to-thread mappings; every other map size runs the generic head
HEADS_32 = ('tc',)
GENERIC_SIZES = ((2, 2), (3, 5), (5, 3), (7, 64), (64, 7), (31, 32), (32, 31), (33, 33), (96, 128))


def head_state_dict(kind):
  """The ten head tensors (fp32) of `synth.make_state_dict(0)` ('synth'), or the 'identity' head:
  hid1 channel 0 is the centre tap with bias +64 (every other hid1 channel is zero), hid2 is the
  centre tap of channel 0 with bias -64, so hid2(relu(hid1(v))) == v for v >= -64.  hid3, hid4
  and occ_out stay synthetic."""
  sd = synth.make_state_dict(0)
  out = {HEAD_PREFIX + n + s: sd[HEAD_PREFIX + n + s].clone().float() for n in HEAD_KEYS
         for s in ('.weight', '.bias')}
  if kind == 'identity':
    w1 = torch.zeros(16, 1, 3, 3)
    w1[0, 0, 1, 1] = 1.0
    b1 = torch.zeros(16)
    b1[0] = 64.0
    w2 = torch.zeros(1, 16, 3, 3)
    w2[0, 0, 1, 1] = 1.0
    out[HEAD_PREFIX + 'hid1.weight'], out[HEAD_PREFIX + 'hid1.bias'] = w1, b1
    out[HEAD_PREFIX + 'hid2.weight'], out[HEAD_PREFIX + 'hid2.bias'] = w2, torch.tensor([-64.0])
  else:
    assert kind == 'synth', kind
  return out


def heat_fp64(sd64, maps, temperature):
  """maps [M, h, w] -> (heat [M, h*w], scale [M]) in float64: the pre-softmax logits of
  tracks_from_cost_volume, and a bound on the magnitude of every term summed into them."""
  m = HEAD_PREFIX
  x = maps.double()[:, None]
  w1, b1, w2, b2 = (sd64[m + k] for k in ('hid1.weight', 'hid1.bias', 'hid2.weight', 'hid2.bias'))
  occ = torch.relu(F.conv2d(x, w1, b1, padding=1))
  heat = F.conv2d(occ, w2, b2, padding=1)[:, 0] * temperature
  occ_abs = F.conv2d(x.abs(), w1.abs(), b1.abs(), padding=1)
  scale = F.conv2d(occ_abs, w2.abs(), b2.abs(), padding=1)[:, 0] * abs(temperature)
  return heat.reshape(len(maps), -1), scale.reshape(len(maps), -1).amax(-1)


def top_two(heat):
  """heat [M, cells] -> (gap between the two largest values, exact tie of the two largest)."""
  v = heat.topk(2, dim=-1).values
  return v[:, 0] - v[:, 1], v[:, 0] == v[:, 1]


def soft_argmax_cells(prob, h, w, include_boundary=False):
  """prob [h*w] (fp64) -> (x, y) in cell units, as utils.soft_argmax; include_boundary counts the
  cells at d^2 == 25 too (the off-by-one a `<=` would make)."""
  ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64),
                          indexing='ij')
  cx, cy = xs.reshape(-1) + 0.5, ys.reshape(-1) + 0.5
  i = int(torch.argmax(prob))
  d2 = (cx - cx[i]) ** 2 + (cy - cy[i]) ** 2
  win = (d2 <= 25.0) if include_boundary else (d2 < 25.0)
  p = prob * win
  return torch.stack([(cx * p).sum(), (cy * p).sum()]) / p.sum()


# ------------------------------------------------------------------------- thread mappings
def owner(head, gh, gw, i):
  """(warp, lane) of the thread that owns flat cell i in a head's pixel-to-thread mapping."""
  y, x = divmod(i, gw)
  if head == 'tc':        # 512 threads: 2 consecutive x per thread, 16 threads per row
    tid = y * 16 + x // 2
  else:                   # generic: cell i belongs to thread i mod 256
    tid = i % 256
  return tid >> 5, tid & 31


def tie_level(head, gh, gw, a, b):
  """Where a head resolves a tie between cells a and b: inside a thread, across the lanes of a
  warp (shuffle) or across warps (shared memory)."""
  (wa, la), (wb, lb) = owner(head, gh, gw, a), owner(head, gh, gw, b)
  if wa != wb:
    return 'warp'
  return 'lane' if la != lb else 'thread'


def mappings(gh, gw):
  return HEADS_32 if (gh, gw) == (32, 32) else ('generic',)


# ------------------------------------------------------------------------- designs
class Design(NamedTuple):
  name: str
  family: str            # flat, tie, peak, radius, saturated, noise
  map: np.ndarray        # [gh, gw] float32, multiples of 1/8 in [-32, 32]
  tie_heads: Tuple[str, ...] = ()   # head weight sets for which the map is a designed tie
  pair: Tuple[int, int] = (-1, -1)  # the designed tied cells (flat indices), if any


def _bump(m, y, x, amp):
  """A 3 x 3 bump with a strict maximum at its centre."""
  m[y - 1:y + 2, x - 1:x + 2] += amp * np.array([[1, 2, 1], [2, 4, 2], [1, 2, 1]], np.float32) / 4


def _pairs(gh, gw, head, bumps):
  """One pair of cells (a < b) per tie level of `head`'s mapping.  bumps: both cells at least 5
  from every border and 8 apart, so the synthetic head sees translated copies of one neighbourhood
  (its maxima then tie exactly, wherever inside the bump they fall)."""
  cells = gh * gw
  if bumps:
    ok = lambda i: 5 <= i // gw < gh - 5 and 5 <= i % gw < gw - 5  # noqa: E731
    far = lambda a, b: max(abs(a // gw - b // gw), abs(a % gw - b % gw)) >= 8  # noqa: E731
  else:
    ok = lambda i: True  # noqa: E731
    far = lambda a, b: True  # noqa: E731
  # prefer pairs in one row (a bump's maximum may sit off its centre: same-row pairs keep their
  # level), starting near the middle of the map
  start = (gh // 3) * gw + gw // 4
  order = list(range(start, cells)) + list(range(start))
  out = {}
  # two bumps never share a thread of the 32 x 32 head (2 consecutive x)
  levels = ('lane', 'warp') if bumps and head in HEADS_32 else ('thread', 'lane', 'warp')
  for level in levels:
    for a in order:
      if not ok(a):
        continue
      cands = [b for b in range(a + 1, cells) if b // gw == a // gw] + \
              [b for b in range(a + 1, cells) if b // gw != a // gw]
      hit = next((b for b in cands if ok(b) and far(a, b) and tie_level(head, gh, gw, a, b) == level),
                 None)
      if hit is not None:
        out[level] = (a, hit)
        break
  return out


def designs(gh, gw):
  """Every designed map that fits a gh x gw map, in a fixed order."""
  cells = gh * gw
  z = lambda: np.zeros((gh, gw), np.float32)  # noqa: E731
  out = [Design('flat0', 'flat', z(), ('identity',), (0, 1)),
         Design('flat_neg', 'flat', z() - 32, ('identity',), (0, 1))]
  # two equal maxima, lower index first, at each tie level of each mapping that runs this size
  for head in mappings(gh, gw):
    for level, (a, b) in _pairs(gh, gw, head, bumps=False).items():
      m = z()
      m.flat[a] = m.flat[b] = 6.0
      out.append(Design(f'cells_{head}_{level}', 'tie', m, ('identity',), (a, b)))
    for level, (a, b) in _pairs(gh, gw, head, bumps=True).items():
      m = z()
      _bump(m, a // gw, a % gw, 8.0)
      _bump(m, b // gw, b % gw, 8.0)
      out.append(Design(f'bumps_{head}_{level}', 'tie', m, HEAD_KINDS, (a, b)))
  # one peak at each corner and each edge midpoint
  spots = {'tl': (0, 0), 'tr': (0, gw - 1), 'bl': (gh - 1, 0), 'br': (gh - 1, gw - 1),
           'top': (0, gw // 2), 'bottom': (gh - 1, gw // 2), 'left': (gh // 2, 0),
           'right': (gh // 2, gw - 1)}
  seen = set()
  for name, (y, x) in spots.items():
    if (y, x) in seen:
      continue
    seen.add((y, x))
    m = z()
    m[y, x] = 4.0
    if gh > 1 and gw > 1:  # a shoulder inside the map so that the window is not symmetric
      m[y + (1 if y == 0 else -1), x] = 3.5
    out.append(Design(f'peak_{name}', 'peak', m))
  # radius-5 window boundary: mass at d^2 == 25 and d^2 in {18, 20} on one side of the peak
  if gh >= 13 and gw >= 13:
    y0, x0 = gh // 2 - 2, gw // 2 - 3
    m = z()
    m[y0, x0] = 8.0
    for dy, dx in ((0, 5), (5, 0), (3, 4), (4, 3), (3, 3), (2, 4), (4, 2)):
      m[y0 + dy, x0 + dx] = 7.875
    out.append(Design('radius', 'radius', m))
  # saturated: one cell stands out by 6 (identity head at temperature 20: a heat gap of 120)
  for name, (y, x) in (('tl', (0, 0)), ('mid', (gh // 2, gw // 2)), ('br', (gh - 1, gw - 1))):
    m = z() - 32
    m[y, x] = -26.0
    out.append(Design(f'saturated_neg_{name}', 'saturated', m))
  m = z()
  m[gh - 1, gw // 2] = 8.0
  out.append(Design('saturated_bottom', 'saturated', m))
  # bf16-exact noise
  g = torch.Generator().manual_seed(1000 + 7 * gh + gw)
  for k in range(4):
    m = (torch.randint(-32, 33, (gh, gw), generator=g).float() / 8.0).numpy()
    out.append(Design(f'noise{k}', 'noise', m))
  for d in out:
    assert d.map.dtype == np.float32 and np.abs(d.map).max() <= 32.0, d.name
  return out


# ------------------------------------------------------------------------- queries
def query_times(T):
  """Query frames: integers, halves (rint rounds them to even, as torch.round does), -0.5 (rounds
  to -0, which matches frame 0), just below it, the last half frame and past the end."""
  return [2.0, 2.5, 3.5, -0.5, -0.51, T - 0.5, T + 3.0, 0.0]


def query_points(B, n, T, ih, iw, seed):
  """[B, n, 3] float32 (t, y, x): t cycles through query_times(T), y and x are anywhere in the
  image (far from the designed peaks, so that a passthrough frame is unmistakable)."""
  g = torch.Generator().manual_seed(seed)
  q = torch.empty(B, n, 3)
  ts = torch.tensor(query_times(T))
  q[..., 0] = ts[torch.arange(n) % len(ts)]
  q[..., 1] = torch.rand(B, n, generator=g) * ih
  q[..., 2] = torch.rand(B, n, generator=g) * iw
  return q


def passthrough(qp, T):
  """[B, n, T] bool: the frames on which the reference puts the query point itself
  (torch.round of the fp32 frame scaled by T / T)."""
  qf = torch.round(qp[..., 0:1].float() * float(T) / float(T))
  return qf == torch.arange(T, dtype=torch.float32)
