"""Split-bf16 plane-pair designs: operands whose planes are independent integer tensors, the exact
models of the plane pairs each GEMM kernel sums, and the plausible wrong pair sets a kernel could
sum instead.

Every dense contraction is a split-bf16 GEMM.  A and B are each held as P bf16 planes, and the
tensor-core kernels (gemm_tc.cu, mma_k_block) sum the plane products A_i . B_j over the pairs
i + j < P; the SIMT kernel (gemm_simt.cu) rebuilds a = sum_i A_i and b = sum_j B_j, so it sums all
P^2 pairs.  No kernel checks that its planes are a real split, so here every plane of A and of B
is its own random integer tensor: each pair (i, j) adds its own nonzero, independent term, and a
kernel that sums any other set of pairs gives different outputs almost everywhere
(tests/test_plane_pairs_host.py states the share).

The exact-accumulator contract of tests/gemm_exact.py holds: sum_k |a_i||b_j| over all P^2 pairs
stays below 2^22, so every partial sum of either model is an integer that fp32 holds exactly, in
any order, and the fp64 model equals the kernel output bit for bit.

A's planes are laid out plane_stride = rows * lda + GAP elements apart, with lda > K, and NaN in
every element between the planes and past column K (gapped_a).  A kernel that reads A with a wrong
plane stride, plane offset or row length sees NaN, not a small error.

The second half of this module designs cost maps for the stage-A cost volume, the one batched and
the one grouped GEMM, whose planes tapir_split_planes makes from fp32 queries and grids (see
cost-volume designs)."""
import numpy as np
import torch

from tests.gemm_exact import choose_conv_tile
from tests.gpu_util import split_like_kernel

f32 = np.float32
EXACT_UNITS = 2.0 ** 22
VMAX = 7      # |v| per plane where K allows it
GAP_ROWS = 128  # NaN rows between A's planes: a whole m-tile
PAD_COLS = 8    # NaN columns past K in each plain A row


def tc_pairs(P):
  """The tensor cores' pair set, in mma_k_block's order."""
  return [(i, j) for i in range(P) for j in range(P - i)]


def all_pairs(P):
  """The SIMT kernel's pair set: (sum_i A_i)(sum_j B_j)."""
  return [(i, j) for i in range(P) for j in range(P)]


def plane_vmax(K, P):
  """The largest |v| <= VMAX per plane for which sum_k over all P^2 pairs of |a_i||b_j| stays
  below 2^22 whatever the values: the bound for both models and every wrong set without repeats."""
  for v in range(VMAX, 0, -1):
    if K * P * P * v * v < EXACT_UNITS:
      return v
  raise ValueError(f'K={K} is too long for exact integer planes')


# ------------------------------------------------------------------------------------ wrong sets
def _key(pairs):
  return tuple(sorted(pairs))


def wrong_sets(P, simt=False):
  """{name: pair list} of the plausible wrong pair sets for P planes, relative to the tensor cores'
  i + j < P (simt=False) or the SIMT kernel's all P^2 pairs.  A pair list may repeat a pair: 'A
  plane q read as plane q - 1' sums A_{q-1} where A_q belongs.  Sets that sum to the same multiset
  share one entry whose name lists them all; the right set itself is left out.  The transposed set
  {(j, i)} is on the list but never shows up: both right sets are their own transposes."""
  right = all_pairs(P) if simt else tc_pairs(P)
  cands = []
  for p in right:
    cands.append((f'drop {p}', [q for q in right if q != p]))
  for p in all_pairs(P):
    if p not in right:
      cands.append((f'add {p}', right + [p]))
  cands.append(('transposed', [(j, i) for i, j in right]))
  cands.append(('all P^2 pairs', all_pairs(P)))
  cands.append(('i + j < P', tc_pairs(P)))
  cands.append((f'the P = {P - 1} set', all_pairs(P - 1) if simt else tc_pairs(P - 1)))
  for q in range(1, P):
    cands.append((f'A plane {q} read as plane {q - 1}', [(q - 1 if i == q else i, j) for i, j in right]))
    cands.append((f'B plane {q} read as plane {q - 1}', [(i, q - 1 if j == q else j) for i, j in right]))
  for q in range(P):
    cands.append((f'A plane {q} read as zero', [(i, j) for i, j in right if i != q]))
    cands.append((f'B plane {q} read as zero', [(i, j) for i, j in right if j != q]))
  out, names = {}, {}
  for name, pairs in cands:
    k = _key(pairs)
    if k == _key(right):
      continue
    if k in names:
      names[k].append(name)
    else:
      names[k] = [name]
      out[k] = pairs
  return {' = '.join(names[k]): pairs for k, pairs in out.items()}


# ------------------------------------------------------------------------------------ designs
class Design:
  """a_pl [P, M, K] (plain) or [P, F, H, W, C] (conv) and w_pl [P, N, K], bf16 on the CPU, each
  plane an independent integer tensor with |v| <= vmax."""

  def __init__(self, name, M, N, K, P, conv=None):
    self.name, self.P, self.conv = name, P, conv
    if conv is not None:
      Fr, H, W, C = conv
      M, K = Fr * H * W, 9 * C
    self.M, self.N, self.K = M, N, K
    self.vmax = plane_vmax(K, P)
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    a_shape = (P, M, K) if conv is None else (P,) + tuple(conv)
    self.a_pl = torch.randint(-self.vmax, self.vmax + 1, a_shape, generator=g).to(torch.bfloat16)
    self.w_pl = torch.randint(-self.vmax, self.vmax + 1, (P, N, K), generator=g).to(torch.bfloat16)
    self._pair = {}

  def pair(self, i, j):
    """A_i . B_j in float64, [M, N]."""
    if (i, j) not in self._pair:
      a, w = self.a_pl[i].double(), self.w_pl[j].double()
      if self.conv is None:
        t = a @ w.t()
      else:
        C = self.conv[3]
        wt = w.reshape(self.N, 3, 3, C).permute(0, 3, 1, 2)
        t = torch.nn.functional.conv2d(a.permute(0, 3, 1, 2), wt, padding=1)
        t = t.permute(0, 2, 3, 1).reshape(self.M, self.N)
      self._pair[(i, j)] = t
    return self._pair[(i, j)]

  def model(self, pairs):
    """sum over `pairs` (repeats counted) of A_i . B_j, float64 [M, N]."""
    acc = torch.zeros(self.M, self.N, dtype=torch.float64)
    for i, j in pairs:
      acc += self.pair(i, j)
    return acc

  def abs_bound(self):
    """max over outputs of sum_k over all P^2 pairs of |a_i||b_j|: what every partial sum of
    either model stays below."""
    a = self.a_pl.double().abs().sum(0)
    w = self.w_pl.double().abs().sum(0)
    if self.conv is None:
      return float((a @ w.t()).max())
    C = self.conv[3]
    wt = w.reshape(self.N, 3, 3, C).permute(0, 3, 1, 2)
    return float(torch.nn.functional.conv2d(a.permute(0, 3, 1, 2), wt, padding=1).max())


# name -> (M, N, K, P, conv).  Ragged M and N everywhere (partial last tiles at BLOCK_N 64 and
# 128); 'small' has M < 128; 'multi' gives some CTAs several tiles at either tile width (plain:
# 70 x 3 or 70 x 5 tiles; conv64_multi: 150 generic, 180 halo tiles on 132 SMs); 'longk' is the
# longest K with |v| = 7 at P = 3 (9 x 1024); 'splitk' splits K into 8 slices.
SPECS = {}
for _P in (1, 2, 3):
  SPECS[f'small_p{_P}'] = (100, 200, 192, _P, None)
  SPECS[f'multi_p{_P}'] = (8923, 300, 320, _P, None)
  SPECS[f'conv64_p{_P}'] = (None, 64, None, _P, (3, 33, 13, 64))
  SPECS[f'conv128_p{_P}'] = (None, 96, None, _P, (2, 20, 24, 128))
for _P in (1, 2):
  SPECS[f'conv64_multi_p{_P}'] = (None, 64, None, _P, (30, 33, 13, 64))
for _P in (2, 3):
  SPECS[f'splitk_p{_P}'] = (300, 389, 2048, _P, None)
SPECS['longk_p3'] = (100, 200, 9216, 3, None)

_DESIGNS = {}


def design(name):
  if name not in _DESIGNS:
    M, N, K, P, conv = SPECS[name]
    _DESIGNS[name] = Design(name, M, N, K, P, conv)
  return _DESIGNS[name]


def gapped_a(a_pl, conv=None, device='cuda'):
  """(buffer, view): a_pl copied into a NaN-filled buffer, planes GAP_ROWS rows further apart than
  they need, plain rows PAD_COLS columns wider than K.  view has a_pl's shape and those strides."""
  P = a_pl.shape[0]
  if conv is None:
    _, M, K = a_pl.shape
    lda = K + PAD_COLS
    stride = (M + GAP_ROWS) * lda
    buf = torch.full((P * stride,), float('nan'), dtype=torch.bfloat16, device=device)
    view = buf.as_strided((P, M, K), (stride, lda, 1))
  else:
    C = conv[3]
    per = a_pl[0].numel()
    stride = per + GAP_ROWS * C
    buf = torch.full((P * stride,), float('nan'), dtype=torch.bfloat16, device=device)
    view = buf.as_strided(tuple(a_pl.shape), (stride,) + tuple(a_pl[0].stride()))
  view.copy_(a_pl)
  return buf, view


# ------------------------------------------------------------------------------- tile coverage
def m_tile_ids(d):
  """[(name, tile id [M])]: the output tiles' rows, plain 128-row tiles, or the generic and the
  halo convolution's pixel tiles."""
  if d.conv is None:
    return [('rows128', np.arange(d.M) // 128)]
  Fr, H, W, _ = d.conv
  f, y, x = np.meshgrid(np.arange(Fr), np.arange(H), np.arange(W), indexing='ij')
  out = []
  for name, (tw, th) in (('generic', choose_conv_tile(H, W)), ('halo', (8, 16))):
    tx = -(-W // tw)
    ty = -(-H // th)
    out.append((name, ((f * ty + y // th) * tx + x // tw).reshape(-1)))
  return out


def untouched_tiles(changed, d):
  """Number of (m-tile, 64-column) output tiles, over every tiling of d, where `changed` [M, N]
  (bool numpy) has no element set."""
  cols = -(-d.N // 64)
  ch = np.zeros((changed.shape[0], cols), bool)
  for c in range(cols):
    ch[:, c] = changed[:, 64 * c:64 * c + 64].any(1)
  missing = 0
  for _, ids in m_tile_ids(d):
    per = np.zeros((ids.max() + 1, cols), bool)
    np.logical_or.at(per, ids, ch)
    missing += int((~per).sum())
  return missing


def fp32_bits(x):
  """float64 torch / numpy -> int32 bits of its fp32 rounding."""
  x = x.numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
  return x.astype(f32).view(np.int32)


def matching_sets(got, d, sets):
  """Names of the sets in `sets` whose fp32 model equals `got` ([M, N] fp32) bit for bit."""
  g = fp32_bits(got)
  return [name for name, pairs in sets.items() if np.array_equal(g, fp32_bits(d.model(pairs)))]


# ------------------------------------------------------------------------ cost-volume designs
# The cost volume cv[n, cell] = sum over the six pairs i + j < 3 of q_i . g_j, where tapir_split_planes
# splits each fp32 query and grid value into three round-to-nearest-even bf16 planes.  Each query n
# of a clip reads four channels 4 n .. 4 n + 3 and nothing else: a probe channel holding
# Q_PROBE = 1 + 2^-9 + 2^-18, whose planes are (1, 2^-9, 2^-18), and three offset channels holding 1.
# Its map at frame t has two candidate cells, a and b; every other cell is 0 on those channels.
# Cell a holds G_A = 32 + 2^-5 + 2^-15 on the probe channel, planes (32, 2^-5, 2^-15), so each pair
# adds its own power of two to cv[a] (PAIR_TERMS).  Cell b holds, depending on the map's kind:
#   'drop (i, j)' (i, j) != (0, 0)  the three bf16 planes of cv[a] - t_ij / 2 on the offset channels,
#                  which only the (0, 0) pair reads: a wins by t_ij / 2 and loses if any pair whose
#                  term is at least t_ij is missing;
#   'drop (0, 0)'  G_B = 28 + 3 * 2^-6 on the probe channel: a leads by 4 in all six pairs, b leads
#                  in the five without (0, 0), which every offset would lose as well;
#   'gain'         the planes of cv[a] + 2^-16 on the offset channels: b wins by 2^-16 and loses to
#                  any extra term a picks up, such as a plane read in the place of a smaller one.
# Every value has at most 22 significant bits between 2^5 and 2^-16: every sum the GEMM forms, and
# v + 64 and v - 64 in the identity head (a 2^-17 grid below v = 64), is exact.  Pairs the tensor
# cores exclude add at most 2^-22 at |v| ~ 32, below fp32's resolution there: only the GEMM designs
# above can see them.
CV_CHANNELS = 4
Q_PROBE = 1 + 2 ** -9 + 2 ** -18
G_A = 32 + 2 ** -5 + 2 ** -15
G_B = 28 + 3 * 2 ** -6
PAIR_TERMS = {(0, 0): 2.0 ** 5, (0, 1): 2.0 ** -5, (0, 2): 2.0 ** -15, (1, 0): 2.0 ** -4,
              (1, 1): 2.0 ** -14, (2, 0): 2.0 ** -13}
CV_KINDS = tuple(f'drop {p}' for p in tc_pairs(3)) + ('gain',)
CV_MARGIN = 2.0 ** -16  # the least heat gap between a map's two candidates, in any kind


def cv_offsets(kind):
  """The fp32 offset-channel values of cell b (three bf16-exact values), or None."""
  s_a = sum(PAIR_TERMS.values())
  if kind == 'gain':
    e = s_a + CV_MARGIN
  elif kind == 'drop (0, 0)':
    return None
  else:
    e = s_a - PAIR_TERMS[tuple(int(c) for c in kind[6:-1].split(','))] / 2
  pl = split_like_kernel(torch.tensor([e], dtype=torch.float32), 3)
  assert pl.double().sum().item() == e, (kind, e)
  return pl.float()[:, 0]


CV_GROUPS = 64  # channel groups of C = 256: query n of a clip reads group n mod 64


class CvDesign:
  """The designed maps of B = len(counts) clips, counts[b] queries in clip b: query features qf
  [sum counts, C] (the clips' queries one after the other; the batched form is counts = [N] * B)
  and grids [B, T, gh, gw, C] (fp32), and per map (query q, frame t) its kind (index into
  CV_KINDS) and candidate cells a, b, [Q, T].

  Query n of a clip reads channel group n mod 64: queries n >= 64 repeat query n mod 64's map and
  so its outputs, bit for bit.  Each clip draws its own candidate cells, and its channels outside
  the groups its queries read hold random values: a query that reads another clip's grid rows
  finds another arg-max.  clip [Q] and rank [Q] are each query's clip and index within it."""

  def __init__(self, counts, T, gh, gw, C=256, seed=0):
    assert C == CV_CHANNELS * CV_GROUPS
    self.counts = [int(n) for n in counts]
    B = len(self.counts)
    self.B, self.T, self.gh, self.gw, self.C = B, T, gh, gw, C
    self.Q = sum(self.counts)
    self.clip = torch.tensor([b for b, n in enumerate(self.counts) for _ in range(n)])
    self.rank = torch.cat([torch.arange(n) for n in self.counts])
    self.group = self.rank % CV_GROUPS
    cells = gh * gw
    g = torch.Generator().manual_seed(seed + 1000 * gh + gw)
    self.qf = _probe_rows(C)[self.group].contiguous()
    # channels no query of the clip reads: any finite values (a query is zero there)
    self.grid = torch.randn(B, T, gh, gw, C, generator=g)
    # per (clip, group, frame); a query's map is that of (its clip, its group)
    kind = torch.zeros(B, CV_GROUPS, T, dtype=torch.int64)
    cell_a, cell_b = torch.zeros_like(kind), torch.zeros_like(kind)
    flat = self.grid.view(B, T, cells, C)
    k = 0
    for b in range(B):
      used = min(self.counts[b], CV_GROUPS)
      flat[b, :, :, :CV_CHANNELS * used] = 0
      for n in range(used):
        for t in range(T):
          kd = CV_KINDS[k % len(CV_KINDS)]
          ca, cb = torch.randperm(cells, generator=g)[:2].tolist()
          c0 = CV_CHANNELS * n
          flat[b, t, ca, c0] = G_A
          if kd == 'drop (0, 0)':
            flat[b, t, cb, c0] = G_B
          else:
            flat[b, t, cb, c0 + 1:c0 + CV_CHANNELS] = cv_offsets(kd)
          kind[b, n, t], cell_a[b, n, t], cell_b[b, n, t] = k % len(CV_KINDS), ca, cb
          k += 1
    self.kind = kind[self.clip, self.group]
    self.cell_a = cell_a[self.clip, self.group]
    self.cell_b = cell_b[self.clip, self.group]

  def winner(self):
    """[Q, T] the cell each map's design makes the arg-max."""
    gain = self.kind == CV_KINDS.index('gain')
    return torch.where(gain, self.cell_b, self.cell_a)

  def _maps(self, acc):
    """[B, 64, T, cells] per (clip, channel group) -> [Q, T, cells] per query."""
    return acc[self.clip, self.group]

  def heat(self, pairs, dtype=torch.float32):
    """The identity head's heat (temperature 1) of every map, [Q, T, cells]: the cost volume
    summed over `pairs` (repeats counted) in fp32, pair by pair in order and channel by channel, as
    the GEMM orders its terms, then fp32(fp32(v + 64) - 64).  dtype float64: the same sums exact."""
    B, T, C = self.B, self.T, self.C
    cells = self.gh * self.gw
    qp = split_like_kernel(_probe_rows(C), 3).to(dtype)
    gp = split_like_kernel(self.grid.reshape(-1, C), 3).to(dtype).view(3, B, T, cells, CV_GROUPS, CV_CHANNELS)
    # [3, 64, 4]: the planes of the channels each group's queries read
    qg = torch.stack([qp[:, n, CV_CHANNELS * n:CV_CHANNELS * (n + 1)] for n in range(CV_GROUPS)], 1)
    acc = torch.zeros(B, T, cells, CV_GROUPS, dtype=dtype)
    for i, j in pairs:
      for c in range(CV_CHANNELS):
        # fp32 products of two bf16 values are exact; each add rounds as the accumulator does
        acc += qg[i, :, c] * gp[j, ..., c]
    return self._maps(((acc + 64.0) - 64.0).permute(0, 3, 1, 2))

  def heat_simt(self):
    """The identity head's heat as the SIMT kernel makes it, [Q, T, cells]: a = sum of the query's
    planes and b = sum of the grid's (both exact: the planes split an fp32 value), then one fp32
    FMA per channel, acc = fp32(a b + acc), channel by channel from 0.  a b + acc is exact in
    float64 here (at most 48 + 2 significant bits), so rounding it once to fp32 is the FMA."""
    B, T, C = self.B, self.T, self.C
    cells = self.gh * self.gw
    q = _probe_rows(C).view(CV_GROUPS, CV_GROUPS, CV_CHANNELS).double()
    qg = torch.stack([q[n, n] for n in range(CV_GROUPS)])  # [64, 4]: the channels each group reads
    gr = self.grid.view(B, T, cells, CV_GROUPS, CV_CHANNELS).double()
    acc = torch.zeros(B, T, cells, CV_GROUPS, dtype=torch.float32)
    for c in range(CV_CHANNELS):
      acc = (qg[:, c] * gr[..., c] + acc.double()).float()
    return self._maps(((acc + 64.0) - 64.0).permute(0, 3, 1, 2))

  @staticmethod
  def argmax(heat):
    """Arg-max over the last dimension, the lowest index winning ties (as the heads)."""
    m = heat.max(-1, keepdim=True).values
    idx = torch.arange(heat.shape[-1]).expand_as(heat)
    return torch.where(heat == m, idx, heat.shape[-1]).min(-1).values


def _probe_rows(C):
  """[64, C] the query feature of each channel group."""
  probe = torch.zeros(CV_GROUPS, C)
  for n in range(CV_GROUPS):
    probe[n, CV_CHANNELS * n] = Q_PROBE
    probe[n, CV_CHANNELS * n + 1:CV_CHANNELS * n + CV_CHANNELS] = 1.0
  return probe

  @staticmethod
  def argmax(heat):
    """Arg-max over the last dimension, the lowest index winning ties (as the heads)."""
    m = heat.max(-1, keepdim=True).values
    idx = torch.arange(heat.shape[-1]).expand_as(heat)
    return torch.where(heat == m, idx, heat.shape[-1]).min(-1).values
