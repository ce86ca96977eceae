"""GEMM operands whose fp32 accumulators are exactly known, the epilogue's arithmetic on them, and a
mirror of gemm_tc.cu's epilogue dispatch.

The exact-accumulator contract.  A is integer-valued with |a| < 2^11 (so most entries above 256
need a second bf16 plane, and none a third), B is bf16-exact, and column n of B is an integer
times 2^-s_n.  B's planes 1 and 2 are zero and so is A's plane 2: only the pairs (0, 0) and (1, 0)
are nonzero, and every kernel that sums those two gives the same accumulator whatever else it sums
or drops.  These designs test the epilogue; tests/plane_pairs.py tests the plane pairs.  Every
product is then an integer times 2^-s_n, and when sum_k |a||b| < 2^(22 - s_n) every partial sum in
any order is exact in fp32 with two bits to spare for the wgmma adder.  So wgmma at either tile
width and schedule, split-K, the halo convolution and the SIMT kernel all hold the same
accumulator, planes_matmul_fp64 of the planes.  The epilogue after it (bias add, residual add, bf16
round-to-nearest-even planes, fp32 statistics partials) is IEEE arithmetic that numpy float32 and
torch's bf16 conversion reproduce, so outputs are known bit for bit.  Only tanh-GELU is not: it
goes through ex2.approx / rcp.approx and is checked against tests/refine_refs.py's bound.

Three design families:
  R (rounding)   accumulator ~ N(0, 20^2) on a 2^-12 grid, random fp32 bias and residual of the
                 same size: (acc + b) + r and (acc + r) + b differ in a sizeable share of elements.
  S (statistics) integer accumulator, bias and residual with |v| <= 1000: the per-warp fp32 partials
                 (16 v^2 < 2^24) and the fp64 atomics are exact, so the fused InstanceNorm sums
                 equal int64 sums.
  G (GELU)       pre-activation v = fp32(acc + b) spans [-12, 12]; a few columns are scaled by 2^8 so
                 that exp overflows (v << 0) or the reciprocal flushes to zero.

The operand planes are built here with torch on the CPU, not by tapir_split_planes, so that these
designs do not depend on the kernel tests/test_gemm_exact_gpu.py also tests."""
import math

import numpy as np
import torch

from tests.backbone_refs import U32
from tests.gpu_util import conv_planes_fp64, planes_matmul_fp64, split_like_kernel
from tests.refine_refs import GELU_K, gelu_exact, gelu_rel_error

f32 = np.float32
A_MAX = 2047     # |a| < 2^11
EXACT_UNITS = 2.0 ** 22  # sum_k |a||b| bound, in units of the column's 2^-s grid
SMS = 132        # H100 SXM: the split-K and tile-width choices below depend on it
LARGE_COLS = 4   # G designs: columns scaled by 2^8


# ------------------------------------------------------------------------------------ designs
class Design:
  """a_pl [P, M, K] bf16 (plain) or [P, F, H, W, C] (conv); w_pl [P, N, K] bf16; bias [N] fp32 or
  None; resid [M, N] fp32 or None; acc [M, N] float64, the exact accumulator; units [N], the
  exponent s_n of column n's grid (acc[:, n] * 2^s_n is an integer); rows_per_frame (statistics)."""

  def __init__(self, **kw):
    self.__dict__.update(kw)

  @property
  def M(self):
    return self.acc.shape[0]

  @property
  def N(self):
    return self.acc.shape[1]

  @property
  def P(self):
    return self.w_pl.shape[0]


def _accumulate(a_pl, w_pl, conv):
  return conv_planes_fp64(a_pl, w_pl) if conv else planes_matmul_fp64(a_pl, w_pl)


def _ib_max(K):
  """The largest |b| integer range 1..7 whose expected sum_k |a||b| stays below 2^21 units."""
  for m in range(7, 0, -1):
    if K * (A_MAX + 1) / 2 * (m * (m + 1) / (2 * m + 1)) <= 2.0 ** 21:
      return m
  return 1


def _a_planes(g, rows, K, P, amax):
  a = torch.randint(-amax, amax + 1, (rows, K), generator=g).float()
  return split_like_kernel(a, P)


def make_design(kind, seed, M, N, K, P, conv=None, rows_per_frame=0):
  """kind 'R', 'S' or 'G'.  conv = (F, H, W, C): then M = F H W and K = 9 C."""
  g = torch.Generator().manual_seed(seed)
  if conv is not None:
    Fr, H, W, C = conv
    M, K = Fr * H * W, 9 * C
  rows, cols = M, (K if conv is None else conv[3])  # conv: A is the NHWC activation
  if kind == 'S':
    a_pl = _a_planes(g, rows, cols, P, 450)
    # two +-1 entries per output column: |acc| <= 900, |bias|, |resid| <= 50
    ib = torch.zeros(N, K)
    for n in range(N):
      k = torch.randperm(K, generator=g)[:2]
      ib[n, k] = torch.randint(0, 2, (2,), generator=g).float() * 2 - 1
    s = torch.zeros(N)
    bias = torch.randint(-50, 51, (N,), generator=g).float()
    resid = torch.randint(-50, 51, (M, N), generator=g).float()
  else:
    a_pl = _a_planes(g, rows, cols, P, A_MAX)
    m = _ib_max(K)
    ib = torch.randint(-m, m + 1, (N, K), generator=g).float()
    # accumulator standard deviation ~ 20 (R) or ~ 5 (G) on the column's grid
    sd = math.sqrt(K) * (A_MAX / math.sqrt(3)) * math.sqrt(m * (m + 1) / 3)
    s = torch.full((N,), float(round(math.log2(sd / (20 if kind == 'R' else 5)))))
    if kind == 'G':
      s[torch.randperm(N, generator=g)[:LARGE_COLS]] -= 8
    if kind == 'R':
      bias = (torch.randn(N, generator=g) * 20).float()
      resid = (torch.randn(M, N, generator=g) * 20).float()
    else:
      bias = (torch.rand(N, generator=g) * 6 - 3).float()
      resid = (torch.randn(M, N, generator=g) * 2).float()
  w = ib * torch.exp2(-s)[:, None]
  w_pl = torch.zeros(P, N, K, dtype=torch.bfloat16)
  w_pl[0] = w.to(torch.bfloat16)
  assert torch.equal(w_pl[0].float(), w), 'B must be bf16-exact'
  if conv is not None:
    a_pl = a_pl.reshape(P, *conv)
  acc = _accumulate(a_pl, w_pl, conv)
  return Design(kind=kind, a_pl=a_pl, w_pl=w_pl, bias=bias, resid=resid, acc=acc, units=s,
                conv=conv, rows_per_frame=rows_per_frame or (M if conv is None else conv[1] * conv[2]))


def abs_sum_units(d):
  """sum_k |a||b| of every output element in units of its column's grid: every partial sum the
  kernels form is bounded by it."""
  a_abs = d.a_pl.float().abs().sum(0, keepdim=True)
  w_abs = d.w_pl[:1].float().abs()
  return _accumulate(a_abs, w_abs, d.conv) * torch.exp2(d.units.double())[None, :]


def plane1_fraction(d):
  """Share of A's elements whose plane 1 is non-zero."""
  return (d.a_pl[1] != 0).double().mean().item() if d.P > 1 else 0.0


# ------------------------------------------------------------------------------------ emulation
def _np(t):
  return t.numpy() if isinstance(t, torch.Tensor) else t


def pre_activation(d, bias):
  """fp32 acc (+ bias): exact accumulator, then one IEEE add."""
  v = _np(d.acc).astype(f32)
  return (v + _np(d.bias)[None, :]).astype(f32) if bias else v


def emulate(d, bias, resid, out_P=0, stats=False, variant=None):
  """The epilogue without GELU on design d, bit for bit: dict(out [M, N] fp32 numpy, planes
  [out_P, M, N] bf16 torch or None, stats [frames, N, 2] float64 or None).

  variant names a deliberate slip that tests/test_gemm_exact_host.py shows the designs detect:
  'resid_first' (residual added before the bias), 'planes_rtz' (planes rounded toward zero),
  'stats_before_resid' (statistics of the value before the residual add)."""
  acc = _np(d.acc).astype(f32)
  b, r = _np(d.bias)[None, :], _np(d.resid)
  if variant == 'resid_first' and bias and resid:
    v = ((acc + r).astype(f32) + b).astype(f32)
  else:
    v = (acc + b).astype(f32) if bias else acc
    pre = v
    v = (v + r).astype(f32) if resid else v
  res = dict(out=v, planes=None, stats=None)
  if out_P:
    vt = torch.from_numpy(v.copy())
    res['planes'] = split_rtz(vt, out_P) if variant == 'planes_rtz' else split_like_kernel(vt, out_P)
  if stats:
    src = pre if variant == 'stats_before_resid' and resid else v
    x = src.astype(np.float64)
    assert np.array_equal(x, np.round(x)) and np.abs(x).max() <= 1000, 'statistics need S designs'
    xi = x.astype(np.int64).reshape(-1, d.rows_per_frame, d.N)
    res['stats'] = np.stack([xi.sum(1), (xi * xi).sum(1)], -1).astype(np.float64)
  return res


def split_rtz(v, planes):
  """split_like_kernel with every plane rounded toward zero (a wrong kernel, for the host test)."""
  out, r = [], v.float().clone()
  for _ in range(planes):
    h = (r.view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16)
    r = r - h.float()
    out.append(h)
  return torch.stack(out)


def order_sensitivity(d):
  """Share of elements where (acc + r) + b differs from (acc + b) + r."""
  a = emulate(d, True, True)['out']
  b = emulate(d, True, True, variant='resid_first')['out']
  return float((a.view(np.int32) != b.view(np.int32)).mean())


def gelu_reference(a):
  """refine_refs.gelu_exact in the equivalent form a * sigmoid(2 k (a + 0.044715 a^3)): float64's
  1 + tanh(z) cancels below a ~ -6 (absolute error ~1e-16 where the value is ~1e-15)."""
  return a * torch.sigmoid(2 * GELU_K * (a + 0.044715 * a ** 3))


def gelu_bound(v, resid=None):
  """(reference, tolerance): the largest |out - (gelu(v) [+ resid])| the kernel's tanh-GELU may
  give is tests/refine_refs.py's relative bound, plus 2^-120 for results the ftz reciprocal
  flushes, plus with a residual the rounding of the final add (which may also be fused with GELU's
  last multiply)."""
  vd = torch.from_numpy(np.asarray(v, dtype=np.float64))
  ge = gelu_reference(vd)
  tol = gelu_rel_error(vd) * ge.abs() + 2.0 ** -120
  want = ge
  if resid is not None:
    rd = torch.from_numpy(np.asarray(resid, dtype=np.float64))
    want = ge + rd
    tol = tol + 2 * U32 * (ge.abs() + rd.abs())
  return want, tol


# ----------------------------------------------------------------------- dispatch mirror
# epilogue()'s whole-tile option sets: (bias, gelu, resid, f32, planes, stats)
FULL_SETS = [(b, True, False, False, 2, False) for b in (True, False)] + [
    (b, False, r, True, 0, s) for b in (True, False) for r in (True, False) for s in (True, False)]


def choose_conv_tile(H, W):
  best = None
  for w in (128, 64, 32, 16, 8):
    h = 128 // w
    tiles = -(-W // w) * -(-H // h)
    if best is None or tiles < best[0]:
      best = (tiles, w, h)
  return best[1], best[2]


def _small_problem(m_tiles, N, sms):
  return m_tiles * -(-N // 128) * 10 < sms * 6


def pick_block_n(m_tiles, N, sms=SMS, force=None):
  if force in (64, 128):
    return force
  if N <= 64:
    return 64
  if _small_problem(m_tiles, N, sms) and m_tiles * -(-N // 128) * 2 <= sms:
    return 64
  return 128


def option_set(bias, gelu, resid, f32_out, out_P, stats):
  return (bool(bias), bool(gelu), bool(resid), bool(f32_out), int(out_P), bool(stats))


def set_name(opts):
  b, g, r, f, pl, s = opts
  parts = [n for n, on in (('bias', b), ('gelu', g), ('resid', r), ('f32', f), ('stats', s)) if on]
  if pl:
    parts.append(f'planes{pl}')
  return '+'.join(parts) or 'none'


def reached(M, N, K, P, opts, conv=None, ld_pad=0, offset=0, block_n=None, splitk=False,
            halo=True, sms=SMS):
  """The epilogue code a gemm_exact GPU run reaches, as a set of labels: 'full/<BLOCK_N>/<set>' for
  an epilogue_full instantiation, 'general/<set>' for the general loop (only lanes that own an
  output element count), 'splitk_reduce/<set>' for split-K's second pass.  The layout follows
  tests/gpu_util.gemm: output, residual and planes share ld = N + ld_pad, and the fp32 output and
  residual start `offset` floats into 256-byte aligned allocations."""
  bias, gelu, resid, f32_out, out_P, stats = opts
  ld = N + ld_pad
  vec_r = resid and ld % 2 == 0 and offset % 2 == 0
  vec_o = f32_out and ld % 2 == 0 and offset % 2 == 0
  vec_p = out_P > 0 and ld % 2 == 0 and (M * ld) % 2 == 0
  nkb = K // 64
  labels = set()
  is_halo = conv is not None and halo and conv[3] == 64 and N == 64 and P <= 2 and out_P == 0
  if conv is not None:
    Fr, H, W, C = conv
    tw, th = (8, 16) if is_halo else choose_conv_tile(H, W)
    tx, ty = -(-W // tw), -(-H // th)
    m_tiles = Fr * tx * ty
  else:
    m_tiles = -(-M // 128)
  bn = 64 if is_halo else pick_block_n(m_tiles, N, sms, block_n)
  # split-K: the first pass stores raw fp32 partials with no other option, the second applies them
  splittable = splitk and not is_halo and not stats and nkb >= 32
  if splittable and bn == 64 and N > 64 and _small_problem(m_tiles, N, sms) and \
      m_tiles * -(-N // 128) * 2 <= sms and block_n is None:
    bn = 128
  n_tiles = -(-N // bn)
  S = 1
  if splittable and m_tiles * n_tiles * 2 <= sms:
    S = min(sms // (m_tiles * n_tiles), 8, nkb // 4)
  if S > 1:
    labels.add('splitk_reduce/' + set_name(opts))
    opts = option_set(False, False, False, True, 0, False)
    bias, gelu, resid, f32_out, out_P, stats = opts
    vec_o, vec_r, vec_p = True, False, False  # the workspace rows are padded to 8 floats
  full_ok = False
  if not gelu and out_P == 0 and vec_o and (not resid or vec_r):
    full_ok = opts in FULL_SETS
  if gelu and not resid and not stats and not f32_out and out_P == 2 and vec_p:
    full_ok = opts in FULL_SETS
  # per lane: rows r0 = r_base + 16 warp + lane / 4 and r0 + 8 of the 128-row tile
  r0 = (np.arange(2)[:, None, None] * 64 + np.arange(4)[None, :, None] * 16 +
        np.arange(8)[None, None, :]).reshape(-1)
  rr = np.stack([r0, r0 + 8])  # [2, 64]
  for mt in range(m_tiles):
    if conv is not None:
      f, t = divmod(mt, tx * ty)
      y = (t // tx) * th + rr // tw
      x = (t % tx) * tw + rr % tw
      ok = (y < H) & (x < W)
    else:
      ok = mt * 128 + rr < M
    both = ok[0] & ok[1]
    some = ok[0] | ok[1]
    for n0 in range(0, N, bn):
      full = both & (n0 + bn <= N) & full_ok
      if full.any():
        labels.add(f'full/{bn}/{set_name(opts)}')
      if (some & ~full).any():
        labels.add('general/' + set_name(opts))
  return labels


# --------------------------------------------------------------------------------- cases
def _sets(*specs):
  return [option_set(*s) for s in specs]


R_SETS = _sets((False, False, False, True, 0, False), (True, False, False, True, 0, False),
               (False, False, True, True, 0, False), (True, False, True, True, 0, False),
               (True, False, True, True, 1, False), (True, False, True, True, 2, False),
               (True, False, True, True, 3, False))
S_SETS = _sets(*[(b, False, r, True, 0, True) for b in (True, False) for r in (True, False)])
G_SETS = _sets((True, True, False, False, 2, False), (False, True, False, False, 2, False),
               (True, True, False, True, 2, False), (True, True, False, False, 1, False),
               (True, True, False, False, 3, False), (True, True, True, True, 0, False))


class Case:
  def __init__(self, cid, kind, M, N, K, P, sets, conv=None, rows_per_frame=0, splitk=False):
    self.cid, self.kind, self.P, self.sets, self.conv, self.splitk = cid, kind, P, sets, conv, splitk
    self.rows_per_frame = rows_per_frame
    if conv is not None:
      M, K = conv[0] * conv[1] * conv[2], 9 * conv[3]
    self.M, self.N, self.K = M, N, K
    self._design = None

  def design(self):
    if self._design is None:
      self._design = make_design(self.kind, sum(map(ord, self.cid)), self.M, self.N, self.K, self.P,
                                 self.conv, self.rows_per_frame)
    return self._design


CASES = [
    Case('plain_r_p1', 'R', 1000, 200, 256, 1, R_SETS),
    Case('plain_r_p2', 'R', 1000, 200, 256, 2, R_SETS),
    Case('plain_r_p3', 'R', 1000, 200, 256, 3, R_SETS),
    Case('plain_s', 'S', 1024, 192, 256, 2, S_SETS, rows_per_frame=256),
    Case('plain_g', 'G', 1000, 256, 512, 2, G_SETS),
    Case('conv_s', 'S', None, 128, None, 2, S_SETS, conv=(2, 20, 24, 64)),
    Case('conv_g', 'G', None, 256, None, 2, G_SETS, conv=(2, 16, 32, 128)),
    Case('halo_s', 'S', None, 64, None, 2, S_SETS, conv=(3, 33, 13, 64)),
    Case('splitk_r', 'R', 300, 512, 2048, 2, R_SETS[3:4], splitk=True),
    Case('splitk_g', 'G', 300, 389, 2048, 2, G_SETS[:1], splitk=True),
]
LAYOUTS = {'aligned': (0, 0), 'unaligned': (1, 1)}  # (ld_pad, offset) of tests/gpu_util.gemm
