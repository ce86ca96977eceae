"""Float64 references of the refinement kernels (local correlation, the mixer's depthwise block,
pyramid pooling, the track update) and the error bounds of their fp32 arithmetic.
tests/test_refine_ops_gpu.py compares the kernels with them; tests/test_refine_refs_host.py checks
the references against the oracle and the bounds against fp32 emulations of the kernels' operation
order.

Every reference takes CPU tensors and returns float64 tensors; every bound is an absolute,
per-element tolerance in the standard model of tests/backbone_refs.py (gamma, U32).  Pooling and
the update replay the reference's operation order, so they have fp32 emulations to compare with
bit for bit instead of bounds."""
import numpy as np
import torch

from tests.backbone_refs import U32, U64, gamma, layernorm_ref

f32 = np.float32
BOX_ROWS = 8       # refine.cu kBoxRows: cell rows of the box path
BOX_COLS_MAX = 16  # refine.cu kBoxColsMax: wider boxes take the per-sample path
PAD = 4            # zero cells around the dot tables (samples far outside clamp into them)
OFFSETS = np.arange(-3, 4)


# ------------------------------------------------------------------------------- coordinates
def pix_f32(p, g, init, gh, size, d):
  """The kernel's fp32 coordinate chain (refine.cu local_corr_kernel), every operation rounded:
  c = p * g / init, then ((2 * ((c + d) / gh) - 1 + 1) * size - 1) / 2.  p fp32 array; g = gw
  (x) or gh (y); size likewise; d the sample offset.  Returns fp32."""
  c = ((p.astype(f32) * f32(g)).astype(f32) / f32(init)).astype(f32)
  a = (c + f32(d)).astype(f32)
  b = (a / f32(gh)).astype(f32)
  g2 = ((f32(2) * b).astype(f32) - f32(1)).astype(f32)
  s = ((g2 + f32(1)).astype(f32) * f32(size)).astype(f32)
  return ((s - f32(1)).astype(f32) / f32(2)).astype(f32)


def pix_exact(p, g, init, gh, size, d):
  """utils.py:76-113's sample position, exactly (fp64; x is normalised by h as well):
  ((2 ((c + d) / gh) - 1 + 1) size - 1) / 2 = (c + d) size / gh - 1/2 with c = p g / init."""
  c = p.astype(np.float64) * g / init
  return (c + d) * size / gh - 0.5


def pix_error(p, g, init, gh, size, d):
  """Bound on |pix_f32 - pix_exact| from running the standard model through the eight-operation
  chain (plus the two of c), to first order, with a 16 u margin for the second-order terms."""
  c = np.abs(p.astype(np.float64) * g / init)
  e = gamma(2) * c
  a = c + abs(d)
  e = e + U32 * a
  b = a / gh
  e = e / gh + U32 * b
  e = 2 * e + U32 * (2 * b + 1)        # 2b exact, - 1 rounds
  e = e + U32 * 2 * b                  # + 1 (back to 2b)
  s = 2 * b * size
  e = e * size + U32 * s               # * size
  e = e + U32 * (s + 1)                # - 1;  / 2 is exact
  return (e / 2) * (1 + 16 * U32) + 8 * U64 * (s + 2)


def kernel_box(py, px, h, w, init_hw):
  """The kernel's cell box of each row: (y0, x0, box_w), from its fp32 chain."""
  ih, iw = init_hw
  y0 = np.floor(pix_f32(py, h, ih, h, h, -3)).astype(np.int64)
  x0 = np.floor(pix_f32(px, w, iw, h, w, -3)).astype(np.int64)
  x_last = np.floor(pix_f32(px, w, iw, h, w, 3)).astype(np.int64) + 1
  return y0, x0, np.maximum(x_last - x0 + 1, 2)


# ------------------------------------------------------------------------------- local corr
def _lookup(table, y, x):
  """table [Q, h + 2 PAD, w + 2 PAD] (zero border), y, x [Q, S] integer cell indices (any
  range) -> [Q, S]."""
  Q, Hp, Wp = table.shape
  yy = torch.clamp(y + PAD, 0, Hp - 1)
  xx = torch.clamp(x + PAD, 0, Wp - 1)
  return torch.gather(table.reshape(Q, -1), 1, yy * Wp + xx)


def local_corr_ref(levels, pos, feats, init_hw, batch, planes=3, query_clip=None):
  """levels: fp32 [batch, T, h, w, C] per level (C 128 for level 0, 256 after); pos [Q, T, 2]
  fp32 (x, y) with Q = batch * N queries (query q reads clip q // N), or, given query_clip
  (int [Q]), any Q queries, query q reading clip query_clip[q]; feats = (hi [Q, T, 128],
  lo [Q, T, 256]) per row.  Returns (corr [Q, T, 49 L], bound), corr in float64.

  The samples are taken at pix_exact's positions (the 7 x 7 offsets in grid cells, zero padding)
  and dotted with the row's feature: tapir_model.py:599-631 in exact arithmetic.  The bound
  assumes the kernel's operation order:
    (a) each cell dot is a lane FMA chain of C / 32 terms and a five-level transpose-reduce:
        gamma(C / 32 + 5) sum |f q|, taken over the 4 x 4 cells around the sample;
    (b) fp32 weights (each within 3 u) and the four-term combine: (12 u + gamma(4)) max |dot|;
    (c) the coordinate chain's rounding (pix_error) times the largest difference between
        neighbouring cell dots along that axis (the interpolant's Lipschitz constant);
    (d) a corner the kernel drops because its row leaves the 8-row box (through fp rounding of
        the chain: see test_refine_refs_host.py): its fp32 weight times |dot|;
    (e) the bf16 split: P planes hold the fp32 value within 2^(-8 P) of its magnitude.
  The fp64 reference's own rounding adds gamma_64(C + 8) sum |f q|."""
  ih, iw = init_hw
  Q, T, _ = pos.shape
  clip = torch.arange(Q) // (Q // batch) if query_clip is None else torch.as_tensor(query_clip).long().cpu()
  dy = torch.from_numpy(np.repeat(OFFSETS, 7)).double()
  dx = torch.from_numpy(np.tile(OFFSETS, 7)).double()
  corr = torch.zeros(Q, T, 49 * len(levels), dtype=torch.float64)
  bound = torch.zeros_like(corr)
  for t in range(T):
    px32, py32 = pos[:, t, 0].numpy().astype(f32), pos[:, t, 1].numpy().astype(f32)
    for li, grid in enumerate(levels):
      _, _, h, w, C = grid.shape
      q = (feats[0] if C == 128 else feats[1])[:, t].double()
      D = torch.empty(Q, h * w, dtype=torch.float64)
      A = torch.empty_like(D)
      for b in range(batch):
        g = grid[b, t].double().reshape(h * w, C)
        D[clip == b] = q[clip == b] @ g.t()
        A[clip == b] = q[clip == b].abs() @ g.abs().t()
      D = torch.nn.functional.pad(D.view(Q, h, w), (PAD, PAD, PAD, PAD))
      A = A.view(Q, h, w)
      A = torch.nn.functional.pad(A, (PAD, PAD, PAD, PAD))
      iy = torch.from_numpy(pix_exact(py32[:, None], h, ih, h, h, dy.numpy()[None]))
      ix = torch.from_numpy(pix_exact(px32[:, None], w, iw, h, w, dx.numpy()[None]))
      fy, fx = torch.floor(iy), torch.floor(ix)
      wy1, wx1 = iy - fy, ix - fx
      y0, x0 = fy.long(), fx.long()
      v = ((1 - wy1) * (1 - wx1) * _lookup(D, y0, x0) + (1 - wy1) * wx1 * _lookup(D, y0, x0 + 1) +
           wy1 * (1 - wx1) * _lookup(D, y0 + 1, x0) + wy1 * wx1 * _lookup(D, y0 + 1, x0 + 1))
      amax = torch.zeros_like(v)
      dmax = torch.zeros_like(v)
      lx = torch.zeros_like(v)
      ly = torch.zeros_like(v)
      for a in range(-1, 3):
        for b in range(-1, 3):
          cell = _lookup(D, y0 + a, x0 + b)
          amax = torch.maximum(amax, _lookup(A, y0 + a, x0 + b))
          dmax = torch.maximum(dmax, cell.abs())
          if b < 2:
            lx = torch.maximum(lx, (_lookup(D, y0 + a, x0 + b + 1) - cell).abs())
          if a < 2:
            ly = torch.maximum(ly, (_lookup(D, y0 + a + 1, x0 + b) - cell).abs())
      ey = torch.from_numpy(pix_error(py32[:, None], h, ih, h, h, dy.numpy()[None]))
      ex = torch.from_numpy(pix_error(px32[:, None], w, iw, h, w, dx.numpy()[None]))
      bd = ((gamma(C // 32 + 5) + 4 * gamma(C + 8, U64)) * amax + (12 * U32 + gamma(4)) * dmax +
            lx * ex + ly * ey)
      # (d): the kernel's own cells and weights, from its fp32 chain
      by0, _, box_w = kernel_box(py32, px32, h, w, init_hw)
      iy32 = pix_f32(py32[:, None], h, ih, h, h, dy.numpy()[None])
      ix32 = pix_f32(px32[:, None], w, iw, h, w, dx.numpy()[None])
      fy32, fx32 = np.floor(iy32), np.floor(ix32)
      wy = [((fy32 + 1) - iy32).astype(f32), (iy32 - fy32).astype(f32)]
      boxed = (box_w <= BOX_COLS_MAX)[:, None]
      ky, kx = torch.from_numpy(fy32.astype(np.int64)), torch.from_numpy(fx32.astype(np.int64))
      for r in (0, 1):
        dropped = torch.from_numpy(boxed & (fy32.astype(np.int64) + r - by0[:, None] >= BOX_ROWS))
        corner = torch.maximum(_lookup(D, ky + r, kx).abs(), _lookup(D, ky + r, kx + 1).abs())
        bd = bd + dropped * torch.from_numpy(wy[r].astype(np.float64)).abs() * corner
      bd = bd + 2.0 ** (-8 * planes) * (v.abs() + bd)
      corr[:, t, 49 * li:49 * (li + 1)] = v
      bound[:, t, 49 * li:49 * (li + 1)] = bd
  return corr, bound


def corr_row_head(occ, expd, feats, ld):
  """The exact columns of the mixer input row [Q, T, ld] (fp32): 0, 0, occ, expd, the 384
  features, then (after the 49 L correlations, left 0 here) zero padding."""
  Q, T = occ.shape
  row = torch.zeros(Q, T, ld)
  row[..., 2] = occ
  row[..., 3] = expd
  row[..., 4:132] = feats[0]
  row[..., 132:388] = feats[1]
  return row


# ------------------------------------------------------------------------------- depthwise block
# gelu_tanh2 (common.cuh): x / (1 + 2^u), u = x (A + B x^2), with these fp32 constants
GELU_A = float(f32(-2.3022081983))
GELU_B = float(f32(-0.1029432396))
GELU_K = float(np.sqrt(2 / np.pi))
# Relative errors of the two MUFU approximations.  These are the one input to the bound not derived
# here: the PTX ISA manual (sections "Floating Point Instructions: ex2" and "...: rcp") gives
# ex2.approx.ftz.f32 within 2 ulp and rcp.approx.ftz.f32 within 1 ulp of the exact result across
# the range of inputs; the bound uses twice those, 2^-21 and 2^-22.
EX2_REL = 2.0 ** -21
RCP_REL = 2.0 ** -22
GELU_LIP = 1.13  # max |d/da gelu_tanh(a)| (1.129 near a = 2.4)


def gelu_exact(a):
  """F.gelu(a, approximate='tanh') in float64 with exact tanh."""
  return 0.5 * a * (1 + torch.tanh(GELU_K * (a + 0.044715 * a ** 3)))


def gelu_rel_error(a):
  """Relative error of gelu_tanh2's fp32 evaluation at a (fp64 tensor): the rounding of u
  (x * x, the FMA, the product: gamma(3)) and of the constants A, B feed 2^u, whose relative error
  ln 2 |du| + EX2_REL reaches the output scaled by 2^u / (1 + 2^u); then 1 + e, rcp and x * r."""
  dA = abs(GELU_A + 2 * GELU_K / np.log(2))
  dB = abs(GELU_B + 2 * GELU_K * 0.044715 / np.log(2))
  u = a * (GELU_A + GELU_B * a * a)
  du = gamma(3) * u.abs() + a.abs() * (dA + dB * a * a)
  s = torch.sigmoid(u * np.log(2))  # 2^u / (1 + 2^u)
  return (np.log(2) * du + EX2_REL) * s + RCP_REL + 2 * U32


def _conv_taps(seq, causal):
  """seq [n, F, C] frames of the conv input, causal: F = T + 2 (frames -2 .. T-1), else F = T
  (zero padded here) -> the three taps [3, n, T, C] of every output frame."""
  if causal:
    T = seq.shape[1] - 2
    return torch.stack([seq[:, k:k + T] for k in range(3)])
  p = torch.nn.functional.pad(seq, (0, 0, 1, 1))
  T = seq.shape[1]
  return torch.stack([p[:, k:k + T] for k in range(3)])


def mixer_dw_ref(block_sd, x, causal, ctx1=None, ctx2=None, planes=3):
  """block_sd: {'ln_w' [512], 'w1' [2048, 1, 3], 'b1', 'w2' [2048, 1, 3], 'b2', 'ln1_w'}; x
  [n, T, 512] fp32; ctx1 [n, 2, 512] / ctx2 [n, 2, 2048] (causal only; None = zero context).
  Returns dict of float64 (value, bound) pairs: 'z', 'planes' (LN_1(z) w1, the sum of the
  planes), 'ctx1', 'ctx2' (the new contexts; causal only).

  nets.py:143-181 as oracle.mixer restates it: y = LN(x) w; causal: [ctx1 | y] with two more zero
  frames in front, else one zero frame each side; h = gelu_tanh(dwconv(y) + b1) (exact tanh);
  causal: [ctx2 | h]; dwconv(h) + b2; z = ((m0 + m1) + m2) + m3 + skip.  The bound follows the
  kernel's order: LN as tests/backbone_refs.layernorm_ref; each conv three FMAs (gamma(3) of
  |b| + sum |w v|, plus sum |w| of its inputs' bounds); GELU 1.13-Lipschitz plus gelu_rel_error;
  the group sum gamma(3), the skip one rounding; LN_1 of z at the kernel's z, which moves by
  e_z: |w| rstd (e_z + max e_z (1 + |z - mu| rstd)); planes as local_corr_ref (e)."""
  n, T, C = x.shape
  y, ey = layernorm_ref(x.reshape(-1, C), block_sd['ln_w'])
  y, ey = y.view(n, T, C), ey.view(n, T, C)
  if causal:
    c1 = ctx1.double() if ctx1 is not None else torch.zeros(n, 2, C, dtype=torch.float64)
    Y = torch.cat([c1, y], 1)
    eY = torch.cat([torch.zeros(n, 2, C, dtype=torch.float64), ey], 1)
  else:
    Y, eY = y, ey
  rep = lambda v: v.repeat_interleave(4, -1)  # noqa: E731  input channel c feeds 4c .. 4c + 3
  w1 = block_sd['w1'].double().reshape(4 * C, 3)
  b1 = block_sd['b1'].double()
  taps, etaps = _conv_taps(rep(Y), causal), _conv_taps(rep(eY), causal)
  a = b1 + sum(w1[:, k] * taps[k] for k in range(3))
  ea = (sum(w1[:, k].abs() * etaps[k] for k in range(3)) +
        gamma(3) * (b1.abs() + sum((w1[:, k] * taps[k]).abs() for k in range(3))))
  h = gelu_exact(a)
  eh = GELU_LIP * ea + gelu_rel_error(a) * (h.abs() + GELU_LIP * ea) + a.abs() * 2.0 ** -120
  if causal:
    c2 = ctx2.double() if ctx2 is not None else torch.zeros(n, 2, 4 * C, dtype=torch.float64)
    H = torch.cat([c2, h], 1)
    eH = torch.cat([torch.zeros(n, 2, 4 * C, dtype=torch.float64), eh], 1)
  else:
    H, eH = h, eh
  w2 = block_sd['w2'].double().reshape(4 * C, 3)
  b2 = block_sd['b2'].double()
  taps, etaps = _conv_taps(H, causal), _conv_taps(eH, causal)
  m = b2 + sum(w2[:, k] * taps[k] for k in range(3))
  em = (sum(w2[:, k].abs() * etaps[k] for k in range(3)) +
        gamma(3) * (b2.abs() + sum((w2[:, k] * taps[k]).abs() for k in range(3))))
  m4, em4 = m.view(n, T, C, 4), em.view(n, T, C, 4)
  s = ((m4[..., 0] + m4[..., 1]) + m4[..., 2]) + m4[..., 3]
  es = em4.sum(-1) + gamma(3) * m4.abs().sum(-1)
  z = s + x.double()
  ez = es + U32 * (z.abs() + es)
  # the kernel layer-norms its own z, within ez of this one: LN's fp32 bound there (1.001 times
  # the bound at fp32(z), which is a relative 1e-6 away) plus LN's change under that shift
  _, ep = layernorm_ref(z.float().reshape(-1, C), block_sd['ln1_w'])
  zc = z.reshape(-1, C)
  p = torch.nn.functional.layer_norm(zc, (C,), block_sd['ln1_w'].double(), None, 1e-5)
  mu = zc.mean(-1, keepdim=True)
  rstd = 1 / torch.sqrt(((zc - mu) ** 2).mean(-1, keepdim=True) + 1e-5)
  ezr = ez.reshape(-1, C) + U32 * zc.abs()  # + the rounding of z to fp32 above
  ezmax = ezr.amax(-1, keepdim=True)
  eprop = block_sd['ln1_w'].double().abs() * rstd * (ezr + ezmax * (1 + (zc - mu).abs() * rstd))
  ep = ep * 1.001 + eprop
  ep = ep + 2.0 ** (-8 * planes) * (p.abs() + ep)
  p_exact = p
  out = {'z': (z, ez), 'planes': (p_exact.view(n, T, C), ep.view(n, T, C))}
  if causal:
    out['ctx1'] = (Y[:, -2:], eY[:, -2:])
    out['ctx2'] = (H[:, -2:], eH[:, -2:])
  return out


def block_weights(seed, scale=1.0):
  """Random weights of one block (what synth.make_state_dict draws, at a chosen scale), fp32."""
  g = torch.Generator().manual_seed(seed)
  return {'ln_w': 1 + 0.5 * torch.randn(512, generator=g),
          'w1': scale * 0.5 * torch.randn(2048, 1, 3, generator=g),
          'b1': scale * 0.3 * torch.randn(2048, generator=g),
          'w2': scale * 0.5 * torch.randn(2048, 1, 3, generator=g),
          'b2': scale * 0.3 * torch.randn(2048, generator=g),
          'ln1_w': 1 + 0.5 * torch.randn(512, generator=g)}


# ------------------------------------------------------------------------------- pooling, update
def pool_emulate(grid):
  """grid [T, h, w, C] fp32 -> [T, h // 2, w // 2, C]: the kernel's (((a + b) + c) + d) * 0.25,
  a, b the top pair, c, d the bottom pair, in fp32 (numpy)."""
  g = grid.numpy().astype(f32)
  T, h, w, C = g.shape
  g = g[:, :h // 2 * 2, :w // 2 * 2]
  a, b = g[:, 0::2, 0::2], g[:, 0::2, 1::2]
  c, d = g[:, 1::2, 0::2], g[:, 1::2, 1::2]
  return torch.from_numpy((((((a + b).astype(f32) + c).astype(f32) + d).astype(f32)) * f32(0.25)).astype(f32))


def update_emulate(res, pos, occ, expd, feats, init_hw, resize_hw, video_hw):
  """tapir_model.py:674-685 and train2orig :435-441 in fp32, in the reference's order: res
  [Q, T, >= 388], pos [Q, T, 2] (x, y), occ, expd [Q, T], feats [Q, T, 384]; video_hw (h, w), or
  one (h, w) per query [Q, 2] (a ragged call's size of each query's clip).  Returns (pos, occ,
  expd, feats, tracks): delta = res[:2] * init / resize (multiply, then divide), pos + delta,
  res[2] + occ, res[3] + expd, res[4:388] + feats, tracks = pos * video / init."""
  r = res.numpy().astype(f32)
  p = pos.numpy().astype(f32)
  ih, iw = init_hw
  rh, rw = resize_hw
  v = np.asarray(video_hw, f32)
  vh, vw = (v[0], v[1]) if v.ndim == 1 else (v[:, None, 0], v[:, None, 1])
  d = np.stack([(r[..., 0] * f32(iw)).astype(f32) / f32(rw), (r[..., 1] * f32(ih)).astype(f32) / f32(rh)], -1)
  newp = (d.astype(f32) + p).astype(f32)
  trk = np.stack([(newp[..., 0] * vw).astype(f32) / f32(iw), (newp[..., 1] * vh).astype(f32) / f32(ih)], -1)
  t = torch.from_numpy
  return (t(newp), t((r[..., 2] + occ.numpy()).astype(f32)), t((r[..., 3] + expd.numpy()).astype(f32)),
          t((r[..., 4:388] + feats.numpy()).astype(f32)), t(trk.astype(f32)))
