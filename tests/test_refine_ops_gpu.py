"""The refinement kernels one at a time through their C entry points, against the float64
references of tests/refine_refs.py on the designs of tests/test_refine_refs_host.py: local
correlation at every pyramid depth, tiny / odd / portrait / panoramic grids, the box width at
which the kernel switches to per-sample dots, positions on cell edges and far outside; pyramid
pooling and the track update bit for bit against fp32 emulations; the mixer's depthwise block at
the causal tile boundaries, with and without context, and at every queries-per-CTA choice.  Every
output sits between NaN guards that must be untouched."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from tapnet_b200 import _lib  # noqa: E402
from tests import gpu_util as U  # noqa: E402
from tests import refine_refs as R  # noqa: E402
from tests.test_backbone_ops_gpu import Guarded, ratio  # noqa: E402
from tests.test_refine_refs_host import (corr_design, corr_feats, corr_positions, mixer_input,  # noqa: E402
                                         pyramid, ragged_corr_design)
from tests.test_stages_gpu import MIXER_QB_CASES  # noqa: E402  every queries-per-CTA count on 132 SMs


def lib():
  return _lib.load()


def _ld(L, extra):
  return (388 + 49 * L + 63) // 64 * 64 + extra


# ------------------------------------------------------------------------------- local corr
def run_local_corr(levels, pos, feats, init_hw, batch, P, ld, per_row, query_clip=None):
  """Returns the planes [P, Q, T, ld] (bf16, cpu).  per_row: the features are [Q, T, 384] rows
  read at stride 384 with the low half 128 floats in (what the refinement loop passes after its
  first iteration); else per-query vectors at stride_t 0 (feats must then be constant over t).
  query_clip: None, or int32 [Q] (tapir_local_corr_ragged: query q reads clip query_clip[q])."""
  Q, T, _ = pos.shape
  rows = Q * T
  grids = [g.cuda().contiguous() for g in levels]
  occ = torch.randn(Q, T, generator=torch.Generator().manual_seed(rows))
  expd = torch.randn(Q, T, generator=torch.Generator().manual_seed(rows + 1))
  pos_d, occ_d, expd_d = pos.cuda().contiguous(), occ.cuda(), expd.cuda()
  if per_row:
    fr = torch.cat(feats, -1).cuda().contiguous()
    fh, fl = fr[..., :128], fr[..., 128:]
  else:
    fh, fl = (f[:, 0].cuda().contiguous()[:, None].expand(Q, T, -1) for f in feats)
  out = Guarded(rows * ld, torch.bfloat16, P)
  args = (grids, pos_d, occ_d, expd_d, fh, fl, out.body().view(P, rows, ld), init_hw)
  if query_clip is not None:
    _lib.local_corr(*args, query_clip=query_clip.cuda())
  elif batch == 1:
    _lib.check(lib().tapir_local_corr(ctypes.byref(_lib.corr_args(*args)), U.stream()), 'tapir_local_corr')
  else:
    _lib.local_corr(*args)
  torch.cuda.synchronize()
  assert out.guards_untouched()
  return out.body().cpu().view(P, Q, T, ld), occ, expd


def check_corr(name, levels, pos, feats, init_hw, batch, P, ld_extra, per_row, query_clip=None):
  L = len(levels)
  ld = _ld(L, ld_extra)
  if not per_row:  # per-query features: the same vector in every frame
    feats = tuple(f[:, :1].expand_as(f).contiguous() for f in feats)
  pl3, occ, expd = run_local_corr(levels, pos, feats, init_hw, batch, 3, ld, per_row, query_clip)
  if P < 3:
    plp, _, _ = run_local_corr(levels, pos, feats, init_hw, batch, P, ld, per_row, query_clip)
    assert torch.equal(plp.view(torch.int16), pl3[:P].view(torch.int16))
  # three planes carry the kernel's fp32 value exactly; every column is that value's split
  v32 = pl3.double().sum(0).float()
  assert torch.equal(pl3.view(torch.int16), U.split_like_kernel(v32, 3).view(torch.int16))
  head = R.corr_row_head(occ, expd, feats, ld)
  kin = 388 + 49 * L
  assert torch.equal(v32[..., :388], head[..., :388])
  assert torch.equal(v32[..., kin:], head[..., kin:])
  Q, T, _ = pos.shape
  ref = torch.empty(Q, T, 49 * L, dtype=torch.float64)
  bound = torch.empty_like(ref)
  for t0 in range(0, T, 8):  # the fp64 reference frame chunk by chunk
    r, b = R.local_corr_ref([g[:, t0:t0 + 8] for g in levels], pos[:, t0:t0 + 8],
                            tuple(f[:, t0:t0 + 8] for f in feats), init_hw, batch, planes=P,
                            query_clip=query_clip)
    ref[:, t0:t0 + 8], bound[:, t0:t0 + 8] = r, b
  err, rr = ratio(pl3[:P].double().sum(0)[..., 388:kin], ref, bound)
  U.record(f'refine_corr_{name}_P{P}_ld+{ld_extra}_{"rows" if per_row else "query"}', err=err, ratio=rr)
  assert rr <= 1.0, (err, rr)


CORR_GPU_CASES = [(name, P, extra, per_row) for name, P, extra, per_row in (
    ('pl0_32x32', 3, 0, False), ('pl1_40x48', 3, 64, True), ('pl2_32x32', 2, 0, True),
    ('pl3_32x32', 1, 64, False), ('pl3_192x320', 3, 0, True), ('pl1_1024', 3, 0, True),
    ('portrait_48x16', 2, 64, True), ('box17_12x29', 3, 0, True), ('pano_24x72', 1, 0, True),
    ('tiny_4x8', 3, 64, False), ('tiny_8x8', 2, 0, True), ('batched_b3', 3, 0, True))]


@pytest.mark.parametrize('name,P,ld_extra,per_row', CORR_GPU_CASES, ids=[c[0] for c in CORR_GPU_CASES])
def test_local_corr(name, P, ld_extra, per_row):
  levels, pos, feats, init_hw, B = corr_design(name)
  check_corr(name, levels, pos, feats, init_hw, B, P, ld_extra, per_row)


# the designs split over 3 to 5 clips by a shuffled query_clip table, at T = 1 and T = 2
RAGGED_CORR_CASES = [c for c in CORR_GPU_CASES if c[0] in ('tiny_4x8', 'box17_12x29', 'pl3_32x32')]
RAGGED_CLIPS = {'tiny_4x8': 3, 'box17_12x29': 4, 'pl3_32x32': 5}


@pytest.mark.parametrize('T', [1, 2])
@pytest.mark.parametrize('name,P,ld_extra,per_row', RAGGED_CORR_CASES, ids=[c[0] for c in RAGGED_CORR_CASES])
def test_local_corr_ragged(name, P, ld_extra, per_row, T):
  """tapir_local_corr_ragged: each query reads the grids of the clip its table entry names; the
  clips' grids differ, so a query that reads another clip's is far outside the bound."""
  clips = RAGGED_CLIPS[name]
  levels, pos, feats, init_hw, table = ragged_corr_design(name, clips, T)
  check_corr(f'{name}_ragged{clips}_T{T}', levels, pos, feats, init_hw, clips, P, ld_extra, per_row, table)


def test_local_corr_production_shape():
  """N = 256 queries, T = 48 frames, three levels (256 x 256 video, pyramid_level 1)."""
  levels = pyramid(1, 48, (64, 64), (32, 32), 1, seed=21)
  pos = corr_positions(256, 48, (256, 256), (32, 32), seed=22)
  feats = corr_feats(256, 48, seed=23)
  check_corr('production_256x48', levels, pos, feats, (256, 256), 1, 2, 0, True)


# ------------------------------------------------------------------------------- pooling
@pytest.mark.parametrize('T,h,w,C', [(2, 3, 5, 128), (3, 2, 3, 256), (1, 2, 2, 256), (4, 40, 48, 256),
                                     (16, 64, 64, 256), (5, 17, 9, 128)])
def test_pool_pyramid(T, h, w, C):
  """T 16 at 64 x 64: 1 M float4 outputs, more than the grid-stride loop's one pass."""
  g = torch.Generator().manual_seed(T * h * w)
  x = torch.randn(T, h, w, C, generator=g)
  xd = x.cuda()
  out = Guarded(T * (h // 2) * (w // 2) * C, torch.float32)
  _lib.check(lib().tapir_pool_pyramid(U.ptr(xd), T, h, w, C, out.ptr(), U.stream()), 'tapir_pool_pyramid')
  torch.cuda.synchronize()
  assert out.guards_untouched()
  got = out.body().cpu().view(T, h // 2, w // 2, C)
  assert torch.equal(got.view(torch.int32), R.pool_emulate(x).view(torch.int32))


# ------------------------------------------------------------------------------- track update
UPDATE_CASES = [  # (n, T, per_row, alias_occ, tracks, init, resize, video)
    (5, 4, True, False, True, (256, 256), (320, 384), (480, 640)),
    (7, 3, False, True, True, (192, 320), (384, 640), (1080, 1920)),
    (9, 2, True, True, False, (256, 256), (256, 256), (256, 256)),
    (700, 100, True, False, True, (320, 384), (512, 640), (720, 1280)),   # 70000 rows > 65535
    # tapir_refine_update_ragged: one (h, w) per clip, a shuffled query_clip table, T = 1
    (11, 1, True, False, True, (256, 256), (320, 384), [(480, 640), (200, 200), (1080, 1920)]),
    (13, 1, False, True, True, (192, 320), (384, 640), [(1080, 1920), (480, 640), (200, 200)]),
]


@pytest.mark.parametrize('n,T,per_row,alias,tracks,init,resize,video', UPDATE_CASES,
                         ids=['5x4_rows', '7x3_query_alias', '9x2_alias_no_tracks', '700x100_rows',
                              '11x1_ragged_rows', '13x1_ragged_query_alias'])
def test_refine_update_bit_exact(n, T, per_row, alias, tracks, init, resize, video):
  g = torch.Generator().manual_seed(n * T)
  ld = 392
  res = torch.randn(n, T, ld, generator=g)
  pos = torch.rand(n, T, 2, generator=g) * 400 - 50
  occ, expd = torch.randn(n, T, generator=g), torch.randn(n, T, generator=g)
  feat = torch.randn(n, T, 384, generator=g)
  if not per_row:
    feat = feat[:, :1].expand(n, T, 384).contiguous()
  d = lambda t: t.cuda().contiguous()  # noqa: E731
  res_d, pos_d, occ_d, expd_d = d(res), d(pos), d(occ), d(expd)
  if per_row:
    fd = d(feat)
    fh, fl = fd[..., :128], fd[..., 128:]
  else:
    fh, fl = (d(f)[:, None].expand(n, T, -1) for f in (feat[:, 0, :128], feat[:, 0, 128:]))
  rows = n * T
  occ_o = None if alias else Guarded(rows, torch.float32)
  expd_o, feat_o = Guarded(rows, torch.float32), Guarded(rows * 384, torch.float32)
  trk = Guarded(rows * 2, torch.float32) if tracks else None
  kw = {}
  if isinstance(video, list):  # per-clip sizes; each query's clip from a shuffled table
    table = (torch.arange(n) % len(video))[torch.randperm(n, generator=g)]
    kw = dict(video_table=torch.tensor(video, dtype=torch.int32, device='cuda'),
              query_clip=table.to(torch.int32).cuda())
  _lib.refine_update(res_d, pos_d, occ_d, expd_d, fh, fl, occ_d if alias else occ_o.body().view(n, T),
                     expd_o.body().view(n, T), feat_o.body().view(n, T, 384),
                     trk.body().view(n, T, 2) if tracks else None, init, resize,
                     (0, 0) if kw else video, **kw)
  torch.cuda.synchronize()
  for o in (occ_o, expd_o, feat_o, trk):
    assert o is None or o.guards_untouched()
  if kw:
    assert not bool((table[1:] >= table[:-1]).all())
    video = torch.tensor(video)[table].numpy()
  p, o, e, f, t = R.update_emulate(res, pos, occ, expd, feat, init, resize, video)
  eq = lambda a, b: torch.equal(a.cpu().reshape(-1).view(torch.int32), b.reshape(-1).view(torch.int32))  # noqa: E731
  assert eq(pos_d, p)
  assert eq(occ_d if alias else occ_o.body(), o)
  assert eq(expd_o.body(), e) and eq(feat_o.body(), f)
  if tracks:
    assert eq(trk.body(), t)


# ------------------------------------------------------------------------------- depthwise block
def queries_per_cta(n, T):
  """mixer_dw's choice (refine.cu): tiles of min(T, 24) frames, 52 rows of shared memory per CTA,
  at most 8 queries, and no more queries per CTA than fill every SM of this device once."""
  sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
  tt = min(T, 24)
  qb = min(max(52 // (2 * tt + 4), 1), 8)
  if qb > 1:
    per_sm = -(-n * -(-T // tt) // sms)
    if per_sm < qb:
      qb = max(per_sm, 2)
  return min(qb, n)


_BLOCKS = {}


def block(seed):
  if seed not in _BLOCKS:
    bs = R.block_weights(seed)
    dev = {k: v.cuda().contiguous() for k, v in bs.items()}
    blk = _lib.MixerBlock()
    blk.ln_w, blk.dw1_w, blk.dw1_b = dev['ln_w'].data_ptr(), dev['w1'].data_ptr(), dev['b1'].data_ptr()
    blk.dw2_w, blk.dw2_b, blk.ln1_w = dev['w2'].data_ptr(), dev['b2'].data_ptr(), dev['ln1_w'].data_ptr()
    _BLOCKS[seed] = (bs, dev, blk)
  return _BLOCKS[seed]


def check_mixer_dw(tag, n, T, causal, ctx_in, ctx_out, in_place=False, seed=0):
  bs, _, blk = block(seed)
  x, c1, c2 = mixer_input(n, T, seed=n * 7 + T + 31 * causal)
  c1, c2 = (c1, c2) if ctx_in else (None, None)
  rows = n * T
  xd = x.cuda()
  z = Guarded(rows * 512, torch.float32)
  pl = Guarded(rows * 512, torch.bfloat16, 3)
  ci1 = Guarded(n * 2 * 512, torch.float32) if ctx_in else None
  ci2 = Guarded(n * 2 * 2048, torch.float32) if ctx_in else None
  if ctx_in:
    ci1.body().copy_(c1.reshape(1, -1))
    ci2.body().copy_(c2.reshape(1, -1))
  if in_place:
    co1, co2 = ci1, ci2
  else:
    co1 = Guarded(n * 2 * 512, torch.float32) if ctx_out else None
    co2 = Guarded(n * 2 * 2048, torch.float32) if ctx_out else None
  p = lambda gb: gb.ptr() if gb is not None else None  # noqa: E731
  _lib.check(lib().tapir_mixer_dw(ctypes.byref(blk), U.ptr(xd), n, T, int(causal), p(ci1), p(ci2), p(co1), p(co2),
                                  z.ptr(), pl.ptr(), pl.stride, 3, U.stream()), 'tapir_mixer_dw')
  torch.cuda.synchronize()
  for gb in (z, pl, ci1, ci2, co1, co2):
    assert gb is None or gb.guards_untouched()
  if ctx_in and not in_place:  # inputs untouched
    assert torch.equal(ci1.body().cpu().view(n, 2, 512), c1) and torch.equal(ci2.body().cpu().view(n, 2, 2048), c2)
  planes = pl.body().cpu().view(3, n, T, 512)
  v32 = planes.double().sum(0).float()
  assert torch.equal(planes.view(torch.int16), U.split_like_kernel(v32, 3).view(torch.int16))
  worst = {}
  for q0 in range(0, n, 64):  # the fp64 reference 64 queries at a time
    sl = slice(q0, q0 + 64)
    ref = R.mixer_dw_ref(bs, x[sl], causal, c1[sl] if ctx_in else None, c2[sl] if ctx_in else None)
    got = {'z': z.body().cpu().view(n, T, 512)[sl], 'planes': v32[sl]}
    if ctx_out:
      got['ctx1'] = co1.body().cpu().view(n, 2, 512)[sl]
      got['ctx2'] = co2.body().cpu().view(n, 2, 2048)[sl]
    for k, g in got.items():
      err, rr = ratio(g, *ref[k])
      e0, r0 = worst.get(k, (0.0, 0.0))
      worst[k] = (max(err, e0), max(rr, r0))
  qb = queries_per_cta(n, T)
  U.record(f'refine_mixer_dw_{tag}', qb=qb, **{f'{k}_err': v[0] for k, v in worst.items()},
           **{f'{k}_ratio': v[1] for k, v in worst.items()})
  for k, (err, rr) in worst.items():
    assert rr <= 1.0, (k, err, rr)


@pytest.mark.parametrize('T', [1, 2, 3, 23, 24, 25, 48, 49, 50])
def test_mixer_dw_noncausal(T):
  check_mixer_dw(f'noncausal_T{T}', 5, T, False, False, False)


@pytest.mark.parametrize('ctx_out', [False, True], ids=['no_out', 'out'])
@pytest.mark.parametrize('ctx_in', [False, True], ids=['no_in', 'in'])
@pytest.mark.parametrize('T', [1, 2, 3, 24, 25, 26, 48, 49])
def test_mixer_dw_causal(T, ctx_in, ctx_out):
  """T = 25, 49: the last tile holds one frame, so the two new-context frames fall in two CTAs."""
  check_mixer_dw(f'causal_T{T}_in{int(ctx_in)}_out{int(ctx_out)}', 5, T, True, ctx_in, ctx_out)


def test_mixer_dw_causal_in_place_single_frame():
  check_mixer_dw('causal_in_place_T1', 6, 1, True, True, True, in_place=True)


@pytest.mark.parametrize('causal', [False, True], ids=['noncausal', 'causal'])
@pytest.mark.parametrize('T,n', MIXER_QB_CASES, ids=[f'T{T}_n{n}' for T, n in MIXER_QB_CASES])
def test_mixer_dw_every_queries_per_cta(T, n, causal):
  check_mixer_dw(f'qb_T{T}_n{n}_{"causal" if causal else "noncausal"}', n, T, causal, causal, causal)


def test_mixer_dw_qb_cases_cover_every_queries_per_cta():
  qbs = sorted(queries_per_cta(n, T) for T, n in MIXER_QB_CASES)
  if torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count == 132:
    assert qbs == list(range(1, 9)), qbs
  assert max(qbs) > 1


def test_mixer_dw_streaming_shape():
  """The online step: 2048 queries, one frame, causal, context updated in place."""
  check_mixer_dw('streaming_n2048_T1', 2048, 1, True, True, True, in_place=True)


def test_mixer_dw_clip_shape():
  """256 queries x 48 frames (two tiles per query), causal with context out."""
  check_mixer_dw('clip_n256_T48', 256, 48, True, True, True)
