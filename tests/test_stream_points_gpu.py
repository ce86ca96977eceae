"""Clips and camera streams with their own point counts: the ragged cost volume (grouped GEMM, both
GEMM paths, up to 64 clips and 65535 queries), local correlation and track update against per-clip
calls (T = 1 and 2, up to 64 clips), estimate_trajectories with points_per_clip against one call per
clip (work groups of whole clips and query chunks, and of more than 64 clips), and the ragged
OnlineTracker against the equal-count tracker, its own eager calls, itself with one stream
disturbed, one-stream trackers and the golden clip, and with 70 streams in one group."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import synth  # noqa: E402
from tapnet_b200 import _lib, streaming, tapir_model  # noqa: E402
from tests import gpu_util as U  # noqa: E402
from tests.conftest import load_golden  # noqa: E402
from tests.test_stages_gpu import _mixer_queries_per_cta, get_model  # noqa: E402
from tests.test_tracker_sizes_gpu import GOLDEN_SLOT, LOGIT_TOL, SIZES, TRACK_TOL, _vis_prob  # noqa: E402

TILE_COUNTS = [1, 63, 64, 65, 127, 128, 129, 200]


def _clip(fg, b):
  return type(fg)(tuple(x[b:b + 1] for x in fg.lowres), tuple(x[b:b + 1] for x in fg.hires),
                  fg.resolutions)


# ------------------------------------------------------------------------- stage A
COUNTS_64 = [(1, 63, 64, 65, 129)[b % 5] for b in range(64)]  # one ragged call of 64 clips


def _stage_a(head, qf, grid, qp, counts, ragged):
  """Stage A of the clips, ragged (one call) or one batched call per clip, into outputs between
  NaN (argmax: -7) guards that must stay untouched; no output may stay unwritten."""
  Q, T = qf.shape[0], grid.shape[1]
  bufs = [U.guarded(Q * T * 2), U.guarded(Q * T), U.guarded(Q * T), U.guarded(Q * T, torch.int32)]
  out = [b[1].view(Q, T, 2) if i == 0 else b[1].view(Q, T) for i, b in enumerate(bufs)]
  if ragged:
    ws = torch.empty(_lib.cost_volume_ragged_workspace_bytes(len(counts), Q, grid.shape),
                     dtype=torch.uint8, device='cuda')
    _lib.cost_volume_tracks_ragged(head, qf, counts, grid, qp, 20.0, (256, 256), *out, ws)
  else:
    q0 = 0
    for b, n in enumerate(counts):
      r = slice(q0, q0 + n)
      ws = torch.empty(_lib.cost_volume_workspace_bytes((1, n), grid[b:b + 1].shape), dtype=torch.uint8,
                       device='cuda')
      _lib.cost_volume_tracks(head, qf[None, r], grid[b:b + 1], None if qp is None else qp[None, r], 20.0,
                              (256, 256), *(o[None, r] for o in out), ws)
      q0 += n
  torch.cuda.synchronize()
  for name, (buf, body) in zip(('points', 'occ', 'expd', 'argmax'), bufs):
    assert U.guards_intact(buf), f'{name}: wrote outside the output'
    assert not (body.isnan().any() if body.is_floating_point() else (body < 0).any()), f'{name}: not written'
  return out


def _stage_a_inputs(counts, T, gh, gw, seed, with_tyx=True):
  Q = sum(counts)
  g = torch.Generator().manual_seed(seed)
  qf = torch.randn(Q, 256, generator=g).cuda()
  grid = torch.randn(len(counts), T, gh, gw, 256, generator=g).cuda()
  qp = torch.cat([torch.rand(Q, 1, generator=g) * T, torch.rand(Q, 2, generator=g) * 256], 1).cuda()
  return qf, grid, qp if with_tyx else None


# (gh, gw, counts, query_tyx): 32 x 32 (the tensor-core head) and 24 x 40, 2 x 2 (the generic
# head's smallest map) and 7 x 64 (more maps than its persistent CTAs) with TILE_COUNTS; 64 clips
# in one call; the last two without query_tyx (no query frame masks the occlusion)
RAGGED_CV_CASES = [pytest.param(32, 32, TILE_COUNTS, True, id='32-32'),
                   pytest.param(24, 40, TILE_COUNTS, True, id='24-40'),
                   pytest.param(32, 32, COUNTS_64, True, id='32-32-64clips'),
                   pytest.param(2, 2, TILE_COUNTS, False, id='2-2-no_tyx'),
                   pytest.param(7, 64, COUNTS_64, False, id='7-64-64clips-no_tyx')]


@pytest.mark.parametrize('gemm', ['tc', 'simt'])
@pytest.mark.parametrize('T', [1, 3])
@pytest.mark.parametrize('gh,gw,counts,with_tyx', RAGGED_CV_CASES)
def test_ragged_cost_volume_equals_per_clip_calls(gemm, T, gh, gw, counts, with_tyx):
  model, _, _ = get_model()
  head = model._pack()['head']
  qf, grid, qp = _stage_a_inputs(counts, T, gh, gw, T * 100 + gh + len(counts), with_tyx)
  with U.switches(TAPIR_B200_GEMM=gemm):
    got = _stage_a(head, qf, grid, qp, counts, True)
    want = _stage_a(head, qf, grid, qp, counts, False)
  for name, x, y in zip(('points', 'occ', 'expd', 'argmax'), got, want):
    assert torch.equal(x, y), name


def test_ragged_cost_volume_query_limit():
  """32 x 32 maps: a ragged call of 65535 queries in all runs and equals its per-clip calls; one of
  65536 is refused before any launch."""
  model, _, _ = get_model()
  head = model._pack()['head']
  counts = [40000, 25535]
  qf, grid, qp = _stage_a_inputs(counts, 1, 32, 32, 5)
  got = _stage_a(head, qf, grid, qp, counts, True)
  want = _stage_a(head, qf, grid, qp, counts, False)
  for name, x, y in zip(('points', 'occ', 'expd', 'argmax'), got, want):
    assert torch.equal(x, y), name
  del got, want
  counts = [40000, 25536]
  qf, grid, qp = _stage_a_inputs(counts, 1, 32, 32, 6)
  out = [torch.empty(65536, 1, 2, device='cuda')] + [torch.empty(65536, 1, device='cuda') for _ in range(2)]
  ws = torch.empty(_lib.cost_volume_ragged_workspace_bytes(2, 65536, grid.shape), dtype=torch.uint8,
                   device='cuda')
  torch.cuda.synchronize()
  before = U.launch_count()
  with pytest.raises(_lib.TapirB200Error, match='65535'):
    _lib.cost_volume_tracks_ragged(head, qf, counts, grid, qp, 20.0, (256, 256), *out, None, ws)
  assert U.launch_count() == before


# ------------------------------------------------------------------------- refinement kernels
COUNTS_4 = [3, 1, 65, 8]
COUNTS_64_SMALL = [(3, 1, 65, 8)[b % 4] for b in range(64)]


def _ragged_local_corr(pyramid_level, T, counts, seed):
  P = 2
  G, Q = len(counts), sum(counts)
  L = 2 + pyramid_level
  gen = torch.Generator().manual_seed(seed)
  levels = [torch.randn(G, T, 64, 64, 128, generator=gen).cuda()]
  h = 32
  for _ in range(L - 1):
    levels.append(torch.randn(G, T, h, h, 256, generator=gen).cuda())
    h //= 2
  pos = (torch.rand(Q, T, 2, generator=gen) * 256).cuda()
  occ, expd = torch.randn(Q, T, generator=gen).cuda(), torch.randn(Q, T, generator=gen).cuda()
  fh, fl = torch.randn(Q, T, 128, generator=gen).cuda(), torch.randn(Q, T, 256, generator=gen).cuda()
  ld = (388 + 49 * L + 63) // 64 * 64
  got = torch.full((P, Q * T, ld), float('nan'), dtype=torch.bfloat16, device='cuda')
  want = got.clone()
  clip = torch.tensor([b for b, n in enumerate(counts) for _ in range(n)], dtype=torch.int32,
                      device='cuda')
  _lib.local_corr(levels, pos, occ, expd, fh, fl, got, (256, 256), query_clip=clip)
  q0 = 0
  for b, n in enumerate(counts):
    r = slice(q0, q0 + n)
    _lib.local_corr([x[b:b + 1] for x in levels], pos[r], occ[r], expd[r], fh[r], fl[r],
                    want[:, q0 * T:(q0 + n) * T], (256, 256))
    q0 += n
  torch.cuda.synchronize()
  assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (pyramid_level, T, G)


@pytest.mark.parametrize('pyramid_level', [0, 1, 2, 3])
def test_ragged_local_corr_equals_per_clip_calls(pyramid_level):
  """Four clips at T = 2 and T = 1 (the tracker's step), and 64 clips (T = 1 at odd levels)."""
  _ragged_local_corr(pyramid_level, 2, COUNTS_4, pyramid_level)
  _ragged_local_corr(pyramid_level, 1, COUNTS_4, 10 + pyramid_level)
  _ragged_local_corr(pyramid_level, 2 - pyramid_level % 2, COUNTS_64_SMALL, 20 + pyramid_level)


def _ragged_refine_update(counts, T, sizes, seed):
  Q = sum(counts)
  g = torch.Generator().manual_seed(seed)
  res = torch.randn(Q, T, 400, generator=g).cuda()
  pos0 = (torch.rand(Q, T, 2, generator=g) * 256).cuda()
  occ, expd = torch.randn(Q, T, generator=g).cuda(), torch.randn(Q, T, generator=g).cuda()
  fhi, flo = torch.randn(Q, T, 128, generator=g).cuda(), torch.randn(Q, T, 256, generator=g).cuda()
  table = torch.tensor(sizes, dtype=torch.int32, device='cuda')
  clip = torch.tensor([b for b, n in enumerate(counts) for _ in range(n)], dtype=torch.int32,
                      device='cuda')

  def run(sl, video_hw, **kw):
    m = sl.stop - sl.start
    pos = pos0[sl].clone()
    outs = [torch.empty(m, T, device='cuda') for _ in range(2)] + [
        torch.empty(m, T, 384, device='cuda'), torch.empty(m, T, 2, device='cuda')]
    _lib.refine_update(res[sl], pos, occ[sl], expd[sl], fhi[sl], flo[sl], *outs, (256, 256),
                       (480, 480), video_hw, **kw)
    return [pos] + outs

  got = run(slice(0, Q), (0, 0), video_table=table, query_clip=clip)
  q0 = 0
  for b, n in enumerate(counts):
    want = run(slice(q0, q0 + n), sizes[b])
    for x, y in zip(got, want):
      assert torch.equal(x[q0:q0 + n], y), f'clip {b} of {len(counts)}, T = {T}'
    q0 += n


def test_ragged_refine_update_equals_per_clip_calls():
  """Three clips at T = 2 and T = 1, and 64 clips of 1 to 9 queries and their own sizes at T = 1."""
  sizes = [(480, 640), (200, 200), (240, 320)]
  _ragged_refine_update([5, 1, 9], 2, sizes, 3)
  _ragged_refine_update([5, 1, 9], 1, sizes, 4)
  _ragged_refine_update([1 + b % 9 for b in range(64)], 1, [(120 + 8 * b, 640 - 4 * b) for b in range(64)], 5)


# ------------------------------------------------------------------------- estimate_trajectories
def _split_qf(qf, r):
  return type(qf)(tuple(x[:, r] for x in qf.lowres), tuple(x[:, r] for x in qf.hires), qf.resolutions)


def _clips_and_queries(model, counts, sizes, T):
  """Videos [B, T, 256, 256, 3], their feature grids, and the clips' queries one after the other:
  query features [1, sum counts, ...] and points [1, sum counts, 3] (clip b's in sizes[b] pixels)."""
  B = len(counts)
  v = torch.cat([synth.make_video(T, seed=1 + 4 * b) for b in range(B)]).cuda()
  qs = [synth.make_queries(n, T, *sizes[b], seed=2 + 4 * b)[0].cuda() for b, n in enumerate(counts)]
  fg = model.get_feature_grids(v, False)
  qfs = [model.get_query_features(v[b:b + 1], False, qs[b][None], _clip(fg, b)) for b in range(B)]
  qf = tapir_model.QueryFeatures(tuple(torch.cat([q.lowres[i] for q in qfs], 1) for i in range(len(qfs[0].lowres))),
                                 tuple(torch.cat([q.hires[i] for q in qfs], 1) for i in range(len(qfs[0].hires))),
                                 qfs[0].resolutions)
  return fg, qf, torch.cat(qs)[None]


def _random_context(model, fg, Q, seed):
  nit = model.num_pips_iter * (len(fg.resolutions) - 1)
  g = torch.Generator().manual_seed(seed)
  return [{k: torch.randn(1, Q, *v.shape[2:], generator=g).cuda() * 0.1 for k, v in d.items()}
          for d in model.construct_initial_causal_state(Q, len(fg.resolutions) - 1)[:nit]]


def _compare_clips(model, sizes, counts, fg, qf, qp, ctx, both, exact):
  """Each clip of `both` (one points_per_clip call) against a one-clip call: bit for bit where
  exact(b), else within TRACK_TOL / LOGIT_TOL and the context within 5e-4.  Returns the largest
  (track, logit, context) differences of the inexact clips."""
  worst = [0.0, 0.0, 0.0]
  q0 = 0
  for b, n in enumerate(counts):
    r = slice(q0, q0 + n)
    kw1 = {}
    if ctx is not None:
      kw1 = dict(causal_context=[{k: v[:, r].contiguous() for k, v in d.items()} for d in ctx],
                 get_causal_context=True)
    one = model.estimate_trajectories(sizes[b], False, _clip(fg, b), _split_qf(qf, r), qp[:, r], **kw1)
    pairs = [(key, i, x[:, r], y) for key in ('tracks', 'occlusion', 'expected_dist')
             for i, (x, y) in enumerate(zip(both[key], one[key]))]
    if ctx is not None:
      pairs += [(f'context {k}', i, d[k][:, r], d1[k]) for i, (d, d1) in
                enumerate(zip(both['causal_context'], one['causal_context'])) for k in d]
    for key, i, x, y in pairs:
      if exact(b):
        assert torch.equal(x, y), f'clip {b}: {key}[{i}]'
      else:
        e = (x - y).abs().max().item()
        slot = 0 if key == 'tracks' else 2 if key.startswith('context') else 1
        worst[slot] = max(worst[slot], e)
    q0 += n
  assert worst[0] <= TRACK_TOL and worst[1] <= LOGIT_TOL and worst[2] <= 5e-4, worst
  return worst


# (causal, rows_bound): every clip in one work group (None); clips 0 and 1 in one group and the
# 130-point clip in query chunks of 22 ('two_clips'); every clip in query chunks of 8
# ('query_chunks').  The same bound applies to the one-clip calls.
PPC_CASES = [pytest.param(False, None, id='False'), pytest.param(True, None, id='True'),
             pytest.param(False, 'two_clips', id='False-two_clips'),
             pytest.param(True, 'two_clips', id='True-two_clips'),
             pytest.param(False, 'query_chunks', id='False-query_chunks'),
             pytest.param(True, 'query_chunks', id='True-query_chunks')]


@pytest.mark.parametrize('causal,rows_bound', PPC_CASES)
def test_points_per_clip_equals_one_call_per_clip(causal, rows_bound, monkeypatch):
  model, _, _ = get_model(causal=causal)
  counts, T = [21, 1, 130], 3
  sizes = [(256, 256), (240, 320), (480, 640)]
  B = len(counts)
  bound = {None: tapir_model._MAX_ROWS_PER_CHUNK, 'two_clips': 22 * T, 'query_chunks': 8 * T}[rows_bound]
  monkeypatch.setattr(tapir_model, '_MAX_ROWS_PER_CHUNK', bound)
  groups = tapir_model._work_groups(counts, T)
  if rows_bound == 'two_clips':
    assert groups[0] == (0, 2, 0, 22) and len(groups) == 1 + 6 and all(g[:2] == (2, 3) for g in groups[1:])
  elif rows_bound == 'query_chunks':
    assert all(g[1] - g[0] == 1 and g[3] - g[2] <= 8 for g in groups)
  fg, qf, qp = _clips_and_queries(model, counts, sizes, T)
  ctx = _random_context(model, fg, sum(counts), 9) if causal else None
  kw = dict(causal_context=ctx, get_causal_context=True) if causal else {}
  both = model.estimate_trajectories(sizes, False, fg, qf, qp, points_per_clip=counts, **kw)
  _compare_clips(model, sizes, counts, fg, qf, qp, ctx, both, lambda b: True)
  U.record(f'points_per_clip_estimate_{rows_bound}' if rows_bound else 'points_per_clip_estimate',
           causal=int(causal), clips=B, frames=T, groups=len(groups), equal=1)


@pytest.mark.parametrize('causal', [False, True])
@pytest.mark.parametrize('clips', [65, 130])
def test_more_than_64_clips_in_one_work_group(clips, causal, monkeypatch):
  """65 and 130 clips of 1 to 9 points in one work group: stage A runs as ceil(G / 64) ragged
  calls while local correlation and the update run one query_clip table over all G clips.
  Non-causal, each clip equals a one-clip call bit for bit (T > 1).  Causal, bit for bit where the
  mixer's queries-per-CTA choice is the same for the group and the clip alone, else within the
  equal-count causal batch's tolerances (the choice decides the bits, DESIGN.md section 7)."""
  model, _, _ = get_model(causal=causal)
  T = 2
  g = torch.Generator().manual_seed(clips)
  counts = (torch.randint(1, 10, (clips,), generator=g)).tolist()
  sizes = [(256, 256)] * clips
  assert tapir_model._work_groups(counts, T) == [(0, clips, 0, sum(counts))] and len(set(counts)) > 1
  fg, qf, qp = _clips_and_queries(model, counts, sizes, T)
  ctx = _random_context(model, fg, sum(counts), clips) if causal else None
  kw = dict(causal_context=ctx, get_causal_context=True) if causal else {}
  calls = []
  real = tapir_model._lib.cost_volume_tracks_ragged

  def counting(head, qfeat, cs, *args):
    calls.append(len(cs))
    return real(head, qfeat, cs, *args)
  monkeypatch.setattr(tapir_model._lib, 'cost_volume_tracks_ragged', counting)
  both = model.estimate_trajectories((256, 256), False, fg, qf, qp, points_per_clip=counts, **kw)
  assert calls == [64] * (clips // 64) + ([clips % 64] if clips % 64 else []), calls
  monkeypatch.undo()
  qb = _mixer_queries_per_cta(sum(counts), T)
  exact = (lambda b: True) if not causal else (lambda b: _mixer_queries_per_cta(counts[b], T) == qb)
  worst = _compare_clips(model, sizes, counts, fg, qf, qp, ctx, both, exact)
  U.record(f'points_per_clip_{clips}_clips', causal=int(causal), points=sum(counts),
           exact_clips=sum(map(exact, range(clips))), ragged_calls=len(calls), tracks=worst[0],
           logits=worst[1], context=worst[2])


# ------------------------------------------------------------------------- OnlineTracker
def _inputs(sizes, counts, T, golden=None):
  frames, queries = [], []
  for s, ((H, W), n) in enumerate(zip(sizes, counts)):
    if golden is not None and s == GOLDEN_SLOT:
      meta = golden['meta']
      frames.append(synth.make_video(T, H, W, seed=meta['video_seed'])[0].cuda())
      queries.append(synth.make_queries(n, T, H, W, seed=meta['query_seed'], frame0_only=True)[0].cuda())
    else:
      frames.append(synth.make_video(T, H, W, seed=40 + 3 * s)[0].cuda())
      queries.append(synth.make_queries(n, T, H, W, seed=41 + 3 * s, frame0_only=True)[0].cuda())
  return frames, queries


@pytest.mark.parametrize('mixed', [False, True])
def test_equal_counts_tracker_equals_the_int_tracker(mixed):
  model, _, _ = get_model(causal=True)
  N, T = 12, 3
  sizes = SIZES if mixed else [(256, 256)] * 3
  S = len(sizes)
  hs, ws = [h for h, _ in sizes], [w for _, w in sizes]
  frames, qs = _inputs(sizes, [N] * S, T)
  a = streaming.OnlineTracker(model, hs, ws, N, num_streams=S)
  b = streaming.OnlineTracker(model, hs, ws, [N] * S, num_streams=S)
  fr0 = [f[0] for f in frames] if mixed else torch.stack([f[0] for f in frames])
  a.init(fr0, torch.stack(qs))
  b.init(fr0, qs)
  for t in range(T):
    if t == 1:
      for trk in (a, b):
        trk.update_query(frames[1][1], torch.tensor([1.0, 60.5, 33.25]), 4, stream=1)
    fr = [f[t] for f in frames] if mixed else torch.stack([f[t] for f in frames])
    ta, va = a.step(fr)
    tb, vb = b.step(fr)
    for s in range(S):
      assert torch.equal(ta[s], tb[s]) and torch.equal(va[s], vb[s]), f'frame {t} stream {s}'
      for x, y in zip(a.last_logits, b.last_logits):
        assert torch.equal(x[s], y[s])
    for ga, gb in zip(a._groups, b._groups):
      for da, db in zip(ga.state, gb.state):
        for k in da:
          assert torch.equal(da[k].reshape(db[k].shape), db[k]), f'frame {t}: state {k}'
  a.close()
  b.close()


COUNTS = [8, 1, 33, 130, 8]  # SIZES[4] (480^2) keeps the golden clip's 8 points


def test_ragged_tracker_replay_singles_golden_and_launches():
  g = load_golden('causal_480x3_n8')
  meta = g['meta']
  assert (meta['H'], meta['W']) == SIZES[GOLDEN_SLOT] and meta['N'] == COUNTS[GOLDEN_SLOT]
  model, _, _ = get_model(causal=True)
  T, S = meta['T'], len(SIZES)
  hs, ws = [h for h, _ in SIZES], [w for _, w in SIZES]
  frames, qs = _inputs(SIZES, COUNTS, T, g)
  trk = streaming.OnlineTracker(model, hs, ws, COUNTS, num_streams=S)
  assert [grp.streams for grp in trk._groups] == [[0], [1], [2, 3], [4]]
  trk.init([f[0] for f in frames], qs)
  singles = [streaming.OnlineTracker(model, H, W, n) for (H, W), n in zip(SIZES, COUNTS)]
  for s in range(S):
    singles[s].init(frames[s][0], qs[s])
  e_t = e_l = 0.0
  vis_mismatch = 0
  gold = [[], [], []]
  for t in range(T):
    if t == 1:
      trk.update_query(frames[2][1], torch.tensor([0.0, 100.5, 37.25]), 30, stream=2)
      singles[2].update_query(frames[2][1], torch.tensor([0.0, 100.5, 37.25]), 30)
    saved = [[{k: v.clone() for k, v in d.items()} for d in grp.state] for grp in trk._groups]
    tracks, vis = trk.step([f[t] for f in frames])
    occ, expd = trk.last_logits
    assert [tuple(x.shape) for x in tracks] == [(n, 1, 2) for n in COUNTS]
    assert [tuple(x.shape) for x in vis] == [(n, 1) for n in COUNTS]
    for grp, st in zip(trk._groups, saved):  # replay == the eager grouped calls, bit for bit
      et, eo, ee = trk._step_group(grp, st)
      for i, s in enumerate(grp.streams):
        r = slice(grp.offsets[i], grp.offsets[i] + COUNTS[s])
        assert torch.equal(tracks[s], et[0, r]), f'frame {t} stream {s}: replay != eager'
        assert torch.equal(occ[s], eo[0, r]) and torch.equal(expd[s], ee[0, r])
      for d, de in zip(grp.state, st):
        for k in d:
          assert torch.equal(d[k], de[k]), f'frame {t}: state {k}'
    for s in range(S):
      t1, v1 = singles[s].step(frames[s][t])
      o1, x1 = singles[s].last_logits
      e_t = max(e_t, (tracks[s] - t1[0]).abs().max().item())
      e_l = max(e_l, (occ[s] - o1[0]).abs().max().item(), (expd[s] - x1[0]).abs().max().item())
      clear = (_vis_prob(o1[0], x1[0]) - 0.5).abs() > 1e-3
      vis_mismatch += int((vis[s][clear] != v1[0][clear]).sum())
    for lst, x in zip(gold, (tracks, occ, expd)):
      lst.append(x[GOLDEN_SLOT].cpu().numpy())
  # launches per step: those of the equal-count tracker with the same groups
  eq = streaming.OnlineTracker(model, hs, ws, 8, num_streams=S)
  eq.init([f[0] for f in frames], torch.stack([synth.make_queries(8, T, H, W, seed=s, frame0_only=True)[0]
                                               for s, (H, W) in enumerate(SIZES)]).cuda())
  counts = []
  for x in (trk, eq):
    x._step_eager()
    torch.cuda.synchronize()
    l0 = U.launch_count()
    x._step_eager()
    counts.append(U.launch_count() - l0)
  for x in singles + [trk, eq]:
    x.close()
  g_t = np.abs(np.concatenate(gold[0], 1) - g['online_tracks']).max()
  g_o = np.abs(np.concatenate(gold[1], 1) - g['online_occlusion']).max()
  g_e = np.abs(np.concatenate(gold[2], 1) - g['online_expected_dist']).max()
  U.record('tracker_ragged_points', streams=S, points=sum(COUNTS), frames=T, tracks_vs_single=e_t,
           logits_vs_single=e_l, vis_mismatch=vis_mismatch, golden_tracks=g_t, golden_occ=g_o,
           golden_expd=g_e, launches=counts[0], launches_equal_counts=counts[1])
  assert e_t <= TRACK_TOL and e_l <= LOGIT_TOL and vis_mismatch == 0
  assert g_t < TRACK_TOL and g_o < LOGIT_TOL and g_e < LOGIT_TOL
  assert counts[0] == counts[1]


def test_ragged_tracker_streams_are_isolated():
  """Changing stream 2's frames and re-targeting one of its points leaves every other stream's
  outputs and causal state bit for bit unchanged."""
  model, _, _ = get_model(causal=True)
  T, S = 3, len(SIZES)
  frames, qs = _inputs(SIZES, COUNTS, T)
  other = synth.make_video(T, 200, 200, seed=77)[0].cuda()

  def run(disturb):
    trk = streaming.OnlineTracker(model, [h for h, _ in SIZES], [w for _, w in SIZES], COUNTS,
                                  num_streams=S)
    fr = [other if disturb and s == 2 else f for s, f in enumerate(frames)]
    trk.init([f[0] for f in fr], qs)
    outs = []
    for t in range(T):
      if disturb and t == 1:
        trk.update_query(fr[2][1], torch.tensor([0.0, 40.5, 150.25]), 9, stream=2)
      tracks, vis = trk.step([f[t] for f in fr])
      outs.append([[x.clone() for x in lst] for lst in (tracks, vis, *trk.last_logits)])
    state = {}
    for s in range(S):
      gi, slot = trk._slot[s]
      grp = trk._groups[gi]
      r = slice(grp.offsets[slot], grp.offsets[slot] + COUNTS[s])
      state[s] = [{k: v[:, r].clone() for k, v in d.items()} for d in grp.state]
    trk.close()
    return outs, state

  (a, sa), (b, sb) = run(False), run(True)
  keep = [s for s in range(S) if s != 2]
  for t in range(T):
    for x, y in zip(a[t], b[t]):
      for s in keep:
        assert torch.equal(x[s], y[s]), f'frame {t} stream {s}'
  assert not torch.equal(a[-1][0][2], b[-1][0][2])
  for s in keep:
    for da, db in zip(sa[s], sb[s]):
      for k in da:
        assert torch.equal(da[k], db[k]), f'stream {s}: {k}'
  U.record('tracker_ragged_isolation', equal=1)


def test_tracker_of_70_streams_runs_two_ragged_stage_a_calls(monkeypatch):
  """70 streams of 256^2 with 1 to 12 points form one group: each step runs two ragged stage-A
  calls (64 + 6 clips) and one query_clip table over all 70 streams.  Over 3 steps, with one
  update_query on stream 64: graph replay equals the eager grouped calls bit for bit, and streams
  0, 63, 64 and 69 are within TRACK_TOL / LOGIT_TOL of one-stream trackers with no visibility flip
  away from 0.5 (T = 1: the mixer GEMMs split K by row count, so the bits may differ)."""
  model, _, _ = get_model(causal=True)
  S, T = 70, 3
  counts = [1 + (7 * s) % 12 for s in range(S)]
  sizes = [(256, 256)] * S
  frames, qs = _inputs(sizes, counts, T)
  trk = streaming.OnlineTracker(model, [256] * S, [256] * S, counts, num_streams=S)
  assert [grp.streams for grp in trk._groups] == [list(range(S))]
  trk.init(torch.stack([f[0] for f in frames]), qs)
  probe = (0, 63, 64, 69)
  singles = {s: streaming.OnlineTracker(model, 256, 256, counts[s]) for s in probe}
  for s in probe:
    singles[s].init(frames[s][0], qs[s])
  calls = []
  real = tapir_model._lib.cost_volume_tracks_ragged

  def counting(head, qfeat, cs, *args):
    calls.append(len(cs))
    return real(head, qfeat, cs, *args)
  monkeypatch.setattr(tapir_model._lib, 'cost_volume_tracks_ragged', counting)
  grp = trk._groups[0]
  e_t = e_l = 0.0
  vis_mismatch = 0
  new_query = torch.tensor([0.0, 100.5, 37.25])
  for t in range(T):
    if t == 1:
      trk.update_query(frames[64][1], new_query, 0, stream=64)
      singles[64].update_query(frames[64][1], new_query, 0)
    saved = [{k: v.clone() for k, v in d.items()} for d in grp.state]
    tracks, vis = trk.step(torch.stack([f[t] for f in frames]))
    occ, expd = trk.last_logits
    del calls[:]
    et, eo, ee = trk._step_group(grp, saved)  # replay == the eager grouped calls, bit for bit
    assert calls == [64, 6], calls
    for i, s in enumerate(grp.streams):
      r = slice(grp.offsets[i], grp.offsets[i] + counts[s])
      assert torch.equal(tracks[s], et[0, r]), f'frame {t} stream {s}: replay != eager'
      assert torch.equal(occ[s], eo[0, r]) and torch.equal(expd[s], ee[0, r])
    for d, de in zip(grp.state, saved):
      for k in d:
        assert torch.equal(d[k], de[k]), f'frame {t}: state {k}'
    for s in probe:
      t1, v1 = singles[s].step(frames[s][t])
      o1, x1 = singles[s].last_logits
      e_t = max(e_t, (tracks[s] - t1[0]).abs().max().item())
      e_l = max(e_l, (occ[s] - o1[0]).abs().max().item(), (expd[s] - x1[0]).abs().max().item())
      clear = (_vis_prob(o1[0], x1[0]) - 0.5).abs() > 1e-3
      vis_mismatch += int((vis[s][clear] != v1[0][clear]).sum())
  for x in list(singles.values()) + [trk]:
    x.close()
  U.record('tracker_70_streams', points=sum(counts), frames=T, tracks_vs_single=e_t,
           logits_vs_single=e_l, vis_mismatch=vis_mismatch)
  assert e_t <= TRACK_TOL and e_l <= LOGIT_TOL and vis_mismatch == 0
