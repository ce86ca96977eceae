"""Clips and camera streams with their own point counts: the ragged cost volume (grouped GEMM, both
GEMM paths), local correlation and track update against per-clip calls, estimate_trajectories with
points_per_clip against one call per clip, and the ragged OnlineTracker against the equal-count
tracker, its own eager calls, itself with one stream disturbed, one-stream trackers and the golden
clip."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import synth  # noqa: E402
from tapnet_b200 import _lib, streaming, tapir_model  # noqa: E402
from tests import gpu_util as U  # noqa: E402
from tests.conftest import load_golden  # noqa: E402
from tests.test_stages_gpu import get_model  # noqa: E402
from tests.test_tracker_sizes_gpu import GOLDEN_SLOT, LOGIT_TOL, SIZES, TRACK_TOL, _vis_prob  # noqa: E402

TILE_COUNTS = [1, 63, 64, 65, 127, 128, 129, 200]


def _clip(fg, b):
  return type(fg)(tuple(x[b:b + 1] for x in fg.lowres), tuple(x[b:b + 1] for x in fg.hires),
                  fg.resolutions)


# ------------------------------------------------------------------------- stage A
def _stage_a(head, qf, grid, qp, counts, ragged):
  Q, T = qf.shape[0], grid.shape[1]
  out = [torch.full(s, float('nan'), device='cuda') for s in ((Q, T, 2), (Q, T), (Q, T))]
  out.append(torch.full((Q, T), -7, dtype=torch.int32, device='cuda'))
  if ragged:
    ws = torch.empty(_lib.cost_volume_ragged_workspace_bytes(len(counts), Q, grid.shape),
                     dtype=torch.uint8, device='cuda')
    _lib.cost_volume_tracks_ragged(head, qf, counts, grid, qp, 20.0, (256, 256), *out, ws)
    return out
  q0 = 0
  for b, n in enumerate(counts):
    r = slice(q0, q0 + n)
    ws = torch.empty(_lib.cost_volume_workspace_bytes((1, n), grid[b:b + 1].shape), dtype=torch.uint8,
                     device='cuda')
    _lib.cost_volume_tracks(head, qf[None, r], grid[b:b + 1], qp[None, r], 20.0, (256, 256),
                            *(o[None, r] for o in out), ws)
    q0 += n
  return out


@pytest.mark.parametrize('gemm', ['tc', 'simt'])
@pytest.mark.parametrize('T', [1, 3])
@pytest.mark.parametrize('gh,gw', [(32, 32), (24, 40)])
def test_ragged_cost_volume_equals_per_clip_calls(gemm, T, gh, gw):
  model, _, _ = get_model()
  head = model._pack()['head']
  counts = TILE_COUNTS
  Q = sum(counts)
  g = torch.Generator().manual_seed(T * 100 + gh)
  qf = torch.randn(Q, 256, generator=g).cuda()
  grid = torch.randn(len(counts), T, gh, gw, 256, generator=g).cuda()
  qp = torch.cat([torch.rand(Q, 1, generator=g) * T, torch.rand(Q, 2, generator=g) * 256], 1).cuda()
  with U.switches(TAPIR_B200_GEMM=gemm):
    got = _stage_a(head, qf, grid, qp, counts, True)
    want = _stage_a(head, qf, grid, qp, counts, False)
  torch.cuda.synchronize()
  for name, x, y in zip(('points', 'occ', 'expd', 'argmax'), got, want):
    assert torch.equal(x, y), name
  assert int((got[3] < 0).sum()) == 0


# ------------------------------------------------------------------------- refinement kernels
@pytest.mark.parametrize('pyramid_level', [0, 1, 2, 3])
def test_ragged_local_corr_equals_per_clip_calls(pyramid_level):
  counts, T, P = [3, 1, 65, 8], 2, 2
  G, Q = len(counts), sum(counts)
  L = 2 + pyramid_level
  gen = torch.Generator().manual_seed(pyramid_level)
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
  assert torch.equal(got.view(torch.int16), want.view(torch.int16))


def test_ragged_refine_update_equals_per_clip_calls():
  counts, T = [5, 1, 9], 2
  Q = sum(counts)
  g = torch.Generator().manual_seed(3)
  res = torch.randn(Q, T, 400, generator=g).cuda()
  pos0 = (torch.rand(Q, T, 2, generator=g) * 256).cuda()
  occ, expd = torch.randn(Q, T, generator=g).cuda(), torch.randn(Q, T, generator=g).cuda()
  fhi, flo = torch.randn(Q, T, 128, generator=g).cuda(), torch.randn(Q, T, 256, generator=g).cuda()
  sizes = [(480, 640), (200, 200), (240, 320)]
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
      assert torch.equal(x[q0:q0 + n], y), f'clip {b}'
    q0 += n


# ------------------------------------------------------------------------- estimate_trajectories
@pytest.mark.parametrize('causal', [False, True])
def test_points_per_clip_equals_one_call_per_clip(causal):
  model, _, _ = get_model(causal=causal)
  counts, T = [21, 1, 130], 3
  sizes = [(256, 256), (240, 320), (480, 640)]
  B = len(counts)
  v = torch.cat([synth.make_video(T, seed=1 + 4 * b) for b in range(B)]).cuda()
  qs = [synth.make_queries(n, T, *sizes[b], seed=2 + 4 * b)[0].cuda() for b, n in enumerate(counts)]
  fg = model.get_feature_grids(v, False)
  qfs = [model.get_query_features(v[b:b + 1], False, qs[b][None], _clip(fg, b)) for b in range(B)]
  qf = tapir_model.QueryFeatures(tuple(torch.cat([q.lowres[i] for q in qfs], 1) for i in range(len(qfs[0].lowres))),
                                 tuple(torch.cat([q.hires[i] for q in qfs], 1) for i in range(len(qfs[0].hires))),
                                 qfs[0].resolutions)
  qp = torch.cat(qs)[None]
  kw = {}
  if causal:
    nit = model.num_pips_iter * (len(fg.resolutions) - 1)
    g = torch.Generator().manual_seed(9)
    ctx = [{k: torch.randn(1, sum(counts), *v.shape[2:], generator=g).cuda() * 0.1 for k, v in d.items()}
           for d in model.construct_initial_causal_state(sum(counts), len(fg.resolutions) - 1)[:nit]]
    kw = dict(causal_context=ctx, get_causal_context=True)
  both = model.estimate_trajectories(sizes, False, fg, qf, qp, points_per_clip=counts, **kw)
  q0 = 0
  for b, n in enumerate(counts):
    r = slice(q0, q0 + n)
    qf1 = type(qf)(tuple(x[:, r] for x in qf.lowres), tuple(x[:, r] for x in qf.hires), qf.resolutions)
    kw1 = {}
    if causal:
      kw1 = dict(causal_context=[{k: v[:, r].contiguous() for k, v in d.items()} for d in ctx],
                 get_causal_context=True)
    one = model.estimate_trajectories(sizes[b], False, _clip(fg, b), qf1, qp[:, r], **kw1)
    for key in ('tracks', 'occlusion', 'expected_dist'):
      for i, (x, y) in enumerate(zip(both[key], one[key])):
        assert torch.equal(x[:, r], y), f'clip {b}: {key}[{i}]'
    if causal:
      for i, (d, d1) in enumerate(zip(both['causal_context'], one['causal_context'])):
        for k in d:
          assert torch.equal(d[k][:, r], d1[k]), f'clip {b}: context {i} {k}'
    q0 += n
  U.record('points_per_clip_estimate', causal=int(causal), clips=B, frames=T, equal=1)


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
