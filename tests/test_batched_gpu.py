"""Several clips per launch sequence: the batched cost volume and local correlation against
per-clip calls of the single-clip entry points, grouped estimate_trajectories against per-clip
calls, and the multi-stream OnlineTracker against single-stream trackers and the golden clip.

The split-K GEMM and the causal mixer's queries-per-CTA choice both depend on the row count, so
results over different row counts are compared bit for bit only where neither can change."""
import ctypes
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import synth  # noqa: E402
from tapnet_b200 import _lib, streaming, tapir_model  # noqa: E402
from tests import gpu_util as U  # noqa: E402
from tests.conftest import load_golden  # noqa: E402
from tests.test_stages_gpu import get_model  # noqa: E402

TRACK_TOL = 1e-3
LOGIT_TOL = 1e-4


def _unit(*shape, seed):
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(*shape, generator=g)
  return x / x.norm(dim=-1, keepdim=True)


# ------------------------------------------------------------------------- entry points
@pytest.mark.parametrize('gh,gw', [(32, 32), (24, 40)])
@pytest.mark.parametrize('T', [1, 3])
@pytest.mark.parametrize('N', [37, 130])
@pytest.mark.parametrize('B', [1, 2, 3, 5])
def test_cost_volume_batched_equals_per_clip(B, N, T, gh, gw):
  model, _, _ = get_model()
  lib = _lib.load()
  pk = model._pack()
  C = 256
  ih, iw = gh * 8, gw * 8
  grid = _unit(B, T, gh, gw, C, seed=11 + B).cuda()
  # queries near grid features so that heat maps are peaked
  g = torch.Generator().manual_seed(12 + N)
  idx = torch.randint(0, T * gh * gw, (B, N), generator=g)
  qf = grid.cpu().reshape(B, -1, C)[torch.arange(B)[:, None], idx] + 0.05 * torch.randn(B, N, C, generator=g)
  qf = (qf / qf.norm(dim=-1, keepdim=True)).cuda().contiguous()
  qp = torch.cat([synth.make_queries(N, T, ih, iw, seed=20 + b) for b in range(B)]).cuda().contiguous()
  outs = {}
  for name, per, dt in (('pts', 2, torch.float32), ('occ', 1, torch.float32), ('expd', 1, torch.float32),
                        ('am', 1, torch.int32)):
    outs[name] = U.guarded(B * N * T * per, dt)
  ws = torch.empty(_lib.cost_volume_workspace_bytes(qf, grid), dtype=torch.uint8, device='cuda')
  _lib.cost_volume_tracks(pk['head'], qf, grid, qp, 20.0, (ih, iw), outs['pts'][1].view(B, N, T, 2),
                          *(outs[k][1].view(B, N, T) for k in ('occ', 'expd', 'am')), ws)
  torch.cuda.synchronize()
  for name, (buf, _) in outs.items():
    assert U.guards_intact(buf), f'{name}: bytes outside the output were written'
  nb1 = lib.tapir_cost_volume_workspace_bytes(N, T, gh, gw, C)
  ws1 = torch.empty(nb1, dtype=torch.uint8, device='cuda')
  for b in range(B):
    pts = torch.empty(N, T, 2, device='cuda')
    occ = torch.empty(N, T, device='cuda')
    expd = torch.empty(N, T, device='cuda')
    am = torch.empty(N, T, dtype=torch.int32, device='cuda')
    _lib.check(lib.tapir_cost_volume_tracks(
        ctypes.byref(pk['head']), U.ptr(qf[b]), U.ptr(grid[b]), N, T, gh, gw, C, U.ptr(qp[b]), 20.0,
        ih, iw, U.ptr(pts), U.ptr(occ), U.ptr(expd), U.ptr(am), U.ptr(ws1), nb1, U.stream()), 'cv')
    torch.cuda.synchronize()
    assert torch.equal(outs['pts'][1].view(B, N, T, 2)[b], pts), f'clip {b}: points'
    assert torch.equal(outs['occ'][1].view(B, N, T)[b], occ), f'clip {b}: occ'
    assert torch.equal(outs['expd'][1].view(B, N, T)[b], expd), f'clip {b}: expd'
    assert torch.equal(outs['am'][1].view(B, N, T)[b], am), f'clip {b}: argmax'


@pytest.mark.parametrize('gh,gw', [(32, 32), (24, 40)])
@pytest.mark.parametrize('pyr', [0, 2])
@pytest.mark.parametrize('T', [1, 3])
@pytest.mark.parametrize('N', [37, 130])
@pytest.mark.parametrize('B', [1, 2, 3, 5])
def test_local_corr_batched_equals_per_clip(B, N, T, pyr, gh, gw):
  lib = _lib.load()
  L = 2 + pyr
  kin = 388 + 49 * L
  kpad = (kin + 63) // 64 * 64
  P = 3
  shapes = [(2 * gh, 2 * gw, 128), (gh, gw, 256)] + [(gh >> l, gw >> l, 256) for l in range(1, pyr + 1)]
  grids = [_unit(B, T, h, w, c, seed=30 + i).cuda() for i, (h, w, c) in enumerate(shapes)]
  g = torch.Generator().manual_seed(40 + B * N)
  pos = (torch.rand(B, N, T, 2, generator=g) * 272 - 8).cuda()  # some samples outside the map
  occ = torch.randn(B, N, T, generator=g).cuda()
  expd = torch.randn(B, N, T, generator=g).cuda()
  per_row = pyr == 2  # per-(query, frame) features (refinement) or per-query ones (first iteration)
  if per_row:
    feat = torch.randn(B, N, T, 384, generator=g).cuda()
    feats = lambda bsl, nq: (feat[bsl].view(nq, T, 384)[..., :128], feat[bsl].view(nq, T, 384)[..., 128:])  # noqa: E731
  else:
    qh = torch.randn(B, N, 128, generator=g).cuda()
    ql = torch.randn(B, N, 256, generator=g).cuda()
    feats = lambda bsl, nq: tuple(q[bsl].reshape(nq, 1, -1).expand(nq, T, -1) for q in (qh, ql))  # noqa: E731

  def args(bsl, nclips):
    rows = nclips * N * T
    buf, body = U.guarded(P * rows * kpad, torch.bfloat16)
    ca = _lib.corr_args([gd[bsl] for gd in grids], pos[bsl], occ[bsl], expd[bsl], *feats(bsl, nclips * N),
                        body.view(P, rows, kpad), (256, 256))
    return ca, buf, body.view(P, nclips, N * T, kpad)

  ca, buf, got = args(slice(0, B), B)
  _lib.check(lib.tapir_local_corr_batched(ctypes.byref(ca), B, U.stream()), 'local_corr_batched')
  torch.cuda.synchronize()
  assert U.guards_intact(buf)
  for b in range(B):
    ca1, buf1, want = args(slice(b, b + 1), 1)
    _lib.check(lib.tapir_local_corr(ctypes.byref(ca1), U.stream()), 'local_corr')
    torch.cuda.synchronize()
    assert U.guards_intact(buf1)
    assert torch.equal(got[:, b].view(torch.int16), want[:, 0].view(torch.int16)), f'clip {b}'


# ------------------------------------------------------------------------- offline model
def _clips(B, T, N, causal=False):
  v = torch.cat([synth.make_video(T, seed=1 + 4 * b) for b in range(B)]).cuda()
  q = torch.cat([synth.make_queries(N, T, seed=2 + 4 * b, frame0_only=causal) for b in range(B)]).cuda()
  return v, q


def _compare(both, one, b, exact):
  errs = []
  for key in ('tracks', 'occlusion', 'expected_dist'):
    x, y = both[key][b], one[key][0]
    if exact:
      assert torch.equal(x, y), f'clip {b}: {key}'
    errs.append((x - y).abs().max().item())
  for key in ('unrefined_tracks', 'unrefined_occlusion'):
    for i, (x, y) in enumerate(zip(both[key], one[key])):
      if exact:
        assert torch.equal(x[b], y[0]), f'clip {b}: {key}[{i}]'
  return errs


@pytest.mark.parametrize('rows_bound', [None, 'two_clips', 'query_chunks'])
def test_forward_batch_of_three_in_work_groups_equals_per_clip_calls(rows_bound):
  """Non-causal: bit for bit, with all clips in one group, with groups of two clips, and with
  every clip split into query chunks (the same bound applied to the per-clip calls)."""
  model, _, _ = get_model()
  B, T, N = 3, 4, 21
  v, q = _clips(B, T, N)
  bound = {None: tapir_model._MAX_ROWS_PER_CHUNK, 'two_clips': 2 * N * T, 'query_chunks': 8 * T}[rows_bound]
  old = tapir_model._MAX_ROWS_PER_CHUNK
  tapir_model._MAX_ROWS_PER_CHUNK = bound
  try:
    groups = tapir_model._work_groups([N] * B, T)
    both = model(v, q)
    ones = [model(v[b:b + 1], q[b:b + 1]) for b in range(B)]
  finally:
    tapir_model._MAX_ROWS_PER_CHUNK = old
  if rows_bound is None:
    assert groups == [(0, 3, 0, 3 * N)]
  elif rows_bound == 'two_clips':
    assert groups == [(0, 2, 0, 2 * N), (2, 3, 2 * N, 3 * N)]
  else:
    assert len(groups) == 3 * 3 and all(g[1] - g[0] == 1 for g in groups)
  for b in range(B):
    _compare(both, ones[b], b, exact=True)
  U.record(f'batched_forward_{rows_bound}', groups=len(groups), equal=1)


def test_one_launch_sequence_for_a_group_of_clips():
  model, _, _ = get_model()
  T, N = 3, 16
  counts = {}
  for B in (1, 3):
    v, q = _clips(B, T, N)
    fg = model.get_feature_grids(v, False)
    qf = model.get_query_features(v, False, q, fg)
    model.estimate_trajectories((256, 256), False, fg, qf, q)  # warm-up (workspaces)
    torch.cuda.synchronize()
    l0 = U.launch_count()
    model.estimate_trajectories((256, 256), False, fg, qf, q)
    torch.cuda.synchronize()
    counts[B] = U.launch_count() - l0
  U.record('batched_offline_launches', b1=counts[1], b3=counts[3])
  assert counts[1] == counts[3] and counts[1] > 40


def test_causal_forward_batch_of_three_within_tolerance():
  """The causal mixer packs several queries per CTA depending on the query count, so B = 3 in one
  group may differ from per-clip calls in the last bits."""
  model, _, _ = get_model(causal=True)
  B, T, N = 3, 5, 24
  v, q = _clips(B, T, N, causal=True)
  both = model(v, q)
  worst = [0.0, 0.0, 0.0]
  for b in range(B):
    errs = _compare(both, model(v[b:b + 1], q[b:b + 1]), b, exact=False)
    worst = [max(w, e) for w, e in zip(worst, errs)]
  U.record('batched_causal_forward', tracks=worst[0], occ=worst[1], expd=worst[2])
  assert worst[0] <= TRACK_TOL and worst[1] <= LOGIT_TOL and worst[2] <= LOGIT_TOL


# ------------------------------------------------------------------------- multi-stream tracker
def _stream_clips(S, T, N, seeds):
  v = torch.cat([synth.make_video(T, seed=s) for s in seeds]).cuda()           # [S, T, H, W, 3]
  q = torch.cat([synth.make_queries(N, T, seed=s + 1, frame0_only=True) for s in seeds]).cuda()
  return v, q


def _vis_prob(occ, expd):
  return (1 - torch.sigmoid(occ)) * (1 - torch.sigmoid(expd))


def test_tracker_multi_stream_equals_eager_and_single_streams():
  model, _, _ = get_model(causal=True)
  S, N, T = 3, 64, 5
  v, q = _stream_clips(S, T, N, seeds=(3, 7, 11))
  trk = streaming.OnlineTracker(model, 256, 256, N, num_streams=S)
  qf = trk.init(v[:, 0], q)
  qf = tapir_model.QueryFeatures(tuple(t.clone() for t in qf.lowres), tuple(t.clone() for t in qf.hires),
                                 qf.resolutions)
  singles = [streaming.OnlineTracker(model, 256, 256, N) for _ in range(S)]
  for s in range(S):
    singles[s].init(v[s, 0], q[s])
  state = [{k: torch.zeros(S, *t.shape[1:], device='cuda') for k, t in d.items()}
           for d in model.construct_initial_causal_state(N, len(qf.resolutions) - 1)]
  e_t = e_l = 0.0
  vis_mismatch = 0
  for t in range(T):
    tracks, vis = trk.step(v[:, t])
    assert tuple(tracks.shape) == (S, N, 1, 2) and tuple(vis.shape) == (S, N, 1)
    occ, expd = trk.last_logits
    gr = model.get_feature_grids(v[:, t:t + 1], False)
    r = model.estimate_trajectories((256, 256), False, gr, qf, None, 64, causal_context=state,
                                    get_causal_context=True)
    state = r['causal_context']
    assert torch.equal(tracks, r['tracks'][-1]), f'frame {t}: graph replay != eager batched call'
    assert torch.equal(occ, r['occlusion'][-1]) and torch.equal(expd, r['expected_dist'][-1])
    for s in range(S):
      t1, v1 = singles[s].step(v[s, t])
      o1, x1 = singles[s].last_logits
      e_t = max(e_t, (tracks[s] - t1[0]).abs().max().item())
      e_l = max(e_l, (occ[s] - o1[0]).abs().max().item(), (expd[s] - x1[0]).abs().max().item())
      clear = (_vis_prob(o1[0], x1[0]) - 0.5).abs() > 1e-3
      vis_mismatch += int((vis[s][clear] != v1[0][clear]).sum())
  for s in singles:
    s.close()
  trk.close()
  U.record('tracker_multi_stream', streams=S, points=N, frames=T, tracks_vs_single=e_t,
           logits_vs_single=e_l, vis_mismatch=vis_mismatch)
  assert e_t <= TRACK_TOL and e_l <= LOGIT_TOL and vis_mismatch == 0


def test_tracker_multi_stream_golden_clip_in_stream_one():
  g = load_golden('causal_256x6_n16')
  meta = g['meta']
  model, _, _ = get_model(causal=True)
  N, T = meta['N'], meta['T']
  gv = synth.make_video(T, meta['H'], meta['W'], seed=meta['video_seed'])
  gq = synth.make_queries(N, T, meta['H'], meta['W'], seed=meta['query_seed'], frame0_only=True)
  ov, oq = _stream_clips(2, T, N, seeds=(21, 25))
  v = torch.cat([ov[:1], gv.cuda(), ov[1:]])
  q = torch.cat([oq[:1], gq.cuda(), oq[1:]])
  trk = streaming.OnlineTracker(model, meta['H'], meta['W'], N, num_streams=3)
  trk.init(v[:, 0], q)
  tr, oc, ex = [], [], []
  for t in range(T):
    tracks, _ = trk.step(v[:, t])
    occ, expd = trk.last_logits
    tr.append(tracks[1].cpu().numpy())
    oc.append(occ[1].cpu().numpy())
    ex.append(expd[1].cpu().numpy())
  trk.close()
  e_t = np.abs(np.concatenate(tr, 1) - g['online_tracks']).max()
  e_o = np.abs(np.concatenate(oc, 1) - g['online_occlusion']).max()
  e_e = np.abs(np.concatenate(ex, 1) - g['online_expected_dist']).max()
  U.record('tracker_multi_stream_golden', tracks_err=e_t, occ_err=e_o, expd_err=e_e)
  assert e_t < TRACK_TOL and e_o < LOGIT_TOL and e_e < LOGIT_TOL


def test_tracker_streams_are_isolated():
  """Changing stream 2's frames and re-targeting one of its points leaves streams 0 and 1 (their
  outputs every frame and their causal state) bit for bit unchanged."""
  model, _, _ = get_model(causal=True)
  S, N, T = 3, 64, 5
  v, q = _stream_clips(S, T, N, seeds=(3, 7, 11))
  other, _ = _stream_clips(1, T, N, seeds=(31,))

  def run(disturb):
    trk = streaming.OnlineTracker(model, 256, 256, N, num_streams=S)
    frames = v.clone()
    if disturb:
      frames[2] = other[0]
    trk.init(frames[:, 0], q)
    outs = []
    for t in range(T):
      if disturb and t == 2:
        trk.update_query(frames[2, 1], torch.tensor([0.0, 40.5, 200.25]), 9, stream=2)
      tracks, vis = trk.step(frames[:, t])
      occ, expd = trk.last_logits
      outs.append([x.clone() for x in (tracks, vis, occ, expd)])
    state = [{k: x[:2].clone() for k, x in d.items()} for d in trk.state]
    trk.close()
    return outs, state

  (a, sa), (b, sb) = run(False), run(True)
  for t in range(T):
    for x, y in zip(a[t], b[t]):
      assert torch.equal(x[:2], y[:2]), f'frame {t}'
  assert any(not torch.equal(x[2], y[2]) for x, y in zip(a[-1], b[-1]))
  for da, db in zip(sa, sb):
    for k in da:
      assert torch.equal(da[k], db[k]), k
  U.record('tracker_stream_isolation', equal=1)


def test_tracker_rejects_wrong_shapes():
  model, _, _ = get_model(causal=True)
  S, N = 3, 8
  v, q = _stream_clips(S, 1, N, seeds=(3, 7, 11))
  trk = streaming.OnlineTracker(model, 256, 256, N, num_streams=S)
  with pytest.raises(ValueError):
    trk.init(v[:2, 0], q[:2])  # two streams
  with pytest.raises(ValueError):
    trk.init(v[:, 0], q[:, :5])  # five points
  with pytest.raises(ValueError):
    trk.init(v[:, 0, :128], q)  # wrong frame size
  trk.init(v[:, 0], q)
  with pytest.raises(ValueError):
    trk.step(v[0, 0])  # one frame for three streams
  with pytest.raises(ValueError):
    trk.update_query(v[0, 0], torch.tensor([0.0, 1.0, 1.0]), 0, stream=3)
  trk.close()


def test_tracker_step_launches():
  """A step over S streams is the launch sequence of a one-stream step; only the split-K reduce
  launches, which depend on the row count, may differ.  They are left out by counting with the
  library's own profiler, which times every launch but those.  (A torch.profiler session here
  would make later sessions in this process miss kernels once CUDA graphs have run in between.)"""
  lib = _lib.load()
  model, _, _ = get_model(causal=True)
  N = 16
  counts, reduces = {}, {}
  for S in (1, 4):
    v, q = _stream_clips(S, 1, N, seeds=tuple(range(3, 3 + 4 * S, 4)))
    trk = streaming.OnlineTracker(model, 256, 256, N, num_streams=S)
    trk.init(v[:, 0], q)
    trk._frame.copy_(v[:, :1])
    trk._step_eager()  # warm-up
    torch.cuda.synchronize()
    l0 = U.launch_count()
    lib.tapir_profile_enable(1)
    trk._step_eager()
    buf = ctypes.create_string_buffer(1 << 16)
    _lib.check(lib.tapir_profile_report(buf, len(buf)), 'tapir_profile_report')
    lib.tapir_profile_enable(0)
    counts[S] = sum(x['launches'] for x in json.loads(buf.value.decode()).values())
    reduces[S] = U.launch_count() - l0 - counts[S]
    trk.close()
  U.record('tracker_step_launches_without_splitk_reduce', s1=counts[1], s4=counts[4],
           reduce_s1=reduces[1], reduce_s4=reduces[4])
  assert counts[1] == counts[4]
