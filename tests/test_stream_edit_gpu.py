"""Point edits inside the online tracker's step: tapir_sample_query_rows against
tapir_sample_query_features bit for bit (one and per-clip video sizes, 1 and 4 levels, shuffled
requests, count 0 and count = capacity, untouched rows, zeroed state rows, CUDA-graph replay with
the table changed between replays), and OnlineTracker.retarget / add_points / remove_points
against update_query + step, the group's own grids, fresh trackers and unedited trackers."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import synth  # noqa: E402
from tapnet_b200 import _lib, streaming  # noqa: E402
from tests import gpu_util as U  # noqa: E402
from tests.conftest import load_golden  # noqa: E402
from tests.test_stages_gpu import get_model  # noqa: E402
from tests.test_stream_points_gpu import COUNTS, _inputs  # noqa: E402
from tests.test_tracker_sizes_gpu import LOGIT_TOL, SIZES, TRACK_TOL  # noqa: E402


def _bits(x):
  return x.contiguous().view(torch.int32)


# ------------------------------------------------------------------------- the kernel
CLIP_SIZES = [(256, 256), (240, 320), (200, 200)]
ROWS = 11
NUM_BLOCKS = 3


def _kernel_inputs(levels, seed):
  g = torch.Generator().manual_seed(seed)
  G = len(CLIP_SIZES)
  # a lowres (256 channels) and a hires (128 channels) grid per level
  dims = [(32, 32, 256), (64, 64, 128), (16, 24, 256), (20, 12, 128), (8, 8, 256), (7, 9, 128),
          (40, 40, 256), (3, 5, 128)][:2 * levels]
  grids = [torch.randn(G, 1, h, w, C, generator=g).cuda() for h, w, C in dims]
  # sentinel rows: every row that is not requested must keep these bits
  outs = [torch.randn(1, ROWS, C, generator=g).cuda() for _, _, C in dims]
  state = [{f'block_{i}_causal_{j}': torch.randn(1, ROWS, 2, width, generator=g).cuda()
            for i in range(NUM_BLOCKS) for j, width in ((1, 512), (2, 2048))} for _ in range(2)]
  return grids, outs, state


def _requests(kind, seed):
  g = torch.Generator().manual_seed(seed)
  G = len(CLIP_SIZES)
  rows = torch.randperm(ROWS, generator=g).tolist()
  if kind == 'none':
    rows = []
  elif kind == 'some':
    rows = rows[:4]
  reqs = []
  for r in rows:
    clip = int(torch.randint(G, (1,), generator=g))
    h, w = CLIP_SIZES[clip]
    t, y, x = torch.rand(3, generator=g).tolist()
    reqs.append((r, clip, 0.0 if r % 2 else 5.0 * t, y * h, x * w))
  return reqs


def _expected(grids, outs, state, reqs, per_clip):
  want_outs = [o.clone() for o in outs]
  want_state = [{k: v.clone() for k, v in d.items()} for d in state]
  for row, clip, t, y, x in reqs:
    vh, vw = CLIP_SIZES[clip] if per_clip else CLIP_SIZES[0]
    q = torch.tensor([[t, y, x]], device='cuda')
    for gr, o in zip(grids, want_outs):
      one = torch.empty(1, gr.shape[-1], device='cuda')
      _lib.sample_query_features(gr[clip].contiguous(), q, (1, vh, vw), one)
      o[0, row] = one[0]
    for d in want_state:
      for v in d.values():
        v[0, row] = 0
  return want_outs, want_state


def _assert_equal(outs, state, want_outs, want_state, what):
  for i, (o, w) in enumerate(zip(outs, want_outs)):
    assert torch.equal(_bits(o), _bits(w)), f'{what}: grid {i}'
  for d, dw in zip(state, want_state):
    for k in d:
      assert torch.equal(_bits(d[k]), _bits(dw[k])), f'{what}: state {k}'


def _video_hw(per_clip):
  if per_clip:
    return torch.tensor(CLIP_SIZES, dtype=torch.int32, device='cuda')
  return CLIP_SIZES[0]


@pytest.mark.parametrize('per_clip', [False, True], ids=['one_size', 'per_clip_sizes'])
@pytest.mark.parametrize('levels', [1, 4])
@pytest.mark.parametrize('kind', ['none', 'some', 'all'])
def test_sample_query_rows_equals_sample_query_features(per_clip, levels, kind):
  seed = 3 * levels + int(per_clip) + 10 * len(kind)
  grids, outs, state = _kernel_inputs(levels, seed)
  reqs = _requests(kind, seed)
  want = _expected(grids, outs, state, reqs, per_clip)
  table = _lib.query_request_table(ROWS, 'cuda')
  host = _lib.query_request_table(ROWS, 'cpu')
  _lib.write_query_requests(host, reqs)
  table.copy_(host)
  _lib.sample_query_rows(grids, outs, _video_hw(per_clip), table,
                         _lib.state_pointer_table(state, ROWS))
  torch.cuda.synchronize()
  _assert_equal(outs, state, *want, f'{kind} requests')


def test_sample_query_rows_skips_requests_out_of_range():
  grids, outs, state = _kernel_inputs(1, 5)
  good = _requests('some', 5)
  bad = [(ROWS, 0, 0.0, 10.0, 10.0), (-1, 0, 0.0, 10.0, 10.0), (2, 3, 0.0, 1.0, 1.0),
         (2, -1, 0.0, 1.0, 1.0)]
  want = _expected(grids, outs, state, good, True)
  host = _lib.query_request_table(ROWS, 'cpu')
  _lib.write_query_requests(host, bad[:2] + good + bad[2:])
  table = host.cuda()
  _lib.sample_query_rows(grids, outs, _video_hw(True), table, _lib.state_pointer_table(state, ROWS))
  torch.cuda.synchronize()
  _assert_equal(outs, state, *want, 'out-of-range requests')


def test_sample_query_rows_replays_in_a_cuda_graph_with_new_tables():
  grids, outs, state = _kernel_inputs(4, 9)
  table = _lib.query_request_table(ROWS, 'cuda')
  ptrs = _lib.state_pointer_table(state, ROWS)
  vhw = _video_hw(True)
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):  # warm-up (module load) with an empty table
    _lib.sample_query_rows(grids, outs, vhw, table, ptrs)
  torch.cuda.current_stream().wait_stream(side)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    _lib.sample_query_rows(grids, outs, vhw, table, ptrs)
  host = _lib.query_request_table(ROWS, 'cpu')
  for step, kind in enumerate(['some', 'none', 'all', 'some']):
    reqs = _requests(kind, 100 + step)
    want = _expected(grids, outs, state, reqs, True)
    _lib.write_query_requests(host, reqs)
    table.copy_(host)
    graph.replay()
    torch.cuda.synchronize()
    _assert_equal(outs, state, *want, f'replay {step} ({kind})')


def test_sample_query_rows_rejects_bad_arguments():
  grids, outs, state = _kernel_inputs(1, 1)
  table = _lib.query_request_table(ROWS, 'cuda')
  with pytest.raises(ValueError):
    _lib.sample_query_rows(grids, outs[:0], CLIP_SIZES[0], table)
  with pytest.raises(ValueError):
    _lib.sample_query_rows(grids, outs, CLIP_SIZES[0], table[:-1])
  with pytest.raises(ValueError):
    _lib.state_pointer_table(state, ROWS + 1)
  with pytest.raises(_lib.TapirB200Error):
    _lib.sample_query_rows(grids, outs, (0, 256), table)


# ------------------------------------------------------------------------- the tracker
def _tracker_state_equal(a, b, what):
  for ga, gb in zip(a._groups, b._groups):
    for da, db in zip(ga.state, gb.state):
      for k in da:
        assert torch.equal(_bits(da[k]), _bits(db[k])), f'{what}: state {k}'


@pytest.mark.parametrize('uint8', [False, True], ids=['float', 'uint8'])
def test_retarget_equals_update_query_then_step(uint8):
  """On a one-stream tracker, retarget before step(frame_k) equals update_query(frame_k) +
  step(frame_k) bit for bit: both sample the one-frame grids of frame_k."""
  model, _, _ = get_model(causal=True)
  T, N = 6, 16
  video = synth.make_video(T, 256, 256, seed=21)[0].cuda()
  if uint8:
    video = ((video + 1) * 127.5).round().clamp(0, 255).to(torch.uint8)
  q = synth.make_queries(N, T, 256, 256, seed=22, frame0_only=True)[0].cuda()
  a = streaming.OnlineTracker(model, 256, 256, N, uint8_frames=uint8)
  b = streaming.OnlineTracker(model, 256, 256, N, uint8_frames=uint8)
  a.init(video[0], q)
  b.init(video[0], q)
  edits = {1: ([3], [[0.0, 100.5, 37.25]]), 2: ([0, 15, 3], [[2.0, 5.0, 250.0], [0.0, 128.0, 128.0],
                                                             [0.0, 1.0, 2.0]]),
           4: ([7, 7], [[0.0, 30.0, 30.0], [0.0, 200.25, 60.75]])}
  for t in range(T):
    if t in edits:
      idx, pts = edits[t]
      a.retarget(torch.tensor(pts), idx)
      for i, p in zip(idx, pts):
        b.update_query(video[t], torch.tensor(p), i)
    ta, va = a.step(video[t])
    tb, vb = b.step(video[t])
    assert torch.equal(_bits(ta), _bits(tb)) and torch.equal(va, vb), f'frame {t}'
    for x, y in zip(a.last_logits, b.last_logits):
      assert torch.equal(_bits(x), _bits(y)), f'frame {t}: logits'
    for x, y in zip(a.query_features.lowres + a.query_features.hires,
                    b.query_features.lowres + b.query_features.hires):
      assert torch.equal(_bits(x), _bits(y)), f'frame {t}: query features'
    _tracker_state_equal(a, b, f'frame {t}')
  # a one-stream tracker keeps an int count: add and remove, outputs [1, N', 1, 2]
  assert a.add_points(torch.tensor([[0.0, 10.0, 10.0], [0.0, 20.0, 20.0]])) == [N, N + 1]
  a.remove_points([0])
  assert a.num_points == N + 1
  tr, vi = a.step(video[0])
  assert tuple(tr.shape) == (1, N + 1, 1, 2) and tuple(vi.shape) == (1, N + 1, 1)
  a.close()
  b.close()


def test_multi_stream_retarget_rows_equal_the_group_grids():
  """On a multi-stream tracker, the rows retarget writes equal get_query_features on the step's
  own group grids bit for bit.  They differ from update_query(frame), which samples a one-frame
  pass of the frame: a group of several streams runs one backbone pass over all of them."""
  model, _, _ = get_model(causal=True)
  T, S = 2, len(SIZES)
  frames, qs = _inputs(SIZES, COUNTS, T)
  trk = streaming.OnlineTracker(model, [h for h, _ in SIZES], [w for _, w in SIZES], COUNTS,
                                num_streams=S)
  trk.init([f[0] for f in frames], qs)
  edits = {2: ([0, 32], [[0.0, 20.5, 100.25], [0.0, 150.0, 3.0]]), 3: ([129], [[0.0, 7.0, 230.0]]),
           4: ([5], [[0.0, 400.0, 17.0]])}
  for s, (idx, pts) in edits.items():
    trk.retarget(torch.tensor(pts), idx, stream=s)
  trk.step([f[1] for f in frames])
  torch.cuda.synchronize()
  for s, (idx, pts) in edits.items():
    gi, slot = trk._slot[s]
    g = trk._groups[gi]
    grids = trk._group_grids(g)  # the static inputs still hold this step's frames
    clip = type(grids)(tuple(x[slot:slot + 1] for x in grids.lowres),
                       tuple(x[slot:slot + 1] for x in grids.hires), grids.resolutions)
    video = torch.empty(1, 1, *SIZES[s], 3, device='cuda')
    want = model.get_query_features(video, False, torch.tensor(pts, device='cuda')[None], clip)
    for got, w in zip(g.query_features.lowres + g.query_features.hires, want.lowres + want.hires):
      rows = [g.offsets[slot] + i for i in idx]
      assert torch.equal(_bits(got[0, rows]), _bits(w[0])), f'stream {s}'
  trk.close()


def test_add_and_remove_points_equal_a_fresh_tracker_and_leave_other_groups():
  """After add_points on stream 1 (its own group) and remove_points on stream 2 (the group of
  streams 2 and 3), later steps equal a fresh tracker of the new counts whose group rows are
  copied from the edited one, bit for bit; streams 0 and 4 (groups without edits) equal those of
  an unedited tracker."""
  model, _, _ = get_model(causal=True)
  T, S = 5, len(SIZES)
  hs, ws = [h for h, _ in SIZES], [w for _, w in SIZES]
  frames, qs = _inputs(SIZES, COUNTS, T)
  edited = streaming.OnlineTracker(model, hs, ws, COUNTS, num_streams=S)
  plain = streaming.OnlineTracker(model, hs, ws, COUNTS, num_streams=S)
  for trk in (edited, plain):
    trk.init([f[0] for f in frames], qs)
    trk.step([f[0] for f in frames])
  new = edited.add_points(torch.tensor([[0.0, 10.0, 20.0], [0.0, 200.0, 300.0], [0.0, 5.5, 6.5]]),
                          stream=1)
  assert new == [1, 2, 3]
  edited.remove_points([0, 17, 32], stream=2)
  edited.retarget(torch.tensor([[0.0, 50.0, 60.0]]), [16], stream=2)  # old point 18
  counts = [8, 4, 30, 130, 8]
  assert edited.num_points == counts
  for trk in (edited, plain):
    trk.step([f[1] for f in frames])
  fresh = streaming.OnlineTracker(model, hs, ws, counts, num_streams=S)
  fresh.init([f[1] for f in frames], [torch.zeros(n, 3, device='cuda') for n in counts])
  for gf, ge in zip(fresh._groups, edited._groups):
    assert gf.counts == ge.counts and gf.offsets == ge.offsets
    for x, y in zip(gf.query_features.lowres + gf.query_features.hires,
                    ge.query_features.lowres + ge.query_features.hires):
      x.copy_(y)
    for dx, dy in zip(gf.state, ge.state):
      for k in dx:
        dx[k].copy_(dy[k])
  for t in range(2, T):
    fr = [f[t] for f in frames]
    te, ve = edited.step(fr)
    le = [[x.clone() for x in lst] for lst in edited.last_logits]
    te, ve = [x.clone() for x in te], [x.clone() for x in ve]
    tf, vf = fresh.step(fr)
    lf = fresh.last_logits
    tp, vp = plain.step(fr)
    lp = plain.last_logits
    for s in range(S):
      assert torch.equal(_bits(te[s]), _bits(tf[s])) and torch.equal(ve[s], vf[s]), f'{t}, {s}'
      for x, y in zip(le, lf):
        assert torch.equal(_bits(x[s]), _bits(y[s])), f'frame {t} stream {s}: logits'
    for s in (0, 4):
      assert torch.equal(_bits(te[s]), _bits(tp[s])) and torch.equal(ve[s], vp[s]), f'{t}, {s}'
      for x, y in zip(le, lp):
        assert torch.equal(_bits(x[s]), _bits(y[s]))
    _tracker_state_equal(edited, fresh, f'frame {t}')
  for trk in (edited, fresh, plain):
    trk.close()


def test_launches_per_step_one_more_per_group_after_an_edit():
  model, _, _ = get_model(causal=True)
  S = len(SIZES)
  frames, qs = _inputs(SIZES, COUNTS, 1)
  trk = streaming.OnlineTracker(model, [h for h, _ in SIZES], [w for _, w in SIZES], COUNTS,
                                num_streams=S)
  trk.init([f[0] for f in frames], qs)

  def launches():
    trk._step_eager()
    torch.cuda.synchronize()
    l0 = U.launch_count()
    trk._step_eager()
    return U.launch_count() - l0
  before = launches()
  assert all(g.edits is None for g in trk._groups)
  trk.retarget(torch.tensor([[0.0, 3.0, 4.0]]), [0], stream=0)
  trk._upload_edits()
  after = launches()
  U.record('stream_edit_launches', unedited=before, edited=after, groups=len(trk._groups))
  assert after == before + len(trk._groups)
  trk.close()


def test_edit_sequence_against_the_reference_golden_and_eager_calls():
  """The golden causal_edit_256x6_n16 (the reference's own functions: re-target point 3 and
  append 4 points at frame 2, remove points 0 and 9 at frame 4) on a one-stream tracker, within
  the streaming goldens' tolerances; each replayed step equals the eager grouped calls bit for bit."""
  g = load_golden('causal_edit_256x6_n16')
  meta, e = g['meta'], g['meta']['edits']
  model, _, _ = get_model(causal=True)
  T, N, H, W = meta['T'], meta['N'], meta['H'], meta['W']
  video = synth.make_video(T, H, W, seed=meta['video_seed'])[0].cuda()
  q = synth.make_queries(N, T, H, W, seed=meta['query_seed'], frame0_only=True)[0].cuda()
  trk = streaming.OnlineTracker(model, H, W, N)
  trk.init(video[0], q)
  grp = trk._groups[0]
  e_t = e_l = 0.0
  for t in range(T):
    if t == e['retarget_frame']:
      trk.retarget(torch.tensor([e['retarget_point']]), [e['retarget_idx']])
    if t == e['add_frame']:
      n = trk.num_points
      assert trk.add_points(torch.tensor(e['add_points'])) == list(range(n, n + len(e['add_points'])))
    if t == e['remove_frame']:
      trk.remove_points(e['remove_idx'])
    assert trk.num_points == meta['counts'][t]
    saved = [{k: v.clone() for k, v in d.items()} for d in grp.state]
    tracks, _ = trk.step(video[t])
    out = [x[0].clone() for x in (tracks,) + tuple(trk.last_logits)]
    state = [{k: v.clone() for k, v in d.items()} for d in grp.state]
    # the eager grouped calls from the same state (the request table still holds this step's edits)
    for d, sv in zip(grp.state, saved):
      for k in d:
        d[k].copy_(sv[k])
    eager = trk._step_group(grp, grp.state)
    for x, y in zip(out, eager):
      assert torch.equal(_bits(x), _bits(y[0])), f'frame {t}: replay != eager'
    for d, sv in zip(grp.state, state):
      for k in d:
        assert torch.equal(_bits(d[k]), _bits(sv[k])), f'frame {t}: state {k}'
    want = [torch.from_numpy(g[f'online_{k}_{t}']) for k in ('tracks', 'occlusion', 'expected_dist')]
    e_t = max(e_t, (out[0].cpu() - want[0]).abs().max().item())
    e_l = max(e_l, (out[1].cpu() - want[1]).abs().max().item(), (out[2].cpu() - want[2]).abs().max().item())
  trk.close()
  U.record('stream_edit_golden', frames=T, counts=str(meta['counts']), tracks=e_t, logits=e_l)
  assert e_t < TRACK_TOL and e_l < LOGIT_TOL
