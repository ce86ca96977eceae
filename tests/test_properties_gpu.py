"""Size-independent properties at BASELINE.json's full sizes (the oracle is too slow there).

c2: 256x256x48, 256 queries; c3: causal streaming, 1024 queries; c5: 1024x1024 (3 refinement
levels) on a reduced clip against the oracle; c4 (multi-GPU): tests/multi_gpu_check.py.
"""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import synth  # noqa: E402
from oracle import tapir_oracle as O  # noqa: E402
from tapnet_b200 import tapir_model  # noqa: E402
from tests import gpu_util as U  # noqa: E402
from tests.test_stages_gpu import get_model  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_c2_chunk_and_permutation_invariance_and_passthrough():
  model, _, _ = get_model()
  T, N = 48, 256
  video = synth.make_video(T).cuda()
  q = synth.make_queries(N, T).cuda()
  out = model(video, q)
  # (a) different chunking + permuted queries: queries are independent, so nothing may change
  perm = torch.randperm(N, generator=torch.Generator().manual_seed(7)).cuda()
  old = tapir_model._MAX_ROWS_PER_CHUNK
  tapir_model._MAX_ROWS_PER_CHUNK = 37 * T  # ragged chunks of 37 queries
  try:
    out_p = model(video, q[:, perm])
  finally:
    tapir_model._MAX_ROWS_PER_CHUNK = old
  e_t = (out_p['tracks'] - out['tracks'][:, perm]).abs().max().item()
  e_o = (out_p['occlusion'] - out['occlusion'][:, perm]).abs().max().item()
  # (b) iteration-0 tracks pass exactly through the query point on the query frame
  # (utils.py:171-191); later iterations move it (SURVEY.md section 4)
  t0 = out['unrefined_tracks'][0][0]  # [N, T, 2]
  qi = q[0, :, 0].long()
  got = t0[torch.arange(N, device='cuda'), qi]
  e_q = (got - torch.flip(q[0, :, 1:3], dims=(-1,))).abs().max().item()
  # (c) stage A of a frame does not depend on the other frames (T-slice independence)
  half = model(video[:, :24], torch.cat([q[..., :1].clamp(max=23), q[..., 1:]], -1))
  sel = (q[0, :, 0] < 24)
  e_s = (half['unrefined_tracks'][0][0, sel] - t0[sel, :24]).abs().max().item()
  e_so = (half['unrefined_occlusion'][0][0, sel] - out['unrefined_occlusion'][0][0, sel, :24]).abs().max().item()
  U.record('c2_properties', chunk_perm_tracks=e_t, chunk_perm_occ=e_o, query_passthrough=e_q,
           tslice_tracks=e_s, tslice_occ=e_so)
  assert e_t <= 1e-4 and e_o <= 1e-5
  assert e_q == 0.0
  assert e_s <= 1e-3 and e_so <= 1e-4
  assert torch.isfinite(out['tracks']).all() and torch.isfinite(out['expected_dist']).all()


def test_c3_streaming_equals_offline_causal_1024_queries():
  """SURVEY.md 3.2: frame-by-frame with causal state == one offline call of the causal model."""
  model, _, _ = get_model(causal=True)
  T, N = 6, 1024
  video = synth.make_video(T).cuda()
  q = synth.make_queries(N, T, frame0_only=True).cuda()
  g0 = model.get_feature_grids(video[:, :1], False)
  qf = model.get_query_features(video[:, :1], False, q, g0)
  state = model.construct_initial_causal_state(N, len(qf.resolutions) - 1)
  state = [{k: v.cuda() for k, v in d.items()} for d in state]
  tr, oc = [], []
  for t in range(T):
    gr = model.get_feature_grids(video[:, t:t + 1], False)
    r = model.estimate_trajectories((256, 256), False, gr, qf, None, 64, causal_context=state,
                                    get_causal_context=True)
    state = r['causal_context']
    tr.append(r['tracks'][-1])
    oc.append(r['occlusion'][-1])
  full = model.get_feature_grids(video, False)
  off = model.estimate_trajectories((256, 256), False, full, qf, None, 64)
  e_t = (torch.cat(tr, 2) - off['tracks'][-1]).abs().max().item()
  e_o = (torch.cat(oc, 2) - off['occlusion'][-1]).abs().max().item()
  U.record('c3_streaming_vs_offline', tracks=e_t, occ=e_o)
  assert e_t <= 1e-3 and e_o <= 1e-4


def test_c5_hires_1024_against_oracle_reduced_clip():
  """1024x1024 -> refinement at 256/512/1024 (12 iterations); one frame, 8 queries."""
  model, sd, cfg = get_model()
  video = synth.make_video(1, 1024, 1024)
  q = synth.make_queries(8, 1, 1024, 1024)
  torch.set_num_threads(min(16, os.cpu_count() or 1))
  with torch.no_grad():
    ref = O.forward(sd, cfg, video, q)
  out = model(video.cuda(), q.cuda())
  assert len(out['unrefined_tracks']) == 12
  e_t = (out['tracks'].cpu() - ref['tracks']).abs().max().item()
  e_o = (out['occlusion'].cpu() - ref['occlusion']).abs().max().item()
  e_e = (out['expected_dist'].cpu() - ref['expected_dist']).abs().max().item()
  U.record('c5_1024_vs_oracle', tracks=e_t, occ=e_o, expd=e_e)
  # tracks are in 1024-pixel units here: 1e-3 px at 256 scale = 4e-3
  assert e_t <= 4e-3 and e_o <= 1e-4 and e_e <= 1e-4


def test_c3_graph_replay_tracker_equals_eager_streaming():
  """tapnet_b200.streaming.OnlineTracker (CUDA-graph replay) == eager per-frame calls, bit for bit."""
  from tapnet_b200 import streaming
  model, _, _ = get_model(causal=True)
  T, N = 5, 64
  video = synth.make_video(T).cuda()
  q = synth.make_queries(N, T, frame0_only=True).cuda()
  trk = streaming.OnlineTracker(model, 256, 256, N)
  qf = trk.init(video[0, 0], q)
  state = model.construct_initial_causal_state(N, len(qf.resolutions) - 1)
  state = [{k: v.cuda().clone() for k, v in d.items()} for d in state]
  for t in range(T):
    tracks, vis = trk.step(video[0, t])
    gr = model.get_feature_grids(video[:, t:t + 1], False)
    r = model.estimate_trajectories((256, 256), False, gr, qf, None, 64, causal_context=state,
                                    get_causal_context=True)
    state = r['causal_context']
    assert torch.equal(tracks, r['tracks'][-1]), f'frame {t}'
    occ, expd = trk.last_logits
    assert torch.equal(occ, r['occlusion'][-1]) and torch.equal(expd, r['expected_dist'][-1])
  U.record('c3_graph_tracker', frames=T, equal=1)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_c4_sharded_equals_single_gpu():
  port = 29500 + os.getpid() % 1000
  cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2',
         '--master-addr', '127.0.0.1', '--master-port', str(port),
         os.path.join(ROOT, 'tests', 'multi_gpu_check.py')]
  p = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
  print(p.stdout[-2000:], p.stderr[-2000:])
  assert p.returncode == 0 and 'MULTI_GPU_OK' in p.stdout


def test_update_query_features_and_tracker_update_query_on_device():
  """`TAPIR.update_query_features` (reference tapir_model.py:774-806) on CUDA tensors and its
  graph-safe twin `OnlineTracker.update_query` (pytorch_live_demo.py:188-200): re-targeting a
  point overwrites exactly that point's query features, zeroes exactly its causal state (through
  every aliased dict), and the following frames equal a tracker that started from scratch with
  the new point at that slot and a zero state for it."""
  from tapnet_b200 import streaming
  model, sd, cfg = get_model(causal=True)
  T, N, idx = 4, 16, 5
  video = synth.make_video(T).cuda()
  q = synth.make_queries(N, T, frame0_only=True).cuda()
  # --- the model method itself, CUDA tensors, against the oracle-free definition
  g0 = model.get_feature_grids(video[:, :1], False)
  qf = model.get_query_features(video[:, :1], False, q, g0)
  qf = tapir_model.QueryFeatures(tuple(t.clone() for t in qf.lowres),
                                 tuple(t.clone() for t in qf.hires), qf.resolutions)
  before_lo = [t.clone() for t in qf.lowres]
  state = model.construct_initial_causal_state(N, len(qf.resolutions) - 1)
  state = [{k: torch.full_like(v, 3.0).cuda() for k, v in d.items()} for d in state]
  new_pt = torch.tensor([[[0.0, 77.25, 130.5]]], device='cuda')
  g1 = model.get_feature_grids(video[:, 1:2], False)
  new_qf = model.get_query_features(video[:, 1:2], False, new_pt, g1)
  qf2, state2 = model.update_query_features(qf, new_qf, idx, state)
  for lvl in range(len(qf2.lowres)):
    assert torch.equal(qf2.lowres[lvl][:, idx], new_qf.lowres[lvl][:, 0])
    assert torch.equal(qf2.hires[lvl][:, idx], new_qf.hires[lvl][:, 0])
    keep = [i for i in range(N) if i != idx]
    assert torch.equal(qf2.lowres[lvl][:, keep], before_lo[lvl][:, keep])
  for d in state2:
    for k, v in d.items():
      assert float(v[:, idx].abs().max()) == 0.0, k
      assert float((v[:, [i for i in range(N) if i != idx]] - 3.0).abs().max()) == 0.0, k
  # --- tracker: re-target after 2 frames, compare frames 2.. with explicit eager calls
  trk = streaming.OnlineTracker(model, 256, 256, N)
  trk.init(video[0, 0], q)
  trk.step(video[0, 0])
  trk.step(video[0, 1])
  trk.update_query(video[0, 1], new_pt[0, 0], idx)
  # eager twin: same features / state, advanced by the model's own methods
  qf_e = tapir_model.QueryFeatures(tuple(t.clone() for t in trk.query_features.lowres),
                                   tuple(t.clone() for t in trk.query_features.hires),
                                   trk.query_features.resolutions)
  st_e = [{k: v.clone() for k, v in d.items()} for d in trk.state]
  assert float(st_e[0]['block_0_causal_1'][:, idx].abs().max()) == 0.0
  assert torch.equal(qf_e.lowres[-1][:, idx], new_qf.lowres[-1][:, 0])
  for t in (2, 3):
    tracks, _ = trk.step(video[0, t])
    gr = model.get_feature_grids(video[:, t:t + 1], False)
    r = model.estimate_trajectories((256, 256), False, gr, qf_e, None, 64, causal_context=st_e,
                                    get_causal_context=True)
    st_e = r['causal_context']
    assert torch.equal(tracks, r['tracks'][-1]), f'frame {t}'
  trk.close()
  U.record('update_query_gpu', ok=1)


def test_zero_queries_and_context_semantics():
  """Edge cases of the reference surface: no query points (empty, correctly shaped outputs), and
  get_causal_context without a causal_context (empty dicts, nets.py:143-176)."""
  model, _, _ = get_model()
  T = 3
  video = synth.make_video(T).cuda()
  q0 = torch.zeros(1, 0, 3, device='cuda')
  out = model(video, q0)
  assert tuple(out['tracks'].shape) == (1, 0, T, 2)
  assert tuple(out['occlusion'].shape) == (1, 0, T)
  assert len(out['unrefined_tracks']) == 4
  q = synth.make_queries(4, T).cuda()
  g = model.get_feature_grids(video, False)
  qf = model.get_query_features(video, False, q, g)
  r = model.estimate_trajectories((256, 256), False, g, qf, q, 64, get_causal_context=True)
  assert len(r['causal_context']) == 4 and all(d == {} for d in r['causal_context'])
  with pytest.raises(ValueError):
    st = [{k: v.cuda() for k, v in d.items()} for d in model.construct_initial_causal_state(4, 1)]
    model.estimate_trajectories((256, 256), False, g, qf, q, 64, causal_context=st)


def test_tracker_survives_workspace_growth():
  """A captured graph bakes raw workspace pointers; a later, larger call on the same model
  replaces the model's workspaces.  The tracker must notice and stay correct (ADVICE r1)."""
  from tapnet_b200 import streaming
  model, _, _ = get_model(causal=True)
  T, N = 4, 32
  video = synth.make_video(T).cuda()
  q = synth.make_queries(N, T, frame0_only=True).cuda()

  def run(disturb):
    trk = streaming.OnlineTracker(model, 256, 256, N)
    trk.init(video[0, 0], q)
    outs = []
    for t in range(T):
      if disturb and t == 2:
        gen = model._ws_generation
        big = synth.make_queries(8192, T).cuda()  # outgrows every workspace of the tracker
        model(video, big)
        assert model._ws_generation != gen and model._ws_retired, 'workspaces were not replaced'
      outs.append(trk.step(video[0, t])[0].clone())
    trk.close()
    return torch.cat(outs, 2)

  a, b = run(False), run(True)
  assert torch.equal(a, b)
  U.record('tracker_workspace_growth', equal=1)


def test_host_clip_streamed_in_equals_device_clip():
  """model(host video, host queries): the clip is copied in frame chunks behind the stem conv;
  results must equal the device-resident call bit for bit (float and uint8 clips)."""
  model, _, _ = get_model()
  T, N = 13, 24   # 13 frames: ragged sub-chunks
  video = synth.make_video(T)
  q = synth.make_queries(N, T)
  ref = model(video.cuda(), q.cuda())
  got = model(video.pin_memory(), q.pin_memory())
  assert torch.equal(ref['tracks'], got['tracks']) and torch.equal(ref['occlusion'], got['occlusion'])
  u8 = ((video + 1) * 127.5).round().clamp(0, 255).to(torch.uint8)
  ref8 = model(u8.cuda(), q.cuda())
  got8 = model(u8.pin_memory(), q)   # pageable queries are fine too
  assert torch.equal(ref8['tracks'], got8['tracks'])
  assert torch.equal(ref8['expected_dist'], got8['expected_dist'])
  # a clip whose first pass resizes (480 -> 256) takes the copy-everything-first route
  v480 = synth.make_video(2, 480, 480)
  q480 = synth.make_queries(6, 2, 480, 480)
  a = model(v480.cuda(), q480.cuda())
  b = model(v480.pin_memory(), q480.pin_memory())
  assert torch.equal(a['tracks'], b['tracks'])
  U.record('host_clip_streaming', equal=1)


def test_batch_of_two_clips_equals_two_calls():
  """B = 2 (the reference's einshape equations carry a batch axis everywhere): same results as
  two B = 1 calls, bit for bit."""
  model, _, _ = get_model()
  T, N = 5, 12
  v = torch.cat([synth.make_video(T, seed=1), synth.make_video(T, seed=5)], 0).cuda()
  q = torch.cat([synth.make_queries(N, T, seed=2), synth.make_queries(N, T, seed=6)], 0).cuda()
  both = model(v, q)
  for b in range(2):
    one = model(v[b:b + 1], q[b:b + 1])
    assert torch.equal(both['tracks'][b], one['tracks'][0])
    assert torch.equal(both['occlusion'][b], one['occlusion'][0])
    assert torch.equal(both['expected_dist'][b], one['expected_dist'][0])
  U.record('batch_two_clips', equal=1)
