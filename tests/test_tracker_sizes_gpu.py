"""Streams of different frame sizes in one OnlineTracker: the multi-frame ingest against per-frame
resample_frames, per-clip video sizes in estimate_trajectories against single-clip calls, and the
mixed-size tracker against one-stream trackers, the golden clip, its own eager calls and itself
with one stream disturbed."""
import ctypes
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import synth  # noqa: E402
from tapnet_b200 import _lib, live, streaming  # noqa: E402
from tests import gpu_util as U  # noqa: E402
from tests.conftest import load_golden  # noqa: E402
from tests.test_stages_gpu import get_model  # noqa: E402
from tests.test_yuv_gpu import make_frames  # noqa: E402

TRACK_TOL = 1e-3
LOGIT_TOL = 1e-4


def _bits(x):
  return x.contiguous().view(torch.int32)


# ------------------------------------------------------------------------- multi-frame ingest
def _ingest_sources():
  """(frame given to ingest_frames_multi, the same frame as resample_frames takes it alone)."""
  g = torch.Generator().manual_seed(5)
  out = []
  u8 = torch.randint(0, 256, (300, 400, 3), generator=g, dtype=torch.uint8).cuda()
  out.append((u8, u8[None]))
  wide = torch.randint(0, 256, (181, 260, 3), generator=g, dtype=torch.uint8).cuda()
  out.append((wide[:, 7:7 + 203], wide[:, 7:7 + 203].contiguous()[None]))  # pitched rows
  out.append((u8[:256, :256].contiguous(), u8[:256, :256].contiguous()[None]))  # same size: copy
  big = torch.randint(0, 256, (517, 333, 3), generator=g, dtype=torch.uint8).cuda()
  out.append((big[:, 11:11 + 301], big[:, 11:11 + 301].contiguous()[None]))  # pitched, upsized
  odd = torch.randint(0, 256, (1, 9, 3), generator=g, dtype=torch.uint8).cuda()
  out.append((odd, odd[None]))  # one row
  for layout, hw, win, seed in (('nv12', (241, 323), (3, 5, 199, 251), 1),
                                ('i420', (480, 640), (0, 80, 480, 480), 2),
                                ('nv12', (97, 131), None, 3)):
    yuv, _ = make_frames(1, 1, *hw, layout, seed=seed, window=win)
    out.append((yuv, yuv))
  return out


def _ingest_check(sources, oh, ow):
  out = torch.full((len(sources), oh, ow, 3), float('nan'), device='cuda')
  _lib.ingest_frames_multi([s for s, _ in sources], out)
  for i, (_, alone) in enumerate(sources):
    want = torch.empty(*alone.shape[:-3], oh, ow, 3, device='cuda')
    _lib.resample_frames(alone, want)
    assert torch.equal(_bits(out[i]), _bits(want.view(oh, ow, 3))), f'frame {i} at {oh}x{ow}'
  return out


@pytest.mark.parametrize('oh,ow', [(256, 256), (480, 480), (96, 136)])
def test_ingest_multi_equals_per_frame_resample(oh, ow):
  sources = _ingest_sources()
  a = _ingest_check(sources, oh, ow)
  b = _ingest_check(sources, oh, ow)  # repeatable
  assert torch.equal(_bits(a), _bits(b))
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    c = _ingest_check(sources, oh, ow)
  torch.cuda.current_stream().wait_stream(side)
  torch.cuda.synchronize()
  assert torch.equal(_bits(a), _bits(c))


def test_ingest_multi_more_frames_than_one_launch():
  sources = _ingest_sources()
  many = [sources[i % len(sources)] for i in range(_lib.INGEST_MAX_FRAMES + 7)]
  torch.cuda.synchronize()
  l0 = U.launch_count()
  out = _ingest_check(many, 64, 72)
  assert U.launch_count() - l0 >= 2
  assert torch.equal(_bits(out[:len(sources)]), _bits(out[len(sources):2 * len(sources)]))


def test_ingest_multi_one_launch():
  sources = _ingest_sources()
  out = torch.empty(len(sources), 256, 256, 3, device='cuda')
  torch.cuda.synchronize()
  l0 = U.launch_count()
  _lib.ingest_frames_multi([s for s, _ in sources], out)
  assert U.launch_count() - l0 == 1


# ------------------------------------------------------------------------- per-clip video sizes
def test_estimate_trajectories_per_clip_video_sizes():
  model, _, _ = get_model()
  B, T, N = 3, 4, 21
  sizes = [(256, 256), (240, 320), (480, 640)]
  v = torch.cat([synth.make_video(T, seed=1 + 4 * b) for b in range(B)]).cuda()
  q = torch.cat([synth.make_queries(N, T, *sizes[b], seed=2 + 4 * b) for b in range(B)]).cuda()
  fg = model.get_feature_grids(v, False)
  qf = model.get_query_features(v, False, q, fg)
  both = model.estimate_trajectories(sizes, False, fg, qf, q)
  for b in range(B):
    fg1 = type(fg)(tuple(x[b:b + 1] for x in fg.lowres), tuple(x[b:b + 1] for x in fg.hires),
                   fg.resolutions)
    qf1 = type(qf)(tuple(x[b:b + 1] for x in qf.lowres), tuple(x[b:b + 1] for x in qf.hires),
                   qf.resolutions)
    one = model.estimate_trajectories(sizes[b], False, fg1, qf1, q[b:b + 1])
    for key in ('tracks', 'occlusion', 'expected_dist'):
      for i, (x, y) in enumerate(zip(both[key], one[key])):
        assert torch.equal(x[b], y[0]), f'clip {b}: {key}[{i}]'
  U.record('per_clip_video_sizes', clips=B, frames=T, equal=1)


def test_refine_update_video_table_equals_per_clip_calls():
  G, n, T = 3, 5, 2
  Q = G * n
  g = torch.Generator().manual_seed(3)
  res = torch.randn(Q, T, 400, generator=g).cuda()
  pos0 = (torch.rand(Q, T, 2, generator=g) * 256).cuda()
  occ, expd = torch.randn(Q, T, generator=g).cuda(), torch.randn(Q, T, generator=g).cuda()
  fhi, flo = torch.randn(Q, T, 128, generator=g).cuda(), torch.randn(Q, T, 256, generator=g).cuda()
  sizes = [(480, 640), (200, 200), (240, 320)]
  table = torch.tensor(sizes, dtype=torch.int32, device='cuda')

  def run(sl, video_hw, video_table=None):
    m = sl.stop - sl.start
    pos = pos0[sl].clone()
    outs = [torch.empty(m, T, device='cuda') for _ in range(2)] + [
        torch.empty(m, T, 384, device='cuda'), torch.empty(m, T, 2, device='cuda')]
    _lib.refine_update(res[sl], pos, occ[sl], expd[sl], fhi[sl], flo[sl], *outs, (256, 256),
                       (480, 480), video_hw, video_table=video_table)
    return [pos] + outs

  got = run(slice(0, Q), (0, 0), table)
  for c in range(G):
    want = run(slice(c * n, (c + 1) * n), sizes[c])
    for x, y in zip(got, want):
      assert torch.equal(x[c * n:(c + 1) * n], y), f'clip {c}'


# ------------------------------------------------------------------------- mixed-size tracker
SIZES = [(256, 256), (240, 320), (200, 200), (240, 240), (480, 480)]
GOLDEN_SLOT = 4


def _mixed_inputs(N, T, golden=None):
  frames, queries = [], []
  for s, (H, W) in enumerate(SIZES):
    if golden is not None and s == GOLDEN_SLOT:
      meta = golden['meta']
      frames.append(synth.make_video(T, H, W, seed=meta['video_seed'])[0].cuda())
      queries.append(synth.make_queries(N, T, H, W, seed=meta['query_seed'], frame0_only=True)[0])
    else:
      frames.append(synth.make_video(T, H, W, seed=40 + 3 * s)[0].cuda())
      queries.append(synth.make_queries(N, T, H, W, seed=41 + 3 * s, frame0_only=True)[0])
  return frames, torch.stack(queries).cuda()


def _vis_prob(occ, expd):
  return (1 - torch.sigmoid(occ)) * (1 - torch.sigmoid(expd))


def test_mixed_size_packed_tracker_against_single_streams_golden_and_eager():
  g = load_golden('causal_480x3_n8')
  meta = g['meta']
  assert (meta['H'], meta['W']) == SIZES[GOLDEN_SLOT]
  model, _, _ = get_model(causal=True)
  N, T, S = meta['N'], meta['T'], len(SIZES)
  frames, q = _mixed_inputs(N, T, g)
  trk = streaming.OnlineTracker(model, [h for h, _ in SIZES], [w for _, w in SIZES], N, num_streams=S)
  assert [grp.streams for grp in trk._groups] == [[0], [1], [2, 3], [4]]
  trk.init([f[0] for f in frames], q)
  singles = [streaming.OnlineTracker(model, H, W, N) for H, W in SIZES]
  for s in range(S):
    singles[s].init(frames[s][0], q[s])
  retarget = (1, torch.tensor([0.0, 100.5, 37.25]), 3)  # stream, (t, y, x), point
  e_t = e_l = 0.0
  vis_mismatch = 0
  gold = [[], [], []]
  for t in range(T):
    if t == 1:
      s, qp, idx = retarget
      trk.update_query(frames[s][1], qp, idx, stream=s)
      singles[s].update_query(frames[s][1], qp, idx)
    saved = [[{k: v.clone() for k, v in d.items()} for d in grp.state] for grp in trk._groups]
    tracks, vis = trk.step([f[t] for f in frames])
    occ, expd = trk.last_logits
    assert tuple(tracks.shape) == (S, N, 1, 2) and tuple(vis.shape) == (S, N, 1)
    # graph replay == the eager grouped calls on the same inputs, bit for bit
    for grp, st in zip(trk._groups, saved):
      et, eo, ee = trk._step_group(grp, st)
      for i, s in enumerate(grp.streams):
        r = slice(grp.offsets[i], grp.offsets[i] + N)
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
  for s in singles:
    s.close()
  trk.close()
  g_t = np.abs(np.concatenate(gold[0], 1) - g['online_tracks']).max()
  g_o = np.abs(np.concatenate(gold[1], 1) - g['online_occlusion']).max()
  g_e = np.abs(np.concatenate(gold[2], 1) - g['online_expected_dist']).max()
  U.record('tracker_mixed_sizes', streams=S, points=N, frames=T, tracks_vs_single=e_t,
           logits_vs_single=e_l, vis_mismatch=vis_mismatch, golden_tracks=g_t, golden_occ=g_o,
           golden_expd=g_e)
  assert e_t <= TRACK_TOL and e_l <= LOGIT_TOL and vis_mismatch == 0
  assert g_t < TRACK_TOL and g_o < LOGIT_TOL and g_e < LOGIT_TOL


def test_mixed_size_packed_streams_are_isolated():
  """Changing stream 2's frames (200^2, grouped with 240^2) and re-targeting one of its points
  leaves every other stream's outputs and causal state bit for bit unchanged."""
  model, _, _ = get_model(causal=True)
  N, T, S = 16, 3, len(SIZES)
  frames, q = _mixed_inputs(N, T)
  other = synth.make_video(T, 200, 200, seed=77)[0].cuda()

  def run(disturb):
    trk = streaming.OnlineTracker(model, [h for h, _ in SIZES], [w for _, w in SIZES], N,
                                  num_streams=S)
    fr = [other if disturb and s == 2 else f for s, f in enumerate(frames)]
    trk.init([f[0] for f in fr], q)
    outs = []
    for t in range(T):
      if disturb and t == 1:
        trk.update_query(fr[2][1], torch.tensor([0.0, 40.5, 150.25]), 9, stream=2)
      trk.step([f[t] for f in fr])
      outs.append([x.clone() for x in (*trk._out[:2], *trk.last_logits)])
    state = {}
    for s in range(S):
      gi, slot = trk._slot[s]
      grp = trk._groups[gi]
      r = slice(grp.offsets[slot], grp.offsets[slot] + N)
      state[s] = [{k: v[:, r].clone() for k, v in d.items()} for d in grp.state]
    trk.close()
    return outs, state

  (a, sa), (b, sb) = run(False), run(True)
  keep = [s for s in range(S) if s != 2]
  for t in range(T):
    for x, y in zip(a[t], b[t]):
      assert torch.equal(x[keep], y[keep]), f'frame {t}'
  assert not torch.equal(a[-1][0][2], b[-1][0][2])
  for s in keep:
    for da, db in zip(sa[s], sb[s]):
      for k in da:
        assert torch.equal(da[k], db[k]), f'stream {s}: {k}'
  U.record('tracker_mixed_sizes_isolation', equal=1)


def _ingest_launches(trk):
  """Launches of the multi-frame ingest in one eager step, by the library's profiler."""
  lib = _lib.load()
  trk._step_eager()  # warm-up
  torch.cuda.synchronize()
  lib.tapir_profile_enable(1)
  trk._step_eager()
  buf = ctypes.create_string_buffer(1 << 16)
  _lib.check(lib.tapir_profile_report(buf, len(buf)), 'tapir_profile_report')
  lib.tapir_profile_enable(0)
  rep = json.loads(buf.value.decode())
  return rep.get('ingest_frames_multi', {}).get('launches', 0)


@pytest.mark.parametrize('fmt', ['uint8', 'nv12'])
def test_one_ingest_launch_per_resampled_pass(fmt):
  """200^2, 240^2 and 250x200 share one resampled 256^2 pass: one ingest launch for it (uint8
  and YUV frames; float frames keep one tapir_bilinear_resize launch each)."""
  model, _, _ = get_model(causal=True)
  sizes = [(200, 200), (240, 240), (250, 200)]
  N = 8
  q = torch.stack([synth.make_queries(N, 1, h, w, seed=s, frame0_only=True)[0]
                   for s, (h, w) in enumerate(sizes)]).cuda()
  if fmt == 'nv12':
    frames = [make_frames(1, 1, h, w, 'nv12', seed=s)[0] for s, (h, w) in enumerate(sizes)]
  else:
    frames = [synth.make_video(1, h, w, seed=s)[0, 0].cuda() for s, (h, w) in enumerate(sizes)]
    if fmt == 'uint8':
      frames = [((f + 1) * 127.5).round().to(torch.uint8) for f in frames]
  trk = streaming.OnlineTracker(model, [h for h, _ in sizes], [w for _, w in sizes], N,
                                uint8_frames=fmt == 'uint8', yuv420=fmt == 'nv12',
                                num_streams=len(sizes))
  assert len(trk._groups) == 1 and not trk._groups[0].uniform
  trk.init(frames, q)
  for s, dst in zip(trk._groups[0].streams, trk._groups[0].sources):
    trk._copy_in(trk._stream_frames([frames[s]], [s])[0], dst)
  n = _ingest_launches(trk)
  trk.close()
  U.record(f'tracker_mixed_ingest_launches_{fmt}', launches=n)
  assert n == 1


def test_yuv_mixed_tracker_equals_uint8_on_converted_frames():
  """Cropped NV12 / I420 streams of different frame sizes track, bit for bit, as a uint8 tracker
  does on the RGB windows the conversion produces."""
  model, _, _ = get_model(causal=True)
  N, T = 8, 2
  geo = [((480, 640), (0, 80, 480, 480), 'nv12'), ((240, 320), (0, 40, 240, 240), 'i420'),
         ((200, 200), None, 'nv12')]
  yuv = [[make_frames(1, 1, *hw, lay, seed=10 * s + t, window=win)[0] for t in range(T)]
         for s, (hw, win, lay) in enumerate(geo)]
  rgb = [[live.yuv420_to_rgb(f)[0, 0] for f in fs] for fs in yuv]
  hws = [f[0].shape[:2] for f in rgb]
  q = torch.stack([synth.make_queries(N, T, *hw, seed=s, frame0_only=True)[0]
                   for s, hw in enumerate(hws)]).cuda()
  ty = streaming.OnlineTracker(model, [hw[0] for hw, _, _ in geo], [hw[1] for hw, _, _ in geo], N,
                               num_streams=3, yuv420=True, window=[w for _, w, _ in geo])
  tu = streaming.OnlineTracker(model, [h for h, _ in hws], [w for _, w in hws], N, num_streams=3,
                               uint8_frames=True)
  assert [g.streams for g in ty._groups] == [g.streams for g in tu._groups] == [[0], [1, 2]]
  ty.init([fs[0] for fs in yuv], q)
  tu.init([fs[0] for fs in rgb], q)
  for t in range(T):
    a = [x.clone() for x in (*ty.step([fs[t] for fs in yuv]), *ty.last_logits)]
    b = [x.clone() for x in (*tu.step([fs[t] for fs in rgb]), *tu.last_logits)]
    for x, y in zip(a, b):
      assert torch.equal(x, y), f'frame {t}'
  with pytest.raises(ValueError, match='yuv420=True'):
    ty.step([fs[0] for fs in rgb])
  ty.close()
  tu.close()
