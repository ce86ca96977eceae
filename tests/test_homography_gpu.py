"""-m gpu: viz.get_homographies_wrt_frame (tapir_homographies_wrt_frame) against the
reference-generated fixture and the numpy oracle.  RANSAC statistics are compared exactly;
homographies (each scaled to unit Frobenius norm with a positive largest entry) to 1e-8; err and
canonical points to 1e-8 within the image's scale and 1e-6 relative beyond it."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import homography_oracle as H  # noqa: E402
from oracle import synth  # noqa: E402
from oracle.make_golden_homography import panning_clip  # noqa: E402
from tapnet_b200 import _lib, viz  # noqa: E402
from tests.test_homography_host import CASES, fixture_cases  # noqa: E402
from tests.test_stages_gpu import get_model  # noqa: E402

TOL = 1e-8


def unit(h):
  h = np.asarray(h, np.float64)
  h = h / np.linalg.norm(h, axis=(-2, -1), keepdims=True)
  flat = h.reshape(len(h), -1)
  sign = np.sign(flat[np.arange(len(h)), np.abs(flat).argmax(1)])
  return h * sign[:, None, None]


def check(got, want, thresh=0.07):
  if 'min_gap' in want:
    # the data must determine every estimate: each system's smallest singular value is separated
    # from the next, so any accurate solver finds the same null vector
    assert want['min_gap'] > 1e-6, want['min_gap']
  homogs, err, canonical, stats = (np.asarray(g.cpu() if isinstance(g, torch.Tensor) else g) for g in got)
  np.testing.assert_array_equal(stats, want['ransac_stats'])
  np.testing.assert_array_equal(err < thresh * thresh, want['err'] < thresh * thresh)
  np.testing.assert_allclose(unit(homogs), unit(want['homogs']), rtol=0, atol=TOL)
  # err and canonical points to 1e-8 within the image's scale (|value| <= 1 in normalised units;
  # every threshold lies far below); beyond it, relative to 1e-6: a point mapped near a
  # homography's line at infinity divides by a small w, which magnifies the last-bit differences
  # of the two sides' homographies by 1 / |w|
  for name, g, w in (('err', err, want['err']), ('canonical', canonical, want['canonical'])):
    near = np.abs(w) <= 1.0
    np.testing.assert_allclose(g[near], w[near], rtol=0, atol=TOL, err_msg=name)
    np.testing.assert_allclose(g[~near], w[~near], rtol=1e-6, atol=0, err_msg=name)


def run(pts, occ, dims, **kw):
  return viz.get_homographies_wrt_frame(pts, occ, dims, return_ransac_stats=True, **kw)


def oracle(pts, occ, dims, **kw):
  with np.errstate(divide='ignore', invalid='ignore'):
    return H.homographies_wrt_frame(pts, occ, dims, **kw)


@pytest.mark.parametrize('name', CASES)
def test_fixture_numpy_and_cuda(name):
  _, c, dims, kw = next(x for x in fixture_cases() if x[0] == name)
  out = run(c['pts'], c['occ'], dims, **kw)
  assert all(isinstance(o, np.ndarray) for o in out) and out[0].dtype == np.float64
  check(out, c, kw.get('thresh', 0.07))
  dev = run(torch.from_numpy(c['pts']).cuda(), torch.from_numpy(c['occ']).cuda(), dims, **kw)
  assert all(o.is_cuda for o in dev)
  check(dev, c, kw.get('thresh', 0.07))


@pytest.mark.parametrize('T,N', [(50, 1024), (200, 4096)])
def test_oracle_at_demo_sizes(T, N):
  rng = np.random.default_rng(T + N)
  pts, occ = panning_clip(rng, T, N, W=256, H_=256)
  want = oracle(pts, occ, (256, 256))
  got = run(torch.from_numpy(pts).cuda(), torch.from_numpy(occ).cuda(), (256, 256))
  check(got, want)
  assert want['ransac_stats'][:, 0].max() >= 1


@pytest.mark.parametrize('ref', [0, 5, 11, None])
@pytest.mark.parametrize('passes', [0, 1, 2, 3])
def test_oracle_reference_frames_and_passes(ref, passes):
  rng = np.random.default_rng(7)
  pts, occ = panning_clip(rng, 12, 300)
  kw = dict(reference_frame=ref, num_refinement_passes=passes)
  check(run(pts, occ, (256, 192), **kw), oracle(pts, occ, (256, 192), **kw))


def test_bool_and_float_occ():
  rng = np.random.default_rng(8)
  pts, occ = panning_clip(rng, 16, 500, dtype=np.float64)
  want = oracle(pts, occ, (256, 192))
  check(run(pts, occ, (256, 192)), want)
  check(run(pts, occ.astype(np.float32), (256, 192)), want)
  dev = run(torch.from_numpy(pts).cuda(), torch.from_numpy(occ.astype(np.float32)).cuda(), (256, 192))
  check(dev, want)


def test_exact_camera_motion_and_foreground():
  """A noise-free planar background under known homographies: the frame-to-reference maps come
  back to 1e-9, and foreground_tracks flags exactly the independent movers."""
  rng = np.random.default_rng(9)
  T, N, W, Hh, ref = 10, 400, 320, 240, 5
  base = np.stack([rng.uniform(0, W, N), rng.uniform(0, Hh, N)], -1)
  true = []
  for t in range(T):
    a = 0.01 * (t - ref)
    true.append(np.array([[np.cos(a), -np.sin(a), 3.0 * (t - ref)], [np.sin(a), np.cos(a), -2.0 * (t - ref)],
                          [1e-5 * (t - ref), 0.0, 1.0]]))
  pts = np.empty((N, T, 2))
  for t in range(T):
    p = np.concatenate([base, np.ones((N, 1))], -1) @ true[t].T
    pts[:, t] = p[:, :2] / p[:, 2:]
  fg = np.zeros(N, bool)
  fg[::10] = True
  # the movers drift 150 px per frame away from the background's motion, so that their squared
  # err (normalised) exceeds even the unsquared 2 thresh the canonical update compares it with
  drift = (np.arange(T) - ref)[None, :, None] * np.array([150.0, -110.0])
  pts[fg] += drift + rng.normal(0, 2.0, (fg.sum(), T, 2))
  occ = np.zeros((N, T), bool)
  homogs, err, _ = viz.get_homographies_wrt_frame(pts, occ, (W, Hh), reference_frame=ref)
  for t in range(T):
    # inv(homogs[ref]) @ homogs[t] maps frame t's background pixels to the reference frame's (the
    # canonical frame itself may drift by a transform common to all frames)
    want = np.linalg.inv(true[t])
    got = np.linalg.solve(homogs[ref], homogs[t])
    got = got / got[2, 2] * want[2, 2]
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-9 * np.abs(want).max())
  np.testing.assert_array_equal(viz.foreground_tracks(err, ~occ), fg)
  fg_dev = viz.foreground_tracks(torch.from_numpy(err).cuda(), torch.from_numpy(~occ).cuda())
  np.testing.assert_array_equal(fg_dev.cpu().numpy(), fg)


def test_model_tracks_on_device_without_sync():
  """The model's tracks[0] / visibles on the device go straight in, with no host sync, and give
  the bits the numpy path gives on the same tracks copied to the host.  (The seeded random weights
  do not track a camera motion: their systems are undetermined, smallest singular gap ~1e-20, so
  the oracle comparisons run on the panning clips above, through CUDA tensors too.)"""
  model, _, _ = get_model()
  T, N = 8, 64
  video = synth.make_video(T)
  q = synth.make_queries(N, T)
  out = model(video.cuda(), q.cuda())
  tracks = out['tracks'][0]
  occ = out['occlusion'][0]
  visibles = occ < occ.median()
  torch.cuda.synchronize()
  torch.cuda.set_sync_debug_mode('error')
  try:
    got = viz.get_homographies_wrt_frame(tracks, ~visibles, (256, 256), return_ransac_stats=True)
    fg = viz.foreground_tracks(got[1], visibles)
  finally:
    torch.cuda.set_sync_debug_mode(0)
  assert all(t.is_cuda for t in got) and fg.is_cuda
  host = viz.get_homographies_wrt_frame(tracks.cpu().numpy(), (~visibles).cpu().numpy(), (256, 256),
                                        return_ransac_stats=True)
  for d, h in zip(got, host):
    np.testing.assert_array_equal(d.cpu().numpy(), h)
  np.testing.assert_array_equal(fg.cpu().numpy(), H.foreground_tracks(host[1], visibles.cpu().numpy()))


def test_repeatable_and_side_stream():
  rng = np.random.default_rng(10)
  pts, occ = panning_clip(rng, 30, 800)
  p, o = torch.from_numpy(pts).cuda(), torch.from_numpy(occ).cuda()
  a = run(p, o, (256, 192))
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    b = run(p, o, (256, 192))
  torch.cuda.current_stream().wait_stream(side)
  for x, y in zip(a, b):
    assert torch.equal(x, y)


def test_random_points_run_until_the_count_term_stops():
  rng = np.random.default_rng(11)
  pts = rng.uniform(0, 256, (300, 3, 2)).astype(np.float32)
  occ = np.zeros((300, 3), bool)
  kw = dict(thresh=1e-5, num_refinement_passes=1)
  got = run(pts, occ, (256, 256), **kw)
  want = oracle(pts, occ, (256, 256), **kw)
  assert want['ransac_stats'][2].tolist() == [295, 4]
  check(got, want, 1e-5)


@pytest.mark.parametrize('kind', ['all_occluded_frames', 'n_below_5', 'never_visible'])
def test_edge_inputs_do_not_fault(kind):
  rng = np.random.default_rng(12)
  pts, occ = panning_clip(rng, 9, 60)
  if kind == 'all_occluded_frames':
    occ[:, [0, 3, 8]] = True   # not the reference frame (4)
  elif kind == 'n_below_5':
    pts, occ = pts[:3], occ[:3]
  else:
    occ[7] = True
    occ[20] = True
  got = run(pts, occ, (256, 192))
  torch.cuda.synchronize()
  if kind == 'n_below_5':
    # every estimate is undetermined (fewer than 4 points): no RANSAC, finite shapes, no fault
    assert np.all(got[3] == 0) and got[0].shape == (9, 3, 3) and got[1].shape == (3, 9)
    return
  want = oracle(pts, occ, (256, 192))
  np.testing.assert_array_equal(got[3], want['ransac_stats'])
  if kind == 'all_occluded_frames':
    # refining an all-occluded frame gives the zero system's e9 on both sides and leaves every
    # canonical point invalid; the estimates after it are undetermined (want['min_gap'] ~ 0), so
    # the whole result is compared on the initial sweep
    assert want['min_gap'] < 1e-12
    pts, occ = pts.copy(), occ.copy()
    got = run(pts, occ, (256, 192), num_refinement_passes=0)
    want = oracle(pts, occ, (256, 192), num_refinement_passes=0)
  check(got, want)


def test_c_abi_errors_name_the_call():
  lib = _lib.load()
  a = _lib.HomographyArgs(N=4, T=2, reference_frame=5)
  assert lib.tapir_homographies_wrt_frame(ctypes.byref(a), None) == 1
  assert b'tapir_homographies_wrt_frame' in lib.tapir_last_error()
