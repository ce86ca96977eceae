"""Camera homographies without a GPU: the numpy oracle against the reference's outputs in
tests/golden/io_homography.npz, the RANSAC stop table and the generator's draws, the C layout of
tapir_homography_args, and argument errors before any CUDA call."""
import ast
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import homography_oracle as H
from tapnet_b200 import _lib, viz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'io_homography.npz')


def fixture_cases():
  g = np.load(GOLDEN)
  dims = tuple(int(v) for v in g['image_dimensions'])
  for name in (str(c) for c in g['cases']):
    kw = dict(ast.literal_eval(bytes(g[f'{name}_kwargs']).decode()))
    yield name, {k: g[f'{name}_{k}'] for k in ('pts', 'occ', 'homogs', 'err', 'canonical',
                                                  'canonical_invalid', 'ransac_stats')}, dims, kw


CASES = [c[0] for c in fixture_cases()]


def run_oracle(c, dims, kw):
  with np.errstate(divide='ignore', invalid='ignore'):
    return H.homographies_wrt_frame(c['pts'], c['occ'], dims, **kw)


@pytest.mark.parametrize('name', CASES)
def test_oracle_equals_fixture(name):
  _, c, dims, kw = next(x for x in fixture_cases() if x[0] == name)
  o = run_oracle(c, dims, kw)
  thresh = kw.get('thresh', 0.07)
  np.testing.assert_array_equal(o['ransac_stats'], c['ransac_stats'])
  np.testing.assert_array_equal(o['err'] < thresh * thresh, c['err'] < thresh * thresh)
  np.testing.assert_array_equal(o['canonical_invalid'], c['canonical_invalid'])
  for k in ('homogs', 'err', 'canonical'):
    np.testing.assert_allclose(o[k], c[k], rtol=0, atol=1e-12, err_msg=k)
  # every system the case solves has a unique null vector, so another solver must find it too
  assert o['min_gap'] > 1e-6


def test_fixture_covers_the_cases():
  cases = {name: (c, kw) for name, c, _, kw in fixture_cases()}
  T = cases['pan'][0]['pts'].shape[1]
  assert {cases['pan_ref0'][1]['reference_frame'], cases['pan_ref_last'][1]['reference_frame']} == {0, T - 1}
  assert 'reference_frame' not in cases['pan'][1]
  assert {cases[n][1].get('num_refinement_passes', 2) for n in cases} >= {0, 1, 2, 3}
  assert cases['t1'][0]['pts'].shape[1] == 1 and cases['n5'][0]['pts'].shape[0] == 5
  assert cases['pan'][0]['pts'].dtype == np.float32 and cases['pan_f64'][0]['pts'].dtype == np.float64
  assert cases['pan_frac0.3'][1]['targ_inlier_frac'] == 0.3
  few = cases['few_visible'][0]
  assert (~few['occ']).sum(0).min() <= 4 and (few['ransac_stats'][:, 0] == 0).sum() >= 3
  # a panning clip: RANSAC stops within a few hypotheses at a high inlier count
  stats = cases['pan'][0]['ransac_stats']
  assert stats[:, 0].max() <= 8 and stats[stats[:, 0] > 0, 1].min() > 40
  # unrelated points, tiny threshold: the first frame of the sweep runs N - 5 hypotheses of 4
  # inliers each (after it, almost every canonical point is invalid)
  rnd = cases['random_tiny_thresh'][0]
  N, T = rnd['pts'].shape[:2]
  assert rnd['ransac_stats'][T // 2 + 1].tolist() == [N - 5, 4]


def test_stop_thresholds_equal_numpy():
  """The C table equals numpy's scalar expression bit for bit.  numpy's array power may take a
  SIMD path that differs by an ulp, but never on the side of an integer: the stop rule compares
  an integer count, so only ceil(thr) matters."""
  for frac in (0.7, 0.3, 0.5, 0.95, 1.0):
    for N in range(1, 4097):
      c = _lib.ransac_stop_thresholds(N, frac)
      if N in (1, 2, 5, 64, 1000, 4096) or N % 97 == 0:
        scalar = np.array([min(1 - (it + 1) / N, frac * 0.99 ** np.float64(it)) * N for it in range(N)])
        np.testing.assert_array_equal(c.view(np.int64), scalar.view(np.int64))
      np.testing.assert_array_equal(np.ceil(c), np.ceil(H.stop_thresholds(N, frac)))
      assert c[-1] == 0.0


def test_hypothesis_draws_are_distinct_usable_indices():
  for m in (4, 5, 6, 17, 1000, 4096):
    r = H.hypothesis_ranks(np.arange(5000), m)
    assert r.min() >= 0 and r.max() < m
    assert all(len(set(row)) == 4 for row in r.tolist())
  # ranks map to usable points in index order
  vis = np.zeros(50, bool)
  vis[[3, 8, 9, 20, 31, 44]] = True
  usable = np.flatnonzero(vis)
  idx = usable[H.hypothesis_ranks(np.arange(200), len(usable))]
  assert np.all(vis[idx])
  u = H.canonical_u(7, 10000)
  assert u.min() >= 0 and u.max() < 1 and abs(u.mean() - 0.5) < 0.02


def test_generator_constants():
  assert int(H.mix(0)) == 0xE220A8397B1DCDAF   # SplitMix64's first output from seed 0
  assert H.hypothesis_ranks(0, 5).tolist() == H.hypothesis_ranks([0], 5).tolist()


def test_homography_args_layout_matches_the_compiler(tmp_path):
  gcc = shutil.which('gcc')
  if gcc is None:
    pytest.skip('no gcc')
  cls = _lib.HomographyArgs
  lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "tapir_b200.h"', 'int main(void) {',
           '  printf("%zu", sizeof(tapir_homography_args));']
  lines += [f'  printf(" %zu", offsetof(tapir_homography_args, {f}));' for f, _ in cls._fields_]
  lines += ['  printf("\\n");', '  return 0;', '}']
  src = tmp_path / 'probe.c'
  src.write_text('\n'.join(lines))
  exe = tmp_path / 'probe'
  subprocess.run([gcc, '-std=c99', '-Wall', '-Werror', '-pedantic', '-I', os.path.join(ROOT, 'include'),
                  str(src), '-o', str(exe)], check=True)
  size, *offsets = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True,
                                                   text=True).stdout.split()]
  assert size == ctypes.sizeof(cls)
  assert offsets == [getattr(cls, f).offset for f, _ in cls._fields_]


def test_c_abi_rejects_bad_arguments():
  """rc 1 and a message naming the call, before any CUDA call (the pointers are never
  dereferenced)."""
  lib = _lib.load()
  p = 0x10000
  N, T = 64, 8
  ws = lib.tapir_homographies_workspace_bytes(T, N)
  assert ws > 0 and lib.tapir_homographies_workspace_bytes(0, N) == 0

  def args(**kw):
    a = dict(tracks=p, tracks_fp64=0, N=N, T=T, reference_frame=4, occluded=p, width=256.0, height=192.0,
             thresh=0.07, outlier_point_threshold=0.95, num_refinement_passes=2, reserved=0,
             stop_thresholds=p, homogs=p, err=p, canonical=p, ransac_stats=None, workspace=p,
             workspace_bytes=ws)
    a.update(kw)
    return _lib.HomographyArgs(**a)

  bad = [dict(N=0), dict(T=0), dict(N=1 << 20, T=1 << 11), dict(tracks_fp64=2), dict(reference_frame=-1),
         dict(reference_frame=T), dict(width=0.0), dict(height=-1.0), dict(width=float('inf')),
         dict(thresh=0.0), dict(thresh=float('nan')), dict(outlier_point_threshold=-0.5),
         dict(num_refinement_passes=-1), dict(tracks=None), dict(occluded=None),
         dict(stop_thresholds=None), dict(homogs=None), dict(err=None), dict(canonical=None),
         dict(workspace=None), dict(workspace_bytes=ws - 1), dict(tracks=p + 2), dict(homogs=p + 4),
         dict(tracks_fp64=1, tracks=p + 4), dict(ransac_stats=p + 2), dict(workspace=p + 16)]
  for kw in bad:
    a = args(**kw)
    assert lib.tapir_homographies_wrt_frame(ctypes.byref(a), None) == 1, kw
    assert b'tapir_homographies_wrt_frame' in lib.tapir_last_error(), kw
  assert lib.tapir_homographies_wrt_frame(None, None) == 1
  out = np.empty(4)
  assert lib.tapir_ransac_stop_thresholds(0, 0.7, out.ctypes.data) == 1
  assert lib.tapir_ransac_stop_thresholds(4, 0.0, out.ctypes.data) == 1
  assert lib.tapir_ransac_stop_thresholds(4, 0.7, None) == 1
  assert b'tapir_ransac_stop_thresholds' in lib.tapir_last_error()


def test_python_rejects_bad_arguments_before_cuda():
  rng = np.random.default_rng(0)
  pts = rng.uniform(0, 100, (20, 6, 2)).astype(np.float32)
  occ = np.zeros((20, 6), bool)
  f = viz.get_homographies_wrt_frame
  for call in (lambda: f(pts[..., :1], occ, (100, 100)),
               lambda: f(pts[0], occ, (100, 100)),
               lambda: f(pts, occ[:, :5], (100, 100)),
               lambda: f(pts, np.full((20, 6), 0.5, np.float32), (100, 100)),
               lambda: f(pts, occ, (100, 0)),
               lambda: f(pts, occ, (100,)),
               lambda: f(pts, occ, (100, 100), reference_frame=6),
               lambda: f(pts, occ, (100, 100), reference_frame=-1),
               lambda: f(pts, occ, (100, 100), thresh=0),
               lambda: f(pts, occ, (100, 100), outlier_point_threshold=-1),
               lambda: f(pts, occ, (100, 100), targ_inlier_frac=0),
               lambda: f(pts, occ, (100, 100), num_refinement_passes=-1),
               lambda: f(np.zeros((0, 6, 2)), np.zeros((0, 6)), (100, 100))):
    with pytest.raises(ValueError):
      call()


def test_foreground_tracks_numpy():
  err = np.array([[0.0, 0.0, 1.0, 1.0], [1.0, 1.0, 1.0, 0.0], [0.0, 0.0, 0.0, 0.0]])
  vis = np.array([[1, 1, 1, 1], [1, 1, 1, 1], [0, 0, 0, 0]], bool)
  # inlier fractions 0.5, 0.25 and 0 (no visible frame)
  np.testing.assert_array_equal(viz.foreground_tracks(err, vis), [True, True, True])
  np.testing.assert_array_equal(viz.foreground_tracks(err, vis, foreground_frac=0.4), [False, True, True])
  np.testing.assert_array_equal(viz.foreground_tracks(err, vis), H.foreground_tracks(err, vis))
