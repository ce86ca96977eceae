"""TEST INFRASTRUCTURE - generates tests/golden/io_homography.npz by executing the reference's own
camera-homography functions (tapnet/utils/viz_utils.py:301-648) on the CPU.

Needs a checkout of the reference (oracle/reference_loader.py, TAPNET_REFERENCE_ROOT):
  python -m oracle.make_golden_homography

viz_utils.py imports jax, matplotlib and mediapy (absent here), so the six FunctionDefs are
compiled unmodified by make_golden_io.reference_functions into a scope where
  * `jnp` is numpy with jnp.float32 mapped to float64 (the whole computation runs in float64);
  * `jax.vmap`, `jax.lax.while_loop` and `jax.lax.cond` are plain Python;
  * `jax.random.choice(PRNGKey(k), N, [4], replace=False, p)` and `np.random.random([N])` draw
    from the generator of oracle/homography_oracle.py (hypothesis k; the c-th call);
  * `print` is silent, and every while_loop's final (it, inliers) is recorded per frame.
The fixture holds inputs and the reference's outputs only.
"""
import os
import types

import numpy as np

from oracle import homography_oracle as H
from oracle import reference_loader
from oracle.make_golden_io import GOLDEN_DIR, reference_functions

FUNCTIONS = ['estimate_homography', 'compute_inliers', 'ransac_homography',
             'maybe_ransac_homography', 'compute_canonical_points', 'get_homographies_wrt_frame']


class _Numpy64(types.ModuleType):
  """numpy, except float32 is float64."""

  def __init__(self):
    super().__init__('jnp')
    self.float32 = np.float64

  def __getattr__(self, name):
    return getattr(np, name)


class _NumpyDrawn(types.ModuleType):
  """numpy, except np.random.random([N]) returns the c-th call's canonical_u."""

  def __init__(self):
    super().__init__('np')
    self.calls = 0
    self.random = types.SimpleNamespace(random=self._random)

  def _random(self, shape):
    self.calls += 1
    (n,) = shape
    return H.canonical_u(self.calls, n)

  def __getattr__(self, name):
    return getattr(np, name)


def _choice(key, n, shape, replace=True, p=None):
  assert not replace and list(shape) == [4] and p is not None
  usable = np.flatnonzero(np.asarray(p) > 0)
  return usable[H.hypothesis_ranks(int(key), len(usable))[0]]


def reference_scope(loops):
  def while_loop(cond, body, state):
    while cond(state):
      state = body(state)
    loops.append((int(state[0]), int(state[1])))
    return state

  jax = types.SimpleNamespace(
      vmap=lambda f: lambda xs: np.stack([f(x) for x in xs]),
      random=types.SimpleNamespace(PRNGKey=lambda k: int(k), choice=_choice),
      lax=types.SimpleNamespace(while_loop=while_loop,
                                cond=lambda pred, a, b: a() if pred else b()))
  scope = dict(np=_NumpyDrawn(), jnp=_Numpy64(), jax=jax, print=lambda *a, **k: None)
  return dict(zip(FUNCTIONS, reference_functions('tapnet/utils/viz_utils.py', FUNCTIONS, scope))), scope


def panning_clip(rng, T, N, W=256, H_=192, fg_frac=0.2, occ_frac=0.1, noise=0.3, dtype=np.float32):
  """A planar background under a slow pan / zoom / tilt, independently moving foreground tracks,
  random occlusions and pixel noise.  Returns pts [N, T, 2], occ [N, T] bool."""
  base = np.stack([rng.uniform(0, W, N), rng.uniform(0, H_, N)], -1)
  pts = np.empty((N, T, 2))
  for t in range(T):
    a = 0.004 * t
    h = np.array([[np.cos(a) * (1 + 0.003 * t), -np.sin(a), 1.5 * t],
                  [np.sin(a), np.cos(a) * (1 + 0.002 * t), -0.8 * t],
                  [2e-5 * t, -1e-5 * t, 1.0]])
    p = np.concatenate([base, np.ones((N, 1))], -1) @ h.T
    pts[:, t] = p[:, :2] / p[:, 2:]
  fg = rng.uniform(size=N) < fg_frac
  walk = np.cumsum(rng.normal(0, 4.0, (N, T, 2)), 1)
  pts[fg] += walk[fg]
  pts += rng.normal(0, noise, pts.shape)
  occ = rng.uniform(size=(N, T)) < occ_frac
  return pts.astype(dtype), occ


def cases():
  rng = np.random.default_rng(23)
  out = []
  pts, occ = panning_clip(rng, 12, 64)
  out.append(('pan', pts, occ, {}))
  out.append(('pan_ref0', pts, occ, dict(reference_frame=0)))
  out.append(('pan_ref_last', pts, occ, dict(reference_frame=11)))
  out.append(('pan_passes0', pts, occ, dict(num_refinement_passes=0)))
  out.append(('pan_passes1', pts, occ, dict(num_refinement_passes=1)))
  out.append(('pan_frac0.3', pts, occ, dict(targ_inlier_frac=0.3)))
  p64, o64 = panning_clip(rng, 9, 48, dtype=np.float64)
  out.append(('pan_f64', p64, o64.astype(np.float32), dict(reference_frame=3, num_refinement_passes=3)))
  p1, o1 = panning_clip(rng, 1, 20)
  out.append(('t1', p1, o1, {}))
  p5, o5 = panning_clip(rng, 6, 5, occ_frac=0.0)
  out.append(('n5', p5, o5, dict(reference_frame=0)))
  # frames 2 and 5 keep 4 visible points each: no RANSAC there, the identity.  (A frame with none
  # at all turns every canonical point invalid in refinement, and the estimates after it are
  # undetermined: the GPU tests cover that input with the initial sweep alone.)
  pf, of = panning_clip(rng, 8, 40)
  of[:, 2] = True
  of[:4, 2] = False
  of[:, 5] = True
  of[10:14, 5] = False
  out.append(('few_visible', pf, of, {}))
  # unrelated random points, tiny threshold: every hypothesis has only its own 4 inliers.  One
  # refinement pass: the reference frame's branch would invert a rank-deficient estimate
  pr = rng.uniform(0, 256, (40, 3, 2)).astype(np.float32)
  out.append(('random_tiny_thresh', pr, np.zeros((40, 3), bool),
              dict(thresh=1e-5, num_refinement_passes=1)))
  return out


def main():
  out, names = {}, []
  for name, pts, occ, kw in cases():
    loops = []
    ref, scope = reference_scope(loops)
    dims = (256, 192)
    frames = []
    maybe = ref['maybe_ransac_homography']

    def recording(*arg, _maybe=maybe, **kwa):
      frames.append(len(loops))
      return _maybe(*arg, **kwa)

    scope['maybe_ransac_homography'] = recording
    canon_ref = ref['compute_canonical_points']
    last = {}

    def canon_recording(*arg, _c=canon_ref, **kwa):
      r = _c(*arg, **kwa)
      last['invalid'] = np.asarray(r[1])
      return r

    scope['compute_canonical_points'] = canon_recording
    with np.errstate(divide='ignore', invalid='ignore'):
      homogs, err, canonical = scope['get_homographies_wrt_frame'](pts, occ, dims, **kw)
    T = pts.shape[1]
    r = kw.get('reference_frame', T // 2)
    order = list(range(r + 1, T)) + list(range(r - 1, -1, -1))
    stats = np.zeros((T, 2), np.int32)
    for i, (fr, before) in enumerate(zip(order, frames)):
      after = frames[i + 1] if i + 1 < len(frames) else len(loops)
      assert after - before in (0, 1)
      if after > before:
        stats[fr] = loops[before]
    out.update({f'{name}_pts': pts, f'{name}_occ': occ, f'{name}_homogs': np.asarray(homogs),
                f'{name}_err': np.asarray(err), f'{name}_canonical': np.asarray(canonical),
                f'{name}_canonical_invalid': last.get('invalid', occ[:, r] != 0).astype(bool),
                f'{name}_ransac_stats': stats,
                f'{name}_kwargs': np.frombuffer(repr(sorted(kw.items())).encode(), np.uint8)})
    names.append(name)
    print(name, pts.shape, 'stats', stats[order].tolist() if len(order) < 12 else stats.sum(0))
  out['cases'] = np.array(names)
  out['image_dimensions'] = np.array([256, 192])
  np.savez_compressed(os.path.join(GOLDEN_DIR, 'io_homography.npz'), **out)
  print('io_homography.npz', names)


if __name__ == '__main__':
  reference_loader.load()
  main()
