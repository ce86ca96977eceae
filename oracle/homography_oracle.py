"""CPU oracle of the camera-homography tools (tapnet/utils/viz_utils.py:301-648,
`get_homographies_wrt_frame` and the five functions it calls), restated in numpy float64.

It is pinned to tests/golden/io_homography.npz (the reference's own functions run through numpy)
and stands in for the reference on sizes the fixture does not hold.  The semantics the CUDA path
(tapnet_b200/csrc/homography.cu) reproduces:

  * points are normalised by (width, height) in float64; a homography is the unit right singular
    vector of the smallest singular value of the 2N x 9 system [a1; a2] * mask, reshaped to 3 x 3;
  * a transform divides by max(1e-12, |w|) * sign(w) (NaN propagates), err = dx^2 + dy^2;
  * RANSAC: hypothesis k draws 4 distinct usable points (`hypothesis_ranks`), is scored by
    sum(err < thresh^2) over all N points, and replaces the kept one only if its count is strictly
    greater; the loop stops after hypothesis k once best >= thr[k + 1] (`stop_thresholds`);
  * canonical points compare the squared err with thresh and 2 thresh unsquared; an invalid point
    is re-initialised from the frame whose visible-count id equals floor(u * count) (`canonical_u`);
  * the frame order and the reference-frame branch of refinement pass j < last follow the
    reference line by line (see `homographies_wrt_frame`).

The generator (mix = SplitMix64's finaliser) replaces jax's PRNG and numpy's global state, which
cannot be reproduced without jax; it is a fixed function of the inputs.
"""
import numpy as np

_M64 = np.uint64
_GAMMA, _C1, _C2 = _M64(0x9E3779B97F4A7C15), _M64(0xBF58476D1CE4E5B9), _M64(0x94D049BB133111EB)


def mix(x):
  """SplitMix64's finaliser of x + gamma, elementwise mod 2^64 (uint64 in, uint64 out)."""
  with np.errstate(over='ignore'):
    z = np.asarray(x, np.uint64) + _GAMMA
    z = (z ^ (z >> _M64(30))) * _C1
    z = (z ^ (z >> _M64(27))) * _C2
    return z ^ (z >> _M64(31))


HYPOTHESIS_SEED = mix(0)
CANONICAL_SEED = mix(1)


def hypothesis_ranks(k, m):
  """[len(k), 4] distinct ranks in 0..m-1 (m >= 4) of hypotheses k, by Floyd's algorithm: for
  d = 0..3 and j = m - 4 + d, r = ((mix(mix(0) ^ (k << 2 | d)) >> 32) * (j + 1)) >> 32, or j if r
  is already taken.  The ranks index the frame's usable points in index order."""
  k = np.atleast_1d(np.asarray(k, np.uint64))
  out = np.empty((k.size, 4), np.int64)
  for d in range(4):
    j = m - 4 + d
    r = (((mix(HYPOTHESIS_SEED ^ ((k << _M64(2)) | _M64(d))) >> _M64(32)) * _M64(j + 1)) >> _M64(32))
    r = r.astype(np.int64)
    taken = np.zeros(k.size, bool)
    for e in range(d):
      taken |= out[:, e] == r
    out[:, d] = np.where(taken, j, r)
  return out


def canonical_u(call, N):
  """u [N] in [0, 1) of call `call` (1-based) of the canonical-point update:
  (mix(mix(1) ^ (call << 32 | n)) >> 11) * 2^-53."""
  n = np.arange(N, dtype=np.uint64)
  bits = mix(CANONICAL_SEED ^ ((_M64(call) << _M64(32)) | n)) >> _M64(11)
  return bits.astype(np.float64) * 2.0 ** -53


def stop_thresholds(N, targ_inlier_frac):
  """thr[it] = min(1 - (it + 1) / N, targ_inlier_frac * 0.99^it) * N, float64, it = 0..N-1."""
  it = np.arange(N)
  return np.minimum(1 - (it + 1) / N, targ_inlier_frac * 0.99 ** it.astype(np.float64)) * N


def solve_homography(targ, src, mask=None, gaps=None):
  """targ = H src for [n, 2] point sets, weighted by mask [n] (default ones): the right singular
  vector of the smallest singular value of the masked 2n x 9 system.  With a list `gaps`, appends
  (s8 - s9) / s1 of the system's singular values (the 9th is 0 below 9 rows): near 0 the null
  vector is undetermined and another solver may pick another one.  The all-zero system (its
  defined answer is e9) appends nothing."""
  m = np.ones(len(targ)) if mask is None else mask
  tx, ty, sx, sy = targ[:, 0], targ[:, 1], src[:, 0], src[:, 1]
  one, zero = np.ones_like(tx), np.zeros_like(tx)
  rows_x = np.stack([sx, sy, one, zero, zero, zero, -tx * sx, -tx * sy, -tx], -1) * m[:, None]
  rows_y = np.stack([zero, zero, zero, sx, sy, one, -ty * sx, -ty * sy, -ty], -1) * m[:, None]
  a = np.concatenate([rows_x, rows_y], 0)
  _, sv, vh = np.linalg.svd(a, full_matrices=a.shape[0] <= 8)
  if gaps is not None and sv[0] > 0:
    s9 = np.zeros(9)
    s9[:len(sv)] = sv
    gaps.append((s9[7] - s9[8]) / s9[0])
  return vh[-1].reshape(3, 3)


def transform(H, src, targ):
  """(tformed [n, 2], err [n]) of src under H against targ."""
  ph = np.concatenate([src, src[:, :1] * 0 + 1], -1).T
  t = (H @ ph).T
  w = t[:, 2:]
  tformed = t[:, :2] / (np.maximum(1e-12, np.abs(w)) * np.sign(w))
  return tformed, np.sum(np.square(targ - tformed), -1)


def ransac(targ, src, vis, thresh, thr, gaps=None):
  """(H, (hypotheses evaluated, best inlier count))."""
  N = len(targ)
  usable = np.flatnonzero(vis)
  t2 = thresh * thresh
  best, best_h, k = 0, np.zeros((3, 3)), 0
  while best < thr[k]:
    idx = usable[hypothesis_ranks(k, len(usable))[0]]
    h = solve_homography(targ[idx], src[idx], gaps=gaps)
    count = int(np.sum(transform(h, src, targ)[1] < t2))
    if count > best:
      best, best_h = count, h
    k += 1
  inliers = transform(best_h, src, targ)[1] < t2
  return solve_homography(targ, src, inliers.astype(np.float64), gaps), (k, best)


def canonical_points(tformed, invalid, err, thresh, outlier_point_threshold, call):
  """compute_canonical_points: (points [N, 2], invalid [N]) from every frame's transformed points
  tformed [T, N, 2], invalid [T, N] bool and err [N] (broadcast over frames) or [T, N]."""
  T, N = invalid.shape
  outlier = invalid | (err > thresh * 2.0)
  inlier = ~invalid & (err < thresh)
  visible = ~invalid
  frac = inlier.sum(0) / np.maximum(1.0, visible.sum(0))
  bad = frac < outlier_point_threshold
  keep = ~outlier
  pts = np.einsum('tnc,tn->nc', tformed, keep) / np.maximum(1.0, keep.sum(0)[:, None])
  # re-initialise: the frame whose 1-based visible count equals floor(u * count), else frame 0
  count = visible.sum(0)
  target = np.floor(canonical_u(call, N) * count)
  ids = np.where(visible, np.cumsum(visible, 0), -1)
  hit = ids == target[None, :]
  frame = np.where(hit.any(0), hit.argmax(0), 0)
  drawn = tformed[frame, np.arange(N)]
  pts = bad[:, None] * drawn + (1 - bad[:, None]) * pts
  return pts, bad


def homographies_wrt_frame(pts, occ, image_dimensions, reference_frame=None, thresh=0.07,
                           outlier_point_threshold=0.95, targ_inlier_frac=0.7,
                           num_refinement_passes=2):
  """get_homographies_wrt_frame: pts [N, T, 2], occ [N, T] (read as occ != 0).  Returns
  dict(homogs [T, 3, 3], err [N, T], canonical [N, 2], canonical_invalid [N],
  ransac_stats [T, 2] int32 (hypotheses evaluated, best inlier count; 0 / 0 for the reference
  frame and frames with <= 4 usable points), min_gap: the smallest (s8 - s9) / s1 of every
  system solved (1.0 when none was); near 0 some estimate was undetermined)."""
  pts = np.transpose(np.asarray(pts), (1, 0, 2)) / np.array(image_dimensions, np.float64)
  occ = np.transpose(np.asarray(occ) != 0)
  T, N = occ.shape
  ref = T // 2 if reference_frame is None else int(reference_frame)
  thr = stop_thresholds(N, targ_inlier_frac)
  calls = [0]

  def update(err):
    calls[0] += 1
    return canonical_points(tformed, invalid, err, thresh, outlier_point_threshold, calls[0])

  canon, canon_bad = pts[ref].copy(), occ[ref].copy()
  tformed = np.zeros_like(pts)
  invalid = np.ones_like(occ)
  all_err = np.zeros(occ.shape)
  tformed[ref], invalid[ref] = canon, canon_bad
  homogs = np.zeros((T, 3, 3))
  homogs[ref] = np.eye(3)
  stats = np.zeros((T, 2), np.int32)
  gaps = [1.0]
  order = list(range(ref + 1, T)) + list(range(ref - 1, -1, -1))
  for i in order:
    vis = ~canon_bad & ~occ[i]
    if vis.sum() > 4:
      h, stats[i] = ransac(canon, pts[i], vis, thresh, thr, gaps)
    else:
      h = np.eye(3)
    tformed[i], err = transform(h, pts[i], canon)
    invalid[i], all_err[i], homogs[i] = occ[i], err, h
    canon, canon_bad = update(err)
  for j in range(num_refinement_passes):
    for fr in [ref] + order:
      err = transform(homogs[fr], pts[fr], canon)[1]
      bad = canon_bad | (err > thresh * thresh) | occ[fr]
      h = solve_homography(canon, pts[fr], (~bad).astype(np.float64), gaps)
      if fr == ref and j != num_refinement_passes - 1:
        # the reference frame stays the identity: every other frame takes inv(h) instead; only
        # the reference frame's row of tformed is rewritten (with the last frame's points)
        h_inv = np.linalg.inv(h)
        for fr2 in range(T):
          homogs[fr2] = h_inv @ homogs[fr2]
        tformed[fr] = transform(homogs[T - 1], pts[T - 1], canon)[0]
        h = np.eye(3)
        canon = update(all_err)[0]
      tformed[fr], err = transform(h, pts[fr], canon)
      all_err[fr], homogs[fr] = err, h
      canon, canon_bad = update(err)
  scale = np.diag(1.0 / np.array(list(image_dimensions) + [1], np.float64))
  return dict(homogs=homogs @ scale, err=all_err.T.copy(), canonical=canon,
              canonical_invalid=canon_bad, ransac_stats=stats, min_gap=min(gaps))


def foreground_tracks(err, visibles, inlier_threshold=0.07, foreground_frac=0.6):
  """The rainbow demo's last step: a track is foreground when at most `foreground_frac` of its
  visible frames have err < inlier_threshold^2."""
  vis = np.asarray(visibles).astype(np.float64)
  inl = (np.asarray(err) < inlier_threshold ** 2) * vis
  return inl.sum(1) / np.maximum(1.0, vis.sum(1)) <= foreground_frac
