"""Offline tracking of clips of any length in bounded GPU memory.

`model(video, query_points)` keeps every frame's feature grids on the device for the whole call,
so the clip length it can take is capped by device memory.  `windowed_forward` returns the same
dict, bit for bit, while holding the grids of a bounded range of frames only.

Why a window can be exact.  Every stage except the PIPs mixer works on one frame at a time
(backbone, stage A, local correlation, pyramid pooling, the track update), and no result depends
on how rows are grouped into launches.  The mixer's blocks each run two depthwise temporal
convolutions of width k: a non-causal convolution reaches (k - 1) / 2 frames to each side, a causal
one k - 1 frames back.  One mixer pass over nb blocks therefore reaches nb (k - 1) frames to each
side (non-causal) or 2 nb (k - 1) back (causal), and a refinement level of num_pips_iter passes
num_pips_iter times that.  At a level boundary the features restart from the query features and
occlusion / expected distance from stage A: only the positions carry over.  So if level l of L runs
on [s - H_l, e + H_l), its positions are exact on [s - H_{l+1}, e + H_{l+1}), with

    H_l = (L - l + 1) * num_pips_iter * nb * (k - 1)         (non-causal, both sides)
    H_l = (L - l + 1) * num_pips_iter * nb * 2 * (k - 1)     (causal, left side only)

and H_{L+1} = 0: the last level is exact on the core [s, e).  Stage A and level 1 use the smallest
grids and the widest range; the last level the largest grids and the narrowest, so each backbone
pass keeps its own buffer sized by the widest level it serves.

The driver, per clip:
  1. Query pre-pass: each query's features are sampled from the two frames its time coordinate
     falls between (`query_tap_frames`), with `tapir_sample_query_features_ex` so that the whole
     clip's length normalises the time axis.  Only those frames go through the backbone.
  2. Sweep: for each core [s, e), every pass's buffer drops the frames the new window no longer
     needs, moves its overlap to the front and runs the backbone on the new frames only (each frame
     goes through each pass once).  Stage A runs over level 1's range, each level l over its own
     range starting from the positions the level before left, and the core frames of every
     iteration's outputs are copied into full-length outputs.
  3. The averages over the levels' last estimates are taken once, on the full-length outputs.
"""
import math
from typing import List, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch

from tapnet_b200 import _lib
from tapnet_b200 import schema
from tapnet_b200 import tapir_model

# share of the free device memory the automatic core length plans for: the rest covers the caching
# allocator's rounding and fragmentation
_MEMORY_SHARE = 0.85


def _mixer_reach(model):
  """(mixer blocks, depthwise kernel width) of the mixer the model runs, read off its weights."""
  sd = dict(model.named_parameters())
  key = 'torch_pips_mixer.blocks.{}.mlp1_up.weight'
  nb = 0
  while key.format(nb) in sd:
    nb += 1
  if nb == 0:
    raise ValueError('the model has no mixer blocks')
  return nb, int(sd[key.format(0)].shape[-1])


def halo_frames(model, video_hw, refinement_resolutions=None) -> List[Tuple[int, int]]:
  """(left, right) halo in frames of each refinement level (level 1 first) of a video_hw video:
  running level l on [s - left, e + right) makes its output positions exact where level l + 1
  runs, and the last level's exact on [s, e).  See the module docstring."""
  plan = tapir_model._pass_plan(video_hw, model.initial_resolution, refinement_resolutions)
  num_levels = len(plan) - 1
  nb, k = _mixer_reach(model)
  if model.use_casual_conv:
    per_level = model.num_pips_iter * nb * 2 * (k - 1)
    return [((num_levels - l + 1) * per_level, 0) for l in range(1, num_levels + 1)]
  per_level = model.num_pips_iter * nb * (k - 1)
  return [((num_levels - l + 1) * per_level,) * 2 for l in range(1, num_levels + 1)]


class Window(NamedTuple):
  """One step of the sweep: the core [start, stop) whose outputs it writes, the frame range of
  each refinement level (level 1 first; stage A runs over level 1's) and of each backbone pass's
  buffer."""
  start: int
  stop: int
  levels: Tuple[Tuple[int, int], ...]
  passes: Tuple[Tuple[int, int], ...]


def pass_levels(plan):
  """For each backbone pass of `plan` (tapir_model._pass_plan), the lowest refinement level among
  the resolutions it serves (the initial resolution, index 0, is served over level 1's range)."""
  return [max(i, 1) for i, step in enumerate(plan) if step.new]


def window_plan(num_frames, window_frames, halos, plan) -> List[Window]:
  """The windows of a sweep over num_frames frames with cores of window_frames frames; halos from
  halo_frames, plan from tapir_model._pass_plan."""
  if window_frames < 1:
    raise ValueError(f'window_frames must be >= 1, got {window_frames}')
  T = int(num_frames)
  owners = pass_levels(plan)
  windows = []
  for s in range(0, T, window_frames):
    e = min(s + window_frames, T)
    levels = tuple(_two_frames(max(0, s - left), min(T, e + right), T) for left, right in halos)
    windows.append(Window(s, e, levels, tuple(levels[l - 1] for l in owners)))
  return windows


def _two_frames(a, z, T):
  """The range a..z-1, widened to two frames when it holds one and the clip has more.  The mixer
  splits K (and so sums in another order) for one-frame calls only, as the whole-clip call does
  for one-frame clips alone; a wider range only adds frames the whole clip also has."""
  if z - a == 1 and T >= 2:
    return (a - 1, z) if a > 0 else (0, 2)
  return (a, z)


def query_tap_frames(t, num_frames):
  """First tap frame t0 of each query time t (the second is t0 + 1 when < num_frames): a float32
  mirror of sample_query_kernel's arithmetic with the clip's own length, border clamp included."""
  t = np.asarray(t, dtype=np.float32)
  f = np.float32(num_frames)
  one, two, half = np.float32(1), np.float32(2), np.float32(0.5)
  c = (t * f) / f + half
  g = two * (c / f) - one
  pix = ((g + one) * f - one) / two
  pix = np.fmin(np.fmax(pix, np.float32(0)), f - one)
  return np.floor(pix).astype(np.int64)


def query_frames(t, num_frames):
  """The frame each query time t marks as its query frame in stage A, with the whole clip's
  float32 arithmetic: rint(t * T / T) (rounding half to even, as rintf)."""
  t = np.asarray(t, dtype=np.float32)
  f = np.float32(num_frames)
  return np.rint((t * f) / f).astype(np.int64)


# ------------------------------------------------------------------------------ byte model
def _f32_bytes(shapes):
  return 4 * sum(math.prod(s) for s in shapes)


def output_bytes(model, video_shape, num_points, refinement_resolutions=None):
  """Bytes of the full-length outputs a call holds: every iteration's occlusion, expected distance
  and tracks, and the averages with their stacking temporaries."""
  B, T, H, W = (int(v) for v in video_shape[:4])
  num_levels = len(tapir_model._pass_plan((H, W), model.initial_resolution,
                                          refinement_resolutions)) - 1
  per = B * num_points * T * 16
  return per * (model.num_pips_iter * num_levels + 1 + num_levels + 1)


def sweep_bytes(model, video_shape, num_points, window_frames, refinement_resolutions=None,
                host_video=False, video_itemsize=1):
  """Device bytes the sweep of one clip needs beyond the full-length outputs, with cores of
  window_frames frames: the pass buffers, the largest backbone step (new frames, their resample and
  the backbone workspace), stage A over level 1's range and the largest refinement level."""
  _, T, H, W = (int(v) for v in video_shape[:4])
  plan = tapir_model._pass_plan((H, W), model.initial_resolution, refinement_resolutions)
  halos = halo_frames(model, (H, W), refinement_resolutions)
  C = min(int(window_frames), T)
  span = [min(T, C + left + right) for left, right in halos]
  steps = [st for st in plan if st.new]
  owners = pass_levels(plan)
  buffers = sum(span[l - 1] * _f32_bytes(tapir_model._grid_shapes(st.h, st.w))
                for st, l in zip(steps, owners))
  backbone = 0
  for st, l in zip(steps, owners):
    new = min(T, C + halos[l - 1][1])  # the first window computes its whole right halo
    b = model._backbone_workspace_bytes(new, st.h, st.w)
    if not st.direct:
      b += new * st.h * st.w * 3 * 4
    if host_video or not st.direct:
      b += new * H * W * 3 * video_itemsize  # the frames staged on the device
    backbone = max(backbone, b)
  # stage A: one query group over level 1's range
  T1 = span[0]
  nq = _group_queries(num_points, T1)
  shapes, stage_a = tapir_model._stage_a_scratch(
      1, nq, T1, tapir_model._grid_shapes(*model.initial_resolution)[0])
  stage_a += _f32_bytes(shapes)
  refine = 0
  for l, (st_i, Tl) in enumerate(zip(plan[1:], span), start=1):
    gh, gw, c = tapir_model._grid_shapes(st_i.h, st_i.w)[0]
    pooled = sum(Tl * (gh >> j) * (gw >> j) * c * 4 for j in range(1, model.pyramid_level + 1))
    level_io = nq * Tl * 16 * (model.num_pips_iter + 2)  # outputs, the cut pos / occ / expd
    specs, mixer_ws = model._refine_scratch(nq, Tl)
    scratch = mixer_ws + sum(math.prod(s) * d.itemsize for s, d in specs)
    refine = max(refine, pooled + level_io + scratch)
  return buffers + max(backbone, stage_a + refine)


def prepass_bytes(model, video_shape, frames, refinement_resolutions=None, host_video=False,
                  video_itemsize=1):
  """Device bytes of the query pre-pass's feature grids over `frames` frames."""
  _, _, H, W = (int(v) for v in video_shape[:4])
  plan = tapir_model._pass_plan((H, W), model.initial_resolution, refinement_resolutions)
  total = frames * H * W * 3 * max(video_itemsize, 4)
  work = 0
  for st in plan:
    if st.new:
      total += frames * _f32_bytes(tapir_model._grid_shapes(st.h, st.w))
      work = max(work, model._backbone_workspace_bytes(frames, st.h, st.w)
                 + (0 if st.direct else frames * st.h * st.w * 3 * 4))
  return total + work


def _group_queries(num_points, frames):
  """Queries per refinement group of one clip over `frames` frames (as estimate_trajectories)."""
  return tapir_model._groups(1, max(1, num_points), max(1, frames))[0][2].stop


def choose_window_frames(model, video_shape, num_points, free_bytes, refinement_resolutions=None,
                         host_video=False, video_itemsize=1):
  """The largest core length whose sweep fits free_bytes next to the full-length outputs."""
  T = int(video_shape[1])
  fixed = output_bytes(model, video_shape, num_points, refinement_resolutions)

  def need(c):
    return fixed + sweep_bytes(model, video_shape, num_points, c, refinement_resolutions,
                               host_video, video_itemsize)
  if need(1) > free_bytes:
    raise ValueError(f'a windowed call on a {tuple(video_shape)} clip with {num_points} queries '
                     f'needs {need(1)} bytes of device memory even with one-frame windows; '
                     f'{free_bytes} are available')
  lo, hi = 1, T
  while lo < hi:
    mid = (lo + hi + 1) // 2
    if need(mid) <= free_bytes:
      lo = mid
    else:
      hi = mid - 1
  return lo


def _free_device_bytes(dev):
  free, _ = torch.cuda.mem_get_info(dev)
  cached = torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
  return int((free + cached) * _MEMORY_SHARE)


# ------------------------------------------------------------------------------ driver
def _check_inputs(model, video, query_points):
  if not isinstance(video, torch.Tensor) or video.dim() != 5 or video.shape[-1] != 3:
    raise ValueError(f'video must be a [B, T, H, W, 3] tensor, got '
                     f'{tuple(video.shape) if isinstance(video, torch.Tensor) else type(video)}')
  if not (video.dtype == torch.uint8 or video.dtype.is_floating_point):
    raise ValueError(f'video must be uint8 or floating point, got {video.dtype}')
  if (not isinstance(query_points, torch.Tensor) or query_points.dim() != 3
      or query_points.shape[0] != video.shape[0] or query_points.shape[-1] != 3):
    raise ValueError(f'query_points must be a [B, N, 3] tensor for {video.shape[0]} clips, got '
                     f'{tuple(query_points.shape) if isinstance(query_points, torch.Tensor) else type(query_points)}')
  dev = model._device_check(None if video.device.type == 'cpu' else video)
  return dev


def _run_pass(model, pk, video, step, a, z, out, dev):
  """Backbone pass `step` over frames a..z-1 of the one-clip video into out (lowres, hires)."""
  src = tapir_model._backbone_frames(video[:, a:z])
  if step.direct and video.device.type == 'cpu':  # streamed in behind the stem convolution
    return model._backbone_pass(pk, torch.empty_like(src, device=dev), src, None, dev, out)
  frames = src.to(dev, non_blocking=True)
  if not step.direct:
    resized = torch.empty(1, z - a, step.h, step.w, 3, dtype=torch.float32, device=dev)
    _lib.resample_frames(frames, resized)
    frames = resized
  model._backbone_pass(pk, frames, None, None, dev, out)


def _alone_frames(step, num_clips, T, b, frames):
  """Which of clip b's `frames` the whole-clip call of num_clips clips of T frames runs through
  pass `step` in a one-frame backbone chunk.  The ExtraConv GEMMs split K for one-frame chunks
  only, which sums in another order, so the driver must run exactly these frames alone.  The
  whole-clip call chunks the num_clips * T frames of the batch in order: every frame is alone when
  a chunk holds one frame, otherwise only the batch's last frame, when it is left over."""
  nf = num_clips * T
  chunk = tapir_model._backbone_chunk(step.h, step.w, nf)
  g = b * T + np.asarray(frames, dtype=np.int64)
  return np.full(g.shape, chunk == 1) | ((g == nf - 1) & (nf % chunk == 1))


def _run_frames(model, pk, video, step, out, alone, dev):
  """Backbone pass `step` over every frame of the one-clip video [1, n, H, W, 3] into out (lowres,
  hires) [1, n, ...]: the frames marked `alone` one per call, every other frame in calls of 2 to
  one chunk of frames, so that the backbone never splits K for them.  A lone unmarked frame runs as
  a two-frame call of itself twice; a short last call starts earlier and recomputes a frame."""
  n = video.shape[1]
  P = tapir_model._backbone_chunk(step.h, step.w, n)
  i = 0
  while i < n:
    if alone[i]:
      _run_pass(model, pk, video, step, i, i + 1, tuple(t[:, i:i + 1] for t in out), dev)
      i += 1
      continue
    j = i
    while j < n and not alone[j]:
      j += 1
    if j - i == 1:
      pair = video[:, i:i + 1].expand(1, 2, *video.shape[2:]).contiguous()
      tmp = tuple(torch.empty((1, 2) + t.shape[2:], dtype=t.dtype, device=dev) for t in out)
      _run_pass(model, pk, pair, step, 0, 2, tmp, dev)
      for t, x in zip(out, tmp):
        t[:, i].copy_(x[:, 0])
    else:
      for a in range(i, j, P):
        a = min(a, j - 2)
        z = min(a + P, j)
        _run_pass(model, pk, video, step, a, z, tuple(t[:, a:z] for t in out), dev)
    i = j


def _query_features(model, pk, video, b, num_clips, qp, plan, max_frames, dev):
  """Query features [N, C] of clip b (video [1, T, H, W, 3]) of num_clips at every resolution of
  `plan` (lowres list, hires list), sampled from the grids of the queries' tap frames only, in
  chunks of at most max_frames frames that keep each query's tap pair together."""
  T, H, W = (int(v) for v in video.shape[1:4])
  steps = [st for st in plan if st.new]
  pass_of = np.cumsum([st.new for st in plan]) - 1
  N = qp.shape[0]
  feats = ([torch.empty(N, schema.LOWRES_DIM, dtype=torch.float32, device=dev) for _ in plan],
           [torch.empty(N, schema.HIRES_DIM, dtype=torch.float32, device=dev) for _ in plan])
  t0 = query_tap_frames(qp[:, 0].cpu().numpy(), T)
  chunks, frames, queries = [], set(), []
  for f0 in np.unique(t0):
    pair = {int(f0)} | ({int(f0) + 1} if f0 + 1 < T else set())
    if frames and len(frames | pair) > max(2, max_frames):
      chunks.append((sorted(frames), queries))
      frames, queries = set(), []
    frames |= pair
    queries.extend(np.nonzero(t0 == f0)[0].tolist())
  if frames:
    chunks.append((sorted(frames), queries))
  for frame_list, query_list in chunks:
    sub = video[:, torch.tensor(frame_list)]
    F = len(frame_list)
    grids = []
    for st in steps:
      g = tuple(torch.empty((1, F) + s, dtype=torch.float32, device=dev)
                for s in tapir_model._grid_shapes(st.h, st.w))
      _run_frames(model, pk, sub, st, g, _alone_frames(st, num_clips, T, b, frame_list), dev)
      grids.append(g)
    slot = torch.full((T,), -1, dtype=torch.int32)
    slot[torch.tensor(frame_list)] = torch.arange(len(frame_list), dtype=torch.int32)
    slot = slot.to(dev)
    idx = torch.tensor(query_list, dtype=torch.long, device=dev)
    q = qp.index_select(0, idx).contiguous()
    for i in range(len(plan)):
      lo, hi = grids[pass_of[i]]
      for grid, dst in ((lo, feats[0][i]), (hi, feats[1][i])):
        out = torch.empty(len(query_list), grid.shape[-1], dtype=torch.float32, device=dev)
        _lib.sample_query_features(grid[0], q, (T, H, W), out, frame_slot=slot)
        dst.index_copy_(0, idx, out)
    del grids
  return feats


def _shift(buf, d, keep):
  """Moves frames d..d+keep-1 of buf [1, F, ...] to 0..keep-1 with forward copies of at most d
  frames each, so no copy reads frames another part of it writes."""
  for j in range(0, keep, d):
    c = min(d, keep - j)
    buf[:, j:j + c].copy_(buf[:, d + j:d + j + c])


def windowed_forward(model, video, query_points, window_frames: Optional[int] = None,
                     refinement_resolutions: Optional[Sequence[Tuple[int, int]]] = None,
                     _halo_trim: Optional[Sequence[int]] = None):
  """`model(video, query_points)` computed window by window in bounded device memory; the returned
  dict (occlusion, tracks, expected_dist and the unrefined_* lists, all full length, on the model's
  device) is bit for bit the whole-clip call's.

  video: [B, T, H, W, 3] uint8 or float, on the model's device or on the host (a pinned host clip
  is streamed in window by window); query_points: [B, N, 3] (t, y, x).  window_frames: the core
  length C; None picks the largest C whose buffers fit the device's free memory (a given C is not
  checked against it; the query pre-pass keeps within both).  The results do not depend on C.  Clips are swept one after another (the batched call computes each clip as its
  single-clip call).  `_halo_trim` (tests only) shortens each level's halo by that many frames."""
  if window_frames is not None and int(window_frames) < 1:
    raise ValueError(f'window_frames must be >= 1, got {window_frames}')
  dev = _check_inputs(model, video, query_points)
  with torch.cuda.device(dev):
    return _windowed(model, video, query_points, window_frames, refinement_resolutions,
                     _halo_trim, dev)


def _windowed(model, video, query_points, window_frames, refinement_resolutions, halo_trim, dev):
  B, T, H, W, _ = (int(v) for v in video.shape)
  N = int(query_points.shape[1])
  host = video.device.type == 'cpu'
  pk = model._pack()
  plan = tapir_model._pass_plan((H, W), model.initial_resolution, refinement_resolutions)
  L = len(plan) - 1
  npi = model.num_pips_iter
  num_iters = npi * L
  halos = halo_frames(model, (H, W), refinement_resolutions)
  if halo_trim is not None:
    halos = [(max(0, a - d), max(0, b - d) if b else 0) for (a, b), d in zip(halos, halo_trim)]
  shape = (B, T, H, W)
  itemsize = video.element_size() if video.dtype == torch.uint8 else 4
  budget = _free_device_bytes(dev)
  if window_frames is None:
    window_frames = choose_window_frames(model, shape, N, budget, refinement_resolutions, host,
                                         itemsize)
  C = min(int(window_frames), max(T, 1))
  # the pre-pass may use what the sweep will, and no more than is free (window_frames may be
  # given larger than fits); two frames, one query's tap pair, at least
  bound = min(budget, sweep_bytes(model, shape, N, C, refinement_resolutions, host, itemsize))
  max_frames = 2
  while (max_frames < T and prepass_bytes(model, shape, max_frames * 2, refinement_resolutions,
                                          host, itemsize) <= bound):
    max_frames *= 2

  occ_out, expd_out, trk_out = tapir_model._new_estimates(num_iters + 1, B, N, T, dev)
  qp_all = query_points.to(device=dev, dtype=torch.float32)
  if N > 0 and T > 0:
    steps = [st for st in plan if st.new]
    pass_of = np.cumsum([st.new for st in plan]) - 1
    for b in range(B):
      clip = video[b:b + 1]
      qp = qp_all[b].contiguous()
      qf_lo, qf_hi = _query_features(model, pk, clip, b, B, qp, plan, max_frames, dev)
      # stage A's query frame, resolved once over the whole clip; each window sees it relative to
      # its own range, so a query outside the range matches no frame
      qframe = torch.from_numpy(query_frames(qp[:, 0].cpu().numpy(), T).astype(np.float32))
      qframe = qframe.to(dev)
      _sweep(model, pk, clip, qp, qframe, qf_lo, qf_hi, plan, steps, pass_of, halos, C, b, B,
             (occ_out, expd_out, trk_out), dev)
  trajectories = dict(occlusion=occ_out, tracks=trk_out, expected_dist=expd_out)
  return dict(
      **tapir_model.refined_average(trajectories, npi),
      unrefined_occlusion=occ_out[:-1],
      unrefined_tracks=trk_out[:-1],
      unrefined_expected_dist=expd_out[:-1],
  )


def _sweep(model, pk, clip, qp, qframe, qf_lo, qf_hi, plan, steps, pass_of, halos, C, b, B,
           outs, dev):
  T, H, W = (int(v) for v in clip.shape[1:4])
  N = qp.shape[0]
  L = len(plan) - 1
  npi = model.num_pips_iter
  windows = window_plan(T, C, halos, plan)
  owners = pass_levels(plan)
  bufs = []
  for st, l in zip(steps, owners):
    cap = max(z - a for w in windows for a, z in [w.levels[l - 1]])
    bufs.append(tuple(torch.empty((1, cap) + s, dtype=torch.float32, device=dev)
                      for s in tapir_model._grid_shapes(st.h, st.w)))
  held = [(0, 0)] * len(steps)
  for win in windows:
    # ---- slide every pass's buffer and run the backbone on the new frames only
    for p, (st, (a, z)) in enumerate(zip(steps, win.passes)):
      a0, z0 = held[p]
      keep = max(0, z0 - a)
      if keep and a > a0:
        for t in bufs[p]:
          _shift(t, a - a0, keep)
      first = a + keep
      if z > first:
        _run_frames(model, pk, clip[:, first:z], st, tuple(t[:, first - a:z - a] for t in bufs[p]),
                    _alone_frames(st, B, T, b, range(first, z)), dev)
      held[p] = (a, z)

    def grid(i, rng, hires=False):
      p = pass_of[i]
      a = held[p][0]
      return bufs[p][1 if hires else 0][:, rng[0] - a:rng[1] - a]

    # pooled pyramid levels of each level's range
    pooled = {l: model._pool_pyramid(grid(l, win.levels[l - 1])) for l in range(1, L + 1)}

    a1, z1 = win.levels[0]
    T1 = z1 - a1
    core = slice(win.start, win.stop)
    for _, _, sl in tapir_model._groups(1, N, T1):
      nq = sl.stop - sl.start
      shapes, _ = tapir_model._stage_a_scratch(1, nq, T1, grid(0, (a1, z1)).shape[2:])
      occ0, expd0, trk0 = (torch.empty(s, dtype=torch.float32, device=dev) for s in shapes[:3])
      qp_w = torch.cat([(qframe[sl] - a1)[:, None], qp[sl, 1:]], dim=1)[None].contiguous()
      pos = model._stage_a(pk, grid(0, (a1, z1)), qf_lo[0][sl][None].contiguous(), qp_w, (H, W),
                           occ0, expd0, trk0, None, dev)
      for full, x in zip(outs, (occ0, expd0, trk0)):
        full[0][b, sl, core] = x[0, :, win.start - a1:win.stop - a1]
      prev = (a1, z1)
      for l in range(1, L + 1):
        al, zl = win.levels[l - 1]
        Tl = zl - al
        pos = pos[:, :, al - prev[0]:zl - prev[0]].contiguous()
        occ0_l = occ0[:, :, al - a1:zl - a1].contiguous()
        expd0_l = expd0[:, :, al - a1:zl - a1].contiguous()
        level_outs = tapir_model._new_estimates(npi, 1, nq, Tl, dev)
        model._refine_level(pk, grid(l, (al, zl), hires=True), grid(l, (al, zl)), pooled[l],
                            qf_hi[l][sl], qf_lo[l][sl], pos, occ0_l, expd0_l,
                            list(zip(*level_outs)), model._refine_buffers(nq, Tl, dev),
                            plan[l][:2], (H, W))
        for full, xs in zip(outs, level_outs):
          for i, x in enumerate(xs):
            full[(l - 1) * npi + i + 1][b, sl, core] = x[0, :, win.start - al:win.stop - al]
        prev = (al, zl)
