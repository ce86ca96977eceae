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

`track_video` runs the same sweep (the same `_slide` and `_track_window` per window) on frames it
asks a reader for: the pre-pass reads only the tap frames, the sweep reads each frame once into a
device ring one window ahead, and each core's outputs are yielded as soon as they are enqueued, so
neither the clip nor full-length outputs ever exist.
"""
import math
from typing import List, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch

from tapnet_b200 import _lib
from tapnet_b200 import live
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

  def staged(st, new):  # the frames staged on the device
    return new * H * W * 3 * video_itemsize if host_video or not st.direct else 0
  buffers, work = _sweep_terms(model, T, (H, W), num_points, window_frames,
                               refinement_resolutions, staged)
  return buffers + work


def _sweep_terms(model, T, hw, num_points, window_frames, refinement_resolutions, staged):
  """(pass buffers, larger of the largest backbone step and stage A + the largest refinement
  level) of a sweep with cores of window_frames frames; staged(step, new) gives the bytes of the
  frames a backbone step over `new` frames stages besides its resample and workspace."""
  plan = tapir_model._pass_plan(hw, model.initial_resolution, refinement_resolutions)
  halos = halo_frames(model, hw, refinement_resolutions)
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
    b += staged(st, new)
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
  return buffers, max(backbone, stage_a + refine)


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
  return tapir_model._work_groups([max(1, num_points)], max(1, frames))[0][3]


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
  return _largest_core(need, free_bytes, T)


def _largest_core(need, free_bytes, T):
  """The largest C in 1..T with need(C) <= free_bytes, need non-decreasing and need(1) fitting."""
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


def _yuv_frames(clip, a, z, repeat=1):
  """Frames a..z-1 of a one-clip YUV clip (each `repeat` times), with its window and matrix."""
  return clip.map_buffers(lambda t: t[:, a:z] if repeat == 1
                          else t[:, a:z].repeat_interleave(repeat, 1))


def _run_pass(model, pk, video, step, a, z, out, dev):
  """Backbone pass `step` over frames a..z-1 of the one-clip video (or device YUV clip) into out
  (lowres, hires)."""
  if isinstance(video, live.YUVFrames):
    frames = _yuv_frames(video, a, z)
  else:
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
      if isinstance(video, live.YUVFrames):
        pair = _yuv_frames(video, i, i + 1, repeat=2)
      else:
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


def _prepass_chunks(t0, T, max_frames):
  """The query pre-pass's chunks as (sorted frames, queries): the tap pairs of the first tap frames
  t0 in frame order, at most max(2, max_frames) frames per chunk, each pair within one chunk."""
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
  return chunks


def _query_features(model, pk, clip_of, video_shape, b, num_clips, qp, plan, max_frames, dev):
  """Query features [N, C] of clip b of num_clips clips of video_shape (T, H, W) at every resolution
  of `plan` (lowres list, hires list), sampled from the grids of the queries' tap frames only, in
  the chunks of _prepass_chunks; clip_of(i, frames) gives chunk i's frames as a one-clip video
  [1, F, H, W, 3] (or a device YUV clip)."""
  T, H, W = (int(v) for v in video_shape)
  steps = [st for st in plan if st.new]
  pass_of = np.cumsum([st.new for st in plan]) - 1
  N = qp.shape[0]
  feats = ([torch.empty(N, schema.LOWRES_DIM, dtype=torch.float32, device=dev) for _ in plan],
           [torch.empty(N, schema.HIRES_DIM, dtype=torch.float32, device=dev) for _ in plan])
  t0 = query_tap_frames(qp[:, 0].cpu().numpy(), T)
  for i, (frame_list, query_list) in enumerate(_prepass_chunks(t0, T, max_frames)):
    sub = clip_of(i, frame_list)
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

  occ_out, expd_out, trk_out = tapir_model._new_estimates(num_iters + 1, (B, N, T), dev)
  qp_all = query_points.to(device=dev, dtype=torch.float32)
  if N > 0 and T > 0:
    steps = [st for st in plan if st.new]
    pass_of = np.cumsum([st.new for st in plan]) - 1
    for b in range(B):
      clip = video[b:b + 1]
      qp = qp_all[b].contiguous()
      qf_lo, qf_hi = _query_features(model, pk, lambda _, fl: clip[:, torch.tensor(fl)],
                                     (T, H, W), b, B, qp, plan, max_frames, dev)
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


def _pass_buffers(windows, plan, dev):
  """One (lowres, hires) buffer per backbone pass of `plan`, sized by the widest range of the level
  it serves over `windows`."""
  bufs = []
  for st, l in zip([st for st in plan if st.new], pass_levels(plan)):
    cap = max(z - a for w in windows for a, z in [w.levels[l - 1]])
    bufs.append(tuple(torch.empty((1, cap) + s, dtype=torch.float32, device=dev)
                      for s in tapir_model._grid_shapes(st.h, st.w)))
  return bufs


def _slide(bufs, held, steps, win, run):
  """Moves every pass's buffer to window `win`'s range and computes its new frames only:
  run(p, step, first, z, out) writes pass p's grids of frames first..z-1 into out.  held: the
  range each buffer holds, updated in place."""
  for p, (st, (a, z)) in enumerate(zip(steps, win.passes)):
    a0, z0 = held[p]
    keep = max(0, z0 - a)
    if keep and a > a0:
      for t in bufs[p]:
        _shift(t, a - a0, keep)
    first = a + keep
    if z > first:
      run(p, st, first, z, tuple(t[:, first - a:z - a] for t in bufs[p]))
    held[p] = (a, z)


def _track_window(model, pk, win, bufs, held, plan, pass_of, qp, qframe, qf_lo, qf_hi, hw, sink,
                  dev):
  """Stage A over level 1's range of window `win` and each refinement level over its own range,
  from the pass buffers.  sink(it, sl, (occ, expd, tracks), a) receives iteration it's estimates
  ([n, frames, ...], frames from a on) of the queries sl; iteration 0 is stage A's."""
  N = qp.shape[0]
  L = len(plan) - 1
  npi = model.num_pips_iter

  def grid(i, rng, hires=False):
    p = pass_of[i]
    a = held[p][0]
    return bufs[p][1 if hires else 0][:, rng[0] - a:rng[1] - a]

  # pooled pyramid levels of each level's range
  pooled = {l: model._pool_pyramid(grid(l, win.levels[l - 1])) for l in range(1, L + 1)}

  a1, z1 = win.levels[0]
  T1 = z1 - a1
  for _, _, q0, q1 in tapir_model._work_groups([N], T1):
    sl, nq = slice(q0, q1), q1 - q0
    shapes, _ = tapir_model._stage_a_scratch(1, nq, T1, grid(0, (a1, z1)).shape[2:])
    occ0, expd0, trk0 = (torch.empty(s, dtype=torch.float32, device=dev) for s in shapes[:3])
    qp_w = torch.cat([(qframe[sl] - a1)[:, None], qp[sl, 1:]], dim=1)
    pos = model._stage_a(pk, grid(0, (a1, z1)), qf_lo[0][sl].contiguous(), [nq], None, qp_w, hw,
                         occ0, expd0, trk0, None, dev)
    sink(0, sl, (occ0, expd0, trk0), a1)
    prev = (a1, z1)
    for l in range(1, L + 1):
      al, zl = win.levels[l - 1]
      Tl = zl - al
      pos = pos[:, al - prev[0]:zl - prev[0]].contiguous()
      occ0_l = occ0[:, al - a1:zl - a1].contiguous()
      expd0_l = expd0[:, al - a1:zl - a1].contiguous()
      level_outs = tapir_model._new_estimates(npi, (nq, Tl), dev)
      model._refine_level(pk, grid(l, (al, zl), hires=True), grid(l, (al, zl)), pooled[l],
                          qf_hi[l][sl], qf_lo[l][sl], pos, occ0_l, expd0_l,
                          list(zip(*level_outs)), model._refine_buffers(nq, Tl, dev),
                          plan[l][:2], hw)
      for i, xs in enumerate(zip(*level_outs)):
        sink((l - 1) * npi + i + 1, sl, xs, al)
      prev = (al, zl)


def _sweep(model, pk, clip, qp, qframe, qf_lo, qf_hi, plan, steps, pass_of, halos, C, b, B,
           outs, dev):
  """The sweep of clip b of B ([1, T, H, W, 3] on the host or the device): each window's core
  outputs go into the full-length outputs `outs` (occlusion, expected distance, tracks lists)."""
  T, H, W = (int(v) for v in clip.shape[1:4])
  windows = window_plan(T, C, halos, plan)
  bufs = _pass_buffers(windows, plan, dev)
  held = [(0, 0)] * len(steps)

  def run(p, st, first, z, out):
    _run_frames(model, pk, clip[:, first:z], st, out, _alone_frames(st, B, T, b, range(first, z)),
                dev)

  for win in windows:
    def sink(it, sl, xs, a, win=win):
      for full, x in zip(outs, xs):
        full[it][b, sl, win.start:win.stop] = x[:, win.start - a:win.stop - a]

    _slide(bufs, held, steps, win, run)
    _track_window(model, pk, win, bufs, held, plan, pass_of, qp, qframe, qf_lo, qf_hi, (H, W),
                  sink, dev)


# ------------------------------------------------------------------------------ frame reader
# track_video runs the same sweep on frames it asks a reader for: each frame is read once, kept in
# a device ring in the reader's format until the last backbone pass that needs it has its grids,
# and every window's core outputs are handed back as soon as they are enqueued.
def _pass_spans(windows):
  """For each window, the frames [lo, hi) its backbone passes still need: from the first frame
  any pass adds to its buffer to the end of the widest range."""
  held = [0] * len(windows[0].passes)
  spans = []
  for win in windows:
    lo, hi = None, 0
    for p, (a, z) in enumerate(win.passes):
      first = max(a, held[p])
      if z > first:
        lo = first if lo is None else min(lo, first)
      hi = max(hi, z)
      held[p] = z
    spans.append((hi if lo is None else lo, hi))
  return spans


def sweep_reads(num_frames, window_frames, halos, plan) -> List[Tuple[int, int]]:
  """The frame range track_video reads for each window of the sweep (halos from halo_frames, plan
  from tapir_model._pass_plan): the frames its passes need that no window before has read.  The
  ranges are consecutive and cover [0, num_frames) once; a window that needs no new frame has an
  empty range and reads nothing."""
  reads, end = [], 0
  for _, hi in _pass_spans(window_plan(num_frames, window_frames, halos, plan)):
    reads.append((end, max(end, hi)))
    end = max(end, hi)
  return reads


def ring_frames(num_frames, window_frames, halos, plan) -> int:
  """Frames of track_video's device ring: the most frames any window's passes still need at once.
  A window's new frames overwrite only frames the window before has run through every pass."""
  return max(hi - lo for lo, hi in _pass_spans(window_plan(num_frames, window_frames, halos, plan)))


def _prepass_reads(t0, T, max_frames):
  """(probe, reads of each _prepass_chunks chunk): the probe is the first tap pair, read before
  anything is sized (it fixes the frame format); each chunk then reads the runs of its frames that
  the frames kept from before (the probe, then the last frame of the chunk before) do not hold."""
  chunks = _prepass_chunks(t0, T, max_frames)
  f0 = chunks[0][0][0]
  probe = (f0, min(f0 + 2, T))
  kept = set(range(*probe))
  reads = []
  for frames, _ in chunks:
    runs = []
    for f in frames:
      if f in kept:
        continue
      if runs and runs[-1][1] == f:
        runs[-1][1] = f + 1
      else:
        runs.append([f, f + 1])
    reads.append([tuple(r) for r in runs])
    kept = {frames[-1]}
  return probe, reads


def prepass_reads(t, num_frames, max_frames) -> List[Tuple[int, int]]:
  """The frame ranges track_video's query pre-pass reads, in order, for queries at times t with
  pre-pass chunks of at most max_frames frames: only the queries' tap frames, each once."""
  probe, reads = _prepass_reads(query_tap_frames(t, num_frames), num_frames, max_frames)
  return [probe] + [r for chunk in reads for r in chunk]


def reader_sweep_bytes(model, video_shape, num_points, window_frames, refinement_resolutions=None,
                       frame_bytes=None):
  """Device bytes of track_video's sweep over a (1, T, H, W) video with cores of window_frames
  frames: the frame ring (frame_bytes per frame, default uint8 RGB), the pass buffers, the larger
  of the largest backbone step and stage A + the largest refinement level, and two windows'
  outputs (the one the caller holds while the next is computed).  No term grows with T once the
  windows reach their full size."""
  _, T, H, W = (int(v) for v in video_shape[:4])
  frame_bytes = H * W * 3 if frame_bytes is None else int(frame_bytes)
  plan = tapir_model._pass_plan((H, W), model.initial_resolution, refinement_resolutions)
  C = min(int(window_frames), T)
  ring = ring_frames(T, C, halo_frames(model, (H, W), refinement_resolutions), plan) * frame_bytes

  def staged(st, new):  # a lone frame's two-frame call of itself: the pair and its grids
    return 2 * frame_bytes + 2 * _f32_bytes(tapir_model._grid_shapes(st.h, st.w))
  buffers, work = _sweep_terms(model, T, (H, W), num_points, C, refinement_resolutions, staged)
  outs = 2 * output_bytes(model, (1, C, H, W), num_points, refinement_resolutions)
  return ring + buffers + work + outs


def choose_reader_window_frames(model, video_shape, num_points, free_bytes,
                                refinement_resolutions=None, frame_bytes=None):
  """The largest core length whose track_video sweep (reader_sweep_bytes) fits free_bytes."""
  def need(c):
    return reader_sweep_bytes(model, video_shape, num_points, c, refinement_resolutions,
                              frame_bytes)
  if need(1) > free_bytes:
    raise ValueError(f'tracking a {tuple(video_shape)} video with {num_points} queries needs '
                     f'{need(1)} bytes of device memory even with one-frame windows; '
                     f'{free_bytes} are available')
  return _largest_core(need, free_bytes, int(video_shape[1]))


def _describe(x):
  """(format string, frame count) of what a reader returned; (None, 0) if it is no frame batch."""
  if isinstance(x, live.YUVFrames):
    if x.y.shape[0] != 1:
      return None, 0
    H, W = x.frame_size
    return (f'YUV {x.layout} {x.bits}-bit {H}x{W} frames, window {x.window}, {x.matrix}, '
            f'{"full" if x.full_range else "limited"} range, on {x.device}'), int(x.y.shape[1])
  if (isinstance(x, torch.Tensor) and x.dim() == 4 and x.shape[-1] == 3
      and (x.dtype == torch.uint8 or x.dtype.is_floating_point)):
    return f'{x.dtype} RGB {x.shape[1]}x{x.shape[2]} frames on {x.device}', int(x.shape[0])
  return None, 0


class _FrameSource:
  """read_frames(start, stop), its result checked against the first call's format.  Keeps what the
  first result looked like, not the frames."""

  def __init__(self, read, dev):
    self.read, self.dev, self.format = read, dev, None

  def __call__(self, a, z):
    x = self.read(a, z)
    what, n = _describe(x)
    if what is None:
      got = tuple(x.shape) if isinstance(x, torch.Tensor) else type(x).__name__
      raise ValueError(f'read_frames({a}, {z}) returned {got}; expected a uint8 or float '
                       f'[{z - a}, H, W, 3] tensor or live.YUVFrames of [1, {z - a}] frames')
    if x.device.type != 'cpu' and x.device != self.dev:
      raise ValueError(f'read_frames({a}, {z}) returned frames on {x.device}; the model is on '
                       f'{self.dev}')
    if self.format is None:
      self.format = what
      self.host = x.device.type == 'cpu'
      if isinstance(x, live.YUVFrames):  # its layout, without its frames
        self.yuv = x.map_buffers(lambda b: torch.empty((1, 0) + tuple(b.shape[2:]), dtype=b.dtype,
                                                       device=b.device))
        self.frame_size = x.frame_size
        self.hw = tuple(int(v) for v in x.shape[2:4])
        self.itemsize = 1
      else:
        self.yuv = None
        self.hw = self.frame_size = (int(x.shape[1]), int(x.shape[2]))
        self.itemsize = 1 if x.dtype == torch.uint8 else 4
    elif what != self.format:
      raise ValueError(f'read_frames({a}, {z}) returned {what}; the first call returned '
                       f'{self.format}')
    if n != z - a:
      raise ValueError(f'read_frames({a}, {z}) returned {n} frames, expected {z - a}')
    return x

  @property
  def frame_bytes(self):
    """Bytes of one frame as the device stores it."""
    H, W = self.frame_size
    if self.yuv is not None:
      return sum(math.prod(b.shape[2:]) * b.element_size() for b in self.yuv.buffers)
    return H * W * 3 * self.itemsize


class _FrameStore:
  """S device frames in a _FrameSource's format: uint8 or float32 RGB [1, S, H, W, 3], or the
  source's YUV buffers [1, S, ...] (dense rows) with its layout, window and matrix."""

  def __init__(self, src, S, dev):
    self.yuv = src.yuv
    if src.yuv is not None:
      self.planes = tuple(torch.empty((1, S) + tuple(b.shape[2:]), dtype=b.dtype, device=dev)
                          for b in src.yuv.buffers)
    else:
      dtype = torch.uint8 if src.itemsize == 1 else torch.float32
      self.planes = (torch.empty((1, S) + src.hw + (3,), dtype=dtype, device=dev),)

  def view(self, s, z):
    """Slots s..z-1 as a one-clip video or YUV clip."""
    if self.yuv is None:
      return self.planes[0][:, s:z]
    return self.yuv.with_buffers([t[:, s:z] for t in self.planes])

  def put(self, s, x, i, n, non_blocking=True):
    """Frames i..i+n-1 of x (a reader's result or another store) into slots s..s+n-1."""
    if isinstance(x, _FrameStore):
      src = [t[0, i:i + n] for t in x.planes]
    elif isinstance(x, live.YUVFrames):
      src = [t[0, i:i + n] for t in x.buffers]
    else:
      src = [x[i:i + n]]
    for dst, t in zip(self.planes, src):
      dst[0, s:s + n].copy_(t, non_blocking=non_blocking)


class _ReaderSweep:
  """The state of one track_video call: prepare() runs the query pre-pass and sizes the sweep,
  window(w) enqueues window w, reads window w + 1's new frames and returns w's outputs, close()
  waits for the copies in flight."""

  def __init__(self, model, read, T, query_points, window_frames, refinement_resolutions,
               unrefined, dev):
    self.model, self.T, self.qp_in, self.dev = model, T, query_points, dev
    self.window_frames, self.refs, self.unrefined = window_frames, refinement_resolutions, unrefined
    self.src = _FrameSource(read, dev)
    self.pending = None  # (reader result, copy-done event) of the next window's frames
    self.cs = self.main = None

  def prepare(self):
    model, T, dev, src = self.model, self.T, self.dev, self.src
    self.pk = model._pack()
    self.main, self.cs = torch.cuda.current_stream(dev), model._copy_stream(dev)
    qp = self.qp_in.to(device=dev, dtype=torch.float32).contiguous()
    times = qp[:, 0].cpu().numpy()
    t0 = query_tap_frames(times, T)
    probe = _prepass_reads(t0, T, 2)[0]
    first = src(*probe)  # fixes the format and the frame size
    H, W = src.hw
    N = qp.shape[0]
    self.plan = plan = tapir_model._pass_plan((H, W), model.initial_resolution, self.refs)
    halos = halo_frames(model, (H, W), self.refs)
    shape = (1, T, H, W)
    budget = _free_device_bytes(dev)
    C = self.window_frames
    if C is None:
      C = choose_reader_window_frames(model, shape, N, budget, self.refs, src.frame_bytes)
    C = min(int(C), T)
    # the pre-pass may use what the sweep will, and no more than is free; two frames at least
    bound = min(budget, reader_sweep_bytes(model, shape, N, C, self.refs, src.frame_bytes))
    max_frames = 2
    while (max_frames < T and prepass_bytes(model, shape, max_frames * 2, self.refs, False,
                                            src.itemsize) <= bound):
      max_frames *= 2
    _, prepass = _prepass_reads(t0, T, max_frames)
    kept = (list(range(*probe)), _FrameStore(src, probe[1] - probe[0], dev))
    kept[1].put(0, first, 0, probe[1] - probe[0], non_blocking=False)
    del first

    def clip_of(i, frames):
      nonlocal kept
      store = _FrameStore(src, len(frames), dev)
      slot = {f: j for j, f in enumerate(frames)}
      for j, f in enumerate(kept[0]):
        if f in slot:
          store.put(slot[f], kept[1], j, 1)
      for a, z in prepass[i]:
        # a blocking copy: the reader may refill its buffer on the next call
        store.put(slot[a], src(a, z), 0, z - a, non_blocking=False)
      last = _FrameStore(src, 1, dev)
      last.put(0, store, len(frames) - 1, 1)
      kept = (frames[-1:], last)
      return store.view(0, len(frames))

    self.qf_lo, self.qf_hi = _query_features(model, self.pk, clip_of, (T, H, W), 0, 1, qp, plan,
                                             max_frames, dev)
    kept = None
    self.qp = qp
    self.qframe = torch.from_numpy(query_frames(times, T).astype(np.float32)).to(dev)
    self.windows = window_plan(T, C, halos, plan)
    self.reads = sweep_reads(T, C, halos, plan)
    self.S = ring_frames(T, C, halos, plan)
    self.ring = _FrameStore(src, self.S, dev)
    self.steps = [st for st in plan if st.new]
    self.pass_of = np.cumsum([st.new for st in plan]) - 1
    self.bufs = _pass_buffers(self.windows, plan, dev)
    self.held = [(0, 0)] * len(self.steps)
    self.pending = self._fetch(0, None)

  def _slots(self, a, z):
    """The ring slots of frames a..z-1 as (first frame, first slot, count) runs (the ring wraps)."""
    f = a
    while f < z:
      s = f % self.S
      n = min(z - f, self.S - s)
      yield f, s, n
      f += n

  def _fetch(self, w, after):
    """Reads window w's new frames and starts their copy into the ring on the copy stream, after
    event `after` (None: after the work enqueued so far)."""
    a, z = self.reads[w]
    if a == z:
      return None
    x = self.src(a, z)
    if after is None:
      self.cs.wait_stream(self.main)
    else:
      self.cs.wait_event(after)
    with torch.cuda.stream(self.cs):
      for f, s, n in self._slots(a, z):
        self.ring.put(s, x, f - a, n)
      done = torch.cuda.Event()
      done.record(self.cs)
    return x, done

  def _run(self, p, st, first, z, out):
    for f, s, n in self._slots(first, z):
      _run_frames(self.model, self.pk, self.ring.view(s, s + n), st,
                  tuple(t[:, f - first:f - first + n] for t in out),
                  _alone_frames(st, 1, self.T, 0, range(f, f + n)), self.dev)

  def window(self, w):
    model, dev, win = self.model, self.dev, self.windows[w]
    if self.pending is not None:
      self.main.wait_event(self.pending[1])
    _slide(self.bufs, self.held, self.steps, win, self._run)
    grids_done = torch.cuda.Event()
    grids_done.record(self.main)  # no pass reads the ring after this
    npi = model.num_pips_iter
    num_iters = npi * (len(self.plan) - 1)
    N, c = self.qp.shape[0], win.stop - win.start
    est = [tuple(x[0] for x in tapir_model._new_estimates(1, (1, N, c), dev))
           if self.unrefined or (it and it % npi == 0) else None for it in range(num_iters + 1)]

    def sink(it, sl, xs, a):
      if est[it] is not None:
        for dst, x in zip(est[it], xs):
          dst[0, sl] = x[:, win.start - a:win.stop - a]

    _track_window(model, self.pk, win, self.bufs, self.held, self.plan, self.pass_of, self.qp,
                  self.qframe, self.qf_lo, self.qf_hi, self.src.hw, sink, dev)
    traj = {k: [e[i] if e is not None else None for e in est]
            for i, k in enumerate(('occlusion', 'expected_dist', 'tracks'))}
    out = tapir_model.refined_average(traj, npi)
    if self.unrefined:
      out.update({f'unrefined_{k}': v[:-1] for k, v in traj.items()})
    # window w's frames are on the device: drop the reader's result before asking for more
    if self.pending is not None:
      self.pending[1].synchronize()
      self.pending = None
    if w + 1 < len(self.windows):
      self.pending = self._fetch(w + 1, grids_done if self.src.host else None)
    return out

  def close(self):
    if self.pending is not None:
      self.pending[1].synchronize()
      self.pending = None
    if self.main is not None:
      self.main.wait_stream(self.cs)  # later work may reuse the ring's memory


def track_video(model, read_frames, num_frames: int, query_points,
                window_frames: Optional[int] = None,
                refinement_resolutions: Optional[Sequence[Tuple[int, int]]] = None,
                unrefined: bool = False):
  """Tracks query_points through a video of num_frames frames that read_frames hands over in
  pieces; yields (start, stop, outputs) window by window in frame order.

  read_frames(start, stop) returns frames start..stop-1: a uint8 or float [stop - start, H, W, 3]
  tensor on the host (pinned or pageable) or on the model's device, or a device live.YUVFrames
  of [1, stop - start] frames whose window is the video.  The first call fixes the frame size and
  format (for YUV also the layout, window, matrix and range); a later call that returns anything else, or
  a wrong frame count, raises ValueError naming its range.  The query pre-pass asks only for the
  queries' tap frames, each once; the sweep then asks for consecutive ranges that cover
  [0, num_frames) once, in order, one window ahead, so the reader decodes while the GPU works.

  query_points: [N, 3] or [1, N, 3] (t, y, x), N >= 1.  outputs: 'tracks' [1, N, stop - start, 2],
  'occlusion' and 'expected_dist' [1, N, stop - start] on the model's device, fresh tensors, and
  with unrefined=True the unrefined_* lists cut to the same frames.  Concatenated over the frame
  axis they equal model(video, query_points) bit for bit.  window_frames: the core length C; None
  picks the largest C whose sweep fits the free device memory.  Host and device memory stay
  bounded whatever num_frames is.  Arguments are checked when the call is made; frames are read
  once the iteration starts."""
  if isinstance(num_frames, bool) or not isinstance(num_frames, (int, np.integer)) or num_frames < 1:
    raise ValueError(f'num_frames must be a positive integer, got {num_frames!r}')
  if window_frames is not None and int(window_frames) < 1:
    raise ValueError(f'window_frames must be >= 1, got {window_frames}')
  if not callable(read_frames):
    raise ValueError(f'read_frames must be callable, got {type(read_frames).__name__}')
  qp = query_points
  if (not isinstance(qp, torch.Tensor) or qp.shape[-1:] != (3,) or qp.dim() not in (2, 3)
      or (qp.dim() == 3 and qp.shape[0] != 1) or qp.shape[-2] == 0):
    raise ValueError('query_points must be an [N, 3] or [1, N, 3] tensor with N >= 1, got '
                     f'{tuple(qp.shape) if isinstance(qp, torch.Tensor) else type(qp).__name__}')
  dev = model._device_check(None if qp.device.type == 'cpu' else qp)
  sweep = _ReaderSweep(model, read_frames, int(num_frames), qp.reshape(-1, 3), window_frames,
                       refinement_resolutions, bool(unrefined), dev)
  return _track_video(sweep, dev)


def _track_video(sweep, dev):
  # the model's device is current while the sweep works, the caller's while it holds a window
  try:
    with torch.cuda.device(dev):
      sweep.prepare()
    for w, win in enumerate(sweep.windows):
      with torch.cuda.device(dev):
        out = sweep.window(w)
      yield win.start, win.stop, out
      del out
  finally:
    with torch.cuda.device(dev):
      sweep.close()
