"""Multi-GPU execution of the TAPIR hot path (SURVEY.md 8(e)), one process per GPU.

Frames are independent in the backbone and queries are independent everywhere, so:
  1. each rank runs the backbone on its own slice of frames,
  2. ONE all-gather of the per-frame feature grids (NCCL over NVLink / NVSwitch),
  3. each rank tracks its own shard of the query points - no collective in the refine loop,
  4. (optional) gather of the [N, T, 4] outputs.
The partitioning helpers are pure functions so they can be tested with gloo on CPU.
"""
from typing import List, Tuple

import torch
import torch.distributed as dist


def frame_shard(num_frames: int, rank: int, world: int) -> Tuple[int, int, int]:
  """Returns (start, stop, padded_per_rank): contiguous frame ranges, last ranks may be short."""
  per = (num_frames + world - 1) // world
  start = min(rank * per, num_frames)
  stop = min(start + per, num_frames)
  return start, stop, per


def query_shard(num_queries: int, rank: int, world: int) -> Tuple[int, int]:
  per = (num_queries + world - 1) // world
  start = min(rank * per, num_queries)
  return start, min(start + per, num_queries)


def all_gather_frames(local: torch.Tensor, num_frames: int, group=None, async_op: bool = False):
  """local: [B, t_local, ...] (this rank's frame slice) -> [B, num_frames, ...] on every rank.

  B == 1 (every demo / benchmark): `[1, t, ...]` IS `[t, ...]` in memory, so the ranks' slices
  are gathered straight into the final layout - no transpose, no zero fill, no copy (the short
  last rank, when the frames do not divide evenly, sends from a padded staging buffer).  With
  async_op the call returns (tensor, work); the tensor is valid after work.wait()."""
  world = dist.get_world_size(group)
  rank = dist.get_rank(group)
  _, _, per = frame_shard(num_frames, rank, world)
  b = local.shape[0]
  rest = tuple(local.shape[2:])
  if b == 1:
    send = local[0].contiguous()
    if send.shape[0] != per:  # short (or empty) last rank
      pad = local.new_zeros((per,) + rest)
      pad[:send.shape[0]] = send
      send = pad
    out = local.new_empty((1, world * per) + rest)
    work = dist.all_gather_into_tensor(out[0], send, group=group, async_op=async_op)
    res = out[:, :num_frames]  # a prefix of the frame axis: still contiguous for B == 1
    return (res, work) if async_op else res
  send = local.new_zeros((per, b) + rest)
  send[:local.shape[1]] = local.transpose(0, 1)
  out = local.new_empty((world * per, b) + rest)
  work = dist.all_gather_into_tensor(out, send.contiguous(), group=group, async_op=async_op)
  if async_op:
    work.wait()
  res = out[:num_frames].transpose(0, 1).contiguous()
  return (res, None) if async_op else res


def gather_queries(local: torch.Tensor, num_queries: int, dim: int = 1, group=None) -> torch.Tensor:
  """Inverse of query_shard along `dim`; every rank receives the full tensor."""
  world = dist.get_world_size(group)
  per = (num_queries + world - 1) // world
  x = local.transpose(0, dim).contiguous()
  send = x.new_zeros((per,) + tuple(x.shape[1:]))
  send[:x.shape[0]] = x
  out = x.new_empty((world * per,) + tuple(x.shape[1:]))
  dist.all_gather_into_tensor(out, send, group=group)
  return out[:num_queries].transpose(0, dim).contiguous()


_SIDE_STREAMS = {}


def _side_stream(device):
  key = str(device)
  if key not in _SIDE_STREAMS:
    _SIDE_STREAMS[key] = torch.cuda.Stream(device=device)
  return _SIDE_STREAMS[key]


def sharded_forward(model, video: torch.Tensor, query_points: torch.Tensor, gather_outputs=True,
                    group=None):
  """model(video, query_points) computed cooperatively by all ranks of `group`.

  `video` [1, T, H, W, 3] and `query_points` [1, N, 3] must be identical on every rank (each
  rank only touches its own frame / query slices).  Returns the same dict as TAPIR.forward
  (on every rank if gather_outputs, else only this rank's query shard).
  """
  from tapnet_b200.tapir_model import FeatureGrids, refined_average  # pylint: disable=g-import-not-at-top
  world = dist.get_world_size(group)
  rank = dist.get_rank(group)
  T = video.shape[1]
  N = query_points.shape[1]
  f0, f1, _ = frame_shard(T, rank, world)
  mdev = next(model.parameters()).device
  on_gpu = mdev.type == 'cuda'
  if on_gpu and query_points.device.type == 'cpu':
    # host buffers in: each rank copies only its own frames (get_feature_grids streams them)
    query_points = query_points.to(mdev, non_blocking=True)
  hires_events = []
  if f1 > f0:
    local = model.get_feature_grids(video[:, f0:f1], False, hires_ready_events=hires_events)
    lo_l, hi_l, res = list(local.lowres), list(local.hires), local.resolutions
  else:  # more ranks than frames: contribute an empty slice with the right trailing shape
    probe = model.get_feature_grids(video[:, :1], False)
    lo_l = [t[:, :0] for t in probe.lowres]
    hi_l = [t[:, :0] for t in probe.hires]
    res = probe.resolutions
  # The hires grid of a resolution is final one third of the way through its backbone pass: its
  # all-gather is issued behind the `hires ready` event on a side stream, so NCCL moves it while
  # ResNet groups 2-3 and the ExtraConvs are still running (SURVEY.md 8(e)).  Only the lowres
  # gather, which needs the end of the backbone, stays exposed.  Every rank issues the
  # collectives in the same order (hires of each distinct resolution, then lowres of each).
  main = torch.cuda.current_stream(mdev) if on_gpu else None
  ready = {h.data_ptr(): ev for h, ev in hires_events}
  side = _side_stream(mdev) if on_gpu else None
  pending_hi, pending_lo, order = {}, {}, []
  for lo, hi in zip(lo_l, hi_l):
    key = (lo.data_ptr(), hi.data_ptr())
    if key in pending_hi:  # equal resolutions alias one tensor: gather it once
      order.append(key)
      continue
    ev = ready.get(hi.data_ptr())
    if side is not None and ev is not None:
      side.wait_event(ev)
      with torch.cuda.stream(side):
        pending_hi[key] = all_gather_frames(hi, T, group, async_op=True)
      hi.record_stream(side)
    else:
      pending_hi[key] = all_gather_frames(hi, T, group, async_op=True)
    order.append(key)
  for lo, hi in zip(lo_l, hi_l):
    key = (lo.data_ptr(), hi.data_ptr())
    if key not in pending_lo:
      pending_lo[key] = all_gather_frames(lo, T, group, async_op=True)
  lowres, hires = [], []
  for key in order:
    for pend in (pending_lo, pending_hi):
      t, work = pend[key]
      if work is not None:
        if main is not None:
          with torch.cuda.stream(main):
            work.wait()
        else:
          work.wait()
        pend[key] = (t, None)
    lowres.append(pending_lo[key][0])
    hires.append(pending_hi[key][0])
  grids = FeatureGrids(tuple(lowres), tuple(hires), tuple(res))
  q0, q1 = query_shard(N, rank, world)
  qp = query_points[:, q0:q1]
  qf = model.get_query_features(video, False, qp, grids)
  tr = model.estimate_trajectories(video.shape[-3:-1], False, grids, qf, qp, None)
  out = refined_average(tr, model.num_pips_iter)
  if gather_outputs and world > 1:
    out = {k: gather_queries(v, N, 1, group) for k, v in out.items()}
  return out
