"""Streaming / online tracking with CUDA-graph replay (BASELINE.json config 3).

`tapnet/pytorch_live_demo.py:44-85` runs, per camera frame,
    feature_grids = model.get_feature_grids(frame)            (one frame)
    model.estimate_trajectories(..., causal_context=state, get_causal_context=True)
which is ~260 small kernel launches: at a few query points the GPU idles between launches
(3.7 ms/frame eager for 8 points).  `OnlineTracker` captures exactly that per-frame step once in
a CUDA graph (fixed frame size and point count) and replays it: same kernels, same results bit for
bit, no per-launch host cost.  The causal state lives in static device buffers that the graph
updates in place; `update_query` mirrors `TAPIR.update_query_features` for re-targeting a point.

With `num_streams=S` one tracker follows S camera streams.  Each stream is
tracked as the reference tracks one camera of its frame size (`height` / `width` / `window` may be
given per stream): the default refinement resolutions of its own size, tracks in its own pixels.
Streams whose backbone passes agree (`tapir_model._pass_plan`) form a group; one captured graph
runs, per group, its passes over the group's frames and one batched estimate_trajectories over its
clips of one frame each (the reference's batch axis, with per-clip video sizes).  Streams of one
frame size form one group whose input is one [S, 1, H, W, 3] batch, so a step is one backbone
pass over the S frames; a group of several sizes resamples its frames in one ingest launch per
pass, whatever their sizes.

With `num_points` a sequence of S counts each stream tracks its own number of points, without
padding.  Either way a group packs its streams' query features, causal state and outputs along the
point axis ([1, sum N, ...]) and runs one estimate_trajectories with `points_per_clip`, so the
per-query stages (stage A, local correlation, the mixer, the track update) run over the streams'
points only.  Each stream's tracks, visibles and logits are slices of its group's packed outputs.

`retarget`, `add_points` and `remove_points` edit a stream's points between steps.  Each edit takes
effect at the next step, on that step's frame: after a tracker's first edit every group's step
runs one `tapir_sample_query_rows` launch that samples the requested rows from the step's own
grids and zeroes their state rows, reading a request table the host uploads before replay.  A
count change re-packs the group's buffers and re-captures the graph.

With `yuv420=True` the tracker takes `live.YUV420Frames` (NV12 / I420 camera or decoder frames),
with `yuv_layout='p010'` (or another `live.YUVFrames` layout) frames of that layout: it keeps static
Y / U / V buffers of the camera frames, a step copies the planes into them and replays the graph,
and the layout, crop windows and colour matrix are fixed at construction.
"""
from typing import List, NamedTuple, Optional, Sequence, Tuple, Union

import torch

from tapnet_b200 import _lib
from tapnet_b200 import live
from tapnet_b200 import tapir_model


class StreamSpec(NamedTuple):
  """One camera stream: its frame size, the crop window it is tracked in (YUV trackers; None for
  the whole frame) and the size of that window, in whose pixels its tracks are."""
  frame_hw: Tuple[int, int]
  window: Optional[Tuple[int, int, int, int]]
  hw: Tuple[int, int]


def _is_window_list(window):
  return window is not None and len(window) > 0 and not isinstance(window[0], int)


def stream_specs(height, width, num_streams: int, yuv420: bool = False,
                 window=None) -> List[StreamSpec]:
  """The StreamSpec of every stream from the constructor's size arguments: `height` and `width`
  are ints or sequences of num_streams ints, `window` (yuv420 only) one (y0, x0, h, w) or a
  sequence of num_streams of them (None entries: the whole frame)."""
  S = int(num_streams)

  def per_stream(v, name):
    if isinstance(v, int):
      return [int(v)] * S
    v = [int(x) for x in v]
    if len(v) != S:
      raise ValueError(f'{name} has {len(v)} entries for {S} streams')
    return v

  if not yuv420 and window is not None:
    raise ValueError('window is only supported with yuv420=True')
  hs, ws = per_stream(height, 'height'), per_stream(width, 'width')
  if _is_window_list(window):
    windows = list(window)
    if len(windows) != S:
      raise ValueError(f'window has {len(windows)} entries for {S} streams')
  else:
    windows = [window] * S
  specs = []
  for s, (H, W, win) in enumerate(zip(hs, ws, windows)):
    if H <= 0 or W <= 0:
      raise ValueError(f'stream {s}: frame size {H}x{W}')
    if win is not None:
      win = tuple(int(a) for a in win)
      y0, x0, h, w = win
      if h <= 0 or w <= 0 or y0 < 0 or x0 < 0 or y0 + h > H or x0 + w > W:
        raise ValueError(f'stream {s}: window {win} outside the {H}x{W} frame')
    specs.append(StreamSpec((H, W), win, (win[2], win[3]) if win is not None else (H, W)))
  return specs


def group_streams(specs: Sequence[StreamSpec], initial_resolution=(256, 256)):
  """Streams that run through one backbone pass sequence and one batched estimate_trajectories:
  a list of (plan, [stream indices]) in order of first appearance.  Streams group by their pass
  plan; a plan with a direct-read pass holds the tracked size, so such a stream only shares a
  group with streams of its size (and, when cropping, of its frame size and window)."""
  from tapnet_b200 import tapir_model as tm  # pylint: disable=g-import-not-at-top
  groups = {}
  for s, spec in enumerate(specs):
    plan = tuple(tm._pass_plan(spec.hw, initial_resolution))
    key = (plan, (spec.frame_hw, spec.window) if any(p.direct for p in plan) else None)
    groups.setdefault(key, (list(plan), []))[1].append(s)
  return list(groups.values())


# -- point edits (OnlineTracker.retarget / add_points / remove_points) as pure functions on one
# stream's pending requests: a dict {point index: (t, y, x)} of the points whose features the next
# step samples, indices in the stream's current points.
def edit_indices(idx, count: int, what: str) -> List[int]:
  """`idx` (an int, a sequence, a 1-D tensor or numpy array) as a list of point indices in
  [0, count)."""
  if isinstance(idx, torch.Tensor):
    if idx.dim() > 1 or idx.dtype.is_floating_point or idx.dtype == torch.bool:
      raise ValueError(f'{what}: idx must be integers, got a {idx.dtype} {list(idx.shape)} tensor')
    idx = idx.reshape(-1).tolist()
  elif hasattr(idx, 'tolist'):  # numpy arrays and scalars (the live demo's np.array([idx]))
    idx = idx.tolist()
  if not isinstance(idx, (list, tuple, range)):
    idx = [idx]
  out = []
  for i in idx:
    if isinstance(i, bool) or not isinstance(i, int):
      raise ValueError(f'{what}: idx must be integers, got {i!r}')
    if not 0 <= i < count:
      raise ValueError(f'{what}: point {i} out of range [0, {count})')
    out.append(int(i))
  return out


def edit_points(query_points, k: Optional[int], what: str) -> List[Tuple[float, float, float]]:
  """`query_points` ([k, 3] or [3]: (t, y, x) in the stream's pixels) as host tuples; k = None
  takes any number."""
  qp = torch.as_tensor(query_points).detach().to('cpu', torch.float32)
  if qp.dim() == 1:
    qp = qp[None]
  if qp.dim() != 2 or qp.shape[1] != 3 or (k is not None and qp.shape[0] != k):
    raise ValueError(f'{what}: query_points must be [{"k" if k is None else k}, 3], got '
                     f'{list(qp.shape)}')
  return [tuple(p) for p in qp.tolist()]


def retarget_requests(pending: dict, count: int, idx, points) -> dict:
  """Pending requests after re-targeting points `idx` at `points`: the last edit of a point wins."""
  idx = edit_indices(idx, count, 'retarget')
  points = edit_points(points, len(idx), 'retarget')
  out = dict(pending)
  out.update(zip(idx, points))
  return out


def add_requests(pending: dict, count: int, points) -> Tuple[dict, int, List[int]]:
  """(pending requests, new count, new indices) after appending `points` to a stream of `count`."""
  points = edit_points(points, None, 'add_points')
  new = list(range(count, count + len(points)))
  out = dict(pending)
  out.update(zip(new, points))
  return out, count + len(points), new


def remove_requests(pending: dict, count: int, idx) -> Tuple[dict, List[int]]:
  """(pending requests, kept indices) after removing points `idx`: the kept points keep their
  order, indices above a removed one shift down, and a removed point's request is dropped.  A
  stream keeps at least one point."""
  idx = edit_indices(idx, count, 'remove_points')
  if len(set(idx)) != len(idx):
    raise ValueError(f'remove_points: idx {idx} has repeated points')
  if len(idx) >= count:
    raise ValueError(f'remove_points: removing {len(idx)} of {count} points; a stream keeps at '
                     'least one')
  gone = set(idx)
  keep = [i for i in range(count) if i not in gone]
  new_index = {old: new for new, old in enumerate(keep)}
  return {new_index[i]: p for i, p in pending.items() if i in new_index}, keep


def packed_offsets(counts: Sequence[int]) -> List[int]:
  """Each stream's first row in a point axis packing streams of `counts` points in turn."""
  return [sum(counts[:i]) for i in range(len(counts))]


class _Edits:
  """A group's request table (tapir_sample_query_rows), sized to its point count: the static
  device table the graph reads, its pinned staging copy, and the event of the last upload."""

  def __init__(self, g, dev, const):
    rows = sum(g.counts)
    self.table = _lib.query_request_table(rows, dev)
    self.staging = _lib.query_request_table(rows, 'cpu', pin_memory=True)
    self.uploaded = torch.cuda.Event()
    self.pending_on_device = False  # the device table holds requests (a nonzero count)
    self.state = _lib.state_pointer_table(g.state, rows)
    self.video_hw = (g.video_size if isinstance(g.video_size, tuple)
                     else const([v for hw in g.video_size for v in hw], dev, torch.int32).view(-1, 2))


class _Group:
  """Streams sharing a pass plan: their static inputs, query features and causal state."""

  def __init__(self, plan, streams, specs, counts):
    self.plan, self.streams = plan, list(streams)
    # stream streams[i]'s points are rows offsets[i] .. offsets[i] + counts[i] - 1 of the group's
    # packed point axis
    self.counts = [counts[s] for s in streams]
    self.offsets = packed_offsets(self.counts)
    self.uniform = len({(specs[s].frame_hw, specs[s].window) for s in streams}) == 1
    sizes = [specs[s].hw for s in streams]
    # one size: estimate_trajectories' one-size call and launches; else per-clip sizes
    self.video_size = sizes[0] if len(set(sizes)) == 1 else sizes
    self.frames = None   # uniform groups: the [G, 1, ...] input of get_feature_grids
    self.sources = None  # otherwise: one one-frame input per stream, resampled together
    self.query_features = None
    self.state = None
    self.edits = None  # after the tracker's first point edit: the group's _Edits


class OnlineTracker:
  """Graph-replayed per-frame step of a causal TAPIR model (`use_casual_conv=True`) over
  `num_streams` camera streams of one frame format, of one frame size or of one size each, with
  one point count or one per stream."""

  def __init__(self, model: 'tapir_model.TAPIR', height: Union[int, Sequence[int]],
               width: Union[int, Sequence[int]], num_points: Union[int, Sequence[int]],
               uint8_frames: bool = False, num_streams: int = 1, yuv420: bool = False, window=None,
               matrix: str = 'bt601', full_range: bool = False, yuv_layout: Optional[str] = None):
    """height x width: the frame size.  With yuv420=True that is the camera frame and `window`
    (y0, x0, h, w; e.g. `live.center_square_window(height, width)`) the crop that is tracked, in
    whose pixels the tracks are; `matrix` / `full_range` describe the YUV frames.  `yuv_layout`
    (a `live.YUVFrames.layout` such as 'p010', 'yuv420p10', 'yuv444', 'yuyv') takes the place of
    yuv420=True for frames of that layout; frames of another layout with the same samples and
    chroma sampling (nv12 and i420; p010 and p016, whose MSB-aligned samples convert alike) are
    accepted too.  `height`,
    `width` and `window` may also give one value per stream: init / step then take a list of
    the streams' frames.  `num_points` may give one count per stream (each >= 1): init then takes
    a list of the streams' [N_s, 3] query points, and step / last_logits return lists of the
    streams' outputs."""
    if not model.use_casual_conv:
      raise ValueError('OnlineTracker needs a causal model: TAPIR(use_casual_conv=True)')
    if int(num_streams) < 1:
      raise ValueError(f'num_streams must be >= 1, got {num_streams}')
    if isinstance(num_points, int):
      counts = [num_points] * int(num_streams)
    else:
      counts = [int(n) for n in num_points]
      if len(counts) != int(num_streams):
        raise ValueError(f'num_points has {len(counts)} counts for {num_streams} streams')
      if min(counts) < 1:
        raise ValueError(f'num_points: every stream needs at least one point, got {counts}')
    if yuv_layout is not None and not live.is_yuv_layout(yuv_layout):
      raise ValueError(f'yuv_layout: unknown layout {yuv_layout!r}')
    if yuv420 and yuv_layout is not None:
      raise ValueError('yuv420 and yuv_layout are exclusive')
    layout = 'yuv420' if yuv420 else yuv_layout
    if layout is not None and uint8_frames:
      raise ValueError('uint8_frames and yuv420 / yuv_layout are exclusive')
    specs = stream_specs(height, width, num_streams, layout is not None, window)
    self.model = model
    self.specs = specs
    self.num_points = num_points if isinstance(num_points, int) else counts
    self._counts = counts
    self.num_streams = len(specs)
    self.dev = next(model.parameters()).device
    if self.dev.type != 'cuda':
      raise RuntimeError('OnlineTracker runs on CUDA only')
    # uint8_frames: frames are raw [0, 255] camera frames (what pytorch_live_demo.py:139-141 holds
    # before preprocess_frames); the normalisation runs inside the stem conv's loads
    self._frame_dtype = torch.uint8 if uint8_frames else torch.float32
    self._yuv = (matrix, bool(full_range)) if layout is not None else None
    self._yuv_layout = layout
    self._groups = [_Group(plan, streams, specs, counts)
                    for plan, streams in group_streams(specs, model.initial_resolution)]
    # streams of one frame size (and window) are one uniform group: init / step take a batch
    self._one_size = len(self._groups) == 1 and self._groups[0].uniform
    self.hw = specs[0].hw if self._one_size else [sp.hw for sp in specs]
    self._slot = {}  # stream -> (group, slot)
    order = []
    for gi, g in enumerate(self._groups):
      G = len(g.streams)
      H, W = specs[g.streams[0]].frame_hw
      if g.uniform:  # one [G, 1, ...] buffer; each stream's input is its slot of it
        g.frames = self._new_input(G, H, W, specs[g.streams[0]].window)
        g.sources = [self._input_slot(g.frames, i) for i in range(G)]
      else:
        g.sources = [self._new_input(1, *specs[s].frame_hw, specs[s].window) for s in g.streams]
      for i, s in enumerate(g.streams):
        self._slot[s] = (gi, i)
        order.append(s)
    # row r of the groups' concatenated outputs is stream order[r]: gather them back in the graph
    self._order = torch.tensor([order.index(s) for s in range(self.num_streams)], device=self.dev)
    self._stream_order = order
    self._pack_rows()
    self._pending = [{} for _ in range(self.num_streams)]  # per stream: point -> (t, y, x)
    # a one-size tracker's input: its group's [S, 1, ...] buffer, into which a step copies the batch
    self._frame = self._groups[0].frames if self._one_size else None
    self._graph = None
    self._graph_sig = None
    self._pinned = False
    self.query_features = None
    self.state = None
    self._out = None

  def _pack_rows(self):
    # stream s's points in the groups' concatenated point axis
    packed = [self._counts[s] for s in self._stream_order]
    offsets = packed_offsets(packed + [0])
    self._rows = {s: slice(offsets[r], offsets[r + 1]) for r, s in enumerate(self._stream_order)}

  def _new_input(self, n, H, W, window):
    if self._yuv is None:
      return torch.zeros(n, 1, H, W, 3, dtype=self._frame_dtype, device=self.dev)
    if self._yuv_layout != 'yuv420':
      return live.YUVFrames.zeros(self._yuv_layout, n, 1, H, W, self.dev, matrix=self._yuv[0],
                                  full_range=self._yuv[1], window=window)
    ch, cw = (H + 1) // 2, (W + 1) // 2
    planes = [torch.zeros(n, 1, *hw, dtype=torch.uint8, device=self.dev)
              for hw in ((H, W), (ch, cw), (ch, cw))]
    return live.YUV420Frames(*planes, matrix=self._yuv[0], full_range=self._yuv[1], window=window)

  @staticmethod
  def _input_slot(frames, i):
    if isinstance(frames, live.YUVFrames):
      return frames.map_buffers(lambda t: t[i:i + 1])
    return frames[i:i + 1]

  def _stream_frames(self, frames, streams):
    """Checks one frame per stream in `streams` (all before any copy): [H, W, 3] tensors (or
    [1, H, W, 3], [1, 1, H, W, 3]) of the stream's size, or one-frame YUVFrames of its frame
    size, window and samples.  Returns them as [1, 1, H, W, 3] tensors / YUV clips."""
    if isinstance(frames, (torch.Tensor, live.YUVFrames)) or len(frames) != len(streams):
      got = len(frames) if isinstance(frames, (list, tuple)) else type(frames).__name__
      raise ValueError(f'expected a list of {len(streams)} frames (one per stream), got {got}')
    out = []
    if self._yuv is not None:
      for s, f in zip(streams, frames):
        sp = self.specs[s]
        self._check_yuv(f, f'stream {s}: ')
        if f.frame_size != sp.frame_hw or f.window != (sp.window or (0, 0) + sp.frame_hw):
          raise ValueError(f'stream {s}: frame {f.frame_size} window {f.window}, expected '
                           f'{sp.frame_hw} window {sp.window}')
        if (f.matrix, f.full_range) != self._yuv:
          raise ValueError(f'stream {s}: {f.matrix}, full_range={f.full_range}; the tracker was '
                           f'built for {self._yuv[0]}, full_range={self._yuv[1]}')
        if tuple(f.y.shape[:2]) != (1, 1) or f.device != self.dev:
          raise ValueError(f'stream {s}: expected one frame on {self.dev}, got '
                           f'{list(f.y.shape[:2])} on {f.device}')
        out.append(f)
      return out
    dtypes = set()
    for s, f in zip(streams, frames):
      if not isinstance(f, torch.Tensor):
        raise ValueError(f'stream {s}: expected a tensor frame, got {type(f).__name__} (one frame '
                         'format per tracker)')
      dtypes.add(f.dtype)
      while f.dim() > 3 and f.shape[0] == 1:
        f = f[0]
      if f.dim() != 3 or tuple(f.shape) != (*self.specs[s].frame_hw, 3):
        raise ValueError(f'stream {s}: frame {tuple(f.shape)}, expected '
                         f'{(*self.specs[s].frame_hw, 3)}')
      out.append(f[None, None])
    if len(dtypes) > 1:
      raise ValueError(f'frames of mixed formats {sorted(map(str, dtypes))}: one per tracker')
    return out

  def _copy_in(self, src, dst):
    if isinstance(dst, live.YUVFrames):
      for d, p in zip((dst.y, dst.u, dst.v), (src.y, src.u, src.v)):
        d.copy_(p if p.dtype == d.dtype else p.view(d.dtype))  # uint16 / int16: the same bits
    else:
      dst.copy_(src)

  def _frames(self, frames):
    """init / step input, all checked before any copy.  A one-size tracker takes one batch:
    [S, H, W, 3], [S, 1, H, W, 3] or, when S = 1, [H, W, 3], returned as [S, 1, H, W, 3] on the
    device; or YUVFrames of [S, 1] frames of its frame size, window, samples and matrix, returned as
    they are.  Other trackers take a list of the streams' frames (`_stream_frames`)."""
    if not self._one_size:
      return self._stream_frames(frames, range(self.num_streams))
    S = self.num_streams
    if self._yuv is not None:
      self._check_yuv(frames, '')
      ref = self._frame
      if frames.frame_size != ref.frame_size:
        raise ValueError(f'frame size {frames.frame_size} != {ref.frame_size}')
      if (frames.window, frames.matrix, frames.full_range) != (ref.window, ref.matrix,
                                                               ref.full_range):
        raise ValueError(f'frames have window {frames.window}, {frames.matrix}, full_range='
                         f'{frames.full_range}; the tracker was built for {ref.window}, '
                         f'{ref.matrix}, full_range={ref.full_range}')
      if frames.device != self.dev:
        raise ValueError(f'frames on {frames.device}, tracker on {self.dev}')
      if tuple(frames.y.shape[:2]) != (S, 1):
        raise ValueError(f'expected YUVFrames of [{S}, 1] frames, got '
                         f'{list(frames.y.shape[:2])}')
      return frames
    frames = frames.to(self.dev, self._frame_dtype, non_blocking=True)
    if frames.dim() == 3:
      frames = frames[None, None]
    elif frames.dim() == 4:
      frames = frames[:, None]
    if frames.dim() != 5 or frames.shape[1] != 1 or frames.shape[4] != 3:
      raise ValueError(f'frames must be [S, H, W, 3], got {tuple(frames.shape)}')
    if frames.shape[0] != S:
      raise ValueError(f'expected {S} frames (one per stream), got {frames.shape[0]}')
    if tuple(frames.shape[2:4]) != self.hw:
      raise ValueError(f'frame size {tuple(frames.shape[2:4])} != {self.hw}')
    return frames

  def _check_yuv(self, f, who):
    """f is a YUV clip whose samples and chroma sampling are those of the tracker's layout."""
    ref = self._groups[0].sources[0]
    if not isinstance(f, live.YUVFrames) or f.sampling != ref.sampling:
      got = f.layout if isinstance(f, live.YUVFrames) else type(f).__name__
      built = ('yuv420=True' if self._yuv_layout == 'yuv420'
               else f'yuv_layout={self._yuv_layout!r}')
      raise ValueError(f'{who}this tracker was built with {built}: pass live.YUVFrames of that '
                       f'layout, got {got} (one frame format per tracker)')

  def _device_frame(self, f):
    return f if isinstance(f, live.YUVFrames) else f.to(self.dev, self._frame_dtype)

  def _query_features_one(self, frame, qp):
    grids = self.model.get_feature_grids(frame, False)
    return self.model.get_query_features(frame, False, qp, grids)

  def _group_grids(self, g):
    if g.uniform:
      return self.model.get_feature_grids(g.frames, False)
    return self.model._feature_grids_of_frames(
        [x if isinstance(x, live.YUVFrames) else x[0, 0] for x in g.sources], g.plan)

  def _step_group(self, g, state):
    """One group's step on its static inputs: its passes and one batched estimate_trajectories
    (B = group size, T = 1) that updates `state` in place; returns (tracks, occ, expd), packed
    [1, sum N, 1, ...].  After the tracker's first edit it first applies the group's request table,
    whose state rows are those of g.state."""
    grids = self._group_grids(g)
    if g.edits is not None:  # the pending point edits, sampled from this frame's grids
      qf = g.query_features
      _lib.sample_query_rows(grids.lowres + grids.hires, qf.lowres + qf.hires, g.edits.video_hw,
                             g.edits.table, g.edits.state)
    r = self.model.estimate_trajectories(g.video_size, False, grids, g.query_features, None, 64,
                                         causal_context=state, get_causal_context=True,
                                         causal_context_out=state, points_per_clip=g.counts)
    return r['tracks'][-1], r['occlusion'][-1], r['expected_dist'][-1]

  def _query_points(self, query_points):
    """init's query points, checked, as a list of S [N_s, 3] float32 tensors on the device: a list
    of the streams' [N_s, 3] points or, with one point count N, a [S, N, 3] tensor ([N, 3] when
    S = 1)."""
    S = self.num_streams
    if isinstance(self.num_points, int) and isinstance(query_points, torch.Tensor):
      qp = query_points.to(self.dev, torch.float32)
      if qp.dim() == 2:
        qp = qp[None]
      if qp.dim() != 3 or qp.shape[0] != S or qp.shape[2] != 3:
        raise ValueError(f'query_points must be [{S}, N, 3], got {tuple(qp.shape)}')
      if qp.shape[1] != self.num_points:
        raise ValueError(f'expected {self.num_points} query points, got {qp.shape[1]}')
      return list(qp)
    if isinstance(query_points, torch.Tensor) or len(query_points) != S:
      got = len(query_points) if isinstance(query_points, (list, tuple)) else type(query_points).__name__
      raise ValueError(f'expected a list of {S} query point tensors (one per stream), got {got}')
    out = []
    for s, (qp, n) in enumerate(zip(query_points, self._counts)):
      if not isinstance(qp, torch.Tensor) or tuple(qp.shape) != (n, 3):
        got = tuple(qp.shape) if isinstance(qp, torch.Tensor) else type(qp).__name__
        raise ValueError(f'stream {s}: query points must be [{n}, 3], got {got}')
      out.append(qp.to(self.dev, torch.float32))
    return out

  # -- pytorch_live_demo.py:44-54 online_model_init
  def init(self, frames: torch.Tensor, query_points: torch.Tensor):
    """frames: [S, H, W, 3] (or [S, 1, H, W, 3]; [H, W, 3] when S = 1) float in [-1, 1];
    query_points [S, N, 3] ([N, 3] when S = 1) as (t, y, x), stream s's on its frame s.  With
    per-stream sizes, frames is a list of the S streams' frames; with per-stream point counts,
    query_points is a list of the S streams' [N_s, 3] points."""
    qps = self._query_points(query_points)
    frames = self._frames(frames)
    # A one-size tracker samples every stream's features from one backbone pass over its batch, as
    # online_model_init on the batch does.  Other trackers compute each stream's as a one-stream
    # tracker of its size does; the two differ in the last bits, as the library splits K for
    # one-frame backbone chunks.
    if self._one_size:
      grids = self.model.get_feature_grids(frames, False)
      per_stream = [self.model.get_query_features(
          frames, False, qps[s][None], tapir_model.FeatureGrids(
              tuple(x[s:s + 1] for x in grids.lowres), tuple(x[s:s + 1] for x in grids.hires),
              grids.resolutions)) for s in range(self.num_streams)]
    else:
      frames = [self._device_frame(f) for f in frames]
      per_stream = [self._query_features_one(frames[s], qps[s][None])
                    for s in range(self.num_streams)]
    for g in self._groups:
      qfs = [per_stream[s] for s in g.streams]
      # private copies: the graph reads these exact buffers on every replay
      g.query_features = tapir_model.QueryFeatures(
          tuple(torch.cat([q.lowres[i] for q in qfs], 1) for i in range(len(qfs[0].lowres))),
          tuple(torch.cat([q.hires[i] for q in qfs], 1) for i in range(len(qfs[0].hires))),
          qfs[0].resolutions)
      init = self.model.construct_initial_causal_state(sum(g.counts), len(g.plan) - 1)
      # [1, sum N, 2, 512 | 2048] per block, one tensor per refinement iteration
      g.state = [{k: v.to(self.dev) for k, v in d.items()} for d in init]
      if g.edits is not None:  # new state buffers: a new pointer table
        g.edits = _Edits(g, self.dev, self.model._const)
    self._pending = [{} for _ in range(self.num_streams)]
    self._publish()
    return self.query_features

  def _publish(self):
    views = [self._published(g) for g in self._groups]
    if self._one_size:
      self.query_features, self.state = views[0]
    else:
      self.query_features, self.state = [v[0] for v in views], [v[1] for v in views]
    self._graph = None

  def _published(self, g):
    """A group's (query features, state) as `query_features` / `state` show them: packed
    [1, sum N, ...] with per-stream point counts, else [G, N, ...] views of the packed buffers
    (writes through them reach the graph)."""
    if not isinstance(self.num_points, int):
      return g.query_features, g.state

    def per_stream(x):
      return x.view(len(g.streams), self.num_points, *x.shape[2:])
    qf = g.query_features
    return (tapir_model.QueryFeatures(tuple(map(per_stream, qf.lowres)),
                                      tuple(map(per_stream, qf.hires)), qf.resolutions),
            [{k: per_stream(v) for k, v in d.items()} for d in g.state])

  def _step_eager(self):
    outs = [self._step_group(g, g.state) for g in self._groups]
    # the groups' packed [1, sum N, 1, ...] outputs, concatenated along the point axis
    tracks, occ, expd = (outs[0][i][0] if len(outs) == 1 else torch.cat([o[i][0] for o in outs])
                         for i in range(3))
    if not isinstance(self.num_points, int):  # each stream's outputs a slice of them
      visibles = live.postprocess_occlusions(occ, expd)
      return tuple([x[self._rows[s]] for s in range(self.num_streams)]
                   for x in (tracks, visibles, occ, expd))
    tracks, occ, expd = (x.view(-1, self.num_points, *x.shape[1:]) for x in (tracks, occ, expd))
    if len(outs) > 1:  # the groups' outputs back in stream order (one group holds them in order)
      tracks, occ, expd = (x.index_select(0, self._order) for x in (tracks, occ, expd))
    visibles = live.postprocess_occlusions(occ, expd)  # pytorch_live_demo.py:57-59
    return tracks, visibles, occ, expd

  def _capture(self):
    # warm-up on a side stream (allocates workspaces, packs weights, fills the constant cache);
    # the state is saved and restored so that warm-up steps do not advance it
    state = [d for g in self._groups for d in g.state]
    saved = [{k: v.clone() for k, v in d.items()} for d in state]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
      for _ in range(2):
        self._step_eager()
    torch.cuda.current_stream().wait_stream(s)
    for d, sv in zip(state, saved):
      for k in d:
        d[k].copy_(sv[k])
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      self._out = self._step_eager()
    for d, sv in zip(state, saved):  # capture does not execute, but be explicit
      for k in d:
        d[k].copy_(sv[k])
    self._graph = g
    # The graph holds RAW pointers into the model's workspaces and packed weight planes.  Pin
    # the workspaces (TAPIR._workspace then parks outgrown buffers instead of freeing them) and
    # remember which buffers / weights the capture saw: step() re-captures when another caller
    # of the same model (a larger offline clip, a second tracker, load_state_dict) replaced them.
    if not self._pinned:
      self.model._pin_workspaces()
      self._pinned = True
    self._graph_sig = self.model._workspace_sig()

  def close(self):
    """Drops the graph and releases the workspace pin."""
    self._graph = None
    if self._pinned:
      self.model._unpin_workspaces()
      self._pinned = False

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint: disable=broad-except
      pass

  # -- pytorch_live_demo.py:62-85 online_model_predict
  def step(self, frames: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """frames: [S, H, W, 3] ([H, W, 3] when S = 1), one per stream.  Returns (tracks [S, N, 1, 2]
    in frame pixels (x, y), visibles [S, N, 1] bool).  The returned tensors are the graph's static
    outputs: copy them if they must outlive the next step.  With per-stream sizes, frames is a
    list of the S streams' frames and each stream's tracks are in its own pixels.  With per-stream
    point counts, tracks and visibles are lists of the S streams' [N_s, 1, 2] and [N_s, 1] views
    into those outputs."""
    if self.query_features is None:
      raise RuntimeError('call init(frame, query_points) first')
    frames = self._frames(frames)
    if self._one_size:  # one copy of the batch (three for YUV planes)
      self._copy_in(frames, self._frame)
    else:
      for g in self._groups:
        for s, dst in zip(g.streams, g.sources):
          self._copy_in(frames[s], dst)
    self._upload_edits()
    if self._graph is not None and self._graph_sig != self.model._workspace_sig():
      self._graph = None  # stale pointers: the model's buffers or weights changed since capture
    if self._graph is None:
      self._capture()
    self._graph.replay()
    return self._out[0], self._out[1]

  def _upload_edits(self):
    """Copies the request tables that changed since the last step (the groups with pending edits,
    and the zero count of those that had some) from their pinned staging to the device."""
    for g in self._groups:
      if g.edits is None:
        continue
      reqs = [(g.offsets[i] + idx, i) + qp for i, s in enumerate(g.streams)
              for idx, qp in sorted(self._pending[s].items())]
      if not reqs and not g.edits.pending_on_device:
        continue
      e = g.edits
      e.uploaded.synchronize()  # the last upload has read the staging buffer
      _lib.write_query_requests(e.staging, reqs)
      n = 1 + _lib.REQUEST_WORDS * len(reqs)
      e.table[:n].copy_(e.staging[:n], non_blocking=True)
      e.uploaded.record()
      e.pending_on_device = bool(reqs)
    self._pending = [{} for _ in range(self.num_streams)]

  # -- point edits: each takes effect at the next step, sampled from that step's frame
  def _edit_stream(self, stream, what):
    if self.query_features is None:
      raise RuntimeError(f'{what}: call init(frame, query_points) first')
    if isinstance(stream, bool) or not isinstance(stream, int) or not 0 <= stream < self.num_streams:
      raise ValueError(f'{what}: stream {stream} out of range [0, {self.num_streams})')
    if what != 'retarget' and isinstance(self.num_points, int) and self.num_streams > 1:
      raise ValueError(f'{what}: a tracker of one point count for {self.num_streams} streams keeps '
                       'it; build it with num_points=[...] (one count per stream) to change counts')

  def _start_editing(self):
    """From the first edit on, every group's step applies its request table."""
    for g in self._groups:
      if g.edits is None:
        g.edits = _Edits(g, self.dev, self.model._const)
        self._graph = None

  def retarget(self, query_points, idx, stream: int = 0):
    """Re-targets points `idx` ([k] or an int) of stream `stream` at query_points ([k, 3] as
    (t, y, x) in that stream's pixels, as update_query takes them; with a one-frame clip t has no
    effect).  At the next step their features are sampled from that step's frame and their causal
    state is zeroed, inside the step (pytorch_live_demo.py:180-206 does both with a second
    backbone pass over the frame).  On a tracker whose step runs several streams through one
    backbone pass, the features come from that pass, so they can differ in the last bits from
    update_query's one-frame pass."""
    self._edit_stream(stream, 'retarget')
    pending = retarget_requests(self._pending[stream], self._counts[stream], idx, query_points)
    if pending:
      self._start_editing()
    self._pending[stream] = pending

  def add_points(self, query_points, stream: int = 0) -> List[int]:
    """Appends query_points ([k, 3], (t, y, x) in the stream's pixels) to stream `stream`'s
    points and returns their indices.  They are tracked from the next step on, their features
    sampled from that step's frame.  The next step captures the graph again."""
    self._edit_stream(stream, 'add_points')
    pending, count, new = add_requests(self._pending[stream], self._counts[stream], query_points)
    if new:
      self._resize(stream, list(range(self._counts[stream])), count)
      self._pending[stream] = pending
    return new

  def remove_points(self, idx, stream: int = 0):
    """Removes points `idx` of stream `stream`: the remaining points keep their order, and
    indices above a removed one shift down.  A stream keeps at least one point.  The next step
    captures the graph again."""
    self._edit_stream(stream, 'remove_points')
    pending, keep = remove_requests(self._pending[stream], self._counts[stream], idx)
    if len(keep) != self._counts[stream]:
      self._resize(stream, keep, len(keep))
      self._pending[stream] = pending

  def _resize(self, stream, keep, count):
    """Re-packs stream `stream`'s group for the stream's kept points `keep` (old indices, in
    order) followed by count - len(keep) new points: their query-feature rows hold zeros until
    the step samples them, their state rows zeros."""
    gi, slot = self._slot[stream]
    g = self._groups[gi]
    total = sum(g.counts)
    src = []  # each new row's old row, or `total` (a zero row) for a new point
    for i, (off, n) in enumerate(zip(g.offsets, g.counts)):
      if i == slot:
        src += [off + k for k in keep] + [total] * (count - len(keep))
      else:
        src += range(off, off + n)
    src = torch.tensor(src, device=self.dev)

    def repack(x):  # [1, total, ...] -> [1, new total, ...]
      return torch.cat([x[0], x.new_zeros(1, *x.shape[2:])]).index_select(0, src)[None]
    qf = g.query_features
    g.query_features = tapir_model.QueryFeatures(tuple(map(repack, qf.lowres)),
                                                 tuple(map(repack, qf.hires)), qf.resolutions)
    g.state = [{k: repack(v) for k, v in d.items()} for d in g.state]
    g.counts[slot] = count
    g.offsets = packed_offsets(g.counts)
    self._counts[stream] = count
    if isinstance(self.num_points, int):  # one stream: the count stays an int
      self.num_points = count
    else:
      self.num_points = list(self._counts)
    self._pack_rows()
    g.edits = None
    self._start_editing()  # a request table of the new size for this group
    self._publish()

  @property
  def last_logits(self):
    """(occlusion, expected_dist) logits of the last step, [S, N, 1] each (with per-stream point
    counts, lists of the S streams' [N_s, 1])."""
    return self._out[2], self._out[3]

  def update_query(self, frame: torch.Tensor, query_point: torch.Tensor, idx: int,
                   stream: int = 0):
    """Re-targets point `idx` of stream `stream` at (t, y, x) = query_point on `frame` ([H, W, 3],
    that stream's frame; pytorch_live_demo.py:188-200): its features are re-sampled and its causal
    state zeroed, in place (graph buffers stay valid).  Other streams are not touched.  It applies
    at once and cancels a pending retarget / add_points request of the point."""
    if self.query_features is None:
      raise RuntimeError('call init(frame, query_points) first')
    if not 0 <= stream < self.num_streams:
      raise ValueError(f'stream {stream} out of range [0, {self.num_streams})')
    n = self._counts[stream]
    if not 0 <= idx < n:
      raise ValueError(f'point {idx} out of range [0, {n}) of stream {stream}')
    frame = self._device_frame(self._stream_frames([frame], [stream])[0])
    new = self._query_features_one(frame, query_point.to(self.dev, torch.float32).reshape(1, 1, 3))
    gi, slot = self._slot[stream]
    g = self._groups[gi]
    row = g.offsets[slot] + idx  # the point's row in the group's packed point axis
    # TAPIR.update_query_features writes [:, idx] of every stream; only this row changes here
    for dst, src in zip(g.query_features.lowres + g.query_features.hires, new.lowres + new.hires):
      dst[0, row] = src[0, 0]
    for d in g.state:
      for v in d.values():
        v[0, row] = 0
    self._pending[stream].pop(idx, None)  # applied now: a pending request of the point is void
