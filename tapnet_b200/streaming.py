"""Streaming / online tracking with CUDA-graph replay (BASELINE.json config 3).

`tapnet/pytorch_live_demo.py:44-85` runs, per camera frame,
    feature_grids = model.get_feature_grids(frame)            (one frame)
    model.estimate_trajectories(..., causal_context=state, get_causal_context=True)
which is ~260 small kernel launches: at a few query points the GPU idles between launches
(3.7 ms/frame eager for 8 points).  `OnlineTracker` captures exactly that per-frame step once in
a CUDA graph (fixed frame size and point count) and replays it: same kernels, same results bit for
bit, no per-launch host cost.  The causal state lives in static device buffers that the graph
updates in place; `update_query` mirrors `TAPIR.update_query_features` for re-targeting a point.

With `num_streams=S` one tracker follows S camera streams (same frame size, same point count): a
step runs the backbone over the S frames in one pass and one batched estimate_trajectories over
the S clips of one frame each (the reference's batch axis), all in one captured graph.

With `yuv420=True` the tracker takes `live.YUV420Frames` (NV12 / I420 camera or decoder frames):
it keeps static Y / U / V buffers of the camera frame, a step copies the 1.5 B/px planes into them
and replays the graph, and the crop window and colour matrix are fixed at construction.
"""
from typing import Optional, Tuple

import torch

from tapnet_b200 import live
from tapnet_b200 import tapir_model


class OnlineTracker:
  """Graph-replayed per-frame step of a causal TAPIR model (`use_casual_conv=True`) over
  `num_streams` camera streams that share one frame size and one point count (pad a stream with
  dummy points if it tracks fewer)."""

  def __init__(self, model: 'tapir_model.TAPIR', height: int, width: int, num_points: int,
               uint8_frames: bool = False, num_streams: int = 1, yuv420: bool = False,
               window: Optional[Tuple[int, int, int, int]] = None, matrix: str = 'bt601',
               full_range: bool = False):
    """height x width: the frame size.  With yuv420=True that is the camera frame and `window`
    (y0, x0, h, w; e.g. `live.center_square_window(height, width)`) the crop that is tracked, in
    whose pixels the tracks are; `matrix` / `full_range` describe the YUV frames."""
    if not model.use_casual_conv:
      raise ValueError('OnlineTracker needs a causal model: TAPIR(use_casual_conv=True)')
    if int(num_streams) < 1:
      raise ValueError(f'num_streams must be >= 1, got {num_streams}')
    if yuv420 and uint8_frames:
      raise ValueError('uint8_frames and yuv420 are exclusive')
    if not yuv420 and window is not None:
      raise ValueError('window is only supported with yuv420=True')
    self.model = model
    self.hw = (int(height), int(width))
    self.num_points = int(num_points)
    self.num_streams = int(num_streams)
    self.dev = next(model.parameters()).device
    if self.dev.type != 'cuda':
      raise RuntimeError('OnlineTracker runs on CUDA only')
    # uint8_frames: frames are raw [0, 255] camera frames (what pytorch_live_demo.py:139-141 holds
    # before preprocess_frames); the normalisation runs inside the stem conv's loads
    self._frame_dtype = torch.uint8 if uint8_frames else torch.float32
    self._yuv = None
    if yuv420:
      H, W = self.hw
      ch, cw = (H + 1) // 2, (W + 1) // 2
      planes = [torch.zeros(self.num_streams, 1, *hw, dtype=torch.uint8, device=self.dev)
                for hw in ((H, W), (ch, cw), (ch, cw))]
      # the graph's input: static planes of the camera frame, fixed window and matrix
      self._yuv = live.YUV420Frames(*planes, matrix=matrix, full_range=full_range, window=window)
      self._frame = self._yuv
      self.hw = tuple(self._yuv.window[2:])
    else:
      self._frame = torch.zeros(self.num_streams, 1, height, width, 3, dtype=self._frame_dtype,
                                device=self.dev)
    self._graph: Optional[torch.cuda.CUDAGraph] = None
    self._graph_sig = None
    self._pinned = False
    self.query_features = None
    self.state = None
    self._out = None

  # -- pytorch_live_demo.py:44-54 online_model_init
  def init(self, frames: torch.Tensor, query_points: torch.Tensor):
    """frames: [S, H, W, 3] (or [S, 1, H, W, 3]; [H, W, 3] when S = 1) float in [-1, 1];
    query_points [S, N, 3] ([N, 3] when S = 1) as (t, y, x), stream s's on its frame s."""
    frame = self._as_frames(frames)
    qp = query_points.to(self.dev, torch.float32)
    if qp.dim() == 2:
      qp = qp[None]
    if qp.dim() != 3 or qp.shape[0] != self.num_streams or qp.shape[2] != 3:
      raise ValueError(f'query_points must be [{self.num_streams}, N, 3], got {tuple(qp.shape)}')
    if qp.shape[1] != self.num_points:
      raise ValueError(f'expected {self.num_points} query points, got {qp.shape[1]}')
    grids = self.model.get_feature_grids(frame, False)
    qf = self.model.get_query_features(frame, False, qp, grids)
    # private copies: the graph reads these exact buffers on every replay
    self.query_features = tapir_model.QueryFeatures(
        tuple(t.clone() for t in qf.lowres), tuple(t.clone() for t in qf.hires), qf.resolutions)
    n_res = len(qf.resolutions) - 1
    init = self.model.construct_initial_causal_state(self.num_points, n_res)
    # [S, N, 2, 512 | 2048] per block, one tensor per refinement iteration
    self.state = [{k: v.to(self.dev).expand(self.num_streams, *v.shape[1:]).clone()
                   for k, v in d.items()} for d in init]
    self._graph = None
    return self.query_features

  def _as_frames(self, frames, num=None):
    """[num, 1, H, W, 3] on the device from [num, H, W, 3], [num, 1, H, W, 3] or, for one
    frame, [H, W, 3].  YUV trackers: YUV420Frames [num, 1, ...] of the camera frame size, in the
    tracker's window and matrix, returned as they are."""
    num = self.num_streams if num is None else num
    if self._yuv is not None:
      return self._check_yuv(frames, num)
    frames = frames.to(self.dev, self._frame_dtype, non_blocking=True)
    if frames.dim() == 3:
      frames = frames[None, None]
    elif frames.dim() == 4:
      frames = frames[:, None]
    if frames.dim() != 5 or frames.shape[1] != 1 or frames.shape[4] != 3:
      raise ValueError(f'frames must be [S, H, W, 3], got {tuple(frames.shape)}')
    if frames.shape[0] != num:
      raise ValueError(f'expected {num} frames (one per stream), got {frames.shape[0]}')
    if tuple(frames.shape[2:4]) != self.hw:
      raise ValueError(f'frame size {tuple(frames.shape[2:4])} != {self.hw}')
    return frames

  def _check_yuv(self, frames, num):
    if not isinstance(frames, live.YUV420Frames):
      raise ValueError('this tracker was built with yuv420=True: pass live.YUV420Frames')
    ref = self._yuv
    if frames.frame_size != ref.frame_size:
      raise ValueError(f'frame size {frames.frame_size} != {ref.frame_size}')
    if (frames.window, frames.matrix, frames.full_range) != (ref.window, ref.matrix,
                                                             ref.full_range):
      raise ValueError(f'frames have window {frames.window}, {frames.matrix}, full_range='
                       f'{frames.full_range}; the tracker was built for {ref.window}, '
                       f'{ref.matrix}, full_range={ref.full_range}')
    if frames.device != self.dev:
      raise ValueError(f'frames on {frames.device}, tracker on {self.dev}')
    if tuple(frames.y.shape[:2]) != (num, 1):
      raise ValueError(f'expected YUV420Frames of [{num}, 1] frames, got '
                       f'{list(frames.y.shape[:2])}')
    return frames

  def _step_eager(self):
    # all streams in one backbone pass and one batched estimate_trajectories (B = S, T = 1)
    grids = self.model.get_feature_grids(self._frame, False)
    # single-frame step: the causal state is updated in place (causal_context_out = state)
    r = self.model.estimate_trajectories(self.hw, False, grids, self.query_features, None, 64,
                                         causal_context=self.state, get_causal_context=True,
                                         causal_context_out=self.state)
    tracks = r['tracks'][-1]
    occ, expd = r['occlusion'][-1], r['expected_dist'][-1]
    visibles = live.postprocess_occlusions(occ, expd)  # pytorch_live_demo.py:57-59
    return tracks, visibles, occ, expd

  def _capture(self):
    # warm-up on a side stream (allocates workspaces, packs weights, fills the constant cache);
    # the state is saved and restored so that warm-up steps do not advance it
    saved = [{k: v.clone() for k, v in d.items()} for d in self.state]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
      for _ in range(2):
        self._step_eager()
    torch.cuda.current_stream().wait_stream(s)
    for d, sv in zip(self.state, saved):
      for k in d:
        d[k].copy_(sv[k])
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      self._out = self._step_eager()
    for d, sv in zip(self.state, saved):  # capture does not execute, but be explicit
      for k in d:
        d[k].copy_(sv[k])
    self._graph = g
    # The graph holds RAW pointers into the model's workspaces and packed weight planes.  Pin
    # the workspaces (TAPIR._workspace then parks outgrown buffers instead of freeing them) and
    # remember which buffers / weights the capture saw: step() re-captures when another caller
    # of the same model (a larger offline clip, a second tracker, load_state_dict) replaced them.
    if not self._pinned:
      self.model._ws_pins += 1
      self._pinned = True
    self._graph_sig = self._model_sig()

  def _model_sig(self):
    return (self.model._ws_generation, self.model._param_sig())

  def close(self):
    """Drops the graph and releases the workspace pin."""
    self._graph = None
    if self._pinned:
      self.model._ws_pins -= 1
      self._pinned = False
      if self.model._ws_pins == 0:
        self.model._ws_retired.clear()

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint: disable=broad-except
      pass

  # -- pytorch_live_demo.py:62-85 online_model_predict
  def step(self, frames: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """frames: [S, H, W, 3] ([H, W, 3] when S = 1), one per stream.  Returns (tracks [S, N, 1, 2]
    in frame pixels (x, y), visibles [S, N, 1] bool).  The returned tensors are the graph's static
    outputs: copy them if they must outlive the next step."""
    if self.query_features is None:
      raise RuntimeError('call init(frame, query_points) first')
    if self._yuv is not None:
      src = self._as_frames(frames)
      for dst, plane in zip((self._yuv.y, self._yuv.u, self._yuv.v), (src.y, src.u, src.v)):
        dst.copy_(plane)
    else:
      self._frame.copy_(self._as_frames(frames))
    if self._graph is not None and self._graph_sig != self._model_sig():
      self._graph = None  # stale pointers: the model's buffers or weights changed since capture
    if self._graph is None:
      self._capture()
    self._graph.replay()
    return self._out[0], self._out[1]

  @property
  def last_logits(self):
    """(occlusion, expected_dist) logits of the last step, [S, N, 1] each."""
    return self._out[2], self._out[3]

  def update_query(self, frame: torch.Tensor, query_point: torch.Tensor, idx: int,
                   stream: int = 0):
    """Re-targets point `idx` of stream `stream` at (t, y, x) = query_point on `frame` ([H, W, 3],
    that stream's frame; pytorch_live_demo.py:188-200): its features are re-sampled and its causal
    state zeroed, in place (graph buffers stay valid).  Other streams are not touched."""
    if self.query_features is None:
      raise RuntimeError('call init(frame, query_points) first')
    if not 0 <= stream < self.num_streams:
      raise ValueError(f'stream {stream} out of range [0, {self.num_streams})')
    if not 0 <= idx < self.num_points:
      raise ValueError(f'point {idx} out of range [0, {self.num_points})')
    frame = self._as_frames(frame, num=1)
    qp = query_point.to(self.dev, torch.float32).reshape(1, 1, 3)
    grids = self.model.get_feature_grids(frame, False)
    new = self.model.get_query_features(frame, False, qp, grids)
    # TAPIR.update_query_features writes [:, idx] of every stream; only [stream, idx] changes here
    for dst, src in zip(self.query_features.lowres + self.query_features.hires,
                        new.lowres + new.hires):
      dst[stream, idx] = src[0, 0]
    for d in self.state:
      for v in d.values():
        v[stream, idx] = 0
