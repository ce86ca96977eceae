"""H100-native TAPIR / BootsTAPIR inference behind the reference's Python surface.

Mirrors `tapnet/torch/tapir_model.py` (reference, 806 LoC): same constructor keywords
(incl. the `use_casual_conv` spelling, :73-89), same methods and argument meaning
(`forward` :139, `get_query_features` :217, `get_feature_grids` :293,
`estimate_trajectories` :394, `construct_initial_causal_state` :763,
`update_query_features` :774), same `FeatureGrids` / `QueryFeatures` tuples (:30-67), same
state-dict keys (218 tensors, `tapnet_b200/schema.py`), same errors.  Underneath, every stage is
a hand-written sm_90a kernel reached through the C ABI of `libtapir_b200.so`
(`include/tapir_b200.h`); PyTorch is used for device memory, streams and (multi-GPU)
`torch.distributed` only.  There is no CPU or eager-PyTorch fallback: tensors must live on a
CUDA device and the shared library must be built, otherwise the calls raise.
"""
import math
from typing import Any, List, Mapping, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import nn

from tapnet_b200 import _lib
from tapnet_b200 import live
from tapnet_b200 import schema


class FeatureGrids(NamedTuple):
  """Per-frame feature grids (reference tapir_model.py:30-45).

  lowres: one [B, T, h/8, w/8, 256] tensor per resolution; hires: [B, T, h/4, w/4, 128];
  resolutions: (h, w) used for each entry (first = TAP-Net initialisation).
  """
  lowres: Sequence[torch.Tensor]
  hires: Sequence[torch.Tensor]
  resolutions: Sequence[Tuple[int, int]]


class QueryFeatures(NamedTuple):
  """Per-query features (reference tapir_model.py:48-67): lowres [B,N,256], hires [B,N,128]."""
  lowres: Sequence[torch.Tensor]
  hires: Sequence[torch.Tensor]
  resolutions: Sequence[Tuple[int, int]]


def generate_default_resolutions(full_size, train_size, num_levels=None):
  """Log-spaced refinement resolutions, multiples of 8 (reference utils.py:275-317)."""
  full_size = tuple(int(v) for v in full_size)
  train_size = tuple(int(v) for v in train_size)
  if all(x == y for x, y in zip(train_size, full_size)):
    return [train_size]
  if num_levels is None:
    size_ratio = np.array(full_size) / np.array(train_size)
    num_levels = int(np.ceil(np.max(np.log2(size_ratio))) + 1)
  if num_levels <= 1:
    return [train_size]
  h, w = full_size[0:2]
  if h % 8 != 0 or w % 8 != 0:
    print('Warning: output size is not a multiple of 8. Final layer will round size down.')
  ll_h, ll_w = train_size[0:2]
  sizes = []
  for i in range(num_levels):
    e = i / (num_levels - 1)
    sizes.append((int(round((ll_h * (h / ll_h) ** e) // 8)) * 8,
                  int(round((ll_w * (w / ll_w) ** e) // 8)) * 8))
  return sizes


def _is_same_res(r1, r2):
  return all(int(x) == int(y) for x, y in zip(r1, r2))


class PassStep(NamedTuple):
  """What get_feature_grids does for one required resolution: `new` starts a backbone pass of
  h x w frames that reads the video itself (`direct`) or its bilinear resample; otherwise the
  level reuses the previous pass's grids."""
  h: int
  w: int
  direct: bool
  new: bool


def _pass_plan(video_hw, initial_resolution, refinement_resolutions=None):
  """The backbone passes of get_feature_grids on a video_hw video (reference tapir_model.py:
  330-360), one PassStep per required resolution (the initial one first); the refinement
  resolutions default to generate_default_resolutions of the video size.  Two videos with the
  same plan have feature grids of the same shapes; a direct-read pass's size is the video's."""
  vh, vw = int(video_hw[0]), int(video_hw[1])
  if refinement_resolutions is None:
    refinement_resolutions = generate_default_resolutions((vh, vw), initial_resolution)
  all_required = [tuple(initial_resolution)] + [tuple(r) for r in refinement_resolutions]
  if any(r[0] % 8 != 0 or r[1] % 8 != 0 for r in all_required):
    raise ValueError('Image resolution must be a multiple of 8.')
  plan = []
  curr_resolution = (-1, -1)
  for resolution in all_required:
    if not _is_same_res(curr_resolution, resolution):
      # reference quirk (:337): the PREVIOUS resolution is compared with the video size
      if _is_same_res(curr_resolution, (vh, vw)):
        h, w = vh, vw
      else:
        h, w = int(resolution[0]), int(resolution[1])
      curr_resolution = resolution
      # align_corners=False resize to the same size is the identity: the pass reads the video
      plan.append(PassStep(h, w, (h, w) == (vh, vw), True))
    else:
      plan.append(plan[-1]._replace(new=False))
  return plan


def _per_clip_sizes(video_size):
  """None for one (h, w); else the list of per-clip (h, w) pairs."""
  if len(video_size) and isinstance(video_size[0], (tuple, list, torch.Size)):
    return [(int(h), int(w)) for h, w in video_size]
  if isinstance(video_size, torch.Tensor) and video_size.dim() == 2:
    return [(int(h), int(w)) for h, w in video_size.tolist()]
  return None


_PRECISIONS = {'bf16': 1, 'bf16x3': 2, 'bf16x6': 3}

# rows (= queries x frames) processed per mixer pass; bounds the workspace to ~1.5 GB
_MAX_ROWS_PER_CHUNK = 98304
# input pixels (frames x H x W) per backbone pass; bounds the workspace to ~2.7 GB
_MAX_BACKBONE_PIXELS = 96 * 256 * 256
# host clips: H2D sub-chunks per backbone pass (each followed by its stem-conv launch)
_H2D_SUBCHUNKS = 6


def _backbone_chunk(h, w, frames):
  """Frames per chunk of a backbone pass over `frames` frames of h x w: it bounds the workspace, as
  the reference's feature_extractor_chunk_size (:346-360) does, and decides bits, as the ExtraConv
  GEMMs split K (and so sum in another order) for one-frame chunks only."""
  return min(max(1, _MAX_BACKBONE_PIXELS // (h * w)), frames)


def _grid_shapes(h, w):
  """Per-frame shapes of the (lowres, hires) feature grids of an h x w backbone pass."""
  return (h // 8, w // 8, schema.LOWRES_DIM), (h // 4, w // 4, schema.HIRES_DIM)


def _backbone_frames(video):
  """A clip as the backbone reads it: contiguous, uint8 kept, any other dtype as float32."""
  return video.contiguous() if video.dtype == torch.uint8 else video.to(torch.float32).contiguous()


def _stage_a_scratch(G, nq, T, grid_shape):
  """Stage A of G clips with nq queries in all, T frames of grid_shape lowres grids: the shapes of
  its float32 occlusion, expected distance, tracks, positions and positions scaled on their way to
  the tracks, and the bytes of its cost-volume workspace."""
  return (((nq, T),) * 2 + ((nq, T, 2),) * 3,
          _lib.cost_volume_ragged_workspace_bytes(G, nq, (G, T, *grid_shape)))


def _new_estimates(count, shape, dev):
  """`count` estimates of queries over T frames as three lists: occlusion and expected distance of
  `shape` (the query dims, then T) and tracks of shape + (2,)."""
  return tuple([torch.empty(s, dtype=torch.float32, device=dev) for _ in range(count)]
               for s in (shape, shape, (*shape, 2)))


def _work_groups(counts, T):
  """Work groups of estimate_trajectories over clips of counts[b] queries, as (b0, b1, q0, q1):
  whole clips b0..b1-1, flattened queries q0..q1-1, while the group's rows (queries x frames) fit
  _MAX_ROWS_PER_CHUNK and its queries one head / mixer launch (65535); a clip whose rows alone
  exceed the bound runs on its own in query chunks.  Each group is one launch sequence over its
  clips.  The groups decide bits: the mixer splits K at T = 1 by row count."""
  out = []
  b0 = q0 = q = 0
  for b, n in enumerate(counts):
    if n * T > _MAX_ROWS_PER_CHUNK or n > 65535:
      if b > b0:
        out.append((b0, b, q0, q))
      chunk_q = max(1, min(n, _MAX_ROWS_PER_CHUNK // T, 65535))
      out += [(b, b + 1, q + c0, q + min(c0 + chunk_q, n)) for c0 in range(0, n, chunk_q)]
      b0, q0 = b + 1, q + n
    elif b > b0 and ((q + n - q0) * T > _MAX_ROWS_PER_CHUNK or q + n - q0 > 65535):
      out.append((b0, b, q0, q))
      b0, q0 = b, q
    q += n
  if len(counts) > b0:
    out.append((b0, len(counts), q0, q))
  return out


def _query_rows(t, q0, q1):
  """Queries q0..q1-1 of t [B, N, ...], counted along its flattened (B, N) point axis: whole clips
  or a range within one clip, as a work group holds them.  One index per tensor, as a group reads
  2 x num_blocks context tensors per iteration and each op costs host time on the online step."""
  n = t.shape[1]
  b, r = divmod(q0, n)
  if r == 0 and (q1 - q0) % n == 0:
    return t[b:b + (q1 - q0) // n]
  return t[b, r:r + q1 - q0]


def _ctx_lists(d, nb, q0, q1, fix=lambda t: t):
  """Queries q0..q1-1 of one iteration's causal context dict as two per-block lists (causal_1,
  causal_2), each passed through `fix`."""
  return ([fix(_query_rows(d[f'block_{i}_causal_1'], q0, q1)) for i in range(nb)],
          [fix(_query_rows(d[f'block_{i}_causal_2'], q0, q1)) for i in range(nb)])


def refined_average(trajectories, num_pips_iter):
  """occlusion / tracks / expected_dist averaged over the estimates that end each refinement
  level, as the reference's forward returns them (tapir_model.py:203-210)."""
  p = num_pips_iter
  return {k: torch.mean(torch.stack(trajectories[k][p::p]), dim=0)
          for k in ('occlusion', 'tracks', 'expected_dist')}


def _on_model_device(fn):
  """Runs a TAPIR method with the model's CUDA device current.  Kernels launch on the current
  device and the C library keeps per-device state (shared-memory attributes, error flag), so
  `build_model(device='cuda:1')` must work without the caller calling torch.cuda.set_device
  (the reference runs on whatever device its tensors live on)."""
  import functools  # pylint: disable=g-import-not-at-top

  @functools.wraps(fn)
  def wrapper(self, *args, **kwargs):
    dev = next(self.parameters()).device
    if dev.type != 'cuda':
      # argument errors are reported in the reference's order; _device_check then raises
      return fn(self, *args, **kwargs)
    with torch.cuda.device(dev):
      return fn(self, *args, **kwargs)
  return wrapper


class TAPIR(nn.Module):
  """TAPIR model (H100 engine).  See the module docstring.

  Extra keyword (not in the reference): `precision` selects the tensor-core arithmetic of the
  dense contractions: 'bf16x3' (default; operands split in two bf16 terms, 3 MMAs, ~16
  mantissa bits, meets the 1e-3 px / 1e-4 logit parity budget), 'bf16x6' (three terms, 6
  MMAs, fp32-equivalent) or 'bf16' (single pass; does NOT meet the parity budget).
  """

  def __init__(
      self,
      bilinear_interp_with_depthwise_conv: bool = False,
      num_pips_iter: int = 4,
      pyramid_level: int = 1,
      mixer_hidden_dim: int = 512,
      num_mixer_blocks: int = 12,
      mixer_kernel_shape: int = 3,
      patch_size: int = 7,
      softmax_temperature: float = 20.0,
      parallelize_query_extraction: bool = False,
      initial_resolution: Tuple[int, int] = (256, 256),
      blocks_per_group: Sequence[int] = (2, 2, 2, 2),
      feature_extractor_chunk_size: int = 10,
      extra_convs: bool = True,
      use_casual_conv: bool = False,
      precision: str = 'bf16x3',
  ):
    super().__init__()
    if precision not in _PRECISIONS:
      raise ValueError(f'precision must be one of {sorted(_PRECISIONS)}')
    self.highres_dim = schema.HIRES_DIM
    self.lowres_dim = schema.LOWRES_DIM
    # stored-but-unused arguments, exactly like the reference (SURVEY.md A.2 quirk 1)
    self.bilinear_interp_with_depthwise_conv = bilinear_interp_with_depthwise_conv
    self.parallelize_query_extraction = parallelize_query_extraction
    self.num_pips_iter = num_pips_iter
    self.pyramid_level = pyramid_level
    self.patch_size = patch_size
    self.softmax_temperature = softmax_temperature
    self.initial_resolution = tuple(initial_resolution)
    self.feature_extractor_chunk_size = feature_extractor_chunk_size
    self.num_mixer_blocks = num_mixer_blocks
    self.use_casual_conv = use_casual_conv
    self.precision = precision
    self._planes = _PRECISIONS[precision]
    self._has_extra = bool(extra_convs)
    if pyramid_level not in (0, 1, 2, 3):
      raise NotImplementedError('pyramid_level must be 0..3 (2 to 5 correlation levels)')

    # Parameters: same names / shapes / order as the reference state dict.
    for key, shape in schema.state_dict_schema(pyramid_level, extra_convs).items():
      self._register(key, self._init_param(key, shape))
    self.extra_convs = self._modules.get('extra_convs', None)
    self._packed = None
    self._packed_sig = None
    self._plist = None
    self._ws = {}
    self._copy_streams = {}
    self._ws_retired = []
    self._ws_pins = 0
    self._ws_generation = 0
    self._consts = {}
    # tests / diagnostics: when True, estimate_trajectories keeps the stage-A arg-max cell of
    # every (query, frame) heat map in `last_stage_a_argmax` ([B, N, T] int32)
    self.capture_stage_a_argmax = False
    self.last_stage_a_argmax = None

  # ------------------------------------------------------------------ parameter plumbing
  def _register(self, key, tensor):
    parts = key.split('.')
    mod = self
    for p in parts[:-1]:
      if p not in mod._modules:
        mod.add_module(p, nn.Module())
      mod = mod._modules[p]
    mod.register_parameter(parts[-1], nn.Parameter(tensor, requires_grad=False))

  @staticmethod
  def _init_param(key, shape):
    is_norm = ('bn_' in key) or ('layer_norm' in key)
    if is_norm:
      return torch.ones(shape) if key.endswith('weight') else torch.zeros(shape)
    wshape = shape if key.endswith('weight') else None
    if wshape is None:
      return torch.zeros(shape)
    fan_in = int(np.prod(shape[1:]))
    bound = 1.0 / math.sqrt(fan_in)
    return (torch.rand(shape) * 2 - 1) * bound

  def _param_sig(self):
    # the module tree is fixed after construction: walk it once (the walk costs ~0.2 ms of host
    # time per call, on the latency path of every public method); `.to()` / `.cuda()` swap the
    # Parameter's .data, which data_ptr() below notices, in-place updates bump _version
    ps = self._plist
    if ps is None:
      ps = self._plist = list(self.parameters())
    return (str(ps[0].device), ps[0].data_ptr(), ps[-1].data_ptr(), sum(p._version for p in ps),
            self._planes)

  def _device_check(self, *tensors):
    dev = next(self.parameters()).device
    if dev.type != 'cuda':
      raise RuntimeError('tapnet_b200.TAPIR runs on CUDA only (no CPU fallback): call '
                         'model.to("cuda") first.')
    for t in tensors:
      if t is not None and t.device != dev:
        raise RuntimeError(f'tensor on {t.device}, model on {dev}')
    return dev

  def _copy_stream(self, dev):
    key = str(dev)
    if key not in self._copy_streams:
      self._copy_streams[key] = torch.cuda.Stream(device=dev)
    return self._copy_streams[key]

  def _const(self, values, dev, dtype=torch.float32):
    """Small constant vectors, cached: creating them per call costs a blocking H2D copy."""
    key = (tuple(float(v) for v in values), str(dev), dtype)
    t = self._consts.get(key)
    if t is None:
      t = torch.tensor(key[0], dtype=dtype, device=dev)
      self._consts[key] = t
    return t

  def _workspace(self, name, nbytes, dev):
    """Grow-only scratch.  A buffer that is outgrown is parked in `_ws_retired` instead of
    being freed while pinned: a captured CUDA graph (streaming.OnlineTracker) holds raw pointers
    into it.  `_ws_generation` changes whenever a buffer is replaced, so graph owners can tell
    (_workspace_sig) that their capture no longer describes the model's current buffers."""
    ws = self._ws.get(name)
    if ws is None or ws.numel() < nbytes or ws.device != dev:
      if ws is not None and self._ws_pins > 0:
        self._ws_retired.append(ws)
      ws = torch.empty(int(nbytes), dtype=torch.uint8, device=dev)
      self._ws[name] = ws
      self._ws_generation += 1
    return ws

  def _pin_workspaces(self):
    """Taken by a captured graph's holder: while pinned, outgrown workspaces are parked."""
    self._ws_pins += 1

  def _unpin_workspaces(self):
    """Releases one pin; the last pin to go frees the parked workspaces."""
    self._ws_pins -= 1
    if self._ws_pins == 0:
      self._ws_retired.clear()

  def _workspace_sig(self):
    """What a captured graph's raw pointers depend on: the workspaces and the packed weights."""
    return self._ws_generation, self._param_sig()

  # ------------------------------------------------------------------ weight packing
  @_on_model_device
  def _pack(self):
    sig = self._param_sig()
    if self._packed is not None and self._packed_sig == sig:
      return self._packed
    sd = {k: v.detach() for k, v in self.state_dict().items()}
    self._packed = _lib.pack_weights(sd, self._planes, self._has_extra,
                                     next(self.parameters()).device)
    self._packed_sig = sig
    return self._packed

  # ------------------------------------------------------------------ public API
  def forward(
      self,
      video: torch.Tensor,
      query_points: torch.Tensor,
      is_training: bool = False,
      query_chunk_size: Optional[int] = 64,
      get_query_feats: bool = False,
      refinement_resolutions: Optional[List[Tuple[int, int]]] = None,
  ) -> Mapping[str, torch.Tensor]:
    """Reference tapir_model.py:139-215."""
    if get_query_feats:
      raise ValueError('Get query feats not supported in TAPIR.')
    pdev = next(self.parameters()).device
    if pdev.type == 'cuda' and video.device.type == 'cpu' and query_points.device.type == 'cpu':
      # host buffers in (extension): the clip is streamed in by get_feature_grids
      query_points = query_points.to(pdev, non_blocking=True)
    feature_grids = self.get_feature_grids(video, is_training, refinement_resolutions)
    query_features = self.get_query_features(video, is_training, query_points, feature_grids,
                                             refinement_resolutions)
    trajectories = self.estimate_trajectories(video.shape[-3:-1], is_training, feature_grids,
                                              query_features, query_points, query_chunk_size)
    return dict(
        **refined_average(trajectories, self.num_pips_iter),
        unrefined_occlusion=trajectories['occlusion'][:-1],
        unrefined_tracks=trajectories['tracks'][:-1],
        unrefined_expected_dist=trajectories['expected_dist'][:-1],
    )

  @_on_model_device
  def get_feature_grids(
      self,
      video: torch.Tensor,
      is_training: bool,
      refinement_resolutions: Optional[List[Tuple[int, int]]] = None,
      hires_ready_events: Optional[list] = None,
  ) -> FeatureGrids:
    """Reference tapir_model.py:293-392.  video: [B, T, H, W, 3] float in [-1, 1] (or uint8
    [0, 255], or a device-resident `live.YUVFrames` clip whose crop window is the video).

    `hires_ready_events` (extension, used by tapnet_b200.distributed): a list that receives one
    (hires tensor, torch.cuda.Event) pair per distinct resolution; the event fires as soon as
    that hires grid is final, while ResNet groups 2-3 and the ExtraConvs are still running."""
    del is_training
    plan = _pass_plan(video.shape[2:4], self.initial_resolution, refinement_resolutions)
    # A HOST clip (ideally pinned) is accepted too (extension): its frames are copied to the
    # device in chunks on a copy stream and the stem convolution - the only reader of the video -
    # runs chunk by chunk behind them, so PCIe time hides behind compute.
    host_video = video.device.type == 'cpu'
    dev = self._device_check(None if host_video else video)
    pk = self._pack()
    # uint8 video = raw [0,255] frames (what the reference's callers hold before
    # preprocess_frames, pytorch_live_demo.py:30-41): normalised inside the stem conv's loads
    # (or inside the resize), so the 4x larger float video never exists.  Extension of the
    # reference surface; float video behaves exactly as before.
    # YUV frames (extension): at the frame's own size the stem conv converts inside its
    # loads; a resized pass converts each bilinear tap in the ingest kernel.  Bit for bit the
    # results of the uint8 RGB frames the conversion produces.
    if not isinstance(video, live.YUVFrames):
      video = _backbone_frames(video)
    n, f, vh, vw, _ = video.shape
    host_src = None
    if host_video:
      host_src = video
      video = torch.empty(video.shape, dtype=video.dtype, device=dev)
      if not plan[0].direct:
        # the first pass resizes the clip: it needs all of it on the device up front
        video.copy_(host_src, non_blocking=True)
        host_src = None
    feature_grid, hires_feats, resize_im_shape = [], [], []
    latent = hires = None
    for h, w, direct, new_pass in plan:
      if new_pass:
        frames = video
        if not direct:
          frames = torch.empty(n, f, h, w, 3, dtype=torch.float32, device=dev)
          _lib.resample_frames(video, frames)
        latent, hires = self._backbone_pass(pk, frames, host_src if frames is video else None,
                                            hires_ready_events, dev)
        if frames is video:
          host_src = None  # the whole clip is on the device now (later passes resize from it)
      feature_grid.append(latent)
      hires_feats.append(hires)
      resize_im_shape.append(torch.Size((h, w)))
    return FeatureGrids(tuple(feature_grid), tuple(hires_feats), tuple(resize_im_shape))

  def _feature_grids_of_frames(self, frames, plan):
    """get_feature_grids of a batch of one-frame clips of different sizes or formats that share
    `plan` (no direct-read pass): frames is a list of [H, W, 3] tensors (float32 in [-1, 1] or
    uint8) or one-frame YUV clips.  Each pass resamples uint8 and YUV frames in one ingest launch;
    float32 frames keep one tapir_bilinear_resize launch each (the multi-frame ingest cannot
    reproduce its rounding bit for bit)."""
    dev = self._device_check(*(None if isinstance(x, live.YUVFrames) else x for x in frames))
    pk = self._pack()
    feature_grid, hires_feats, resize_im_shape = [], [], []
    latent = hires = None
    for h, w, direct, new_pass in plan:
      if direct:
        raise ValueError('_feature_grids_of_frames: a direct-read pass needs frames of one size')
      if new_pass:
        batch = torch.empty(len(frames), 1, h, w, 3, dtype=torch.float32, device=dev)
        if any(isinstance(x, torch.Tensor) and x.dtype == torch.float32 for x in frames):
          for x, out in zip(frames, batch):
            _lib.resample_frames(x[None], out)
        else:
          _lib.ingest_frames_multi(frames, batch.view(len(frames), h, w, 3))
        latent, hires = self._backbone_pass(pk, batch, None, None, dev)
      feature_grid.append(latent)
      hires_feats.append(hires)
      resize_im_shape.append(torch.Size((h, w)))
    return FeatureGrids(tuple(feature_grid), tuple(hires_feats), tuple(resize_im_shape))

  def _backbone_pass(self, pk, frames, host_src, hires_ready_events, dev, out=None):
    """Feature grids (lowres, hires) of every frame of `frames` ([B, T, h, w, 3] on the device, or
    a YUV clip).  host_src: the host clip whose copy `frames` is yet to be, streamed in here.
    out: None, or the contiguous (lowres, hires) tensors to write the grids into."""
    n, f, h, w, _ = frames.shape
    nf = n * f
    shapes = [(n, f) + s for s in _grid_shapes(h, w)]
    if out is None:
      out = [torch.empty(s, dtype=torch.float32, device=dev) for s in shapes]
    else:
      for name, t, shape in zip(('lowres', 'hires'), out, shapes):
        if (t.shape != shape or t.dtype != torch.float32 or t.device != dev
            or not t.is_contiguous()):
          raise ValueError(f'grids_out {name} must be a contiguous float32 {list(shape)} tensor '
                           f'on {dev}, got {t.dtype} {tuple(t.shape)} on {t.device}')
    latent, hires = out
    src = frames if isinstance(frames, live.YUVFrames) else frames.view(nf, h, w, 3)
    flat_lo, flat_hi = (t.view(nf, *s[2:]) for t, s in zip(out, shapes))
    chunk = _backbone_chunk(h, w, nf)
    ws = self._workspace('backbone', self._backbone_workspace_bytes(nf, h, w), dev)
    ev = None
    if hires_ready_events is not None:
      ev = torch.cuda.Event()
      ev.record(torch.cuda.current_stream(dev))  # materialises the CUDA event handle
      hires_ready_events.append((hires, ev))
    streamed = host_src is not None
    if streamed:
      main = torch.cuda.current_stream(dev)
      cs = self._copy_stream(dev)
      cs.wait_stream(main)  # the staging buffer's previous owner is done
      host_flat = host_src.view(nf, h, w, 3)
    for s0 in range(0, nf, chunk):
      c = min(chunk, nf - s0)
      if streamed:
        # sub-chunks of >= ~4 MB (each costs ~70 us of host time: copy, event, stem launch),
        # at most _H2D_SUBCHUNKS per pass
        nsub = max(1, min(_H2D_SUBCHUNKS, (c * h * w * 3 * src.element_size()) >> 22))
        sub = max(1, -(-c // nsub))
        for a in range(s0, s0 + c, sub):
          b = min(a + sub, s0 + c)
          with torch.cuda.stream(cs):
            src[a:b].copy_(host_flat[a:b], non_blocking=True)
            arrived = torch.cuda.Event()
            arrived.record(cs)
          main.wait_event(arrived)
          _lib.backbone_stem(pk['backbone'], src[a:b], c, a - s0, ws)
      _lib.backbone_forward(pk['backbone'], src, flat_lo[s0:s0 + c], flat_hi[s0:s0 + c], ws,
                            ev if s0 + c >= nf else None, frame0=s0, stem_done=streamed)
    return latent, hires

  def _backbone_workspace_bytes(self, frames, h, w):
    """Workspace bytes of a backbone pass over `frames` frames of h x w."""
    return _lib.backbone_workspace_bytes(_backbone_chunk(h, w, frames), h, w, self._has_extra,
                                         self._planes)

  @_on_model_device
  def get_query_features(
      self,
      video: torch.Tensor,
      is_training: bool,
      query_points: torch.Tensor,
      feature_grids: Optional[FeatureGrids] = None,
      refinement_resolutions: Optional[List[Tuple[int, int]]] = None,
  ) -> QueryFeatures:
    """Reference tapir_model.py:217-291.  query_points: [B, N, 3] as (t, y, x)."""
    if feature_grids is None:
      feature_grids = self.get_feature_grids(video, is_training, refinement_resolutions)
    dev = self._device_check(query_points)
    qp = query_points.to(torch.float32).contiguous()
    b, nq, _ = qp.shape
    query_feats, hires_query_feats = [], []
    cache = {}
    for i, _ in enumerate(feature_grids.resolutions):
      lo_grid, hi_grid = feature_grids.lowres[i], feature_grids.hires[i]
      key = (lo_grid.data_ptr(), hi_grid.data_ptr())
      if key not in cache:  # identical grids give identical features (reference recomputes)
        outs = []
        for grid in (lo_grid, hi_grid):
          grid = grid.contiguous()
          out = torch.empty(b, nq, grid.shape[-1], dtype=torch.float32, device=dev)
          for bi in range(b if nq > 0 else 0):
            _lib.sample_query_features(grid[bi], qp[bi], video.shape[1:4], out[bi])
          outs.append(out)
        cache[key] = outs
      query_feats.append(cache[key][0])
      hires_query_feats.append(cache[key][1])
    return QueryFeatures(tuple(query_feats), tuple(hires_query_feats),
                         tuple(feature_grids.resolutions))

  @_on_model_device
  def estimate_trajectories(
      self,
      video_size: Tuple[int, int],
      is_training: bool,
      feature_grids: FeatureGrids,
      query_features: QueryFeatures,
      query_points_in_video: Optional[torch.Tensor],
      query_chunk_size: Optional[int] = None,
      causal_context: Optional[list] = None,
      get_causal_context: bool = False,
      causal_context_out: Optional[list] = None,
      points_per_clip: Optional[Sequence[int]] = None,
  ) -> Mapping[str, Any]:
    """Reference tapir_model.py:394-578.

    `points_per_clip` (extension): None, or the query counts of the B clips of feature_grids, each
    >= 1.  query_features, query_points_in_video and the causal context then hold the clips'
    queries one clip after the other along the point axis ([1, sum N, ...]; the context
    [1, sum N, 2, 512 | 2048]) and so do the outputs ([1, sum N, T, ...]).  Each clip's results
    equal a single-clip call with its queries, bit for bit, at T > 1.

    `video_size` (extension): one (h, w) for every clip, or a sequence of B (h, w) pairs, clip b's
    tracks (and query points) then being in its own video's pixels; each clip's results equal a
    single-clip call with its size, bit for bit.

    `causal_context_out` (extension, optional): list of dicts of preallocated [B, N, 2, 512|2048]
    tensors that receive the new causal context instead of fresh allocations.  For single-frame
    steps (T == 1, the streaming case) it may be `causal_context` itself: the state is then
    updated in place, which saves a 1 GB copy per frame at 1024 points.

    `query_chunk_size` only bounds memory in the reference (queries are independent,
    SURVEY.md 2.2); here chunks are sized by rows (queries x frames) to keep all 132 SMs busy
    and the argument is accepted for compatibility.  No query shuffling is done (the
    reference's randperm only changes chunk membership).
    """
    del is_training, query_chunk_size
    dev = self._device_check(query_features.lowres[0])
    pk = self._pack()
    per_clip = _per_clip_sizes(video_size)
    video_hw = None if per_clip is not None else (int(video_size[0]), int(video_size[1]))
    num_levels_total = len(feature_grids.lowres)
    num_iters = self.num_pips_iter * (num_levels_total - 1)
    B, N = query_features.lowres[0].shape[:2]  # [1, sum N] with points_per_clip
    T = feature_grids.lowres[0].shape[1]
    nb = pk['num_blocks']
    if points_per_clip is None:
      counts = [N] * B
    else:
      counts = self._check_points_per_clip(points_per_clip, feature_grids, query_features,
                                           query_points_in_video)
    video_table = None
    if per_clip is not None:
      if len(per_clip) != len(counts):
        raise ValueError(f'video_size has {len(per_clip)} (h, w) pairs for {len(counts)} clips')
      # [clips, 2] (h, w): the track update's table
      video_table = self._const([v for hw in per_clip for v in hw], dev,
                                torch.int32).view(len(counts), 2)

    occ_out, expd_out, trk_out = _new_estimates(num_iters + 1, (B, N, T), dev)
    new_ctx = self._new_causal_context(causal_context, get_causal_context, causal_context_out,
                                       num_iters, nb, B, N, T, dev)
    write_ctx = get_causal_context and causal_context is not None
    am_out = None
    if self.capture_stage_a_argmax:
      am_out = torch.empty(B, N, T, dtype=torch.int32, device=dev)
      self.last_stage_a_argmax = am_out
    out = dict(occlusion=occ_out, tracks=trk_out, expected_dist=expd_out)
    if get_causal_context:
      out['causal_context'] = new_ctx
    if N == 0 or T == 0:
      # nothing to track (the reference fails in torch.cat on an empty chunk list,
      # tapir_model.py:556-559; returning correctly shaped empty tensors is the useful behaviour)
      return out

    # pooled pyramid levels: once per resolution level over all B*T frames (the reference
    # recomputes them every iteration of every chunk, tapir_model.py:519-527)
    pooled = {level: self._pool_pyramid(feature_grids.lowres[level].contiguous())
              for level in range(1, num_levels_total)}

    for b0, b1, q0, q1 in _work_groups(counts, T):
      bs = slice(b0, b1)
      gcounts = [q1 - q0] if b1 - b0 == 1 else counts[b0:b1]
      query_clip = None
      if len(set(gcounts)) > 1:
        # [nq] int32 clip (within the group) of each query: cached, so a captured step uploads nothing
        query_clip = self._const([b for b, n in enumerate(gcounts) for _ in range(n)], dev,
                                 torch.int32)

      def rows(t):  # the group's queries of a per-query tensor; outputs are written in place
        return _query_rows(t, q0, q1)

      occ0, expd0 = rows(occ_out[0]), rows(expd_out[0])
      pos = self._stage_a(pk, feature_grids.lowres[0][bs].contiguous(),
                          rows(query_features.lowres[0]).contiguous(), gcounts, query_clip,
                          rows(query_points_in_video) if query_points_in_video is not None else None,
                          video_hw if video_table is None else per_clip[b0:b1], occ0, expd0,
                          rows(trk_out[0]), rows(am_out) if am_out is not None else None, dev)

      # ---- refinement iterations, one level at a time
      bufs = self._refine_buffers(q1 - q0, T, dev)
      npi = self.num_pips_iter
      for level in range(1, num_levels_total):
        its = range((level - 1) * npi, level * npi)
        ctxs = []
        for it in its:
          ctx = [None] * 4
          if causal_context is not None:
            ctx[:2] = _ctx_lists(causal_context[it], nb, q0, q1,
                                 lambda t: t.to(device=dev, dtype=torch.float32).contiguous())
          if write_ctx:
            ctx[2:] = _ctx_lists(new_ctx[it], nb, q0, q1)
          ctxs.append(ctx)
        outs = [(rows(occ_out[it + 1]), rows(expd_out[it + 1]), rows(trk_out[it + 1])) for it in its]
        self._refine_level(pk, feature_grids.hires[level][bs], feature_grids.lowres[level][bs],
                           [g[bs] for g in pooled[level]], rows(query_features.hires[level]),
                           rows(query_features.lowres[level]), pos, occ0, expd0, outs, bufs,
                           feature_grids.resolutions[level],
                           video_hw if video_table is None else video_table[bs], ctxs, query_clip)
    return out

  @staticmethod
  def _check_points_per_clip(points_per_clip, feature_grids, query_features, query_points):
    """estimate_trajectories' points_per_clip as a list of ints, checked against the clips of
    feature_grids and the [1, sum N, ...] queries (ValueError before any launch)."""
    counts = [int(n) for n in points_per_clip]
    B = feature_grids.lowres[0].shape[0]
    if len(counts) != B:
      raise ValueError(f'points_per_clip has {len(counts)} counts for {B} clips')
    if min(counts, default=0) < 1:
      raise ValueError(f'points_per_clip: every clip needs at least one point, got {counts}')
    want = (1, sum(counts))
    for name, t in [('query_features', f) for f in query_features.lowres + query_features.hires] + [
        ('query_points_in_video', query_points)]:
      if t is not None and tuple(t.shape[:2]) != want:
        raise ValueError(f'{name} has shape {tuple(t.shape)}; points_per_clip {counts} needs '
                         f'[1, {want[1]}, ...]')
    return counts

  def _new_causal_context(self, causal_context, get_causal_context, causal_context_out, num_iters,
                          nb, B, N, T, dev):
    """Checks the causal context arguments of estimate_trajectories; returns the list of dicts the
    call fills with the new context (None when get_causal_context is False)."""
    # Causal context bookkeeping follows nets.py:143-176: a block only produces a new context
    # when it was GIVEN one (new_causal_context is filled inside `if causal_context is not None`),
    # so get_causal_context without causal_context yields empty dicts, exactly like the reference.
    if causal_context is not None:
      if not self.use_casual_conv:
        raise ValueError('causal_context needs a causal model (use_casual_conv=True); the '
                         'reference would run its non-causal convolutions over the context rows')
      if len(causal_context) < num_iters:
        raise ValueError(f'causal_context has {len(causal_context)} entries, {num_iters} needed')
      for d in causal_context[:num_iters]:
        for i in range(nb):
          for key, width in ((f'block_{i}_causal_1', 512), (f'block_{i}_causal_2', 2048)):
            if tuple(d[key].shape) != (B, N, 2, width):
              raise ValueError(f'causal_context[{key}] has shape {tuple(d[key].shape)}, expected '
                               f'{(B, N, 2, width)}')
    if get_causal_context and causal_context is not None and causal_context_out is not None:
      if T != 1 and any(causal_context_out[it][k].data_ptr() == causal_context[it][k].data_ptr()
                        for it in range(num_iters) for k in causal_context[it]):
        raise ValueError('causal_context_out may alias causal_context only for single-frame steps')
      new_ctx = [dict(d) for d in causal_context_out[:num_iters]]
      for d in new_ctx:
        for k, v in d.items():
          if not (v.is_contiguous() and v.dtype == torch.float32 and v.device == dev):
            raise ValueError(f'causal_context_out[{k}] must be a contiguous fp32 tensor on {dev}')
      return new_ctx
    if not get_causal_context:
      return None
    new_ctx = [{} for _ in range(num_iters)]
    if causal_context is not None:
      for d in new_ctx:
        for i in range(nb):
          d[f'block_{i}_causal_1'] = torch.empty(B, N, 2, 512, dtype=torch.float32, device=dev)
          d[f'block_{i}_causal_2'] = torch.empty(B, N, 2, 2048, dtype=torch.float32, device=dev)
    return new_ctx

  def _stage_a(self, pk, grid, qfeat, counts, query_clip, query_points, video_hw, occ, expd,
               tracks, argmax, dev):
    """Stage A for one group of clips: the global cost volume and the track / occlusion head of
    the group's nq queries, counts[b] of clip b one clip after the other, against grid
    [G, T, h, w, 256].  qfeat [.., 256] (contiguous), query_points [.., 3] or None, occ, expd
    [.., T], tracks [.., T, 2] (video pixels) and argmax (or None) hold the nq queries in any
    leading dims.  query_clip (see _refine) None: one batched call on [G, n, ...] views, the
    scalings broadcast per clip; else calls of at most MAX_RAGGED_CLIPS clips on [nq, ...], the
    scalings per query.  Returns the positions [nq, T, 2] in initial-resolution pixels."""
    G, T = grid.shape[:2]
    nq = occ.numel() // T
    ih, iw = self.initial_resolution
    lead = (G, nq // G) if query_clip is None else (nq,)
    if isinstance(video_hw[0], tuple):  # one (h, w) per clip: per-clip or per-query scales
      if query_clip is not None:
        video_hw = [hw for hw, n in zip(video_hw, counts) for _ in range(n)]
      dims = (len(video_hw),) + (1,) * (len(lead) - 1)
      to_init = self._const([v for h, w in video_hw for v in (T, h, w)], dev).view(*dims, 3)
      to_video = self._const([v for h, w in video_hw for v in (w, h)], dev).view(*dims, 1, 2)
    else:
      vh, vw = video_hw
      to_init, to_video = self._const([T, vh, vw], dev), self._const([vw, vh], dev)
    qp = None
    if query_points is not None:
      qp = query_points.to(torch.float32).reshape(*lead, 3)
      # utils.convert_grid_coordinates (coords * out / in), tapir_model.py:488-493
      qp = (qp * self._const([T, ih, iw], dev) / to_init).contiguous()
    qfeat, occ, expd = qfeat.view(*lead, -1), occ.view(*lead, T), expd.view(*lead, T)
    argmax = argmax.view(*lead, T) if argmax is not None else None
    pos = torch.empty(*lead, T, 2, dtype=torch.float32, device=dev)
    if query_clip is None:
      ws = self._workspace('cost_volume', _stage_a_scratch(G, nq, T, grid.shape[2:])[1], dev)
      _lib.cost_volume_tracks(pk['head'], qfeat, grid, qp, self.softmax_temperature, (ih, iw), pos,
                              occ, expd, argmax, ws)
    else:
      step = _lib.MAX_RAGGED_CLIPS
      for c0 in range(0, G, step):
        cs = counts[c0:c0 + step]
        r0 = sum(counts[:c0])
        r = slice(r0, r0 + sum(cs))
        ws = self._workspace('cost_volume',
                             _stage_a_scratch(len(cs), r.stop - r0, T, grid.shape[2:])[1], dev)
        _lib.cost_volume_tracks_ragged(pk['head'], qfeat[r], cs, grid[c0:c0 + len(cs)],
                                       qp[r] if qp is not None else None, self.softmax_temperature,
                                       (ih, iw), pos[r], occ[r], expd[r],
                                       argmax[r] if argmax is not None else None, ws)
    # train2orig (tapir_model.py:435-441)
    torch.div(pos * to_video, self._const([iw, ih], dev), out=tracks.view(*lead, T, 2))
    return pos.view(nq, T, 2)

  def _refine_scratch(self, nq, T):
    """The refinement of nq queries over T frames: the (shape, dtype) of the mixer's input planes,
    its output rows and the two feature buffers the iterations alternate between, and the bytes of
    the mixer workspace."""
    x_planes = (self._planes, nq * T, _lib.padded_k(schema.mixer_input_dim(self.pyramid_level)))
    f32 = torch.float32
    return ([(x_planes, torch.bfloat16), ((nq, T, schema.mixer_output_dim()), f32)]
            + [((nq, T, schema.HIRES_DIM + schema.LOWRES_DIM), f32)] * 2,
            _lib.mixer_workspace_bytes(x_planes))

  def _refine_buffers(self, nq, T, dev):
    """The _refine_scratch of nq queries over T frames: (x_planes, res, feats, mixer workspace)."""
    specs, ws_bytes = self._refine_scratch(nq, T)
    x_planes, res, *feats = (torch.empty(s, dtype=d, device=dev) for s, d in specs)
    return x_planes, res, feats, self._workspace('mixer', ws_bytes, dev)

  def _pool_pyramid(self, grid):
    """The pooled levels of lowres grids [..., h, w, C], each the 2 x 2 mean of the one before."""
    pooled = []
    for _ in range(self.pyramid_level):
      *lead, h, w, c = grid.shape
      pooled.append(torch.empty(*lead, h // 2, w // 2, c, dtype=torch.float32, device=grid.device))
      _lib.pool_pyramid(grid, pooled[-1])
      grid = pooled[-1]
    return pooled

  def _refine_level(self, pk, hires, lowres, pooled, qf_hi, qf_lo, pos, occ0, expd0, outs, bufs,
                    resize_hw, video_hw, ctxs=None, query_clip=None):
    """The num_pips_iter refinement iterations of one level (reference tapir_model.py:529-552)
    for nq queries over T frames.  hires, lowres [G, T, h, w, C]: the level's grids, pooled: the
    _pool_pyramid of lowres; qf_hi / qf_lo: the query features [..., 128 | 256] of the nq queries;
    pos [..., T, 2] is moved in place; occ0 / expd0: the stage-A estimates the level starts from;
    outs: one (occ, expd, tracks) output view per iteration; bufs: _refine_buffers; ctxs: one mixer
    context list per iteration (see _refine), or None; query_clip: see _refine.  Only pos carries over to the next level:
    features restart from the query and occlusion / expected distance from stage A."""
    levels = [hires.contiguous(), lowres.contiguous()] + pooled
    qfeat = (qf_hi.contiguous(), qf_lo.contiguous())
    x_planes, res, feats, mws = bufs
    nq, T = res.shape[:2]
    occ, expd = occ0, expd0
    fsrc = None  # the previous iteration's features; None: start from the query features
    for i, (occ_n, expd_n, trk_n) in enumerate(outs):
      if fsrc is not None:
        feat = (fsrc[..., :128], fsrc[..., 128:])
      else:
        feat = tuple(q.view(nq, 1, -1).expand(nq, T, -1) for q in qfeat)
      fdst = feats[1] if fsrc is feats[0] else feats[0]
      self._refine(pk, levels, pos, occ, expd, feat, x_planes, res,
                   ctxs[i] if ctxs is not None else [None] * 4, mws, occ_n, expd_n, fdst, trk_n,
                   resize_hw, video_hw, query_clip)
      fsrc, occ, expd = fdst, occ_n, expd_n

  def _refine(self, pk, levels, pos, occ, expd, feat, x_planes, res, ctx, mws, occ_out, expd_out,
              feat_out, tracks_out, resize_hw, video_hw, query_clip=None):
    """One refinement iteration (the refine_pips call, reference tapir_model.py:529-542): local correlation around pos
    over the pyramid `levels`, the mixer, and the update of pos (in place), occlusion, expected
    distance, features (hi, lo views `feat` -> feat_out) and tracks.  ctx: the mixer's causal
    context lists (ctx1_in, ctx2_in, ctx1_out, ctx2_out), None where absent.  video_hw: one
    (h, w), or an int32 [G, 2] table of per-clip sizes.  query_clip: None (clips of equal query
    counts), or the int32 [nq] clip of each query."""
    _lib.local_corr(levels, pos, occ, expd, *feat, x_planes, self.initial_resolution,
                    query_clip=query_clip)
    _lib.mixer_forward(pk['mixer'], x_planes, res, self.use_casual_conv, *ctx, mws)
    if isinstance(video_hw, torch.Tensor):
      _lib.refine_update(res, pos, occ, expd, *feat, occ_out, expd_out, feat_out, tracks_out,
                         self.initial_resolution, resize_hw, (0, 0), video_table=video_hw,
                         query_clip=query_clip)
    else:
      _lib.refine_update(res, pos, occ, expd, *feat, occ_out, expd_out, feat_out, tracks_out,
                         self.initial_resolution, resize_hw, video_hw)

  def construct_initial_causal_state(self, num_points, num_resolutions=1):
    """Reference tapir_model.py:763-772 (the same dict object repeated, CPU tensors)."""
    value_shapes = {}
    for i in range(self.num_mixer_blocks):
      value_shapes[f'block_{i}_causal_1'] = (1, num_points, 2, 512)
      value_shapes[f'block_{i}_causal_2'] = (1, num_points, 2, 2048)
    fake_ret = {k: torch.zeros(v, dtype=torch.float32) for k, v in value_shapes.items()}
    return [fake_ret] * num_resolutions * 4

  def update_query_features(self, query_features, new_query_features, idx_to_update,
                            causal_state=None):
    """Reference tapir_model.py:774-806: in-place overwrite of the given query slots."""
    if isinstance(idx_to_update, int):
      idx_to_update = tuple([idx_to_update])
    idx_to_update = np.array(idx_to_update)

    def apply_update_idx(s1, s2):
      s1[:, idx_to_update] = s2.to(s1.device) if isinstance(s2, torch.Tensor) else s2
      return s1

    query_features = QueryFeatures(
        lowres=tuple(apply_update_idx(a, b) for a, b in
                     zip(query_features.lowres, new_query_features.lowres)),
        hires=tuple(apply_update_idx(a, b) for a, b in
                    zip(query_features.hires, new_query_features.hires)),
        resolutions=query_features.resolutions,
    )
    if causal_state is not None:
      init_causal_state = self.construct_initial_causal_state(
          len(idx_to_update), len(query_features.resolutions) - 1)
      causal_state = [
          {k: apply_update_idx(v, init_causal_state[i][k]) for k, v in d.items()}
          for i, d in enumerate(causal_state)
      ]
      return query_features, causal_state
    return query_features


def build_model(checkpoint_path: Optional[str] = None, device: str = 'cuda', **tapir_kwargs):
  """BASELINE.json north_star names a `build_model`; the reference spells it out at each call
  site as TAPIR(...) + load_state_dict(torch.load(path)) + .to(device).eval()
  (tapnet/pytorch_live_demo.py:110-117).  This is that sequence."""
  if checkpoint_path is not None and str(checkpoint_path).endswith('.npy'):
    # Haiku parameter tree (the format "Online TAPIR" is published in, README.md:165, and what
    # robotap/tapir_clustering.py:track_many_points is handed): convert, then the usual sequence
    from tapnet_b200 import convert  # pylint: disable=g-import-not-at-top
    import numpy as _np  # pylint: disable=g-import-not-at-top
    ckpt = _np.load(checkpoint_path, allow_pickle=True).item()
    params = ckpt['params'] if 'params' in ckpt else ckpt
    kwargs = convert.infer_model_kwargs(params)  # pyramid_level / extra_convs from the tree
    kwargs.update(tapir_kwargs)
    state_dict = convert.convert_haiku_params(params, kwargs['pyramid_level'],
                                              kwargs['extra_convs'])
    model = TAPIR(**kwargs)
    model.load_state_dict(state_dict)
    return model.to(device).eval()
  model = TAPIR(**tapir_kwargs)
  if checkpoint_path is not None:
    model.load_state_dict(torch.load(checkpoint_path, map_location='cpu'))
  return model.to(device).eval()
