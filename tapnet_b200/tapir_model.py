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
import ctypes
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


_PRECISIONS = {'bf16': 1, 'bf16x3': 2, 'bf16x6': 3}

# rows (= queries x frames) processed per mixer pass; bounds the workspace to ~1.5 GB
_MAX_ROWS_PER_CHUNK = 98304
# input pixels (frames x H x W) per backbone pass; bounds the workspace to ~2.7 GB
_MAX_BACKBONE_PIXELS = 96 * 256 * 256
# host clips: H2D sub-chunks per backbone pass (each followed by its stem-conv launch)
_H2D_SUBCHUNKS = 6


def _ptr(t):
  return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _groups(B, N, T):
  """Work groups of estimate_trajectories as (b0, b1, query slice): whole clips b0..b1-1 with all
  their queries while the group's rows (clips x queries x frames) fit _MAX_ROWS_PER_CHUNK and its
  queries fit one head / mixer launch (65535); a clip whose rows alone exceed the bound runs on its
  own in query chunks.  Each group is one launch sequence over its clips."""
  if N * T <= _MAX_ROWS_PER_CHUNK and N <= 65535:
    g = max(1, min(B, _MAX_ROWS_PER_CHUNK // (N * T), 65535 // N))
    return [(b0, min(b0 + g, B), slice(0, N)) for b0 in range(0, B, g)]
  chunk_q = max(1, min(N, _MAX_ROWS_PER_CHUNK // T, 65535))
  return [(bi, bi + 1, slice(q0, min(q0 + chunk_q, N)))
          for bi in range(B) for q0 in range(0, N, chunk_q)]


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

  def _stream(self, dev=None):
    # the current stream OF THE MODEL'S DEVICE (every public method runs its launches inside
    # `torch.cuda.device(dev)`, so the C side's per-device caches and the pointers agree)
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)

  def _copy_stream(self, dev):
    key = str(dev)
    if key not in self._copy_streams:
      self._copy_streams[key] = torch.cuda.Stream(device=dev)
    return self._copy_streams[key]

  def _const(self, values, dev):
    """Small constant vectors, cached: creating them per call costs a blocking H2D copy."""
    key = (tuple(float(v) for v in values), str(dev))
    t = self._consts.get(key)
    if t is None:
      t = torch.tensor(key[0], dtype=torch.float32, device=dev)
      self._consts[key] = t
    return t

  def _workspace(self, name, nbytes, dev):
    """Grow-only scratch.  A buffer that is outgrown is parked in `_ws_retired` instead of
    being freed while `_ws_pins` > 0: a captured CUDA graph (streaming.OnlineTracker) holds raw
    pointers into it.  `_ws_generation` changes whenever a buffer is replaced, so graph owners
    can tell that their capture no longer describes the model's current buffers."""
    ws = self._ws.get(name)
    if ws is None or ws.numel() < nbytes or ws.device != dev:
      if ws is not None and self._ws_pins > 0:
        self._ws_retired.append(ws)
      ws = torch.empty(int(nbytes), dtype=torch.uint8, device=dev)
      self._ws[name] = ws
      self._ws_generation += 1
    return ws

  # ------------------------------------------------------------------ weight packing
  @_on_model_device
  def _pack(self):
    sig = self._param_sig()
    if self._packed is not None and self._packed_sig == sig:
      return self._packed
    lib = _lib.load()
    sd = {k: v.detach() for k, v in self.state_dict().items()}
    dev = next(self.parameters()).device
    P = self._planes
    keep = []  # tensors referenced by raw pointers below
    stream = self._stream(dev)

    def f32(t):
      t = t.to(device=dev, dtype=torch.float32).contiguous().clone()
      keep.append(t)
      return t

    def linear(w2d, bias, planes=P):
      w2d = f32(w2d)
      n, k = w2d.shape
      kp = (k + 63) // 64 * 64
      dst = torch.empty(planes, n, kp, dtype=torch.bfloat16, device=dev)
      keep.append(dst)
      _lib.check(lib.tapir_split_planes(_ptr(w2d), k, _ptr(dst), kp, n * kp, n, k, kp, planes,
                                        stream), 'tapir_split_planes')
      b = f32(bias) if bias is not None else None
      return _lib.Linear(w=dst.data_ptr(), bias=(b.data_ptr() if b is not None else None), N=n,
                         K=kp, planes=planes, k_logical=k)

    def conv(wkey, bkey=None):
      w = sd[wkey]
      co = w.shape[0]
      w2d = w.permute(0, 2, 3, 1).reshape(co, -1)  # K order (ky, kx, cin)
      return linear(w2d, sd[bkey] if bkey else None)

    bw = _lib.BackboneWeights()
    stem = f32(sd['resnet_torch.initial_conv.weight'].permute(2, 3, 1, 0))  # [7,7,3,64]
    bw.stem_w = stem.data_ptr()
    cin = 64
    bi = 0
    for g, (cout, stride) in enumerate(zip(schema.GROUP_CHANNELS, schema.GROUP_STRIDES)):
      for b in range(2):
        p = f'resnet_torch.block_groups.{g}.blocks.{b}.'
        blk = bw.blocks[bi]
        blk.cin = cin if b == 0 else cout
        blk.cout = cout
        blk.stride = stride if b == 0 else 1
        blk.has_proj = 1 if b == 0 else 0
        if b == 0:
          blk.proj = conv(p + 'proj_conv.weight')
        blk.conv0 = conv(p + 'conv_0.weight')
        blk.conv1 = conv(p + 'conv_1.weight')
        blk.bn0_w = f32(sd[p + 'bn_0.weight']).data_ptr()
        blk.bn0_b = f32(sd[p + 'bn_0.bias']).data_ptr()
        blk.bn1_w = f32(sd[p + 'bn_1.weight']).data_ptr()
        blk.bn1_b = f32(sd[p + 'bn_1.bias']).data_ptr()
        bi += 1
      cin = cout
    bw.num_extra = schema.NUM_EXTRA_CONV_BLOCKS if self._has_extra else 0
    for i in range(bw.num_extra):
      p = f'extra_convs.blocks.{i}.'
      eb = bw.extra[i]
      eb.ln_w = f32(sd[p + 'layer_norm.weight']).data_ptr()
      eb.ln_b = f32(sd[p + 'layer_norm.bias']).data_ptr()
      eb.conv = conv(p + 'conv.weight', p + 'conv.bias')
      eb.conv1 = conv(p + 'conv_1.weight', p + 'conv_1.bias')
    bw.planes = P

    hw = _lib.HeadWeights()
    m = 'torch_cost_volume_track_mods.'
    for name, key in (('hid1', 'hid1'), ('hid2', 'hid2'), ('hid3', 'hid3'), ('hid4', 'hid4'),
                      ('occ', 'occ_out')):
      setattr(hw, name + '_w', f32(sd[m + key + '.weight']).data_ptr())
      setattr(hw, name + '_b', f32(sd[m + key + '.bias']).data_ptr())

    mw = _lib.MixerWeights()
    x = 'torch_pips_mixer.'
    mw.linear = linear(sd[x + 'linear.weight'], sd[x + 'linear.bias'])
    mw.linear_1 = linear(sd[x + 'linear_1.weight'], sd[x + 'linear_1.bias'])
    mw.ln_w = f32(sd[x + 'layer_norm.weight']).data_ptr()
    nb = len([k for k in sd if k.startswith(x + 'blocks.') and k.endswith('.layer_norm.weight')])
    mw.num_blocks = nb
    mw.planes = P
    for i in range(nb):
      p = f'{x}blocks.{i}.'
      blk = mw.blocks[i]
      blk.ln_w = f32(sd[p + 'layer_norm.weight']).data_ptr()
      blk.dw1_w = f32(sd[p + 'mlp1_up.weight']).data_ptr()
      blk.dw1_b = f32(sd[p + 'mlp1_up.bias']).data_ptr()
      blk.dw2_w = f32(sd[p + 'mlp1_up_1.weight']).data_ptr()
      blk.dw2_b = f32(sd[p + 'mlp1_up_1.bias']).data_ptr()
      blk.ln1_w = f32(sd[p + 'layer_norm_1.weight']).data_ptr()
      blk.up = linear(sd[p + 'conv_channels_mixer.mlp2_up.weight'],
                      sd[p + 'conv_channels_mixer.mlp2_up.bias'])
      blk.down = linear(sd[p + 'conv_channels_mixer.mlp2_down.weight'],
                        sd[p + 'conv_channels_mixer.mlp2_down.bias'])
    self._packed = dict(backbone=bw, head=hw, mixer=mw, keep=keep,
                        mixer_in=int(mw.linear.K), num_blocks=nb)
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
    p = self.num_pips_iter
    return dict(
        occlusion=torch.mean(torch.stack(trajectories['occlusion'][p::p]), dim=0),
        tracks=torch.mean(torch.stack(trajectories['tracks'][p::p]), dim=0),
        expected_dist=torch.mean(torch.stack(trajectories['expected_dist'][p::p]), dim=0),
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
    [0, 255], or a device-resident `live.YUV420Frames` clip whose crop window is the video).

    `hires_ready_events` (extension, used by tapnet_b200.distributed): a list that receives one
    (hires tensor, torch.cuda.Event) pair per distinct resolution; the event fires as soon as
    that hires grid is final, while ResNet groups 2-3 and the ExtraConvs are still running."""
    del is_training
    if refinement_resolutions is None:
      refinement_resolutions = generate_default_resolutions(video.shape[2:4],
                                                            self.initial_resolution)
    all_required = [tuple(self.initial_resolution)] + [tuple(r) for r in refinement_resolutions]
    for resolution in all_required:
      if resolution[0] % 8 != 0 or resolution[1] % 8 != 0:
        raise ValueError('Image resolution must be a multiple of 8.')
    # A HOST clip (ideally pinned) is accepted too (extension): its frames are copied to the
    # device in chunks on a copy stream and the stem convolution - the only reader of the video -
    # runs chunk by chunk behind them, so PCIe time hides behind compute.
    host_video = video.device.type == 'cpu'
    dev = self._device_check(None if host_video else video)
    lib = _lib.load()
    pk = self._pack()
    # uint8 video = raw [0,255] frames (what the reference's callers hold before
    # preprocess_frames, pytorch_live_demo.py:30-41): normalised inside the stem conv's loads
    # (or inside the resize), so the 4x larger float video never exists.  Extension of the
    # reference surface; float video behaves exactly as before.
    # YUV 4:2:0 frames (extension): at the frame's own size the stem conv converts inside its
    # loads; a resized pass converts each bilinear tap in the ingest kernel.  Bit for bit the
    # results of the uint8 RGB frames the conversion produces.
    yuv = isinstance(video, live.YUV420Frames)
    video_u8 = not yuv and video.dtype == torch.uint8
    if not yuv:
      video = video.contiguous() if video_u8 else video.to(torch.float32).contiguous()
    n, f, vh, vw, _ = video.shape
    host_src = None
    if host_video:
      host_src = video
      video = torch.empty(video.shape, dtype=video.dtype, device=dev)
      if tuple(all_required[0]) != (vh, vw):
        # the first pass resizes the clip: it needs all of it on the device up front
        video.copy_(host_src, non_blocking=True)
        host_src = None
    feature_grid, hires_feats, resize_im_shape = [], [], []
    curr_resolution = (-1, -1)
    latent = hires = None
    shape_hw = None
    stream = self._stream(dev)
    for resolution in all_required:
      if resolution[0] % 8 != 0 or resolution[1] % 8 != 0:
        raise ValueError('Image resolution must be a multiple of 8.')
      if not _is_same_res(curr_resolution, resolution):
        # reference quirk (:337): the PREVIOUS resolution is compared with the video size
        if _is_same_res(curr_resolution, video.shape[-3:-1]):
          h, w = vh, vw
          frames_src = video
        else:
          h, w = int(resolution[0]), int(resolution[1])
          if (h, w) == (vh, vw):
            frames_src = video  # align_corners=False resize to the same size is the identity
          else:
            frames_src = torch.empty(n, f, h, w, 3, dtype=torch.float32, device=dev)
            if yuv:
              desc = video.c_struct()
              _lib.check(lib.tapir_ingest_frames_yuv420(ctypes.byref(desc), n * f,
                                                        _ptr(frames_src), h, w, stream),
                         'tapir_ingest_frames_yuv420')
            elif video_u8:
              _lib.check(lib.tapir_ingest_frames(_ptr(video), n * f, vh, vw, 0, 0, vh, vw,
                                                 _ptr(frames_src), h, w, stream),
                         'tapir_ingest_frames')
            else:
              _lib.check(lib.tapir_bilinear_resize(_ptr(video), n * f, vh, vw, 3,
                                                   _ptr(frames_src), h, w, stream),
                         'tapir_bilinear_resize')
        if h % 8 != 0 or w % 8 != 0:
          raise ValueError('Image resolution must be a multiple of 8.')
        curr_resolution = resolution
        shape_hw = (h, w)
        nf = n * f
        latent = torch.empty(n, f, h // 8, w // 8, self.lowres_dim, dtype=torch.float32, device=dev)
        hires = torch.empty(n, f, h // 4, w // 4, self.highres_dim, dtype=torch.float32, device=dev)
        src_yuv = frames_src is video and yuv
        flat_src = None if src_yuv else frames_src.view(nf, h, w, 3)
        flat_lo = latent.view(nf, h // 8, w // 8, self.lowres_dim)
        flat_hi = hires.view(nf, h // 4, w // 4, self.highres_dim)
        # frames are independent in the backbone (InstanceNorm per frame, LayerNorm per
        # pixel), so the frame-chunk size only bounds the workspace; the reference's
        # feature_extractor_chunk_size (:346-360) has the same role.
        chunk = max(1, _MAX_BACKBONE_PIXELS // (h * w))
        chunk = min(chunk, nf)
        nbytes = lib.tapir_backbone_workspace_bytes(chunk, h, w, int(self._has_extra), self._planes)
        ws = self._workspace('backbone', nbytes, dev)
        ev = None
        if hires_ready_events is not None:
          ev = torch.cuda.Event()
          ev.record(torch.cuda.current_stream(dev))  # materialises the CUDA event handle
          hires_ready_events.append((hires, ev))
        streamed = host_src is not None and frames_src is video
        if streamed:
          main = torch.cuda.current_stream(dev)
          cs = self._copy_stream(dev)
          cs.wait_stream(main)  # the staging buffer's previous owner is done
          host_flat = host_src.view(nf, h, w, 3)
        for s0 in range(0, nf, chunk):
          c = min(chunk, nf - s0)
          last = s0 + c >= nf
          if streamed:
            # sub-chunks of >= ~4 MB (each costs ~70 us of host time: copy, event, stem launch),
            # at most _H2D_SUBCHUNKS per pass
            nsub = max(1, min(_H2D_SUBCHUNKS, (c * h * w * 3 * flat_src.element_size()) >> 22))
            sub = max(1, -(-c // nsub))
            for a in range(s0, s0 + c, sub):
              b = min(a + sub, s0 + c)
              with torch.cuda.stream(cs):
                flat_src[a:b].copy_(host_flat[a:b], non_blocking=True)
                arrived = torch.cuda.Event()
                arrived.record(cs)
              main.wait_event(arrived)
              _lib.check(lib.tapir_backbone_stem(
                  ctypes.byref(pk['backbone']), _ptr(flat_src[a:]), int(video_u8), c, h, w, a - s0,
                  b - a, _ptr(ws), ws.numel(), stream), 'tapir_backbone_stem')
          ready = ctypes.c_void_p(ev.cuda_event) if (ev is not None and last) else None
          if src_yuv:
            desc = video.c_struct(s0)
            _lib.check(lib.tapir_backbone_forward_yuv420(
                ctypes.byref(pk['backbone']), ctypes.byref(desc), c, _ptr(flat_lo[s0:]),
                _ptr(flat_hi[s0:]), _ptr(ws), ws.numel(), ready, stream),
                       'tapir_backbone_forward_yuv420')
            continue
          _lib.check(lib.tapir_backbone_forward_ex(
              ctypes.byref(pk['backbone']), None if streamed else _ptr(flat_src[s0:]),
              int(flat_src.dtype == torch.uint8),
              c, h, w, _ptr(flat_lo[s0:]), _ptr(flat_hi[s0:]), _ptr(ws), ws.numel(),
              ready, stream),
                     'tapir_backbone_forward')
        if streamed:
          host_src = None  # the whole clip is on the device now (later passes resize from it)
      feature_grid.append(latent)
      hires_feats.append(hires)
      resize_im_shape.append(torch.Size(shape_hw))
    return FeatureGrids(tuple(feature_grid), tuple(hires_feats), tuple(resize_im_shape))

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
    lib = _lib.load()
    stream = self._stream(dev)
    shape = video.shape
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
          _, t, gh, gw, c = grid.shape
          out = torch.empty(b, nq, c, dtype=torch.float32, device=dev)
          for bi in range(b if nq > 0 else 0):
            _lib.check(lib.tapir_sample_query_features(
                _ptr(grid[bi]), t, gh, gw, c, _ptr(qp[bi]), nq, int(shape[1]), int(shape[2]),
                int(shape[3]), _ptr(out[bi]), stream), 'tapir_sample_query_features')
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
  ) -> Mapping[str, Any]:
    """Reference tapir_model.py:394-578.

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
    lib = _lib.load()
    pk = self._pack()
    stream = self._stream(dev)
    P = self._planes
    ih, iw = self.initial_resolution
    vh, vw = int(video_size[0]), int(video_size[1])
    num_levels_total = len(feature_grids.lowres)
    num_iters = self.num_pips_iter * (num_levels_total - 1)
    B, N = query_features.lowres[0].shape[:2]
    T = feature_grids.lowres[0].shape[1]
    L = self.pyramid_level + 2
    kin = pk['mixer_in']
    nb = pk['num_blocks']

    def new(*shape, dtype=torch.float32):
      return torch.empty(*shape, dtype=dtype, device=dev)

    occ_out = [new(B, N, T) for _ in range(num_iters + 1)]
    expd_out = [new(B, N, T) for _ in range(num_iters + 1)]
    trk_out = [new(B, N, T, 2) for _ in range(num_iters + 1)]
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
    new_ctx = None
    if get_causal_context and causal_context is not None and causal_context_out is not None:
      if T != 1 and any(causal_context_out[it][k].data_ptr() == causal_context[it][k].data_ptr()
                        for it in range(num_iters) for k in causal_context[it]):
        raise ValueError('causal_context_out may alias causal_context only for single-frame steps')
      new_ctx = [dict(d) for d in causal_context_out[:num_iters]]
      for d in new_ctx:
        for k, v in d.items():
          if not (v.is_contiguous() and v.dtype == torch.float32 and v.device == dev):
            raise ValueError(f'causal_context_out[{k}] must be a contiguous fp32 tensor on {dev}')
    elif get_causal_context:
      new_ctx = [{} for _ in range(num_iters)]
      if causal_context is not None:
        for d in new_ctx:
          for i in range(nb):
            d[f'block_{i}_causal_1'] = new(B, N, 2, 512)
            d[f'block_{i}_causal_2'] = new(B, N, 2, 2048)
    write_ctx = get_causal_context and causal_context is not None
    am_out = None
    if self.capture_stage_a_argmax:
      am_out = torch.empty(B, N, T, dtype=torch.int32, device=dev)
      self.last_stage_a_argmax = am_out
    if N == 0 or T == 0:
      # nothing to track (the reference fails in torch.cat on an empty chunk list,
      # tapir_model.py:556-559; returning correctly shaped empty tensors is the useful behaviour)
      out = dict(occlusion=occ_out, tracks=trk_out, expected_dist=expd_out)
      if get_causal_context:
        out['causal_context'] = new_ctx
      return out

    # pooled pyramid levels: once per resolution level over all B*T frames (the reference
    # recomputes them every iteration of every chunk, tapir_model.py:519-527); each is the 2x2
    # average of the one before it
    pooled = {}
    for level in range(1, num_levels_total):
      g = feature_grids.lowres[level].contiguous()
      outs = []
      for _ in range(self.pyramid_level):
        _, t, gh, gw, c = g.shape
        out = new(B, t, gh // 2, gw // 2, c)
        _lib.check(lib.tapir_pool_pyramid(_ptr(g), B * t, gh, gw, c, _ptr(out), stream),
                   'tapir_pool_pyramid')
        outs.append(out)
        g = out
      pooled[level] = outs

    for b0, b1, sl in _groups(B, N, T):
      G = b1 - b0
      n = sl.stop - sl.start
      nq = G * n  # queries of the group, flattened over its clips
      rows = nq * T
      bs = slice(b0, b1)
      # every [bs, sl] slice below is contiguous: either whole clips or a query chunk of one clip
      # ---- stage A: global cost volume + track / occlusion head
      grid0 = feature_grids.lowres[0][bs].contiguous()
      _, _, gh0, gw0, c0 = grid0.shape
      qf0 = query_features.lowres[0][bs, sl].contiguous()
      qp = None
      if query_points_in_video is not None:
        qp = query_points_in_video[bs, sl].to(torch.float32)
        # utils.convert_grid_coordinates (coords * out / in), tapir_model.py:488-493
        qp = (qp * self._const([T, ih, iw], dev) / self._const([T, vh, vw], dev)).contiguous()
      pos = new(nq, T, 2)
      # outputs are written in place
      occ0, expd0 = occ_out[0][bs, sl], expd_out[0][bs, sl]
      nbytes = lib.tapir_cost_volume_batched_workspace_bytes(G, n, T, gh0, gw0, c0)
      ws = self._workspace('cost_volume', nbytes, dev)
      _lib.check(lib.tapir_cost_volume_tracks_batched(
          ctypes.byref(pk['head']), _ptr(qf0), _ptr(grid0), G, n, T, gh0, gw0, c0, _ptr(qp),
          float(self.softmax_temperature), ih, iw, _ptr(pos), _ptr(occ0), _ptr(expd0),
          _ptr(am_out[bs, sl]) if am_out is not None else None,
          _ptr(ws), ws.numel(), stream), 'tapir_cost_volume_tracks_batched')
      # train2orig (tapir_model.py:435-441)
      torch.div(pos.view(G, n, T, 2) * self._const([vw, vh], dev), self._const([iw, ih], dev),
                out=trk_out[0][bs, sl])

      # ---- refinement iterations
      x_planes = new(P, rows, kin, dtype=torch.bfloat16)
      res = new(rows, 388)
      feats = [new(nq, T, 384), new(nq, T, 384)]
      occ, expd = occ0, expd0
      nbytes = lib.tapir_mixer_workspace_bytes(rows, P)
      mws = self._workspace('mixer', nbytes, dev)
      have_feats = False
      cur = 0
      for it in range(num_iters):
        level = it // self.num_pips_iter + 1
        hires_g = feature_grids.hires[level][bs].contiguous()
        lowres_g = feature_grids.lowres[level][bs].contiguous()
        ca = _lib.CorrArgs()
        grids = [hires_g, lowres_g] + [g[bs] for g in pooled[level]]
        for li, g in enumerate(grids):
          ca.levels[li].grid = g.data_ptr()
          ca.levels[li].h, ca.levels[li].w, ca.levels[li].C = g.shape[2], g.shape[3], g.shape[4]
        ca.num_levels = L
        ca.num_points, ca.num_frames = n, T
        ca.init_h, ca.init_w = ih, iw
        ca.planes = P
        ca.pos, ca.occ, ca.expd = pos.data_ptr(), occ.data_ptr(), expd.data_ptr()
        if have_feats:
          fsrc = feats[cur]
          fh = (fsrc.data_ptr(), T * 384, 384)
          fl = (fsrc.data_ptr() + 128 * 4, T * 384, 384)
        else:
          qh = query_features.hires[level][bs, sl].contiguous()
          ql = query_features.lowres[level][bs, sl].contiguous()
          fh = (qh.data_ptr(), 128, 0)
          fl = (ql.data_ptr(), 256, 0)
        ca.feat_hi, ca.feat_hi_stride_n, ca.feat_hi_stride_t = fh
        ca.feat_lo, ca.feat_lo_stride_n, ca.feat_lo_stride_t = fl
        ca.out_planes = x_planes.data_ptr()
        ca.out_plane_stride = rows * kin
        ca.ld = kin
        _lib.check(lib.tapir_local_corr_batched(ctypes.byref(ca), G, stream),
                   'tapir_local_corr_batched')

        io = _lib.MixerIO()
        io.x_planes = x_planes.data_ptr()
        io.x_plane_stride = rows * kin
        io.ldx = kin
        io.num_points, io.num_frames = nq, T
        io.causal = int(self.use_casual_conv)
        holders = []
        if causal_context is not None:
          c1 = [causal_context[it][f'block_{i}_causal_1'][bs, sl].to(device=dev, dtype=torch.float32).contiguous()
                for i in range(nb)]
          c2 = [causal_context[it][f'block_{i}_causal_2'][bs, sl].to(device=dev, dtype=torch.float32).contiguous()
                for i in range(nb)]
          holders += c1 + c2
          io.ctx1_in = (ctypes.c_void_p * nb)(*[t.data_ptr() for t in c1])
          io.ctx2_in = (ctypes.c_void_p * nb)(*[t.data_ptr() for t in c2])
        o1 = o2 = None
        if write_ctx:
          o1 = [new_ctx[it][f'block_{i}_causal_1'][bs, sl] for i in range(nb)]
          o2 = [new_ctx[it][f'block_{i}_causal_2'][bs, sl] for i in range(nb)]
          io.ctx1_out = (ctypes.c_void_p * nb)(*[t.data_ptr() for t in o1])
          io.ctx2_out = (ctypes.c_void_p * nb)(*[t.data_ptr() for t in o2])
        io.out = res.data_ptr()
        io.ldo = 388
        _lib.check(lib.tapir_mixer_forward(ctypes.byref(pk['mixer']), ctypes.byref(io), _ptr(mws),
                                           mws.numel(), stream), 'tapir_mixer_forward')

        ua = _lib.UpdateArgs()
        ua.res, ua.ld_res = res.data_ptr(), 388
        ua.num_points, ua.num_frames = nq, T
        ua.init_h, ua.init_w = ih, iw
        rh, rw = feature_grids.resolutions[level]
        ua.resize_h, ua.resize_w = int(rh), int(rw)
        ua.video_h, ua.video_w = vh, vw
        ua.feat_hi, ua.feat_hi_stride_n, ua.feat_hi_stride_t = fh
        ua.feat_lo, ua.feat_lo_stride_n, ua.feat_lo_stride_t = fl
        nxt = 1 - cur if have_feats else cur
        trk_i = trk_out[it + 1][bs, sl]
        occ_n, expd_n = occ_out[it + 1][bs, sl], expd_out[it + 1][bs, sl]
        ua.pos = pos.data_ptr()
        ua.occ_in, ua.expd_in = occ.data_ptr(), expd.data_ptr()
        ua.occ_out, ua.expd_out = occ_n.data_ptr(), expd_n.data_ptr()
        ua.feat_out = feats[nxt].data_ptr()
        ua.tracks_out = trk_i.data_ptr()
        _lib.check(lib.tapir_refine_update(ctypes.byref(ua), stream), 'tapir_refine_update')
        cur = nxt
        have_feats = True
        occ, expd = occ_n, expd_n
        if (it + 1) % self.num_pips_iter == 0:
          # level boundary (tapir_model.py:549-552): features restart from the query,
          # occlusion / expected_dist revert to the stage-A estimate, positions carry over
          have_feats = False
          occ, expd = occ0, expd0
        del holders

    out = dict(occlusion=occ_out, tracks=trk_out, expected_dist=expd_out)
    if get_causal_context:
      out['causal_context'] = new_ctx
    return out

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
