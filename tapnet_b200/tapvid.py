"""TAP-Vid evaluation on the GPU (DESIGN section 10, row f6).

The names are those of `tapnet/tapvid/evaluation_datasets.py`, whose module imports TensorFlow,
tensorflow_datasets and mediapy; here the pickles are read with plain `open` / `glob`, the frames
are resized on the device and the metrics are reduced there (`metrics.compute_tapvid_metrics`):

    from tapnet_b200 import tapir_model, tapvid
    model = tapir_model.build_model('bootstapir_checkpoint_v2.pt')
    ds = tapvid.create_davis_dataset('tapvid_davis.pkl', query_mode='strided')
    mean, per_video = tapvid.evaluate(model, ds, 'strided')
    print(tapvid.latex_table(mean))

or `python -m tapnet_b200.tapvid --dataset davis --path tapvid_davis.pkl --checkpoint C.pt`.

`evaluate(..., redetection=True)` adds AJ_RD, the re-detection Average Jaccard of
`tapnet/tapnextpp/metrics/aj_rd.py` (`metrics.compute_redetection_metrics`), which the reference
reports on RoboTAP (`create_robotap_dataset`); `window_frames` tracks long clips in bounded memory
(`windowed.windowed_forward`).

`resize_video` is the reference's `media.resize_video` on uint8 frames, assuming (mediapy is not
a dependency) that mediapy sends a uint8 3-channel frame to
`PIL.Image.fromarray(frame).resize((w, h), resample=LANCZOS)`: PIL's 8-bit Lanczos resampler,
bit for bit (`tapir_resize_lanczos_u8`; the arithmetic is in include/tapir_b200.h).  mediapy's
float per-channel path is not provided.

One difference from the reference readers: `video` is the resized uint8 clip [1, T, h, w, 3] on
the current CUDA device, not the float clip in [-1, 1].  `frames / 255 * 2 - 1` in float32 gives
the reference's clip exactly, and TAPIR's uint8 input path computes bit for bit what its float
path computes on that clip.
"""
import argparse
import glob
import io
import json
import os
import pickle

import numpy as np
import torch

from tapnet_b200 import _lib, metrics

_MODES = ('first', 'strided')
_TABLES = {}   # (in, out, device) -> (bounds, taps, event after their upload)


# ------------------------------------------------------------------------------ resize
def _tables(n_in, n_out, dev):
  """The device copies of one axis's Lanczos tables, uploaded once per (in, out, device); the
  current stream waits for the upload (no host sync)."""
  key = (n_in, n_out, str(dev))
  if key not in _TABLES:
    bounds, taps = _lib.lanczos_weights(n_in, n_out)
    d = [torch.from_numpy(a).pin_memory().to(dev, non_blocking=True) for a in (bounds, taps)]
    ev = torch.cuda.Event()
    ev.record()
    _TABLES[key] = (d[0], d[1], ev)
  bounds, taps, ev = _TABLES[key]
  torch.cuda.current_stream(dev).wait_event(ev)
  return bounds, taps


def _size(v, what):
  if not 1 <= v <= _lib.MAX_RESIZE_SIDE:
    raise ValueError(f'resize_video: {what} {v} outside 1..{_lib.MAX_RESIZE_SIDE}')
  return v


def resize_video(video, output_size):
  """uint8 video [T, H, W, 3] -> [T, h, w, 3], output_size = (h, w), with PIL's Lanczos.

  A numpy array gives a numpy array; a CUDA tensor gives a CUDA tensor on its device, computed
  on the current stream without a host sync."""
  on_device = isinstance(video, torch.Tensor) and video.is_cuda
  if not on_device:
    video = np.asarray(video)
  if video.dtype != (torch.uint8 if on_device else np.uint8):
    raise ValueError(f'resize_video: only uint8 frames are supported, got {video.dtype}')
  if video.ndim != 4 or video.shape[3] != 3:
    raise ValueError(f'resize_video: video must be [T, H, W, 3], got {tuple(video.shape)}')
  T, H, W = (int(v) for v in video.shape[:3])
  h, w = (int(v) for v in output_size)
  _size(h, 'output height'), _size(w, 'output width')
  if T:
    _size(H, 'height'), _size(W, 'width')
  if not torch.cuda.is_available():
    raise RuntimeError('resize_video needs a CUDA device (tapnet_b200 has no CPU fallback)')
  dev = video.device if on_device else torch.device('cuda', torch.cuda.current_device())
  with torch.cuda.device(dev):
    src = video.contiguous() if on_device else torch.from_numpy(np.ascontiguousarray(video)).pin_memory().to(
        dev, non_blocking=True)
    out = torch.empty(T, h, w, 3, dtype=torch.uint8, device=dev)
    if T:
      ws_bytes = int(_lib.load().tapir_resize_lanczos_u8_workspace_bytes(T, H, W, h, w))
      ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev) if ws_bytes else None
      _lib.resize_lanczos_u8(src, out, _tables(W, w, dev) if W != w else None,
                             _tables(H, h, dev) if H != h else None, ws)
  return out if on_device else out.cpu().numpy()


# ------------------------------------------------------------------------------ queries
def sample_queries_strided(target_occluded, target_points, frames, query_stride=5):
  """Queries at every query_stride-th frame where a track is visible (evaluation_datasets.py
  sample_queries_strided): dict(video [1, T, ...], query_points [1, Q, 3] (t, y, x) float64,
  target_points [1, Q, T, 2], occluded [1, Q, T], trackgroup [1, Q] int64), queries ordered by
  frame, then by track."""
  starts = np.arange(0, target_occluded.shape[1], query_stride)
  visible = target_occluded[:, starts] == 0                 # [tracks, strides]
  s, n = np.nonzero(visible.T)
  t = starts[s]
  query = np.stack([t.astype(np.float64), target_points[n, t, 1], target_points[n, t, 0]], -1)
  return {
      'video': frames[None],
      'query_points': query[None],
      'target_points': target_points[n][None],
      'occluded': target_occluded[n][None],
      'trackgroup': n.astype(np.int64)[None],
  }


def sample_queries_first(target_occluded, target_points, frames):
  """One query per track at its first visible frame; tracks never visible are dropped
  (evaluation_datasets.py sample_queries_first): dict(video, query_points [1, Q, 3] (t, y, x),
  target_points [1, Q, T, 2], occluded [1, Q, T])."""
  valid = np.sum(~target_occluded, axis=1) > 0
  points, occluded = target_points[valid], target_occluded[valid]
  if not len(points):
    raise ValueError('sample_queries_first: no track is ever visible')
  t = np.argmax(occluded == 0, axis=1)
  rows = np.arange(len(t))
  query = np.stack([t, points[rows, t, 1], points[rows, t, 0]], -1)
  return {
      'video': frames[None],
      'query_points': query[None],
      'target_points': points[None],
      'occluded': occluded[None],
  }


def _sample(query_mode, target_occluded, target_points, frames):
  if query_mode == 'strided':
    return sample_queries_strided(target_occluded, target_points, frames)
  return sample_queries_first(target_occluded, target_points, frames)


def _check_mode(query_mode):
  if query_mode not in _MODES:
    raise ValueError(f'Unknown query mode {query_mode}.')


# ------------------------------------------------------------------------------ readers
class _Staging:
  """One pinned host buffer reused for every video of a reader: a clip is copied in and sent to
  the device with a stream-ordered copy; the next clip waits only for that copy."""

  def __init__(self):
    self.buf = None
    self.copied = None

  def to_device(self, frames):
    frames = np.ascontiguousarray(frames)
    if frames.dtype != np.uint8 or frames.ndim != 4 or frames.shape[3] != 3:
      raise ValueError(f'TAP-Vid frames must be uint8 [T, H, W, 3], got {frames.dtype} {frames.shape}')
    if self.copied is not None:
      self.copied.synchronize()
    if self.buf is None or self.buf.numel() < frames.nbytes:
      self.buf = torch.empty(frames.nbytes, dtype=torch.uint8, pin_memory=True)
    host = self.buf[:frames.nbytes].view(frames.shape)
    host.numpy()[...] = frames
    dev = torch.device('cuda', torch.cuda.current_device())
    out = torch.empty(frames.shape, dtype=torch.uint8, device=dev)
    out.copy_(host, non_blocking=True)
    self.copied = torch.cuda.Event()
    self.copied.record()
    return out


def _clip(frames, resolution, staging):
  """Native uint8 frames -> the clip on the device, resized when `resolution` differs."""
  video = staging.to_device(frames)
  if resolution is not None and tuple(resolution) != tuple(video.shape[1:3]):
    video = resize_video(video, resolution)
  return video


def _scaled(points, video):
  return points * np.array([video.shape[2], video.shape[1]])


def _davis_format_videos(path, key, query_mode, resolution, staging):
  """Yields {key: converted} per video of one pickle in TAP-Vid-DAVIS's format (a dict of
  videos, read in its key order)."""
  with open(path, 'rb') as f:
    data = pickle.load(f)
  for name in data.keys():
    video = _clip(data[name]['video'], resolution, staging)
    points = _scaled(data[name]['points'], video)
    yield {key: _sample(query_mode, data[name]['occluded'], points, video)}


def create_davis_dataset(davis_points_path, query_mode='strided', full_resolution=False,
                         resolution=(256, 256)):
  """Yields {'davis': converted} per video of the TAP-Vid-DAVIS pickle, in its key order."""
  _check_mode(query_mode)
  if full_resolution:
    raise NotImplementedError('full_resolution reads davis/full_resolution through '
                              'tensorflow_datasets, which tapnet_b200 does not use')
  yield from _davis_format_videos(davis_points_path, 'davis', query_mode, resolution, _Staging())


def create_robotap_dataset(robotap_path, query_mode='strided', resolution=(256, 256)):
  """Yields {'robotap': converted} per video of RoboTAP.  RoboTAP ships as pickles in
  TAP-Vid-DAVIS's dict format (the reference's tapvid/README.md), and each video is read exactly
  as create_davis_dataset reads one.  robotap_path is one pickle, or a directory whose `*.pkl`
  files are read in sorted order.  The reference has no RoboTAP reader; this one is the DAVIS
  reader's loop over those files."""
  _check_mode(query_mode)
  paths = (sorted(glob.glob(os.path.join(robotap_path, '*.pkl'))) if os.path.isdir(robotap_path)
           else [robotap_path])
  staging = _Staging()
  for path in paths:
    yield from _davis_format_videos(path, 'robotap', query_mode, resolution, staging)


def create_rgb_stacking_dataset(robotics_points_path, query_mode='strided', resolution=(256, 256)):
  """Yields {'robotics': converted} per example of the TAP-Vid-RGB-Stacking pickle."""
  _check_mode(query_mode)
  with open(robotics_points_path, 'rb') as f:
    data = pickle.load(f)
  staging = _Staging()
  for example in data:
    video = _clip(example['video'], resolution, staging)
    points = _scaled(example['points'], video)
    yield {'robotics': _sample(query_mode, example['occluded'], points, video)}


def _decode_jpeg(frame):
  from PIL import Image  # pylint: disable=g-import-not-at-top
  return np.array(Image.open(io.BytesIO(frame)))


def create_kinetics_dataset(kinetics_path, query_mode='strided', resolution=(256, 256)):
  """Yields {'kinetics': converted} per video of the `*_of_0010.pkl` shards under kinetics_path
  (shards in sorted order).  JPEG frames are decoded on the host with PIL, as the reference does;
  the points are scaled in place, so they keep the pickle's dtype."""
  _check_mode(query_mode)
  staging = _Staging()
  for shard in sorted(glob.glob(os.path.join(kinetics_path, '*_of_0010.pkl'))):
    with open(shard, 'rb') as f:
      data = pickle.load(f)
    if isinstance(data, dict):
      data = list(data.values())
    for example in data:
      frames = example['video']
      if isinstance(frames[0], bytes):
        frames = np.array([_decode_jpeg(fr) for fr in frames])
      video = _clip(frames, resolution, staging)
      points = example['points']
      points *= np.array([video.shape[2], video.shape[1]])
      yield {'kinetics': _sample(query_mode, example['occluded'], points, video)}


# ------------------------------------------------------------------------------ evaluation
def _upload(a, dtype, dev):
  return torch.from_numpy(np.ascontiguousarray(a, dtype)).pin_memory().to(dev, non_blocking=True)


def evaluate(model, dataset, query_mode='strided', *, redetection=False, window_frames=None):
  """Runs `model(video, query_points)` on each video of a reader and its TAP-Vid metrics on the
  device; returns (mean_scalars, per_video).

  per_video: one {metric: float} dict per video (compute_tapvid_metrics' float64 values).
  mean_scalars: {metric: np.float32}, the reference's dataset mean
  (training/supervised_point_prediction.py:937-948): each video's scalar rounded to float32,
  summed in video order in float32, divided by the video count.

  The prediction counts as visible where (1 - sigmoid(occlusion)) (1 - sigmoid(expected_dist))
  > 0.5, the torch demo's postprocess_occlusions; the reference's training evaluation takes
  1 - (1 - sigmoid(occlusion)) (1 - sigmoid(expected_dist)) > 0.5 as occluded, which differs only
  for a visibility within one float32 ulp of 0.5.  Ground-truth tracks go to the counters as
  float32: exact at 256 x 256 for float32 pickle points (points x 256); at other sizes the float64
  product is rounded to float32 once.  The host waits for the device once, at the end.

  redetection=True adds compute_redetection_metrics' scalar keys (AJ_RD_D{D}_dmin{d},
  AJ_RD_dmin{d}, AJ_RD; default thresholds) to each video's dict, from the same predictions
  (visible as above), ground-truth visibility = not occluded and the same float32 ground truth;
  the TAP-Vid keys and the single sync are unchanged.  The reference defines no dataset mean for
  AJ_RD, and a video without a reappearance has NaN there; so an AJ_RD key's mean is taken over
  the videos where it is not NaN (float32, in video order, as dataset_mean), and
  mean_scalars['<key>/videos'] counts them (NaN mean when there are none).

  window_frames: None runs `model(video, query_points)`; an integer core length, or 'auto' (the
  largest core that fits free device memory), runs windowed.windowed_forward instead, whose
  outputs are bit for bit the whole-clip call's: for clips whose whole-clip grids would not fit."""
  _check_mode(query_mode)
  if window_frames is not None and window_frames != 'auto' and (
      isinstance(window_frames, bool) or not isinstance(window_frames, int) or window_frames < 1):
    raise ValueError(f"evaluate: window_frames must be None, 'auto' or an integer >= 1, got {window_frames!r}")
  keys, rows, events = None, [], []
  with torch.no_grad():
    for sample in dataset:
      (ex,) = sample.values()
      video = ex['video']
      dev = video.device
      qp = _upload(ex['query_points'], np.float32, dev)
      if window_frames is None:
        out = model(video, qp)
      else:
        from tapnet_b200 import windowed  # pylint: disable=g-import-not-at-top
        out = windowed.windowed_forward(model, video, qp, None if window_frames == 'auto' else window_frames)
      occluded, target = _upload(ex['occluded'], np.uint8, dev), _upload(ex['target_points'], np.float32, dev)
      logits = (out['occlusion'], out['expected_dist'])
      m = metrics.compute_tapvid_metrics(qp, occluded, target, None, out['tracks'], query_mode,
                                         pred_logits=logits)
      keys = keys or list(m)
      rows.append(torch.cat([m[k].reshape(1) for k in keys]))
      if redetection:
        ev = metrics.redetection_events(out['tracks'], None, target, occluded == 0,
                                        metrics.DIST_THRESHOLDS, pred_logits=logits)
        host = torch.empty(ev.shape, dtype=ev.dtype, pin_memory=True)
        host.copy_(ev, non_blocking=True)   # stream-ordered before the table's copy below
        events.append(host)
  if not rows:
    raise ValueError('evaluate: the dataset is empty')
  table = torch.stack([r.to(rows[0].device) for r in rows]).cpu().numpy()   # the one sync
  per_video = [{k: float(v) for k, v in zip(keys, row)} for row in table]
  if not redetection:
    return dataset_mean(per_video), per_video
  mean = dataset_mean(per_video)
  for m, host in zip(per_video, events):
    m.update({k: float(v) for k, v in metrics.redetection_metrics_from_events(host.numpy(), 1).items()})
  for k in per_video[0]:
    if k.startswith('AJ_RD'):
      vals = [{k: m[k]} for m in per_video if not np.isnan(m[k])]
      mean[k] = dataset_mean(vals)[k] if vals else np.float32(np.nan)
      mean[f'{k}/videos'] = len(vals)
  return mean, per_video


def dataset_mean(per_video):
  """{metric: np.float32} mean of per-video {metric: value} dicts as the reference's evaluation
  loop forms it: values rounded to float32, summed in list order in float32, divided by the count."""
  total = {k: np.float32(v) for k, v in per_video[0].items()}
  for m in per_video[1:]:
    total = {k: np.float32(total[k] + np.float32(m[k])) for k in total}
  return {k: np.float32(v / np.float32(len(per_video))) for k, v in total.items()}


def latex_table(mean_scalars):
  """The reference's two-line latex table of TAP-Vid (or PCK) scalars, values x 100 to 3
  significant digits."""
  if 'average_jaccard' in mean_scalars:
    fields = ['average_jaccard', 'average_pts_within_thresh', 'occlusion_accuracy']
    fields += [f'jaccard_{t}' for t in metrics.THRESHOLDS] + [f'pts_within_{t}' for t in metrics.THRESHOLDS]
    header = ' & '.join(['AJ', '$<\\delta^{x}_{avg}$', 'OA']
                        + [f'Jac. $\\delta^{{{i}}}$' for i in range(5)]
                        + [f'$<\\delta^{{{i}}}$' for i in range(5)])
  else:
    fields = [f'PCK@0.{i}' for i in range(1, 6)]
    header = ' & '.join(fields)
  return header + '\n' + ' & '.join(f'{float(np.asarray(mean_scalars[k] * 100)):.3}' for k in fields)


# ------------------------------------------------------------------------------ CLI
_READERS = {'davis': create_davis_dataset, 'kinetics': create_kinetics_dataset,
            'rgb_stacking': create_rgb_stacking_dataset, 'robotap': create_robotap_dataset}


def _model_kwargs(path):
  """pyramid_level / extra_convs of a torch state dict, from its key set and mixer width (a Haiku
  .npy tree is inferred by build_model itself)."""
  if str(path).endswith('.npy'):
    return {}
  from tapnet_b200 import schema  # pylint: disable=g-import-not-at-top
  sd = torch.load(path, map_location='cpu')
  extra = any(k.startswith('extra_convs.') for k in sd)
  din = int(sd['torch_pips_mixer.linear.weight'].shape[1])
  for level in range(4):
    if schema.mixer_input_dim(level) == din:
      return dict(pyramid_level=level, extra_convs=extra)
  raise ValueError(f'{path}: unexpected mixer input width {din}')


def _window_frames(v):
  if v == 'auto':
    return v
  if not v.isdigit() or int(v) < 1:
    raise argparse.ArgumentTypeError(f"expected an integer >= 1 or 'auto', got {v!r}")
  return int(v)


def main(argv=None):
  p = argparse.ArgumentParser(description='TAP-Vid evaluation of a TAPIR checkpoint on the GPU')
  p.add_argument('--dataset', required=True, choices=sorted(_READERS))
  p.add_argument('--path', required=True, help='the pickle (davis, rgb_stacking, robotap), the shard '
                 'directory (kinetics) or a directory of pickles (robotap)')
  p.add_argument('--checkpoint', required=True, help='torch state dict (.pt) or Haiku tree (.npy)')
  p.add_argument('--query-mode', default='strided', choices=_MODES)
  p.add_argument('--resolution', type=int, nargs=2, default=(256, 256), metavar=('H', 'W'))
  p.add_argument('--redetection', action='store_true',
                 help='add the AJ_RD re-detection metrics and, per key, the videos its mean is over')
  p.add_argument('--window-frames', type=_window_frames, default=None, metavar='N|auto',
                 help='track each clip in temporal windows of N core frames (auto: fit free memory)')
  a = p.parse_args(argv)
  from tapnet_b200 import tapir_model  # pylint: disable=g-import-not-at-top
  model = tapir_model.build_model(a.checkpoint, **_model_kwargs(a.checkpoint))
  mean, per_video = evaluate(model, _READERS[a.dataset](a.path, a.query_mode, resolution=tuple(a.resolution)),
                             a.query_mode, redetection=a.redetection, window_frames=a.window_frames)

  def clean(v):
    if isinstance(v, int):   # the AJ_RD means' video counts
      return v
    return None if np.isnan(v) else float(v)

  print(json.dumps(dict(dataset=a.dataset, query_mode=a.query_mode, resolution=list(a.resolution),
                        card=torch.cuda.get_device_name(), videos=len(per_video),
                        mean={k: clean(v) for k, v in mean.items()},
                        per_video=[{k: clean(v) for k, v in m.items()} for m in per_video])))
  print(latex_table(mean))


if __name__ == '__main__':
  main()
