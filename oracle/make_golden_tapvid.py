"""TEST INFRASTRUCTURE - generates tests/golden/io_tapvid_eval.npz from the reference's own
TAP-Vid evaluation front end (tapnet/tapvid/evaluation_datasets.py).

Run in the build container only (needs /root/reference and Pillow):
    python -m oracle.make_golden_tapvid

The module imports TensorFlow, tensorflow_datasets and mediapy, so, as in make_golden_io, its
FunctionDefs are compiled unmodified into a scope that provides `tf.io.gfile.GFile = open`,
`tf.io.gfile.glob` = sorted glob.glob, `media.resize_video` = PIL Lanczos on each uint8 frame
(what mediapy does with uint8 RGB frames), `Image`, `io`, `pickle` and `path`.  The fixture holds
the seeded pickles' arrays (Kinetics JPEG bytes as one uint8 array with offsets), the readers'
outputs for both query modes, `latex_table` strings, and PIL's Lanczos outputs over a size matrix.
"""
import glob
import io
import json
import os
import pickle
import tempfile
import types
from os import path
from typing import Iterable, Mapping, Optional, Tuple, Union

import numpy as np
import PIL
from PIL import Image

from oracle import reference_loader
from oracle.make_golden_io import GOLDEN_DIR, reference_functions

# (H, W) -> (h, w): up, down, one axis, identity, 1-pixel sides, ratios up to 15x
RESIZE_CASES = [((16, 24), (40, 56)), ((90, 120), (32, 40)), ((30, 64), (30, 21)),
                ((64, 30), (17, 30)), ((20, 20), (20, 20)), ((1, 1), (5, 7)), ((1, 37), (4, 1)),
                ((23, 1), (1, 9)), ((15, 150), (1, 10)), ((4, 3), (60, 45)), ((37, 53), (21, 90))]
DAVIS_RES = (16, 24)
KINETICS_RES = (20, 28)
FUNCTIONS = ['resize_video', 'latex_table', 'sample_queries_strided', 'sample_queries_first',
             'create_davis_dataset', 'create_rgb_stacking_dataset', 'create_kinetics_dataset']


def pil_resize_video(video, output_size):
  h, w = output_size
  return np.stack([np.asarray(Image.fromarray(f).resize((w, h), resample=Image.Resampling.LANCZOS))
                   for f in video])


def reference_scope():
  gfile = types.SimpleNamespace(GFile=open, glob=lambda p: sorted(glob.glob(p)))
  scope = dict(np=np, Image=Image, io=io, pickle=pickle, path=path,
               tf=types.SimpleNamespace(io=types.SimpleNamespace(gfile=gfile)),
               media=types.SimpleNamespace(resize_video=pil_resize_video), tfds=None,
               Iterable=Iterable, Mapping=Mapping, Optional=Optional, Tuple=Tuple, Union=Union)
  scope['DatasetElement'] = Mapping[str, Mapping[str, Union[np.ndarray, str]]]
  fns = reference_functions('tapnet/tapvid/evaluation_datasets.py', FUNCTIONS, scope)
  return dict(zip(FUNCTIONS, fns))


def _smooth_frames(rng, T, H, W):
  """Frames with some spatial structure (so that JPEG round trips and resizes are not noise)."""
  y, x = np.mgrid[0:H, 0:W]
  base = np.stack([(x * 7 + y * 3) % 256, (x * 2 + y * 9) % 256, (x * y) % 256], -1)
  noise = rng.integers(0, 40, (T, H, W, 3))
  return ((base[None] + noise + np.arange(T)[:, None, None, None] * 11) % 256).astype(np.uint8)


def _tracks(rng, N, T):
  """float32 points in [0, 1] and bool occlusion with: track 0 occluded on every stride frame
  (0, 5, 10, ...) but visible elsewhere, track 1 never visible, the others random."""
  points = rng.uniform(0, 1, (N, T, 2)).astype(np.float32)
  occluded = rng.uniform(size=(N, T)) < 0.3
  occluded[0] = False
  occluded[0, ::5] = True
  occluded[1] = True
  occluded[2, :3] = True   # first visible frame after the start
  return points, occluded


def make():
  ref = reference_scope()
  rng = np.random.default_rng(23)
  out, meta = {}, {'pillow': PIL.__version__, 'resize_cases': RESIZE_CASES}

  for i, ((H, W), (h, w)) in enumerate(RESIZE_CASES):
    src = rng.integers(0, 256, (2, H, W, 3), dtype=np.uint8)
    out[f'resize{i}_src'] = src
    out[f'resize{i}_out'] = ref['resize_video'](src, (h, w))

  # DAVIS: dict of two videos (T = 12 and 7, not multiples of 5)
  davis = {}
  for name, (T, H, W) in (('bear', (12, 36, 48)), ('goat', (7, 30, 40))):
    points, occluded = _tracks(rng, 6, T)
    davis[name] = {'video': _smooth_frames(rng, T, H, W), 'points': points, 'occluded': occluded}
  # RGB-Stacking: list of one example already at its evaluation size (no resize)
  T, H, W = 8, 16, 24
  points, occluded = _tracks(rng, 5, T)
  robotics = [{'video': _smooth_frames(rng, T, H, W), 'points': points, 'occluded': occluded}]
  # Kinetics: two shards (a list and a dict) of JPEG-encoded videos
  kinetics = {}
  for shard, (T, H, W) in (('0000_of_0010', (6, 24, 32)), ('0001_of_0010', (11, 18, 30))):
    frames = []
    for f in _smooth_frames(rng, T, H, W):
      buf = io.BytesIO()
      Image.fromarray(f).save(buf, format='JPEG', quality=90)
      frames.append(buf.getvalue())
    points, occluded = _tracks(rng, 6, T)
    kinetics[shard] = {'video': frames, 'points': points, 'occluded': occluded}

  for name, ex in davis.items():
    for k, v in ex.items():
      out[f'pkl_davis_{name}_{k}'] = v
  for k, v in robotics[0].items():
    out[f'pkl_robotics_0_{k}'] = v
  for shard, ex in kinetics.items():
    lens = np.array([len(b) for b in ex['video']])
    out[f'pkl_kinetics_{shard}_jpeg'] = np.frombuffer(b''.join(ex['video']), np.uint8)
    out[f'pkl_kinetics_{shard}_jpeg_offsets'] = np.concatenate([[0], np.cumsum(lens)])
    out[f'pkl_kinetics_{shard}_points'] = ex['points']
    out[f'pkl_kinetics_{shard}_occluded'] = ex['occluded']
  meta.update(davis=list(davis), kinetics=list(kinetics), davis_resolution=DAVIS_RES,
              kinetics_resolution=KINETICS_RES)

  with tempfile.TemporaryDirectory() as tmp:
    with open(os.path.join(tmp, 'davis.pkl'), 'wb') as f:
      pickle.dump(davis, f)
    with open(os.path.join(tmp, 'robotics.pkl'), 'wb') as f:
      pickle.dump(robotics, f)
    for j, (shard, ex) in enumerate(kinetics.items()):
      with open(os.path.join(tmp, f'{shard}.pkl'), 'wb') as f:
        pickle.dump([ex] if j == 0 else {'v': ex}, f)
    readers = {
        'davis': lambda mode: ref['create_davis_dataset'](os.path.join(tmp, 'davis.pkl'), mode,
                                                          resolution=DAVIS_RES),
        'robotics': lambda mode: ref['create_rgb_stacking_dataset'](
            os.path.join(tmp, 'robotics.pkl'), mode, resolution=(16, 24)),
        'kinetics': lambda mode: ref['create_kinetics_dataset'](tmp, mode, resolution=KINETICS_RES),
    }
    counts = {}
    for reader, make_ds in readers.items():
      for mode in ('strided', 'first'):
        n = 0
        for n, sample in enumerate(make_ds(mode)):
          (key,) = sample.keys()
          assert key == reader, key
          for k, v in sample[key].items():
            out[f'{reader}_{mode}_{n}_{k}'] = np.asarray(v)
        counts[f'{reader}_{mode}'] = n + 1
    meta['videos'] = counts

  # the samplers with a non-default stride
  ex = davis['bear']
  pts = ex['points'] * np.array([48, 36])
  for k, v in ref['sample_queries_strided'](ex['occluded'], pts, ex['video'], query_stride=3).items():
    out[f'stride3_{k}'] = np.asarray(v)

  # latex_table on float32 means (as the evaluation loop forms them) and on PCK scalars
  keys = ['average_jaccard', 'average_pts_within_thresh', 'occlusion_accuracy'] + \
      [f'{p}_{t}' for p in ('jaccard', 'pts_within') for t in (1, 2, 4, 8, 16)]
  tables = []
  for i in range(4):
    vals = rng.uniform(0, 1, len(keys)).astype(np.float32)
    if i == 1:
      vals[:3] = [0.0, 1.0, 0.12345]
    out[f'latex{i}_values'] = vals
    tables.append(ref['latex_table'](dict(zip(keys, vals))))
  pck = rng.uniform(0, 1, 5)
  out['latex_pck_values'] = pck
  tables.append(ref['latex_table']({f'PCK@0.{i + 1}': v for i, v in enumerate(pck)}))
  out['latex_tables'] = np.array(tables)
  meta['latex_keys'] = keys

  out['meta'] = np.frombuffer(json.dumps(meta).encode(), np.uint8)
  dst = os.path.join(GOLDEN_DIR, 'io_tapvid_eval.npz')
  np.savez_compressed(dst, **out)
  print(dst, os.path.getsize(dst), 'bytes,', len(out), 'arrays')


if __name__ == '__main__':
  reference_loader.load()
  make()
