"""TAP-Vid evaluation front end without a GPU: the C ABI's Lanczos tables against the numpy oracle,
the oracle against PIL (fixture and, when Pillow imports, directly), the query samplers and the
dataset readers against the reference's outputs in tests/golden/io_tapvid_eval.npz, latex_table
and the dataset mean, and argument checks that fire before any CUDA call."""
import json
import os
import pickle

import numpy as np
import pytest

from oracle import tapvid_oracle as O
from tapnet_b200 import _lib, tapvid

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'io_tapvid_eval.npz')
OUTS = (1, 3, 64, 255, 256, 257, 512, 720)


def golden():
  g = dict(np.load(GOLDEN))
  g['meta'] = json.loads(bytes(g['meta']).decode())
  return g


def write_pickles(g, d):
  """The fixture's seeded DAVIS, RGB-Stacking and Kinetics pickles, written under directory d;
  returns (davis path, robotics path, kinetics directory)."""
  meta = g['meta']
  davis = {n: {k: g[f'pkl_davis_{n}_{k}'] for k in ('video', 'points', 'occluded')} for n in meta['davis']}
  robotics = [{k: g[f'pkl_robotics_0_{k}'] for k in ('video', 'points', 'occluded')}]
  paths = (os.path.join(d, 'davis.pkl'), os.path.join(d, 'robotics.pkl'), d)
  for p, obj in zip(paths, (davis, robotics)):
    with open(p, 'wb') as f:
      pickle.dump(obj, f)
  for j, shard in enumerate(meta['kinetics']):
    raw, off = g[f'pkl_kinetics_{shard}_jpeg'].tobytes(), g[f'pkl_kinetics_{shard}_jpeg_offsets']
    ex = {'video': [raw[a:b] for a, b in zip(off[:-1], off[1:])],
          'points': g[f'pkl_kinetics_{shard}_points'], 'occluded': g[f'pkl_kinetics_{shard}_occluded']}
    with open(os.path.join(d, f'{shard}.pkl'), 'wb') as f:
      pickle.dump([ex] if j == 0 else {'v': ex}, f)
  return paths


def readers(paths, meta):
  davis, robotics, kinetics = paths
  return {
      'davis': lambda mode: tapvid.create_davis_dataset(davis, mode, resolution=tuple(meta['davis_resolution'])),
      'robotics': lambda mode: tapvid.create_rgb_stacking_dataset(robotics, mode, resolution=(16, 24)),
      'kinetics': lambda mode: tapvid.create_kinetics_dataset(kinetics, mode,
                                                              resolution=tuple(meta['kinetics_resolution'])),
  }


def check_converted(g, prefix, converted, video=None):
  """converted equals the fixture's reference sample `prefix` in keys, values and dtypes (the
  video by `video(converted['video'])`, or skipped when None)."""
  want = {k[len(prefix) + 1:] for k in g if k.startswith(prefix + '_')}
  assert set(converted) == want
  for k, v in converted.items():
    ref = g[f'{prefix}_{k}']
    if k == 'video':
      if video is not None:
        got = video(v)
        assert got.dtype == ref.dtype and got.shape == ref.shape
        np.testing.assert_array_equal(got, ref)
      continue
    assert v.dtype == ref.dtype and v.shape == ref.shape, (prefix, k, v.dtype, ref.dtype)
    np.testing.assert_array_equal(v, ref)


@pytest.mark.parametrize('out_size', OUTS)
def test_c_weights_equal_oracle(out_size):
  for in_size in range(1, 1101):
    bounds, taps = _lib.lanczos_weights(in_size, out_size)
    ob, ot = O.lanczos_weights(in_size, out_size)
    assert bounds.dtype == np.int32 and taps.dtype == np.int32
    np.testing.assert_array_equal(bounds, ob, err_msg=f'{in_size} -> {out_size}')
    np.testing.assert_array_equal(taps, ot, err_msg=f'{in_size} -> {out_size}')


def test_weights_of_large_ratios():
  # 2160 x 3840 -> 256^2: 53 taps per output row, 91 per output column
  assert _lib.lanczos_weights(2160, 256)[1].shape == (256, 53)
  assert _lib.lanczos_weights(3840, 256)[1].shape == (256, 91)
  for n_in, n_out in ((2160, 256), (3840, 256), (1, 256), (65535, 1)):
    b, t = _lib.lanczos_weights(n_in, n_out)
    ob, ot = O.lanczos_weights(n_in, n_out)
    np.testing.assert_array_equal(b, ob)
    np.testing.assert_array_equal(t, ot)


def test_oracle_equals_fixture_pil():
  g = golden()
  assert g['meta']['pillow']
  for i, ((H, W), (h, w)) in enumerate(g['meta']['resize_cases']):
    src, ref = g[f'resize{i}_src'], g[f'resize{i}_out']
    assert src.shape[1:3] == (H, W) and ref.shape[1:3] == (h, w)
    np.testing.assert_array_equal(O.resize(src, h, w), ref, err_msg=f'{(H, W)} -> {(h, w)}')


def test_oracle_equals_pil_on_random_sizes():
  Image = pytest.importorskip('PIL.Image')
  rng = np.random.default_rng(3)
  for _ in range(12):
    H, W, h, w = (int(v) for v in rng.integers(1, 160, 4))
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    ref = np.asarray(Image.fromarray(img).resize((w, h), resample=Image.Resampling.LANCZOS))
    np.testing.assert_array_equal(O.resize(img, h, w), ref, err_msg=f'{(H, W)} -> {(h, w)}')


def test_samplers_equal_fixture():
  g = golden()
  ex = {k: g[f'pkl_davis_bear_{k}'] for k in ('video', 'points', 'occluded')}
  pts = ex['points'] * np.array([48, 36])
  check_converted(g, 'stride3', tapvid.sample_queries_strided(ex['occluded'], pts, ex['video'], query_stride=3),
                  video=lambda v: v)


def test_readers_equal_fixture(tmp_path, monkeypatch):
  """Keys, dtypes, values and video order of every reader in both query modes; the clip is
  resized here by the numpy oracle (the device clip is checked by test_tapvid_gpu.py)."""
  g = golden()
  meta = g['meta']

  def host_clip(frames, resolution, staging):
    frames = np.asarray(frames)
    if resolution is not None and tuple(resolution) != frames.shape[1:3]:
      frames = O.resize(frames, *resolution)
    return frames

  monkeypatch.setattr(tapvid, '_clip', host_clip)
  for reader, make_ds in readers(write_pickles(g, str(tmp_path)), meta).items():
    for mode in ('strided', 'first'):
      samples = list(make_ds(mode))
      assert len(samples) == meta['videos'][f'{reader}_{mode}']
      for n, sample in enumerate(samples):
        assert list(sample) == [reader]
        check_converted(g, f'{reader}_{mode}_{n}', sample[reader],
                        video=lambda v: v[None].astype(np.float32) / 255.0 * 2.0 - 1.0
                        if v.ndim == 4 else v.astype(np.float32) / 255.0 * 2.0 - 1.0)


def test_latex_table_equals_fixture():
  g = golden()
  keys = g['meta']['latex_keys']
  tables = [str(t) for t in g['latex_tables']]
  for i in range(4):
    assert tapvid.latex_table(dict(zip(keys, g[f'latex{i}_values']))) == tables[i]
  pck = {f'PCK@0.{i + 1}': v for i, v in enumerate(g['latex_pck_values'])}
  assert tapvid.latex_table(pck) == tables[4]


def test_dataset_mean_equals_restatement():
  rng = np.random.default_rng(8)
  keys = ['average_jaccard', 'occlusion_accuracy', 'jaccard_1']
  for videos in (1, 2, 7, 30):
    per_video = [{k: float(v) for k, v in zip(keys, rng.uniform(0, 1, len(keys)))} for _ in range(videos)]
    got, want = tapvid.dataset_mean(per_video), O.mean_scalars(per_video)
    assert list(got) == keys
    for k in keys:
      assert got[k].dtype == np.float32 and got[k] == want[k]
  # float32 rounding of each video's value matters: a float64 mean can differ
  per_video = [{'a': 0.1}, {'a': 0.2}, {'a': 0.7}]
  assert tapvid.dataset_mean(per_video)['a'] == (np.float32(0.1) + np.float32(0.2) + np.float32(0.7)) / np.float32(3)


def test_bad_inputs_raise_before_cuda(tmp_path):
  good = np.zeros((2, 8, 8, 3), np.uint8)
  with pytest.raises(ValueError, match='uint8'):
    tapvid.resize_video(good.astype(np.float32), (4, 4))
  with pytest.raises(ValueError, match=r'\[T, H, W, 3\]'):
    tapvid.resize_video(good[..., :2], (4, 4))
  with pytest.raises(ValueError, match=r'\[T, H, W, 3\]'):
    tapvid.resize_video(good[0], (4, 4))
  with pytest.raises(ValueError, match='outside'):
    tapvid.resize_video(good, (0, 4))
  with pytest.raises(ValueError, match='outside'):
    tapvid.resize_video(good, (4, 70000))
  with pytest.raises(ValueError, match='outside'):
    _lib.lanczos_weights(0, 5)
  assert _lib.load().tapir_resize_lanczos_u8_workspace_bytes(1, 0, 8, 4, 4) == 0
  p = tmp_path / 'x.pkl'
  p.write_bytes(pickle.dumps({}))
  with pytest.raises(ValueError, match='query mode'):
    next(tapvid.create_davis_dataset(str(p), 'middle'))
  with pytest.raises(NotImplementedError):
    next(tapvid.create_davis_dataset(str(p), full_resolution=True))
  with pytest.raises(ValueError, match='query mode'):
    next(tapvid.create_kinetics_dataset(str(tmp_path), 'middle'))
  with pytest.raises(ValueError, match='query mode'):
    tapvid.evaluate(None, [], 'middle')
  with pytest.raises(ValueError, match='ever visible'):
    tapvid.sample_queries_first(np.ones((2, 4), bool), np.zeros((2, 4, 2)), good)
