"""-m gpu: the Lanczos resize kernel (tapir_resize_lanczos_u8) against PIL's outputs in
tests/golden/io_tapvid_eval.npz and the numpy oracle, bit for bit; the readers' device clips;
and `evaluate` against compute_tapvid_metrics on the reference's float clips."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import tapvid_oracle as O  # noqa: E402
from tapnet_b200 import _lib, metrics, tapvid  # noqa: E402
from tests.test_stages_gpu import get_model  # noqa: E402
from tests.test_tapvid_host import check_converted, golden, readers, write_pickles  # noqa: E402


def _random(seed, T, H, W):
  return np.random.default_rng(seed).integers(0, 256, (T, H, W, 3), dtype=np.uint8)


def test_fixture_numpy_and_cuda():
  g = golden()
  for i, (_, (h, w)) in enumerate(g['meta']['resize_cases']):
    src, ref = g[f'resize{i}_src'], g[f'resize{i}_out']
    got = tapvid.resize_video(src, (h, w))
    assert isinstance(got, np.ndarray) and got.dtype == np.uint8
    np.testing.assert_array_equal(got, ref)
    d = torch.from_numpy(src).cuda()
    got = tapvid.resize_video(d, (h, w))
    assert got.is_cuda and got.dtype == torch.uint8
    np.testing.assert_array_equal(got.cpu().numpy(), ref)


@pytest.mark.parametrize('case', [
    (1, 480, 854, 256, 256), (1, 720, 1280, 256, 256), (1, 1080, 1920, 256, 256),
    (1, 2160, 3840, 256, 256), (2, 100, 130, 256, 256), (2, 1, 1, 256, 256),
    (3, 64, 300, 64, 256), (3, 300, 64, 256, 64), (2, 48, 80, 48, 80), (3, 37, 53, 21, 90),
    (250, 72, 128, 64, 64)])
def test_kernel_equals_oracle(case):
  T, H, W, h, w = case
  src = _random(sum(case), T, H, W)
  got = tapvid.resize_video(torch.from_numpy(src).cuda(), (h, w)).cpu().numpy()
  np.testing.assert_array_equal(got, O.resize(src, h, w))


def test_side_stream_and_repeat():
  src = torch.from_numpy(_random(5, 4, 480, 854)).cuda()
  first = tapvid.resize_video(src, (256, 256))
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    outs = [tapvid.resize_video(src, (256, 256)) for _ in range(3)]
  torch.cuda.current_stream().wait_stream(side)
  for o in outs:
    assert torch.equal(o, first)
  assert torch.equal(tapvid.resize_video(src, (256, 256)), first)


def test_c_abi_bad_arguments_return_1():
  lib = _lib.load()
  T, H, W, h, w = 2, 48, 64, 24, 40
  src = torch.zeros(T, H, W, 3, dtype=torch.uint8, device='cuda')
  dst = torch.zeros(T, h, w, 3, dtype=torch.uint8, device='cuda')
  xb, xt = (torch.from_numpy(a).cuda() for a in _lib.lanczos_weights(W, w))
  yb, yt = (torch.from_numpy(a).cuda() for a in _lib.lanczos_weights(H, h))
  need = lib.tapir_resize_lanczos_u8_workspace_bytes(T, H, W, h, w)
  assert 0 < need <= T * H * w * 3
  ws = torch.zeros(need + 64, dtype=torch.uint8, device='cuda')
  p = _lib.ptr
  s = _lib.stream()

  def call(**kw):
    a = dict(src=p(src), dst=p(dst), frames=T, H=H, W=W, h=h, w=w, xb=p(xb), xt=p(xt), xk=xt.shape[1],
             yb=p(yb), yt=p(yt), yk=yt.shape[1], ws=p(ws), wsb=need)
    a.update(kw)
    return lib.tapir_resize_lanczos_u8(a['src'], a['dst'], a['frames'], a['H'], a['W'], a['h'], a['w'],
                                       a['xb'], a['xt'], a['xk'], a['yb'], a['yt'], a['yk'], a['ws'],
                                       a['wsb'], s)

  assert call() == 0
  torch.cuda.synchronize()
  bad = [dict(frames=0), dict(H=0), dict(w=-1), dict(h=70000), dict(src=None), dict(dst=None),
         dict(xb=None), dict(yt=None), dict(xk=xt.shape[1] + 1), dict(yk=1), dict(ws=None),
         dict(wsb=need - 1), dict(ws=ctypes.c_void_p(ws.data_ptr() + 8)),
         dict(dst=p(src)), dict(dst=ctypes.c_void_p(src.data_ptr() + 100)), dict(ws=p(src))]
  for kw in bad:
    assert call(**kw) == 1, kw
    assert lib.tapir_last_error()
  torch.cuda.synchronize()


def test_readers_device_clips_equal_reference(tmp_path):
  g = golden()
  meta = g['meta']

  def to_float(v):
    assert v.is_cuda and v.dtype == torch.uint8
    return v.cpu().numpy().astype(np.float32) / 255.0 * 2.0 - 1.0   # numpy: an IEEE division

  for reader, make_ds in readers(write_pickles(g, str(tmp_path)), meta).items():
    for mode in ('strided', 'first'):
      samples = list(make_ds(mode))
      assert len(samples) == meta['videos'][f'{reader}_{mode}']
      for n, sample in enumerate(samples):
        check_converted(g, f'{reader}_{mode}_{n}', sample[reader], video=to_float)


@pytest.mark.parametrize('mode', ['strided', 'first'])
def test_evaluate_equals_metrics_on_reference_clips(tmp_path, mode):
  g = golden()
  meta = g['meta']
  model = get_model()[0]
  davis, _, kinetics = write_pickles(g, str(tmp_path))
  for reader, ds in (('davis', tapvid.create_davis_dataset(davis, mode, resolution=tuple(meta['davis_resolution']))),
                     ('kinetics', tapvid.create_kinetics_dataset(kinetics, mode,
                                                                 resolution=tuple(meta['kinetics_resolution'])))):
    mean, per_video = tapvid.evaluate(model, ds, mode)
    assert len(per_video) == meta['videos'][f'{reader}_{mode}']
    for n, got in enumerate(per_video):
      pre = f'{reader}_{mode}_{n}'
      qp = torch.from_numpy(g[f'{pre}_query_points'].astype(np.float32)).cuda()
      with torch.no_grad():
        out = model(torch.from_numpy(g[f'{pre}_video']).cuda(), qp)
      want = metrics.compute_tapvid_metrics(qp, g[f'{pre}_occluded'], g[f'{pre}_target_points'], None,
                                            out['tracks'], mode,
                                            pred_logits=(out['occlusion'], out['expected_dist']))
      assert list(got) == list(want)
      for k, v in want.items():
        assert np.array_equal(np.float64(got[k]), v.item(), equal_nan=True), (pre, k, got[k], v.item())
    ref_mean = O.mean_scalars(per_video)
    assert all(mean[k] == ref_mean[k] or (np.isnan(mean[k]) and np.isnan(ref_mean[k])) for k in mean)
    assert tapvid.latex_table(mean) == tapvid.latex_table(ref_mean)
