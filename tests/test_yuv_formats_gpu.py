"""-m gpu: YUV frames of every layout (P010 / P016, yuv420p10 / 12, YUV444 8 / 16-bit, YUYV, UYVY,
NV12, I420).  The conversion kernel equals the integer oracle on every 8-bit triple of the 4:2:2 and
4:4:4 layouts and on every 10-bit triple of the 4:2:0 ones; the same content in every layout gives
the same bytes; and every model path fed a layout equals, bit for bit, the same path fed the uint8
RGB frames the conversion produces, with the launch counts of NV12."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import synth  # noqa: E402
from tapnet_b200 import _lib, live, streaming  # noqa: E402
from tests.test_stages_gpu import get_model  # noqa: E402
from tests.test_tracker_sizes_gpu import _ingest_check  # noqa: E402
from tests.test_video_reader_gpu import _check  # noqa: E402
from tests.test_windowed_gpu import _assert_equal, _queries, _whole  # noqa: E402
from tests.test_yuv_formats_host import CHROMA, KR_KB, MATRICES  # noqa: E402
from tests.test_yuv_gpu import _assert_grids_equal  # noqa: E402

LAYOUTS = ['nv12', 'i420', 'p010', 'p016', 'yuv420p10', 'yuv420p12', 'yuv444', 'yuv444p16',
           'yuyv', 'uyvy']


def oracle16(Y16, U16, V16, matrix, full_range):
  """The 16-bit contract restated in torch int64 on the device: uint8 RGB [..., 3]."""
  cr, gu, gv, bu = CHROMA[(matrix, bool(full_range))]
  k, off = (256, 0) if full_range else (298, 4096)
  L = k * (Y16.long() - off) + 32768
  D, E = U16.long() - 32768, V16.long() - 32768
  rgb = torch.stack([(L + cr * E) >> 16, (L - gu * D - gv * E) >> 16, (L + bu * D) >> 16], -1)
  return rgb.clamp(0, 255).to(torch.uint8)


def float16(Y16, U16, V16, matrix, full_range):
  kr, kb = KR_KB[matrix]
  kg = 1.0 - kr - kb
  ys, cs = (1.0, 1.0) if full_range else (255.0 / 219.0, 255.0 / 224.0)
  L = (Y16.double() / 256 - (0 if full_range else 16)) * ys
  D, E = (U16.double() / 256 - 128) * cs, (V16.double() / 256 - 128) * cs
  return torch.stack([L + 2 * (1 - kr) * E, L - 2 * (1 - kb) * kb / kg * D - 2 * (1 - kr) * kr / kg * E,
                      L + 2 * (1 - kb) * D], -1).clamp(0, 255)


def make_layout(layout, Y, U, V, pad=0, **kw):
  """A clip of `layout` (a live.YUV_LAYOUTS name) from 16-bit-normalised sample planes (int64 on
  the device) Y [B, T, H, W] and U, V of the layout's chroma size, rows padded by `pad` samples.
  8-bit layouts take the high bytes, LSB-aligned layouts the top `bits` bits, MSB-aligned layouts
  the samples."""
  spec = live.YUV_LAYOUTS[layout]
  B, T, H, W = Y.shape
  sh = 8 if spec.dtype == torch.uint8 else (16 - spec.bits if spec.lsb_aligned else 0)

  def store(x):  # 16-bit samples >= 2^15 go into int16 as the same bits
    x = x >> sh
    buf = torch.zeros(*x.shape[:3], x.shape[3] + pad, *x.shape[4:], dtype=spec.dtype,
                      device=x.device)[:, :, :, :x.shape[3]]
    buf.copy_(x.to(torch.uint8) if spec.dtype == torch.uint8 else
              ((x + 32768) % 65536 - 32768).to(torch.int16))
    return buf

  if spec.form == 'semi':
    return spec.make(store(Y), store(torch.stack([U, V], -1)), **kw)
  if spec.form == 'planar':
    return spec.make(store(Y), store(U), store(V), **kw)
  # packed 4:2:2: Y0 U Y1 V (yuyv) or U Y0 V Y1 (uyvy) per pixel pair
  p = torch.zeros(B, T, H, 2 * W + pad, dtype=torch.uint8, device=Y.device)[..., :2 * W]
  yo, uo, vo = (0, 1, 3) if layout == 'yuyv' else (1, 0, 2)
  p[..., yo::2] = (Y >> 8).to(torch.uint8)
  p[..., uo::4] = (U >> 8).to(torch.uint8)
  p[..., vo::4] = (V >> 8).to(torch.uint8)
  return spec.make(p, **kw)


def shift_of(layout):
  return live.YUV_LAYOUTS[layout].chroma_shift


def quantise(layout, x):
  """16-bit samples as the layout stores them, normalised back to 16 bits."""
  spec = live.YUV_LAYOUTS[layout]
  keep = 8 if spec.dtype == torch.uint8 else (spec.bits if spec.lsb_aligned else 16)
  return (x >> (16 - keep)) << (16 - keep)


def random_clip(layout, B, T, H, W, seed, pad=0, **kw):
  """Random content in `layout`: (clip, 16-bit Y, U, V planes of what it stores)."""
  g = torch.Generator(device='cuda').manual_seed(seed)
  sx, sy = shift_of(layout)
  ch, cw = -(-H // (1 << sy)), -(-W // (1 << sx))
  Y, U, V = (quantise(layout, torch.randint(0, 65536, s, generator=g, device='cuda'))
             for s in ((B, T, H, W), (B, T, ch, cw), (B, T, ch, cw)))
  return make_layout(layout, Y, U, V, pad, **kw), (Y, U, V)


def planes_oracle(layout, Y, U, V, window, matrix, full_range):
  """RGB of the window from the stored samples: chroma sample (r >> sy, c >> sx), nearest."""
  sx, sy = shift_of(layout)
  y0, x0, h, w = window
  r = torch.arange(y0, y0 + h, device=Y.device)
  c = torch.arange(x0, x0 + w, device=Y.device)
  pick = lambda P, rr, cc: P[:, :, rr][:, :, :, cc]  # noqa: E731
  return oracle16(pick(Y, r, c), pick(U, r >> sy, c >> sx), pick(V, r >> sy, c >> sx), matrix,
                  full_range)


# ------------------------------------------------------------------------------ conversion
@pytest.mark.parametrize('layout', ['yuyv', 'uyvy', 'yuv444'])
def test_8bit_layouts_exact_on_every_triple(layout):
  """64 frames of 512^2 pixels hold all 2^24 8-bit triples once: pixel pair p carries the chroma
  pair p mod 2^16 and the two Y values 2 (p >> 16) and 2 (p >> 16) + 1."""
  F, S = 64, 512
  p = torch.arange(F * S * S // 2, device='cuda').view(1, F, S, S // 2)
  Yp = (2 * (p >> 16)).repeat_interleave(2, 3) + torch.arange(S, device='cuda') % 2
  Uc, Vc = (p & 0xffff) >> 8, p & 0xff
  if layout == 'yuv444':
    Uc, Vc = Uc.repeat_interleave(2, 3), Vc.repeat_interleave(2, 3)
  for matrix, full in MATRICES:
    f = make_layout(layout, Yp << 8, Uc << 8, Vc << 8, pad=40, matrix=matrix, full_range=full)
    got = live.yuv_to_rgb(f)
    assert torch.equal(got, planes_oracle(layout, Yp << 8, Uc << 8, Vc << 8, (0, 0, S, S), matrix,
                                          full)), (matrix, full)


@pytest.mark.parametrize('layout', ['p010', 'yuv420p10'])
@pytest.mark.parametrize('matrix,full_range', MATRICES)
def test_10bit_exact_on_every_triple(layout, matrix, full_range):
  """All 2^30 10-bit triples in 16 slices of 256 frames of 512^2: one chroma pair per 2x2 block,
  block b of the clip carries chroma pair b mod 2^20 and Y = 4 (b >> 20) + its position."""
  F, S = 256, 512
  q = ((torch.arange(S, device='cuda')[:, None] % 2) * 2 + torch.arange(S, device='cuda')[None] % 2)
  worst = 0.0
  for s in range(16):
    b = s * F * (S // 2) ** 2 + torch.arange(F * (S // 2) ** 2, device='cuda').view(1, F, S // 2, S // 2)
    c = b & 0xfffff
    U, V = (c >> 10) << 6, (c & 1023) << 6
    Y = ((4 * (b >> 20)).repeat_interleave(2, 2).repeat_interleave(2, 3) + q) << 6
    frames = make_layout(layout, Y, U, V, pad=24, matrix=matrix, full_range=full_range)
    got = live.yuv_to_rgb(frames)
    up = lambda P: P.repeat_interleave(2, 2).repeat_interleave(2, 3)  # noqa: E731
    assert torch.equal(got, oracle16(Y, up(U), up(V), matrix, full_range)), s
    worst = max(worst, float((got.double() - float16(Y, up(U), up(V), matrix, full_range)).abs().max()))
    del frames, got, b, c, U, V, Y
  assert worst <= 1.0, worst


@pytest.mark.parametrize('layout', ['p016', 'yuv444p16', 'yuv420p12', 'yuv420p10', 'yuyv', 'uyvy',
                                    'yuv444', 'nv12', 'i420'])
@pytest.mark.parametrize('matrix,full_range', MATRICES)
def test_random_samples_odd_windows_pitched_rows(layout, matrix, full_range):
  even = layout in ('yuyv', 'uyvy')
  W, win = (54, (3, 6, 31, 42)) if even else (53, (3, 5, 31, 41))
  clip, (Y, U, V) = random_clip(layout, 2, 3, 37, W, seed=LAYOUTS.index(layout), pad=13,
                                matrix=matrix, full_range=full_range, window=win)
  assert torch.equal(live.yuv_to_rgb(clip), planes_oracle(layout, Y, U, V, win, matrix, full_range))


def test_lsb_aligned_samples_ignore_the_bits_above():
  """yuv420p12: the 4 bits above the sample are masked off, as the contract states."""
  clip, (Y, U, V) = random_clip('yuv420p12', 1, 2, 30, 40, seed=5)
  want = live.yuv_to_rgb(clip)
  g = torch.Generator(device='cuda').manual_seed(6)
  for t in clip.buffers:
    t.bitwise_or_(torch.randint(0, 16, t.shape, generator=g, device='cuda', dtype=torch.int16) << 12)
  assert torch.equal(live.yuv_to_rgb(clip), want)


def test_every_layout_of_one_content_converts_to_the_same_bytes():
  """8-bit content as NV12, I420, YUV444 (chroma repeated), YUYV / UYVY (chroma repeated
  vertically), P016 and 16-bit YUV444 (samples shifted into the high byte)."""
  g = torch.Generator(device='cuda').manual_seed(7)
  B, T, H, W = 2, 3, 38, 54
  Y = torch.randint(0, 256, (B, T, H, W), generator=g, device='cuda') << 8
  U, V = (torch.randint(0, 256, (B, T, H // 2, W // 2), generator=g, device='cuda') << 8 for _ in range(2))
  win = (2, 4, 30, 40)
  want = live.yuv_to_rgb(make_layout('nv12', Y, U, V, window=win))
  rep = {(1, 1): lambda P: P, (1, 0): lambda P: P.repeat_interleave(2, 2),
         (0, 0): lambda P: P.repeat_interleave(2, 2).repeat_interleave(2, 3)}
  for layout in LAYOUTS:
    f = rep[shift_of(layout)]
    got = live.yuv_to_rgb(make_layout(layout, Y, f(U), f(V), pad=6, window=win))
    assert torch.equal(got, want), layout


def test_conversion_on_a_side_stream_and_in_a_cuda_graph():
  clip, _ = random_clip('p010', 1, 4, 72, 128, seed=8, window=(4, 8, 64, 96))
  want = live.yuv_to_rgb(clip)
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    got = live.yuv_to_rgb(clip)
  torch.cuda.current_stream().wait_stream(side)
  assert torch.equal(got, want)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    out = live.yuv_to_rgb(clip)
  other, _ = random_clip('p010', 1, 4, 72, 128, seed=9, window=(4, 8, 64, 96))
  for dst, src in zip(clip.buffers, other.buffers):
    dst.copy_(src)
  graph.replay()
  torch.cuda.synchronize()
  assert torch.equal(out, live.yuv_to_rgb(other))


def _tensors(x):
  """The tensors of a tracker output (tensors, or lists of per-stream tensors), flattened."""
  if isinstance(x, torch.Tensor):
    return [x]
  return [t for y in x for t in _tensors(y)]


# ------------------------------------------------------------------------------ model paths
@pytest.mark.parametrize('layout', LAYOUTS)
def test_feature_grids_bit_identical(layout):
  """The stem loader at the model's resolution (odd frame size for planar layouts, odd window
  origin) and the ingest resize path (480x640 and 720x1280 centre windows)."""
  model, _, _ = get_model()
  W, win = (264, (3, 4, 256, 256)) if layout in ('yuyv', 'uyvy') else (263, (3, 5, 256, 256))
  clip, _ = random_clip(layout, 1, 2, 261, W, seed=11, pad=8, window=win)
  _assert_grids_equal(model.get_feature_grids(clip, False),
                      model.get_feature_grids(live.yuv_to_rgb(clip), False))
  for H, W in ((480, 640), (720, 1280)):
    clip, _ = random_clip(layout, 1, 2, H, W, seed=12, matrix='bt709',
                          window=live.center_square_window(H, W))
    a = model.get_feature_grids(clip, False)
    assert len(a.resolutions) > 1
    _assert_grids_equal(a, model.get_feature_grids(live.yuv_to_rgb(clip), False))


@pytest.mark.parametrize('layout', ['p010', 'yuv420p12', 'yuv444p16', 'yuyv'])
def test_end_to_end_bit_identical(layout):
  model, _, _ = get_model()
  clip, _ = random_clip(layout, 1, 8, 256, 256, seed=13, matrix='bt2020')
  g = torch.Generator().manual_seed(5)
  q = torch.cat([torch.randint(0, 8, (1, 16, 1), generator=g).float(),
                 torch.rand(1, 16, 2, generator=g) * 255], -1).cuda()
  a = model(clip, q)
  b = model(live.yuv_to_rgb(clip), q)
  assert sorted(a) == sorted(b) and any(k.startswith('unrefined') for k in a)
  for k in a:
    if isinstance(a[k], (list, tuple)):
      assert len(a[k]) == len(b[k]) > 0
      for x, y in zip(a[k], b[k]):
        assert torch.equal(x, y), k
    else:
      assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize('layout', ['p010', 'yuyv', 'yuv444p16'])
@pytest.mark.parametrize('S', [1, 3])
def test_online_tracker_equals_uint8_tracker(layout, S):
  """6 graph-replayed steps at 256 x 320 (centre window), a retarget at step 2 and an add_points
  at step 4, against a uint8 tracker on the converted frames."""
  model, _, _ = get_model(causal=True)
  H, W, N = 256, 320, 8
  window = live.center_square_window(H, W)
  clip, _ = random_clip(layout, S, 6, H, W, seed=20 + S, window=window)

  def frame(t):
    return clip.map_buffers(lambda b: b[:, t:t + 1])

  g = torch.Generator().manual_seed(S)
  qp = torch.cat([torch.zeros(S, N, 1), torch.rand(S, N, 2, generator=g) * 255], -1).cuda()
  counts = N if S == 1 else [N] * S  # per-stream counts: add_points may change one
  a = streaming.OnlineTracker(model, H, W, counts, num_streams=S, yuv_layout=layout, window=window)
  b = streaming.OnlineTracker(model, 256, 256, counts, uint8_frames=True, num_streams=S)
  if S > 1:
    qp = list(qp)
  try:
    a.init(frame(0), qp)
    b.init(live.yuv_to_rgb(frame(0)), qp)
    for t in range(6):
      if t == 2:
        for trk in (a, b):
          trk.retarget(torch.tensor([[0.0, 100.5, 37.25]]), [3], stream=S - 1)
      if t == 4:
        for trk in (a, b):
          assert trk.add_points(torch.tensor([[0.0, 10.0, 10.0]]), stream=0) == [N]
      got = [x.clone() for x in _tensors(a.step(frame(t)))]
      want = _tensors(b.step(live.yuv_to_rgb(frame(t))))
      assert len(got) == len(want) and all(torch.equal(x, y) for x, y in zip(got, want)), t
      got, want = _tensors(a.last_logits), _tensors(b.last_logits)
      assert len(got) == len(want) and all(torch.equal(x, y) for x, y in zip(got, want)), t
    with pytest.raises(ValueError):
      a.step(frame(0).with_window(None))
    with pytest.raises(ValueError):
      a.step(live.yuv_to_rgb(frame(0)))
  finally:
    a.close()
    b.close()


def test_track_video_with_a_p010_reader():
  """A crop window of 256 x 384 out of 270 x 400 frames: a resampled and a direct pass."""
  model = get_model()[0]
  T = 97
  clip, _ = random_clip('p010', 1, T, 270, 400, seed=23, matrix='bt709', window=(6, 9, 256, 384))
  q = _queries([0, 96, 33, 34.5, 70, 12.25], 256, 384)
  want = _check(model, clip, q, read=lambda a, z: clip.map_buffers(lambda b: b[:, a:z]),
                window_frames=40, unrefined=True)
  _assert_equal(want, _whole(model, live.yuv_to_rgb(clip), q))


# ------------------------------------------------------------------------------ launch counts
@pytest.mark.parametrize('layout', [x for x in LAYOUTS if x != 'nv12'])
def test_launch_counts_equal_nv12(layout):
  model, _, _ = get_model(causal=True)
  lib = _lib.load()

  def count(fn):
    fn()  # workspaces, packed weights and graphs exist
    n0 = lib.tapir_launch_count()
    fn()
    return lib.tapir_launch_count() - n0

  for H, W, win in ((256, 256, None), (480, 640, live.center_square_window(480, 640))):
    ours, _ = random_clip(layout, 1, 2, H, W, seed=30, window=win)
    nv12, _ = random_clip('nv12', 1, 2, H, W, seed=30, window=win)
    n_ours = count(lambda: model.get_feature_grids(ours, False))
    assert n_ours == count(lambda: model.get_feature_grids(nv12, False)) > 0, (H, W)
    assert count(lambda: live.ingest_frames(ours, None, (128, 96))) == 1
  H, W, N = 720, 1280, 16
  window = live.center_square_window(H, W)
  counts = []  # init and the first step, which captures the step's graph
  qp = torch.rand(1, N, 3, device='cuda') * torch.tensor([0, 255, 255], device='cuda')
  for lay in (layout, 'nv12'):
    clip, _ = random_clip(lay, 1, 1, H, W, seed=31, window=window)
    trk = streaming.OnlineTracker(model, H, W, N, yuv_layout=lay, window=window)
    try:
      n0 = lib.tapir_launch_count()
      trk.init(clip, qp)
      trk.step(clip)
      counts.append(lib.tapir_launch_count() - n0)
    finally:
      trk.close()
  assert counts[0] == counts[1] > 0


# ------------------------------------------------------------------------------ mixed tables
def _uint16(clip):
  """The clip over torch.uint16 views of its 16-bit buffers (decoders hand back either type)."""
  return clip.map_buffers(lambda b: b.view(torch.uint16) if b.dtype == torch.int16 else b)


@pytest.mark.parametrize('oh,ow', [(256, 256), (96, 136)])
def test_ingest_multi_mixes_layouts_and_sample_sizes(oh, ow):
  """One tapir_ingest_frames_multi table of P010 (int16 and uint16 planes), yuv420p12, 16-bit
  YUV444, YUYV, UYVY and NV12 frames of different sizes and windows, and uint8 frames: each output
  row equals, bit for bit, its frame's own resample."""
  geo = [('p010', 270, 400, (6, 9, 256, 384)), ('yuv420p12', 181, 243, (1, 3, 150, 200)),
         ('yuv444p16', 120, 96, None), ('yuyv', 200, 300, (10, 20, 180, 240)),
         ('p010', 97, 131, (7, 11, 80, 100)), ('uyvy', 64, 64, (0, 2, 60, 60)),
         ('nv12', 240, 320, (0, 40, 240, 240)), ('p016', 50, 70, None)]
  sources = []
  for i, (layout, H, W, win) in enumerate(geo):
    clip, _ = random_clip(layout, 1, 1, H, W, seed=40 + i, pad=6, matrix='bt2020' if i % 2 else 'bt709',
                          window=win)
    if i == 4:
      clip = _uint16(clip)
    sources.append((clip, clip))
    if i % 3 == 0:  # a uint8 frame with pitched rows between the YUV ones
      g = torch.Generator(device='cuda').manual_seed(i)
      rgb = torch.randint(0, 256, (H, W + 5, 3), generator=g, device='cuda', dtype=torch.uint8)
      sources.append((rgb[:, :W], rgb[:, :W].contiguous()[None]))
  lib = _lib.load()
  n0 = lib.tapir_launch_count()
  _ingest_check(sources, oh, ow)
  assert lib.tapir_launch_count() - n0 == 1 + len(sources)  # one multi launch, one per frame alone


def test_uint16_planes_read_as_their_int16_bits():
  for layout in ('p010', 'yuv420p12', 'yuv444p16'):
    clip, _ = random_clip(layout, 1, 2, 37, 53, seed=50, window=(3, 5, 31, 41))
    assert torch.equal(live.yuv_to_rgb(_uint16(clip)), live.yuv_to_rgb(clip)), layout


@pytest.mark.parametrize('layout', ['p010', 'yuyv'])
def test_mixed_size_tracker_equals_uint8_on_converted_frames(layout):
  """Cropped streams of different frame sizes in one yuv_layout tracker (a direct-read group and a
  resampled group of two sizes, whose frames go through one multi-frame ingest table) track, bit
  for bit, as a uint8 tracker on the RGB windows.  P010 streams hand over uint16 planes, and the
  last stream gives P016 frames to the P010 tracker."""
  model, _, _ = get_model(causal=True)
  N, T = 8, 3
  geo = [((480, 640), (0, 80, 480, 480)), ((240, 320), (0, 40, 240, 240)), ((200, 200), None)]

  def frame(s, t):
    (H, W), win = geo[s]
    lay = 'p016' if layout == 'p010' and s == 2 else layout
    clip, _ = random_clip(lay, 1, 1, H, W, seed=10 * s + t, pad=4, window=win)
    return _uint16(clip) if layout == 'p010' else clip

  yuv = [[frame(s, t) for t in range(T)] for s in range(len(geo))]
  rgb = [[live.yuv_to_rgb(f)[0, 0] for f in fs] for fs in yuv]
  hws = [f[0].shape[:2] for f in rgb]
  q = torch.stack([synth.make_queries(N, T, *hw, seed=s, frame0_only=True)[0]
                   for s, hw in enumerate(hws)]).cuda()
  ty = streaming.OnlineTracker(model, [hw[0] for hw, _ in geo], [hw[1] for hw, _ in geo], N,
                               num_streams=3, yuv_layout=layout, window=[w for _, w in geo])
  tu = streaming.OnlineTracker(model, [h for h, _ in hws], [w for _, w in hws], N, num_streams=3,
                               uint8_frames=True)
  try:
    assert [g.streams for g in ty._groups] == [g.streams for g in tu._groups]
    assert any(not g.uniform and len(g.streams) > 1 for g in ty._groups)
    ty.init([fs[0] for fs in yuv], q)
    tu.init([fs[0] for fs in rgb], q)
    for t in range(T):
      a = [x.clone() for x in (*ty.step([fs[t] for fs in yuv]), *ty.last_logits)]
      b = [x.clone() for x in (*tu.step([fs[t] for fs in rgb]), *tu.last_logits)]
      assert len(a) == len(b)
      for x, y in zip(a, b):
        assert torch.equal(x, y), f'frame {t}'
    with pytest.raises(ValueError, match='yuv_layout'):
      ty.step([fs[0] for fs in rgb])
    other = 'nv12' if layout == 'p010' else 'p010'
    with pytest.raises(ValueError, match='yuv_layout'):
      ty.step([random_clip(other, 1, 1, *hw, seed=0, window=w)[0] for hw, w in geo])
  finally:
    ty.close()
    tu.close()
