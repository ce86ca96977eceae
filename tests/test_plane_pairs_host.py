"""The plane-pair designs of tests/plane_pairs.py hold what they claim: their models are exact in
fp32 whatever the summation order, and every plausible wrong pair set changes a large share of
the outputs and every output tile, so a kernel that sums one of them cannot pass
tests/test_plane_pairs_gpu.py by luck.  The cost-volume designs flip their arg-max as designed.
CPU only."""
import copy

import pytest
import torch

from tests import plane_pairs as PP

NAMES = sorted(PP.SPECS)
MIN_CHANGED = 0.99  # share of fp32 outputs every wrong set must change (the least is 0.998)
MODELS = ('tc', 'simt')


def _right(d, model):
  return PP.tc_pairs(d.P) if model == 'tc' else PP.all_pairs(d.P)


def _im2col(d):
  """A's planes as [P, M, K] (conv: 3 x 3 patches, zero padding, K ordered (ky, kx, c))."""
  if d.conv is None:
    return d.a_pl.float()
  P, (Fr, H, W, C) = d.P, d.conv
  x = torch.nn.functional.pad(d.a_pl.float(), (0, 0, 1, 1, 1, 1))
  taps = [x[:, :, ky:ky + H, kx:kx + W, :] for ky in range(3) for kx in range(3)]
  return torch.stack(taps, 4).reshape(P, Fr * H * W, 9 * C)


def _fp32_sum(a, w, pairs, order):
  """sum over pairs of A_i . B_j in fp32, one rounding per add, in the given order."""
  K = a.shape[2]
  acc = torch.zeros(a.shape[1], w.shape[1], dtype=torch.float32)
  if order == 'kblock_major':  # the wgmma kernels: k-block, then pair, then k
    for k0 in range(0, K, 64):
      for i, j in pairs:
        for k in range(k0, k0 + 64):
          acc += a[i, :, k, None] * w[j, None, :, k]
    return acc
  ks = range(K - 1, -1, -1) if order == 'k_descending' else range(K)
  if order == 'pair_major':
    for i, j in pairs:
      for k in ks:
        acc += a[i, :, k, None] * w[j, None, :, k]
    return acc
  for k in ks:
    for i, j in pairs:
      acc += a[i, :, k, None] * w[j, None, :, k]
  return acc


@pytest.mark.parametrize('name', NAMES)
def test_designs_are_exact(name):
  d = PP.design(name)
  for pl in (d.a_pl, d.w_pl):
    v = pl.float()
    assert torch.equal(v, v.round()) and v.abs().max() <= d.vmax
    # every plane is its own tensor: mostly nonzero, and no plane repeats another
    assert all((v[q] != 0).double().mean() > 0.8 for q in range(d.P))
    assert all(not torch.equal(v[p], v[q]) for p in range(d.P) for q in range(p))
  assert d.abs_bound() < PP.EXACT_UNITS
  # with at most 2^22 units every fp32 partial sum is exact: a few orders on some of the outputs
  a, w = _im2col(d), d.w_pl.float()
  rows = torch.linspace(0, d.M - 1, 48).long()
  a, cols = a[:, rows], torch.arange(min(d.N, 40))
  w = w[:, cols]
  for model in MODELS:
    want = d.model(_right(d, model))[rows][:, cols]
    for order in ('k_ascending', 'k_descending', 'pair_major', 'kblock_major'):
      got = _fp32_sum(a, w, _right(d, model), order)
      assert torch.equal(got.double(), want), (model, order)


@pytest.mark.parametrize('model', MODELS)
@pytest.mark.parametrize('name', NAMES)
def test_every_wrong_set_changes_most_outputs_and_every_tile(name, model):
  d = PP.design(name)
  right = PP.fp32_bits(d.model(_right(d, model)))
  sets = PP.wrong_sets(d.P, simt=model == 'simt')
  assert sets
  for set_name, pairs in sets.items():
    changed = PP.fp32_bits(d.model(pairs)) != right
    assert changed.mean() >= MIN_CHANGED, (set_name, changed.mean())
    assert PP.untouched_tiles(changed, d) == 0, set_name


def test_wrong_sets_name_the_likely_slips():
  tc3 = PP.wrong_sets(3)
  # mma_k_block at P = 3 skipping (1, 1); skipping (0, 2), so that B's plane 2 is never read; and
  # looping j < P instead of j < P - i
  for slip in ('drop (1, 1)', 'drop (0, 2) = B plane 2 read as zero', 'all P^2 pairs'):
    assert slip in tc3, sorted(tc3)
  assert sorted(tc3['all P^2 pairs']) == PP.all_pairs(3)
  assert 'add (1, 1) = all P^2 pairs' in PP.wrong_sets(2)
  assert 'drop (1, 1) = i + j < P' in PP.wrong_sets(2, simt=True)
  # both right sets are their own transposes: the transposed set is never a wrong one
  for P in (1, 2, 3):
    for right in (PP.tc_pairs(P), PP.all_pairs(P)):
      assert sorted((j, i) for i, j in right) == sorted(right)
    assert not any('transposed' in n for n in list(PP.wrong_sets(P)) + list(PP.wrong_sets(P, True)))
  assert len(PP.wrong_sets(3)) == 19 and len(PP.wrong_sets(3, simt=True)) == 21


def test_matching_sets_names_what_was_summed():
  d = PP.design('small_p3')
  sets = PP.wrong_sets(3)
  assert len(sets['drop (1, 1)']) == 5
  got = d.model(sets['drop (1, 1)']).float().numpy()
  assert PP.matching_sets(got, d, sets) == ['drop (1, 1)']
  assert PP.matching_sets(d.model(PP.tc_pairs(3)).float().numpy(), d, sets) == []


@pytest.mark.parametrize('conv', [None, (2, 5, 7, 64)])
def test_gapped_layout_holds_nan_outside_the_planes(conv):
  P = 3
  a = torch.arange(P * 70 * 64 if conv is None else P * 2 * 5 * 7 * 64).float().to(torch.bfloat16)
  a = a.view(P, 70, 64) if conv is None else a.view(P, *conv)
  buf, view = PP.gapped_a(a, conv, device='cpu')
  assert torch.equal(view.float(), a.float())
  assert view.stride(0) > a[0].numel() + PP.GAP_ROWS - 1
  if conv is None:
    assert view.stride(1) == 64 + PP.PAD_COLS and view.stride(1) % 8 == 0
  assert view.stride(0) % 8 == 0
  inside = torch.zeros(buf.numel(), dtype=torch.bool)
  idx = torch.arange(buf.numel()).as_strided(view.shape, view.stride())
  inside[idx.reshape(-1)] = True
  assert torch.isnan(buf[~inside].float()).all() and not torch.isnan(buf[inside].float()).any()
  assert int((~inside).sum()) >= P * PP.GAP_ROWS * 64


# ------------------------------------------------------------------------------ cost volume
# (counts, T, gh, gw): the batched form (counts = [N] * B) and ragged ones: counts around the
# 128-row m-tile, a clip of one query between two of more than 128, and 64 clips (one grouped call
# of TAPIR_MAX_RAGGED_CLIPS) mixing 1, 63, 64, 65 and 129
COUNTS_64 = [(1, 63, 64, 65, 129)[b % 5] for b in range(64)]
CV_DESIGNS = {
    '32x32': ([40, 40], 2, 32, 32),
    '25x39': ([40, 40], 3, 25, 39),
    'ragged5_32x32': ([1, 40, 127, 128, 129], 3, 32, 32),
    'ragged3_25x39': ([200, 1, 129], 1, 25, 39),
    'ragged64_32x32': (COUNTS_64, 1, 32, 32),
}


@pytest.fixture(scope='module', params=sorted(CV_DESIGNS))
def cv(request):
  return PP.CvDesign(*CV_DESIGNS[request.param])


def test_cv_values_split_as_designed():
  pl = lambda v: PP.split_like_kernel(torch.tensor([v], dtype=torch.float32), 3)[:, 0].double().tolist()  # noqa: E731
  assert pl(PP.Q_PROBE) == [1.0, 2.0 ** -9, 2.0 ** -18]
  assert pl(PP.G_A) == [32.0, 2.0 ** -5, 2.0 ** -15]
  assert pl(PP.G_B) == [28.0, 3 * 2.0 ** -6, 0.0]
  q, g = pl(PP.Q_PROBE), pl(PP.G_A)
  assert {(i, j): q[i] * g[j] for i, j in PP.tc_pairs(3)} == PP.PAIR_TERMS
  for kind in PP.CV_KINDS:
    e = PP.cv_offsets(kind)
    if e is not None:  # bf16-exact: only the (0, 0) pair reads them
      assert torch.equal(e.to(torch.bfloat16).float(), e)


def test_cv_design_picks_its_winner(cv):
  heat = cv.heat(PP.tc_pairs(3))
  # the fp32 sums and the head's +-64 are exact
  assert torch.equal(heat.double(), cv.heat(PP.tc_pairs(3), torch.float64))
  assert torch.equal(PP.CvDesign.argmax(heat), cv.winner())
  top = heat.topk(2, -1).values
  assert ((top[..., 0] - top[..., 1]) >= PP.CV_MARGIN).all()
  # the cells outside the candidates are far below them
  rest = heat.clone()
  for c in (cv.cell_a, cv.cell_b):
    rest.scatter_(-1, c[..., None], float('-inf'))
  assert rest.max() <= 0 and top[..., 1].min() >= 28
  # every kind is on every clip of at least one map per kind, at both index orders of its
  # candidates
  for k in range(len(PP.CV_KINDS)):
    m = cv.kind == k
    for b, n in enumerate(cv.counts):
      if min(n, PP.CV_GROUPS) * cv.T >= len(PP.CV_KINDS):
        assert m[cv.clip == b].any(), (b, PP.CV_KINDS[k])
    assert (cv.cell_a[m] < cv.cell_b[m]).any() and (cv.cell_a[m] > cv.cell_b[m]).any()


def test_cv_each_pair_flips_its_maps(cv):
  sets = PP.wrong_sets(3)
  for pair in PP.tc_pairs(3):
    name = next(n for n in sets if n.split(' = ')[0] == f'drop {pair}')
    am = PP.CvDesign.argmax(cv.heat(sets[name]))
    mine = cv.kind == PP.CV_KINDS.index(f'drop {pair}')
    assert (am[mine] == cv.cell_b[mine]).all(), pair


# the wrong sets the cost-volume designs must see: all but the added pairs, whose terms are
# below fp32's resolution at the designs' magnitude
CV_UNSEEN = ('add (1, 2)', 'add (2, 1)', 'add (2, 2)', 'all P^2 pairs')


def test_cv_designs_see_every_wrong_set_but_the_added_pairs(cv):
  win = cv.winner()
  for name, pairs in PP.wrong_sets(3).items():
    flipped = int((PP.CvDesign.argmax(cv.heat(pairs)) != win).sum())
    if name in CV_UNSEEN:
      assert flipped == 0, name
    else:
      assert flipped >= 2 * cv.B, (name, flipped)


def test_cv_queries_past_64_repeat_their_map(cv):
  """Query n of a clip reads channel group n mod 64: its features and map are query n mod 64's."""
  heat = cv.heat(PP.tc_pairs(3))
  q0 = 0
  for n in cv.counts:
    for r in range(PP.CV_GROUPS, n):
      src = q0 + r % PP.CV_GROUPS
      assert torch.equal(cv.qf[q0 + r], cv.qf[src]) and torch.equal(heat[q0 + r], heat[src])
    q0 += n


def test_cv_another_clips_grid_moves_maps_of_every_clip(cv):
  """A clip whose queries read the next clip's grid rows (a wrong B offset in the grouped GEMM)
  picks another cell on at least one map of every clip: each clip has its own candidate cells."""
  if cv.B < 2:
    pytest.skip('one clip')
  other = copy.copy(cv)
  other.grid = cv.grid.roll(-1, 0)
  moved = PP.CvDesign.argmax(other.heat(PP.tc_pairs(3))) != cv.winner()
  for b in range(cv.B):
    assert moved[cv.clip == b].any(), b


def test_cv_simt_all_pairs_keep_the_winner(cv):
  """The SIMT kernel sums a b with a, b the planes' fp32 sums: its products round (by at most
  2^-19 near 32, half an ulp there) and it adds the pairs the tensor cores leave out (at most
  2^-22).  Every kind's margin of 2^-16 holds through both, on the host model of its FMA chain."""
  heat = cv.heat_simt()
  assert torch.equal(PP.CvDesign.argmax(heat), cv.winner())
  top = heat.topk(2, -1).values
  assert ((top[..., 0] - top[..., 1]) >= PP.CV_MARGIN).all()
