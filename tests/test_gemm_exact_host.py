"""The exact-accumulator GEMM designs of tests/gemm_exact.py hold what they claim, the GPU cases
reach every epilogue path, and the emulation would notice the slips an epilogue rewrite could make.
CPU only."""
import numpy as np
import pytest
import torch

from tests import gemm_exact as E

CASES = {c.cid: c for c in E.CASES}


@pytest.mark.parametrize('cid', sorted(CASES))
def test_accumulator_is_exact_in_fp32(cid):
  d = CASES[cid].design()
  assert float(E.abs_sum_units(d).max()) < E.EXACT_UNITS
  # B carries no low planes: only the pairs (i, 0) are nonzero (tests/plane_pairs.py tells the
  # pair sets apart)
  assert not d.w_pl[1:].float().any()
  # acc is on its columns' grids and therefore held exactly by fp32
  scaled = d.acc * torch.exp2(d.units.double())[None, :]
  assert torch.equal(scaled, scaled.round())
  assert torch.equal(d.acc.float().double(), d.acc)
  if d.kind == 'S':
    assert torch.equal(d.acc, d.acc.round())
    for bias in (False, True):
      for resid in (False, True):
        assert np.abs(E.emulate(d, bias, resid)['out']).max() <= 1000


@pytest.mark.parametrize('cid', sorted(c.cid for c in E.CASES if c.P > 1))
def test_a_uses_its_second_plane(cid):
  assert E.plane1_fraction(CASES[cid].design()) > 0.15


@pytest.mark.parametrize('cid', sorted(c.cid for c in E.CASES if c.kind == 'R'))
def test_r_designs_are_order_sensitive(cid):
  assert E.order_sensitivity(CASES[cid].design()) >= 0.05


@pytest.mark.parametrize('cid', sorted(c.cid for c in E.CASES if c.kind == 'G'))
def test_g_designs_span_the_gelu_range(cid):
  d = CASES[cid].design()
  for bias in (False, True):
    v = E.pre_activation(d, bias)
    inner = v[np.abs(v) <= 12]
    assert inner.min() < -11 and inner.max() > 11 and inner.size > 0.8 * v.size
    # e^u overflows to inf (rcp gives 0) and flushes to 0 (the result is x)
    assert v.min() < -100 and v.max() > 100


def _coverage():
  """Every label E.reached gives, over the runs tests/test_gemm_exact_gpu.py makes."""
  seen = set()
  for c in E.CASES:
    for opts in c.sets:
      for ld_pad, offset in E.LAYOUTS.values():
        for bn in (64, 128):
          for splitk in ((False, True) if c.splitk else (False,)):
            seen |= E.reached(c.M, c.N, c.K, c.P, opts, c.conv, ld_pad, offset, bn, splitk)
  return seen


def test_every_full_tile_instantiation_is_reached():
  seen = _coverage()
  want = {f'full/{bn}/{E.set_name(s)}' for bn in (64, 128) for s in E.FULL_SETS}
  assert len(want) == 20
  assert want <= seen, sorted(want - seen)


def test_every_full_tile_option_set_also_reaches_the_general_loop():
  seen = _coverage()
  missing = [E.set_name(s) for s in E.FULL_SETS if 'general/' + E.set_name(s) not in seen]
  assert not missing, missing
  assert 'splitk_reduce/bias+resid+f32' in seen


def test_mirror_follows_the_dispatch_rules():
  gelu_planes = E.option_set(True, True, False, False, 2, False)
  f32 = E.option_set(True, False, True, True, 0, False)
  # aligned whole tiles take epilogue_full, the ragged last row / column tiles the general loop
  assert E.reached(1000, 256, 512, 2, gelu_planes, block_n=128) == \
      {'full/128/bias+gelu+planes2', 'general/bias+gelu+planes2'}
  assert E.reached(1024, 256, 512, 2, gelu_planes, block_n=128) == {'full/128/bias+gelu+planes2'}
  # an odd leading dimension or a 4-byte aligned output sends every tile to the general loop
  assert E.reached(1024, 256, 512, 2, gelu_planes, ld_pad=1) == {'general/bias+gelu+planes2'}
  assert E.reached(1024, 256, 512, 2, f32, offset=1) == {'general/bias+resid+f32'}
  assert E.reached(1024, 256, 512, 2, f32, ld_pad=2, offset=2, block_n=64) == {'full/64/bias+resid+f32'}
  # sets outside the table never take a whole-tile epilogue
  assert E.reached(1024, 256, 512, 2, E.option_set(True, True, False, True, 2, False)) == \
      {'general/bias+gelu+f32+planes2'}
  # the C = 64 -> 64 halo convolution runs 64-wide tiles of 8 x 16 pixels
  stats = E.option_set(True, False, True, True, 0, True)
  assert E.reached(None, 64, 576, 2, stats, conv=(1, 16, 8, 64)) == {'full/64/bias+resid+f32+stats'}
  assert E.choose_conv_tile(20, 24) == (32, 4) and E.choose_conv_tile(33, 13) == (16, 8)
  # split-K: 300 x 512 x 2048 fills 24 of 132 SMs with 128-wide tiles: five k-slices
  assert E.reached(300, 512, 2048, 2, f32, splitk=True) == \
      {'splitk_reduce/bias+resid+f32', 'full/128/f32', 'general/f32'}


@pytest.mark.parametrize('variant,cid,opts', [
    ('resid_first', 'plain_r_p2', (True, True, 0, False)),
    ('resid_first', 'splitk_r', (True, True, 0, False)),
    ('planes_rtz', 'plain_r_p1', (True, True, 2, False)),
    ('planes_rtz', 'plain_r_p3', (True, True, 3, False)),
    ('stats_before_resid', 'plain_s', (True, True, 0, True)),
    ('stats_before_resid', 'conv_s', (False, True, 0, True)),
    ('stats_before_resid', 'halo_s', (True, True, 0, True)),
])
def test_emulation_detects_epilogue_slips(variant, cid, opts):
  d = CASES[cid].design()
  bias, resid, out_P, stats = opts
  good = E.emulate(d, bias, resid, out_P, stats)
  bad = E.emulate(d, bias, resid, out_P, stats, variant=variant)
  if variant == 'resid_first':
    diff = (good['out'].view(np.int32) != bad['out'].view(np.int32)).mean()
  elif variant == 'planes_rtz':
    diff = (good['planes'].view(torch.int16) != bad['planes'].view(torch.int16)).any(0).double().mean()
  else:
    diff = (good['stats'] != bad['stats']).mean()
  assert diff > 0.05, diff


def test_split_rtz_is_a_different_rounding():
  v = torch.tensor([1 + 2 ** -8 + 2 ** -20, -(1 + 2 ** -7 + 2 ** -9)], dtype=torch.float32)
  assert not torch.equal(E.split_rtz(v, 1).view(torch.int16), E.split_like_kernel(v, 1).view(torch.int16))
  # both reconstruct v exactly with three planes
  for pl in (E.split_rtz(v, 3), E.split_like_kernel(v, 3)):
    assert torch.equal(pl.double().sum(0), v.double())



def test_gelu_reference_is_the_tanh_formula():
  a = torch.linspace(-4, 12, 4001, dtype=torch.float64)
  ref = E.gelu_reference(a)
  assert ((ref - E.gelu_exact(a)).abs() <= 1e-15 * (1 + ref.abs())).all()
  # where 1 + tanh cancels, the sigmoid form keeps its relative accuracy
  a = torch.tensor([-7.0, -9.0, -11.0], dtype=torch.float64)
  z = E.GELU_K * (a + 0.044715 * a ** 3)
  assert torch.allclose(E.gelu_reference(a), a * torch.exp(2 * z) / (1 + torch.exp(2 * z)), rtol=1e-14, atol=0)
