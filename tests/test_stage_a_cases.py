"""The designed stage-A cost maps can catch the bugs they target (CPU only, float64 reference).

tests/test_stage_a_gpu.py runs these designs through the two track heads.  Here each family is
checked on its own: tie maps really tie, the radius plateau really moves the point when the
d^2 == 25 cells are counted, the query times really separate rint from round-half-away, and the
saturated maps really underflow exp in fp32."""
import numpy as np
import pytest
import torch

from tests import stage_a_designs as D

SIZES = ((32, 32),) + D.GENERIC_SIZES


def _sd64(kind):
  return {k: v.double() for k, v in D.head_state_dict(kind).items()}


def _maps(ds):
  return torch.tensor(np.stack([d.map for d in ds]))


@pytest.mark.parametrize('gh,gw', SIZES)
def test_design_values_are_exact_in_bf16(gh, gw):
  for d in D.designs(gh, gw):
    m = torch.from_numpy(d.map)
    assert torch.equal(m.to(torch.bfloat16).float(), m), d.name
    assert torch.equal(m * 8, (m * 8).round()) and m.abs().max() <= 32, d.name


@pytest.mark.parametrize('kind', D.HEAD_KINDS)
def test_tie_designs_tie_exactly_at_every_level(kind):
  """Every designed tie has two exactly equal maximal probabilities in float64, the lower index
  first.  Together the tie maps reach every tie level of every head's pixel-to-thread mapping:
  inside a thread, across lanes and across warps (the synthetic head needs two separated bumps,
  which never share a thread of the 32 x 32 head)."""
  sd64 = _sd64(kind)
  covered = set()
  for gh, gw in SIZES:
    ds = [d for d in D.designs(gh, gw) if kind in d.tie_heads]
    for temp in D.TEMPERATURES if ds else ():
      heat, _ = D.heat_fp64(sd64, _maps(ds), float(np.float32(temp)))
      prob = torch.softmax(heat, -1)
      for d, p in zip(ds, prob):
        tied = (p == p.max()).nonzero().flatten().tolist()
        assert len(tied) >= 2, (gh, gw, temp, d.name)
        a, b = tied[:2]
        assert int(torch.argmax(p)) == a
        assert (a, b) == d.pair, (gh, gw, temp, d.name, (a, b))
        if d.family == 'tie':
          for head in D.mappings(gh, gw):
            covered.add((head, D.tie_level(head, gh, gw, a, b)))
  want = {(h, l) for h in D.HEADS_32 + ('generic',) for l in ('thread', 'lane', 'warp')}
  if kind == 'synth':
    want -= {('tc', 'thread')}
  assert want <= covered, sorted(want - covered)


@pytest.mark.parametrize('temp', D.TEMPERATURES)
@pytest.mark.parametrize('gh,gw', [s for s in SIZES if min(s) >= 13])
def test_radius_plateau_moves_the_point_if_the_boundary_counts(gh, gw, temp):
  """Counting the d^2 == 25 cells (a `<=` for the `<` of utils.soft_argmax) moves the identity
  head's point by more than ten times the track budget."""
  ds = [d for d in D.designs(gh, gw) if d.family == 'radius']
  assert len(ds) == 1
  heat, _ = D.heat_fp64(_sd64('identity'), _maps(ds), float(np.float32(temp)))
  prob = torch.softmax(heat[0], -1)
  inside = D.soft_argmax_cells(prob, gh, gw)
  with_boundary = D.soft_argmax_cells(prob, gh, gw, include_boundary=True)
  px = (inside - with_boundary).abs() * torch.tensor([256.0 / gw, 256.0 / gh], dtype=torch.float64)
  assert px.max() > 10 * D.POINT_TOL, px


@pytest.mark.parametrize('T', [1, 3, 5])
def test_query_times_separate_rint_from_round_half_away(T):
  """The heads round the query frame with rintf (half to even, as torch.round).  roundf (half away
  from zero) would move the passthrough frame of some chosen query time; -0.5 must round to -0,
  which matches frame 0."""
  ts = np.array(D.query_times(T), np.float32)
  rint = np.rint(ts)
  away = np.sign(ts) * np.floor(np.abs(ts) + np.float32(0.5))
  frames = np.arange(T)
  match_rint, match_away = rint[:, None] == frames[None], away[:, None] == frames[None]
  assert (match_rint != match_away).any()
  ref = D.passthrough(torch.from_numpy(ts)[None, :, None].expand(1, -1, 3).contiguous(), T)[0]
  assert torch.equal(ref, torch.from_numpy(match_rint))
  assert ref[list(ts).index(np.float32(-0.5)), 0]


@pytest.mark.parametrize('gh,gw', SIZES)
def test_saturated_designs_underflow_exp_with_the_identity_head(gh, gw):
  """At temperature 20 every cell but the peak is more than SATURATED_GAP below it, so fp32 exp
  gives exactly 0 there and the peak probability is exactly 1."""
  assert np.exp(np.float32(-D.SATURATED_GAP + 2)) == 0  # margin for the kernels' fp32 heat
  ds = [d for d in D.designs(gh, gw) if d.family == 'saturated']
  heat, _ = D.heat_fp64(_sd64('identity'), _maps(ds), 20.0)
  gap, tie = D.top_two(heat)
  assert (gap > D.SATURATED_GAP).all() and not tie.any(), gap


def test_identity_head_heat_is_temperature_times_map():
  ds = D.designs(32, 32)
  maps = _maps(ds)
  for temp in D.TEMPERATURES:
    heat, _ = D.heat_fp64(_sd64('identity'), maps, temp)
    assert torch.equal(heat, maps.double().reshape(len(ds), -1) * temp)
