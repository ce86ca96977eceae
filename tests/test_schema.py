import json
import os

import pytest

from tapnet_b200 import schema

SURFACE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_surface.json')


def test_param_counts():
  s = schema.state_dict_schema()
  n = sum(int(__import__('numpy').prod(v)) for v in s.values())
  assert len(s) == 218 and n == 54699335  # SURVEY.md 8(a1)
  s0 = schema.state_dict_schema(0, False)
  assert len(s0) == 188


@pytest.mark.parametrize('kw', [dict(pyramid_level=1), dict(pyramid_level=0, extra_convs=False)])
def test_schema_matches_reference_module(kw):
  """Same keys, order and shapes as the reference TAPIR(**kw).state_dict(), whose digest
  oracle/make_golden_surface.py stored."""
  with open(SURFACE) as fh:
    ref = next(d for d in json.load(fh)['schemas'] if d['kwargs'] == kw)
  from oracle.make_golden_surface import schema_digest
  s = schema.state_dict_schema(kw.get('pyramid_level', 1), kw.get('extra_convs', True))
  assert len(s) == ref['num_keys']
  assert schema_digest(s.items()) == ref['sha256']
