"""TEST INFRASTRUCTURE - generates tests/golden/reference_surface.json from the UNMODIFIED reference.

Run where the reference is importable (see oracle/reference_loader.py):
  python -m oracle.make_golden_surface
Stores what the host-side surface tests compare against: the reference TAPIR's state-dict keys and
shapes (as a digest) for two constructor configurations, and its generate_default_resolutions over a sweep of
frame sizes.
"""
import contextlib
import hashlib
import io
import json
import os

from oracle import reference_loader

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'tests', 'golden', 'reference_surface.json')

SCHEMA_CONFIGS = [dict(pyramid_level=1), dict(pyramid_level=0, extra_convs=False)]
RESOLUTION_SIZES = [(256, 256), (240, 240), (480, 480), (480, 640), (360, 640), (512, 512), (720, 1280),
                    (1024, 1024), (1080, 1920), (264, 264), (250, 500), (2048, 1024)]


def schema_digest(items):
  """sha256 of the ordered (key, shape) list of a state dict."""
  return hashlib.sha256(json.dumps([[k, list(v)] for k, v in items]).encode()).hexdigest()


def main():
  tapir_model = reference_loader.load()
  from tapnet.torch import utils as ref_utils  # pylint: disable=g-import-not-at-top
  schemas = []
  for kw in SCHEMA_CONFIGS:
    sd = tapir_model.TAPIR(**kw).state_dict()
    schemas.append(dict(kwargs=kw, num_keys=len(sd),
                        sha256=schema_digest([(k, list(v.shape)) for k, v in sd.items()])))
  resolutions = []
  for hw in RESOLUTION_SIZES:
    with contextlib.redirect_stdout(io.StringIO()):
      r = ref_utils.generate_default_resolutions(hw, (256, 256))
    resolutions.append(dict(size=list(hw), resolutions=[[int(v) for v in x] for x in r]))
  with open(OUT, 'w') as fh:
    json.dump(dict(schemas=schemas, default_resolutions=resolutions), fh)
    fh.write('\n')
  print(f'wrote {OUT}')


if __name__ == '__main__':
  main()
