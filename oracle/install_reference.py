"""TEST INFRASTRUCTURE - installs the UNMODIFIED reference into oracle/_ref (git-ignored).

`__graft_entry__.build()` calls install() so that bench.py's CPU arm runs the reference's own torch
path wherever the built tree goes: an offline `pip install --no-index --no-deps --target` of the
checkout found by oracle/reference_loader.py (einshape and dm-tree come from oracle/shims).
Without a readable checkout it does nothing and the CPU arm uses the oracle port (`kind`).
"""
import os
import shutil
import subprocess
import sys
import tempfile

from oracle import reference_loader

TARGET = os.path.join(os.path.dirname(os.path.abspath(__file__)), '_ref')


def install() -> bool:
  """Returns True when oracle/_ref holds the reference's torch model afterwards."""
  model = os.path.join(TARGET, 'tapnet', 'torch', 'tapir_model.py')
  if os.path.isfile(model):
    return True
  if not reference_loader.available():
    return False
  tmp = TARGET + '.tmp'
  shutil.rmtree(tmp, ignore_errors=True)
  with tempfile.TemporaryDirectory() as src:
    # build from a private copy: the checkout may be read-only for this user
    src = os.path.join(src, 'tapnet')
    shutil.copytree(reference_loader.REFERENCE_ROOT, src,
                    ignore=shutil.ignore_patterns('.git', 'assets', 'colabs', 'build', '*.egg-info'))
    for d, _, _ in os.walk(src):  # copytree keeps the checkout's read-only modes
      os.chmod(d, 0o755)
    r = subprocess.run([sys.executable, '-m', 'pip', 'install', '--quiet', '--no-index', '--no-deps',
                        '--no-build-isolation', '--no-cache-dir', '--target', tmp, src],
                       capture_output=True, text=True)
  if r.returncode != 0 or not os.path.isfile(os.path.join(tmp, 'tapnet', 'torch', 'tapir_model.py')):
    shutil.rmtree(tmp, ignore_errors=True)
    sys.stderr.write(f'oracle/_ref: reference install failed, the CPU arm will use the oracle port\n'
                     f'{r.stderr[-2000:]}\n')
    return False
  os.replace(tmp, TARGET)
  return True


if __name__ == '__main__':
  print(TARGET if install() else 'reference not available')
