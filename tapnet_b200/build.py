"""Builds tapnet_b200/libtapir_b200.so (sm_90a only) with nvcc, in-tree."""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libtapir_b200.so')
SOURCES = ['common.cu', 'gemm_tc.cu', 'gemm_simt.cu', 'backbone.cu', 'stage_a.cu', 'refine.cu',
           'frames_io.cu', 'paint.cu', 'resample.cu', 'homography.cu', 'api.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '-Xcompiler', '-fPIC']


def _nvcc():
  for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
    if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
      return cand
  return 'nvcc'


def _digest():
  h = hashlib.sha256()
  files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))]
  files.append(os.path.join(os.path.dirname(HERE), 'include', 'tapir_b200.h'))
  for f in files:
    with open(f, 'rb') as fh:
      h.update(f.encode())
      h.update(fh.read())
  h.update(' '.join(NVCC_FLAGS).encode())
  return h.hexdigest()


def build(force=False, verbose=False):
  """Compiles every CUDA source and links the shared library; returns its path."""
  stamp = LIB + '.stamp'
  digest = _digest()
  if not force and os.path.exists(LIB) and os.path.exists(stamp):
    with open(stamp) as fh:
      if fh.read().strip() == digest:
        return LIB
  objdir = os.path.join(HERE, 'build')
  os.makedirs(objdir, exist_ok=True)
  nvcc = _nvcc()
  procs = []
  objs = []
  for src in SOURCES:
    obj = os.path.join(objdir, src.replace('.cu', '.o'))
    objs.append(obj)
    cmd = [nvcc] + NVCC_FLAGS + ['-c', os.path.join(CSRC, src), '-o', obj]
    if verbose:
      print(' '.join(cmd))
    procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
  failed = False
  for src, p in procs:
    out, _ = p.communicate()
    if p.returncode != 0:
      failed = True
      sys.stderr.write(f'--- nvcc failed for {src}\n{out.decode()}\n')
    elif verbose and out:
      print(out.decode())
  if failed:
    raise RuntimeError('nvcc compilation failed')
  cmd = [nvcc, '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a', '-ldl']
  subprocess.check_call(cmd)
  with open(stamp, 'w') as fh:
    fh.write(digest)
  return LIB


if __name__ == '__main__':
  print(build(force='--force' in sys.argv, verbose=True))
