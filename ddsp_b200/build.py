"""Builds libddsp_b200.so in-tree with nvcc for sm_90a (H100) only."""
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, 'csrc')
LIB_PATH = os.path.join(_HERE, 'libddsp_b200.so')
# the nvcc command line that built LIB_PATH: other flags or another arch rebuild
CMD_PATH = LIB_PATH + '.cmd'

NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a',
    '-O3', '-lineinfo', '-std=c++17',
    '-Xcompiler', '-fPIC', '-shared',
]


def _sources():
  return [os.path.join(CSRC, 'capi.cu')]


def _newest_mtime():
  newest = 0.0
  for root in (CSRC, os.path.join(_HERE, '..', 'include')):
    for name in os.listdir(root):
      if name.endswith(('.cu', '.cuh', '.h', '.inc')):
        newest = max(newest, os.path.getmtime(os.path.join(root, name)))
  return newest


def _command(verbose=False):
  nvcc = os.environ.get('NVCC', 'nvcc')
  return [nvcc] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + [
      '-o', LIB_PATH] + _sources()


def _built_with():
  try:
    with open(CMD_PATH) as f:
      return f.read()
  except OSError:
    return None


def is_stale():
  """True if the library is missing, older than its sources, or was built by
  another nvcc command line (compiler, flags, arch)."""
  return (not os.path.exists(LIB_PATH) or
          os.path.getmtime(LIB_PATH) < _newest_mtime() or
          _built_with() != ' '.join(_command()))


def build(force=False, verbose=False):
  """Compiles the CUDA library if missing, older than its sources or built with
  another command line."""
  if not force and not is_stale():
    return LIB_PATH
  cmd = _command(verbose)
  proc = subprocess.run(cmd, capture_output=True, text=True)
  if proc.returncode != 0:
    raise RuntimeError('nvcc failed:\n%s\n%s' % (' '.join(cmd), proc.stderr))
  with open(CMD_PATH, 'w') as f:
    f.write(' '.join(_command()))
  if verbose:
    sys.stderr.write(proc.stderr)
  return LIB_PATH


if __name__ == '__main__':
  print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
