"""Builds libddsp_b200.so in-tree with nvcc for sm_90a (H100) only: one nvcc -c per
unit of csrc/, run concurrently, then one link."""
import concurrent.futures
import os
import subprocess
import sys
import tempfile

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, 'csrc')
LIB_PATH = os.path.join(_HERE, 'libddsp_b200.so')
# the nvcc command lines that built LIB_PATH: other flags or another arch rebuild
CMD_PATH = LIB_PATH + '.cmd'
# stands for the temporary object directory in the recorded command lines
_OBJ = '$OBJ'

NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a',
    '-O3', '-lineinfo', '-std=c++17',
    '-Xcompiler', '-fPIC',
]


def _sources():
  return sorted(os.path.join(CSRC, n) for n in os.listdir(CSRC) if n.endswith('.cu'))


def _newest_mtime():
  newest = 0.0
  for root in (CSRC, os.path.join(_HERE, '..', 'include')):
    for name in os.listdir(root):
      if name.endswith(('.cu', '.cuh', '.h', '.inc')):
        newest = max(newest, os.path.getmtime(os.path.join(root, name)))
  return newest


def _commands(out, flags=(), obj_dir=_OBJ, verbose=False):
  """The compile command of every unit, objects in obj_dir, and the link into out."""
  nvcc = [os.environ.get('NVCC', 'nvcc')] + NVCC_FLAGS + list(flags)
  compiles, objs = [], []
  for src in _sources():
    obj = os.path.join(obj_dir, os.path.basename(src)[:-len('.cu')] + '.o')
    compiles.append(nvcc + (['-Xptxas', '-v'] if verbose else []) + ['-c', '-o', obj, src])
    objs.append(obj)
  return compiles, nvcc + ['-shared', '-o', out] + objs


def _record(out, flags=()):
  compiles, link = _commands(out, flags)
  return '\n'.join(' '.join(cmd) for cmd in compiles + [link])


def _built_with():
  try:
    with open(CMD_PATH) as f:
      return f.read()
  except OSError:
    return None


def is_stale():
  """True if the library is missing, older than its sources, or was built by
  other nvcc command lines (compiler, flags, arch, units)."""
  return (not os.path.exists(LIB_PATH) or
          os.path.getmtime(LIB_PATH) < _newest_mtime() or
          _built_with() != _record(LIB_PATH))


def _run(cmd):
  proc = subprocess.run(cmd, capture_output=True, text=True)
  if proc.returncode != 0:
    raise RuntimeError('nvcc failed:\n%s\n%s' % (' '.join(cmd), proc.stderr))
  return proc.stderr


def build(force=False, verbose=False, out=LIB_PATH, flags=()):
  """Compiles the CUDA library if missing, older than its sources or built with
  other command lines.  `out` and extra nvcc `flags` (e.g. -D switches) build a
  variant of it, always from scratch."""
  if out == LIB_PATH and not flags and not force and not is_stale():
    return out
  with tempfile.TemporaryDirectory() as obj_dir:
    compiles, link = _commands(out, flags, obj_dir, verbose)
    with concurrent.futures.ThreadPoolExecutor(os.cpu_count() or 1) as pool:
      logs = list(pool.map(_run, compiles))
    _run(link)
  with open(out + '.cmd', 'w') as f:
    f.write(_record(out, flags))
  if verbose:
    sys.stderr.write(''.join(logs))
  return out


if __name__ == '__main__':
  print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
