"""ctypes binding of libddsp_b200.so, derived at import from its C ABI,
include/ddsp_b200.h: every `ddsp_b200_*` prototype becomes an entry of SIGNATURES,
and every `DDSP_B200_*` enum value or integer #define a module attribute without
the prefix (E_INVALID, PAD_SAME, HMM_MAX_STATES, ...).

There is NO fallback: if the shared library is missing or fails to load, every
op raises.  Build it with `python -m ddsp_b200.build` (needs nvcc, not a GPU).
"""
import ctypes
import os
import re
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libddsp_b200.so')
HEADER_PATH = os.path.join(_HERE, '..', 'include', 'ddsp_b200.h')

_sz = ctypes.c_size_t   # the type of every workspace size

# C types of the header, spelled without `const` and whitespace.  Device pointers
# travel as integers.
_SCALARS = {
    'int': ctypes.c_int,
    'int64_t': ctypes.c_int64,
    'uint64_t': ctypes.c_uint64,
    'size_t': _sz,
    'float': ctypes.c_float,
    'double': ctypes.c_double,
}


def _ctype(spelling, is_return=False):
  """The ctypes type of a C type as the header spells it; an unknown type raises, so
  that a new type in the header is never bound by a guess."""
  t = re.sub(r'\bconst\b|\s', '', spelling)
  if is_return and t == 'char*':
    return ctypes.c_char_p
  if t in ('ddsp_b200_host_pipeline**', 'ddsp_b200_gru**'):
    return ctypes.POINTER(ctypes.c_void_p)
  if t.endswith('*') and not t.endswith('**'):
    return ctypes.c_void_p
  if t in _SCALARS:
    return _SCALARS[t]
  raise TypeError(f'ddsp_b200: the C type {spelling.strip()!r} in the ABI header has no '
                  'ctypes binding in ddsp_b200/_lib.py')


def parse_header(text):
  """(signatures, constants) of the C header `text`: {name: (restype, argtypes)} for
  every ddsp_b200_* prototype and {NAME: value} for every DDSP_B200_NAME enum value
  or integer #define."""
  text = re.sub(r'/\*.*?\*/|//[^\n]*', ' ', text, flags=re.S)
  constants = {m[1]: int(m[2]) for m in
               re.finditer(r'^\s*#\s*define\s+DDSP_B200_(\w+)\s+(-?\d+)\s*$', text, re.M)}
  for body in re.findall(r'\benum\s*\{([^}]*)\}', text):
    for item in body.split(','):
      m = re.fullmatch(r'\s*DDSP_B200_(\w+)\s*=\s*(-?\d+)\s*', item)
      if not m:
        raise ValueError(f'ddsp_b200: enumerator {item.strip()!r} of the ABI header is '
                         'not DDSP_B200_NAME = integer')
      constants[m[1]] = int(m[2])
  text = re.sub(r'^\s*#[^\n]*', ' ', text, flags=re.M)
  signatures = {}
  for m in re.finditer(r'([\w\s*]+?)\b(ddsp_b200_\w+)\s*\(([^()]*)\)\s*;', text):
    params = [p.strip() for p in m[3].split(',')]
    if params == ['void']:
      params = []
    # a parameter is its type and a name: drop the name
    argtypes = [_ctype(re.sub(r'\w+$', '', p)) for p in params]
    signatures[m[2]] = (_ctype(m[1], is_return=True), argtypes)
  return signatures, constants


def _read_header():
  if not os.path.exists(HEADER_PATH):
    raise RuntimeError(
        'ddsp_b200: %s is missing. The C ABI header declares what the binding '
        'calls; it belongs next to the package, in the source tree.' % HEADER_PATH)
  with open(HEADER_PATH) as f:
    return f.read()


SIGNATURES, _CONSTANTS = parse_header(_read_header())
globals().update(_CONSTANTS)
PADDING = {name[len('PAD_'):].lower(): value for name, value in _CONSTANTS.items()
           if name.startswith('PAD_')}

_lib = None
_lock = threading.Lock()


def bind(path):
  """Opens the library at `path` and gives each C entry point its header signature."""
  lib = ctypes.CDLL(path)
  for name, (restype, argtypes) in SIGNATURES.items():
    fn = getattr(lib, name)  # AttributeError if the .so lacks a symbol
    fn.restype = restype
    fn.argtypes = argtypes
  return lib


def load():
  """Loads the library once; raises RuntimeError loudly if it is absent."""
  global _lib
  if _lib is not None:
    return _lib
  with _lock:
    if _lib is not None:
      return _lib
    if not os.path.exists(LIB_PATH):
      raise RuntimeError(
          'ddsp_b200: %s is missing. The CUDA extension is the product - '
          'there is no CPU fallback. Build it with `python -m ddsp_b200.build` '
          '(or __graft_entry__.build()).' % LIB_PATH)
    _lib = bind(LIB_PATH)
  return _lib


def check(rc):
  """Maps a C status to the reference's Python error convention."""
  if rc == OK:
    return
  msg = load().ddsp_b200_last_error().decode('utf-8', 'replace')
  if rc == E_INVALID:
    raise ValueError(msg)
  if rc == E_UNSUPPORTED:
    raise NotImplementedError(msg)
  raise RuntimeError('ddsp_b200 (status %d): %s' % (rc, msg))
