"""The ctypes binding derived from include/ddsp_b200.h (`_lib.parse_header`), and the
library's pure-host shape queries that the Python routing asks instead of restating
the launchers' rules."""
import ctypes
import os
import re

import pytest

from ddsp_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
  with open(os.path.join(ROOT, 'include', 'ddsp_b200.h')) as f:
    return f.read()


def test_every_declaration_is_bound():
  """As many prototypes as the comment-stripped header declares; the comments also
  mention calls such as ddsp_b200_ir_size(nb, window_size)."""
  code = re.sub(r'/\*.*?\*/|//[^\n]*', ' ', _header(), flags=re.S)
  declared = re.findall(r'\b(ddsp_b200_\w+)\s*\(', code)
  assert len(declared) == len(set(declared)) == len(_lib.SIGNATURES)
  assert set(declared) == set(_lib.SIGNATURES)


def test_spot_types():
  sig = _lib.SIGNATURES
  for name, r in (('ddsp_b200_wasserstein_forward', 5), ('ddsp_b200_wasserstein_backward', 9)):
    assert sig[name][1][r] is ctypes.c_int64, name
  for name in ('ddsp_b200_hmm_log_prob', 'ddsp_b200_hmm_log_prob_backward',
               'ddsp_b200_hmm_viterbi'):
    assert sig[name][1][-3:-1] == [ctypes.c_double, ctypes.c_double], name
  assert sig['ddsp_b200_host_pipeline_create'][1][0] is ctypes.POINTER(ctypes.c_void_p)
  assert sig['ddsp_b200_last_error'] == (ctypes.c_char_p, [])
  assert sig['ddsp_b200_version'] == (ctypes.c_int, [])
  assert sig['ddsp_b200_launch_count'] == (ctypes.c_uint64, [])
  assert sig['ddsp_b200_add'][1] == [ctypes.c_void_p] * 3 + [ctypes.c_int64,
                                                             ctypes.c_void_p]
  assert sig['ddsp_b200_sinusoidal_workspace'][0] is ctypes.c_size_t


def test_constants():
  assert (_lib.OK, _lib.E_INVALID, _lib.E_UNSUPPORTED, _lib.E_CUDA, _lib.E_WORKSPACE) == (
      0, -1, -2, -3, -4)
  assert _lib.PADDING == {'same': 0, 'valid': 1, 'center': 2}
  assert _lib.VERSION == 200


def test_parser_on_a_small_header():
  sig, const = _lib.parse_header("""
      #define DDSP_B200_X 7 /* seven */
      enum { DDSP_B200_A = -1, DDSP_B200_B = 2 };
      /* ddsp_b200_not_a_declaration(x) */
      const char* ddsp_b200_name(void);
      size_t ddsp_b200_f(const float* x, int64_t n,
                         double d, void* stream);""")
  assert const == {'X': 7, 'A': -1, 'B': 2}
  assert sig == {'ddsp_b200_name': (ctypes.c_char_p, []),
                 'ddsp_b200_f': (ctypes.c_size_t, [ctypes.c_void_p, ctypes.c_int64,
                                                   ctypes.c_double, ctypes.c_void_p])}


@pytest.mark.parametrize('decl', ['int ddsp_b200_f(unsigned n);',
                                  'int ddsp_b200_f(short n);',
                                  'void ddsp_b200_f(int n);',
                                  'int ddsp_b200_f(float** p);'])
def test_an_unknown_type_raises(decl):
  with pytest.raises(TypeError, match='no ctypes binding'):
    _lib.parse_header(decl)


def _query(name, *args):
  """The query's answer, checked to launch nothing and leave the last error alone."""
  lib = _lib.load()
  assert lib.ddsp_b200_add(None, None, None, 4, None) == _lib.E_INVALID
  before = (lib.ddsp_b200_last_error(), lib.ddsp_b200_launch_count())
  took = getattr(lib, 'ddsp_b200_' + name)(*args)
  assert (lib.ddsp_b200_last_error(), lib.ddsp_b200_launch_count()) == before
  assert took in (0, 1)
  return took


@pytest.mark.parametrize('f,nb,n,ws,takes', [
    (10, 65, 640, 0, 1), (1000, 65, 64000, 257, 1), (33, 33, 3293, 257, 1),
    (10, 65, 640, 2, 0),              # one tap: nothing to compensate the delay with
    (2, 65, 2048, 0, 0),              # 32 frames of 1024 samples do not fit one CTA
    (20, 129, 10240, 0, 0),
    (10, 1, 640, 0, 0), (1000, 65, 999, 0, 0)])   # one band; frames do not tile
def test_filtered_noise_backward_takes(f, nb, n, ws, takes):
  assert _query('filtered_noise_backward_takes', f, nb, n, ws) == takes


@pytest.mark.parametrize('b,f,n,takes', [
    (1, 10, 640, 1), (1, 10, 1280, 1), (1, 1, 8192, 1), (65535, 10, 640, 1),
    (1, 10, 650, 0), (1, 10, 960, 0), (1, 1, 8256, 0), (65536, 10, 640, 0),
    (1, 10, 5, 0), (1, 0, 640, 0)])
def test_harmonic_backward_takes(b, f, n, takes):
  assert _query('harmonic_backward_takes', b, f, n) == takes


@pytest.mark.parametrize('t,k,takes', [
    (1000, 1024, 1), (10000, 128, 1), (1551, 1024, 1), (1552, 1024, 0),
    (10240, 128, 1), (10241, 128, 0), (1, 1024, 1), (0, 128, 0)])
def test_hmm_viterbi_takes(t, k, takes):
  assert _query('hmm_viterbi_takes', t, k) == takes
