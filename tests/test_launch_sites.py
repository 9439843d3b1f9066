"""Every kernel of the C library starts through one helper, `launch` in common.cuh, which
reserves dynamic shared memory, launches, counts the launch for
ddsp_b200_launch_count() and turns a launch error into E_CUDA.  The only other launch
is noise_ring.cuh's programmatic dependent launch (cudaLaunchKernelEx).  Each entry
point states its overlap rule in one check_overlap call."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'ddsp_b200', 'csrc')


def _code():
  """{file name: source without comments} of every unit and header of the library."""
  code = {}
  for name in sorted(os.listdir(CSRC)):
    if name.endswith(('.cu', '.cuh')):
      with open(os.path.join(CSRC, name)) as f:
        code[name] = re.sub(r'/\*.*?\*/|//[^\n]*', ' ', f.read(), flags=re.S)
  return code


def _uses(pattern):
  """{file name: count} of the files where `pattern` occurs."""
  counts = {name: len(re.findall(pattern, text)) for name, text in _code().items()}
  return {name: n for name, n in counts.items() if n}


def _helper():
  m = re.search(r'\nint launch\(.*?\n}\n', _code()['common.cuh'], flags=re.S)
  assert m, 'common.cuh defines no launch helper'
  return m.group(0)


def test_only_the_helper_uses_launch_syntax():
  assert _uses(r'<<<') == {'common.cuh': 1}
  assert '<<<' in _helper()


def test_one_launch_outside_the_helper():
  assert _uses(r'\bcudaLaunchKernelEx\b') == {'noise_ring.cuh': 1}


def test_only_the_helper_and_noise_ring_reserve_and_check():
  # common.cuh: the definition and the helper's use
  for name in ('set_smem', 'DDSP_CHECK_LAUNCH'):
    assert _uses(r'\b%s\(' % name) == {'common.cuh': 2, 'noise_ring.cuh': 1}, name
    assert name + '(' in _helper(), name


def test_no_pairwise_overlap_macros():
  assert _uses(r'\bDDSP_REQUIRE_(SAME_OR_)?DISJOINT\b') == {}
