"""Randomised cross-check of the oracle against the UNMODIFIED reference (CPU).

The golden fixtures pin the oracle on the path's configurations; this sweeps the
argument space around them - shapes, paddings, delays, odd / even / degenerate filter
windows, every amplitude resampling method, both phase accumulators, sample rates,
optional arguments - in the reference's "wide" mode (its own code evaluated in float64)
against the oracle's float64 mode.  It is how the odd-window Hann discrepancy was found.
The cases are drawn from fixed seeds by tests/golden/make_golden.py::fuzz_cases, which
also wrote the reference's results to tests/golden/reference_fuzz.npz.
"""
import os

import numpy as np
import pytest

from oracle import ddsp_oracle as o
from tests.golden import make_golden as mg

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CASES = mg.fuzz_cases()


@pytest.fixture(scope='module')
def want():
  return np.load(os.path.join(GOLD, 'reference_fuzz.npz'))


def _close(got, want, tol, what):
  got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
  assert got.shape == want.shape, (what, got.shape, want.shape)
  if got.size:
    assert np.abs(got - want).max() <= tol * max(1.0, np.abs(want).max()), what


def _check_group(group, want):
  """Every case of `group` against the stored reference result; the number of
  cases the reference accepted."""
  stored_cases = {k[:len(group) + 4] for k in want.files if k.startswith(group + '_')}
  assert len(stored_cases) == len(CASES[group]), (group, len(stored_cases))
  accepted = 0
  for i, (tag, tol, _, oracle_fn) in enumerate(CASES[group]):
    key = '%s_%03d' % (group, i)
    if key + '_raises' in want.files:
      with pytest.raises(Exception):
        oracle_fn(o)
      continue
    got = oracle_fn(o)
    stored = sorted(k[len(key) + 1:] for k in want.files if k.startswith(key + '_'))
    assert stored == sorted(got), (tag, stored, sorted(got))
    for name, value in got.items():
      ref = want['%s_%s' % (key, name)]
      if name == 'phase':
        d = np.angle(np.exp(1j * (np.asarray(value, np.float64) - ref)))
        assert np.abs(d).max() <= tol, tag
      else:
        _close(value, ref, tol, (tag, name))
    accepted += 1
  return accepted


def test_fft_convolve_shapes_paddings_delays(want):
  assert _check_group('fft_convolve', want) >= 12


def test_frequency_filter_windows(want):
  _check_group('frequency_filter', want)


def test_harmonic_synthesis_argument_space(want):
  _check_group('harmonic_synthesis', want)


def test_controls_oscillators_streaming_and_scalers(want):
  _check_group('controls_oscillators_streaming_and_scalers', want)
