"""Writes tests/golden/sinc.npz: outputs of the UNMODIFIED REFERENCE's
core.sinc_impulse_response and core.sinc_filter (core.py:1576-1625, 1658-1690) on
seeded inputs, run on the NumPy TensorFlow shim in wide float64 (and, for
sinc_filter, narrow float32 too).

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_sinc_golden.py          # rewrite the fixture
  python tests/golden/make_sinc_golden.py --check  # regenerate in memory and compare

tests/test_sinc_filter.py reads the fixture; the inputs come from the generators below.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests.golden.make_golden import _both, compare   # noqa: E402

PATH = os.path.join(HERE, 'sinc.npz')

WINDOWS = (0, 1, 2, 7, 8, 255, 256, 257, 512, 1024, 2048)
CUTOFFS = (0.0, 1e-3, 0.25, 0.5, 1.0, 1.5, -0.3)          # normalised (f / nyquist)
SAMPLE_RATES = (None, 16000, 44100)
# sinc_filter cases: (B, N, cutoff shape, window, padding, high_pass, sample_rate)
FILTER_CASES = [
    (2, 300, (2, 1, 1), 64, 'same', False, None),
    (2, 300, (2, 1, 1), 64, 'valid', True, None),
    (2, 300, (2, 7, 1), 33, 'same', False, 16000),        # ragged: frames of 43
    (2, 300, (1, 7, 1), 33, 'valid', True, None),
    (2, 120, (2, 120, 1), 16, 'same', True, 44100),        # one frame per sample
    (2, 120, (120, 1), 16, 'valid', False, None),          # [F, 1]: shared, F frames
    (1, 50, (), 20, 'same', False, None),                  # scalar cutoff
    (2, 300, (2, 1, 1), 1, 'same', False, None),           # one tap: empty crop
]


def ir_cases():
  """(window, high_pass, sample_rate, cutoff) of the impulse-response fixture: every
  cutoff as a [7, 1] column at each window and setting, at every rate up to 512 taps,
  plus the scalar, [B, F, 1] and [1, F, 1] shapes."""
  cases = []
  col = np.asarray(CUTOFFS, np.float32)[:, None]
  for ws in WINDOWS:
    for hp in (False, True):
      for sr in (SAMPLE_RATES if ws <= 512 else (None,)):
        c = col if sr is None else (col * np.float32(sr / 2.0)).astype(np.float32)
        cases.append((ws, hp, sr, c))
  rng = np.random.default_rng(77)
  cases.append((64, False, None, np.float32(0.3)))
  cases.append((64, True, 16000, rng.uniform(100, 7000, (3, 5, 1)).astype(np.float32)))
  cases.append((33, False, None, rng.uniform(0, 1, (1, 4, 1)).astype(np.float32)))
  return cases


def filter_inputs():
  """Seeded (audio, cutoff) of each FILTER_CASES entry."""
  rng = np.random.default_rng(78)
  out = []
  for b, n, cshape, _, _, _, sr in FILTER_CASES:
    audio = rng.standard_normal((b, n)).astype(np.float32)
    c = rng.uniform(0.05, 0.95, cshape).astype(np.float32)
    if sr is not None:
      c = (c * np.float32(sr / 2.0)).astype(np.float32)
    out.append((audio, c))
  return out


def sinc():
  ddsp = ref_on_shim.load()
  out = {}
  for i, (ws, hp, sr, c) in enumerate(ir_cases()):
    # the reference scales with `*=`: hand it a copy
    _, w = _both(lambda: ddsp.core.sinc_impulse_response(
        np.array(c, copy=True), window_size=ws, sample_rate=sr, high_pass=hp))
    out['ir_wide_%03d' % i] = w.astype(np.float64)
  for i, (case, (audio, c)) in enumerate(zip(FILTER_CASES, filter_inputs())):
    _, _, _, ws, padding, hp, sr = case
    n, w = _both(lambda: ddsp.core.sinc_filter(
        audio, np.array(c, copy=True), window_size=ws, sample_rate=sr, padding=padding,
        high_pass=hp))
    out['filter_f32_%02d' % i] = n
    out['filter_wide_%02d' % i] = w.astype(np.float64)
  return out


if __name__ == '__main__':
  got = sinc()
  if '--check' in sys.argv:
    compare('sinc', got, np.load(PATH))
    print('ok    sinc')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote sinc %.0f kB' % (os.path.getsize(PATH) / 1e3))
