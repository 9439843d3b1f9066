"""Writes tests/golden/sinusoidal_to_harmonic.npz: outputs of the UNMODIFIED REFERENCE's
core.sinusoidal_to_harmonic (core.py:733-781) on seeded inputs, run on the NumPy
TensorFlow shim in narrow float32 and in wide float64.

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_sinusoidal_to_harmonic_golden.py          # rewrite the fixture
  python tests/golden/make_sinusoidal_to_harmonic_golden.py --check  # regenerate and compare

tests/test_sinusoidal_to_harmonic.py reads the fixture; the inputs come from the seeded
generator below.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests.golden.make_golden import _both, compare   # noqa: E402

PATH = os.path.join(HERE, 'sinusoidal_to_harmonic.npz')

# (name, B, T, S, K, harmonic_width, sample_rate, normalize)
CASES = [
    ('default', 2, 4, 5, 8, 0.1, 16000, False),
    ('default_norm', 2, 4, 5, 8, 0.1, 16000, True),
    ('pretrain', 2, 3, 100, 100, 0.1, 16000, False),
    ('pretrain_norm', 2, 3, 100, 100, 0.1, 16000, True),
    ('narrow', 2, 3, 100, 100, 0.03, 44100, False),
    ('narrow_norm', 2, 3, 100, 8, 0.03, 16000, True),
    ('wide', 2, 3, 5, 100, 1.0, 44100, False),
    ('wide_norm', 2, 3, 100, 100, 1.0, 16000, True),
    ('k1', 3, 2, 5, 1, 0.1, 44100, False),
    ('k1_norm', 3, 2, 100, 1, 1.0, 16000, True),
    ('s1', 2, 3, 1, 8, 0.03, 16000, False),
    ('s1_norm', 2, 3, 1, 100, 0.1, 44100, True),
]


def inputs(i, b=None, t=None, s=None):
  """Seeded (sin_amps, sin_freqs, f0_hz) of CASES[i] (or of the given shape):
  noisy harmonics of f0 in 80 .. 400 Hz, a few far from any harmonic, and in the
  frames that exist:
    (0, 0)   f0 = 0, with a 0 Hz sinusoid (weight 1 to every harmonic);
    (0, 1)   f0 = 3000 Hz: most harmonics at or above Nyquist, the sinusoids near its
             harmonics 1 .. 4;
    (0, 2)   f0 = 200 Hz with sinusoids exactly on harmonics 1, 2, ... and, from
             S = 3 on, a second one on harmonic 1 (its weights sum to 2 > 1);
    (-1, -1) all-zero amplitudes;
    (-1, 0)  a 0 Hz sinusoid under a nonzero f0."""
  if b is None:
    _, b, t, s, *_ = CASES[i]
  rng = np.random.default_rng(2100 + i)
  f0 = np.exp(rng.uniform(np.log(80.0), np.log(400.0), (b, t, 1)))
  n = rng.integers(1, 12, (b, t, s))
  freqs = f0 * n * np.exp(rng.normal(0.0, 0.02, (b, t, s)))
  far = rng.uniform(size=(b, t, s)) < 0.2
  freqs = np.where(far, rng.uniform(20.0, 9000.0, (b, t, s)), freqs)
  amps = rng.uniform(0.05, 1.0, (b, t, s))
  f0, freqs, amps = (v.astype(np.float32) for v in (f0, freqs, amps))
  if s >= 1:
    f0[0, 0, 0] = 0.0
    freqs[0, 0, 0] = 0.0
    if t > 1:
      f0[0, 1, 0] = 3000.0
      freqs[0, 1, :] = 3000.0 * (n[0, 1] % 4 + 1) + rng.normal(0.0, 30.0, s)
    if t > 2:
      f0[0, 2, 0] = 200.0
      freqs[0, 2, :] = 200.0 * np.arange(1, s + 1, dtype=np.float32)
      if s >= 3:
        freqs[0, 2, 2] = 200.0
    if b * t > 1:
      freqs[-1, 0, 0] = 0.0
    amps[-1, -1, :] = 0.0
  return amps, freqs, f0


def sinusoidal_to_harmonic():
  ddsp = ref_on_shim.load()
  out = {}
  for i, (name, *_, width, sr, norm) in enumerate(CASES):
    a, f, f0 = inputs(i)
    k = CASES[i][4]
    narrow, wide = _both(lambda: ddsp.core.sinusoidal_to_harmonic(
        a, f, f0, harmonic_width=width, n_harmonics=k, sample_rate=sr, normalize=norm))
    out[name + '_amp_f32'], out[name + '_dist_f32'] = narrow
    out[name + '_amp_wide'], out[name + '_dist_wide'] = (np.asarray(v, np.float64)
                                                         for v in wide)
  return out


if __name__ == '__main__':
  got = sinusoidal_to_harmonic()
  if '--check' in sys.argv:
    compare('sinusoidal_to_harmonic', got, np.load(PATH))
    print('ok    sinusoidal_to_harmonic')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote sinusoidal_to_harmonic %.0f kB' % (os.path.getsize(PATH) / 1e3))
