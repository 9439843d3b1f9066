"""Writes tests/golden/spectral_terms.npz: losses.SpectralLoss of the UNMODIFIED
REFERENCE with each spectrogram term alone and all five together, 'L1' and 'L2', run
on the NumPy TensorFlow shim in its float64 (wide) mode.

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_spectral_terms_golden.py          # rewrite the fixture
  python tests/golden/make_spectral_terms_golden.py --check  # regenerate and compare

tests/test_spectral_loss_terms.py reads the fixture, inputs included.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests.golden.make_golden import _both, compare   # noqa: E402

PATH = os.path.join(HERE, 'spectral_terms.npz')

TERMS = ('mag', 'delta_time', 'delta_freq', 'cumsum_freq', 'logmag')
DEFAULT_SIZES = (2048, 1024, 512, 256, 128, 64)
# (name, signal, fft_sizes, weights): every term alone and all five together at the
# default sizes, all five at 4096 and 16, and a single frame (N <= the 256-sample hop
# of the 1024-point STFT), where delta_time is the mean of nothing
ALL = dict(mag=1.0, delta_time=0.7, delta_freq=1.3, cumsum_freq=0.05, logmag=0.4)
CASES = ([(t, 'long', DEFAULT_SIZES, {t: 1.0}) for t in TERMS] +
         [('all', 'long', DEFAULT_SIZES, ALL), ('all_4096_16', 'long', (4096, 16), ALL),
          ('one_frame', 'short', (1024,), ALL)])
LOSS_TYPES = ('L1', 'L2')


def signals():
  """(target, audio) float32: [2, 6000] for 'long' (a 220 Hz tone at two levels plus
  noise against noise), [2, 200] for 'short'."""
  rng = np.random.default_rng(4242)
  out = {}
  for name, n in (('long', 6000), ('short', 200)):
    target = (0.1 * rng.standard_normal((2, n))).astype(np.float32)
    t = np.arange(n) / 16000.0
    audio = (0.3 * np.sin(2 * np.pi * 220.0 * t)[None, :] * np.array([[1.0], [0.5]])
             + 0.05 * rng.standard_normal((2, n))).astype(np.float32)
    out[name] = (target, audio)
  return out


def spectral_terms():
  ddsp = ref_on_shim.load()
  sig = signals()
  out = {}
  for name, (target, audio) in sig.items():
    out[name + '_target'] = target
    out[name + '_audio'] = audio
  for case, name, sizes, weights in CASES:
    kw = {t + '_weight': weights.get(t, 0.0) for t in TERMS}
    target, audio = sig[name]
    for loss_type in LOSS_TYPES:
      loss = ddsp.losses.SpectralLoss(fft_sizes=sizes, loss_type=loss_type, **kw)
      out[f'{loss_type}_{case}'] = np.float64(_both(lambda: loss(target, audio))[1])
  return out


if __name__ == '__main__':
  got = spectral_terms()
  if '--check' in sys.argv:
    compare('spectral_terms', got, np.load(PATH))
    print('ok    spectral_terms')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote spectral_terms %.0f kB' % (os.path.getsize(PATH) / 1e3))
