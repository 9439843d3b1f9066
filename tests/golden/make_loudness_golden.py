"""Writes tests/golden/loudness.npz: outputs of the UNMODIFIED REFERENCE's
spectral_ops.compute_loudness (spectral_ops.py:254-324), compute_power
(spectral_ops.py:234-249) and losses.SpectralLoss with a loudness term
(losses.py:130-243) on seeded inputs, run on the NumPy TensorFlow shim in its float64
(wide) mode.  The shim's librosa stub has no fft_frequencies or A_weighting, so
`loudness()` installs tests/loudness_ref.py's restatements of librosa's closed forms
on it for the run.

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_loudness_golden.py          # rewrite the fixture
  python tests/golden/make_loudness_golden.py --check  # regenerate in memory and compare

tests/test_loudness.py reads the fixture; the inputs come from the seeded generators
below.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests.golden.make_golden import _both, compare   # noqa: E402

PATH = os.path.join(HERE, 'loudness.npz')

# compute_loudness cases: (sample_rate, n_fft, padding, N, 1-D input); hop = sr // 250
LOUD = [(16000, 512, 'center', 4000, False), (16000, 512, 'same', 4001, False),
        (16000, 512, 'valid', 4000, False), (16000, 2048, 'center', 8000, False),
        (16000, 64, 'center', 1000, False), (16000, 64, 'valid', 1003, False),
        (16000, 64, 'same', 999, False), (24000, 1024, 'same', 6000, False),
        (24000, 512, 'valid', 5000, False), (44100, 1024, 'center', 5000, False),
        (44100, 2048, 'same', 10000, False), (48000, 2048, 'valid', 9000, False),
        (48000, 512, 'center', 7001, False), (16000, 2048, 'center', 1500, False),
        (16000, 1024, 'same', 300, False), (16000, 512, 'center', 3000, True),
        (44100, 512, 'valid', 2000, True)]
# compute_power cases: (sample_rate, frame_size, padding, N, 1-D input)
POWER = [(16000, 64, 'center', 4000, False), (16000, 512, 'center', 4000, False),
         (16000, 1000, 'same', 4001, False), (16000, 1024, 'valid', 4000, False),
         (44100, 1000, 'center', 5000, False), (48000, 1024, 'same', 7001, False),
         (24000, 64, 'valid', 3000, False), (16000, 512, 'center', 2500, True)]
LOSS_N = 4000
B = 3


def audio_input(seed, n, is_1d):
  """Seeded noise rows at three levels (1, 0.03, 1e-4 of full scale)."""
  rng = np.random.default_rng(seed)
  x = rng.uniform(-1.0, 1.0, (B, n)) * np.array([[1.0], [0.03], [1e-4]])
  x = x.astype(np.float32)
  return x[0] if is_1d else x


def loud_input(i):
  return audio_input(1000 + i, LOUD[i][3], LOUD[i][4])


def power_input(i):
  return audio_input(1100 + i, POWER[i][3], POWER[i][4])


def loss_inputs():
  rng = np.random.default_rng(1200)
  target = rng.uniform(-1.0, 1.0, (2, LOSS_N)).astype(np.float32)
  audio = (0.5 * target + 0.1 * rng.standard_normal((2, LOSS_N))).astype(np.float32)
  return target, audio


def wide(fn):
  return np.asarray(_both(fn)[1], np.float64)


def _install_weighting(ddsp):
  """Gives the shim's librosa module (the one the reference imported) the two
  functions compute_loudness calls."""
  from tests import loudness_ref
  librosa = ddsp.spectral_ops.librosa
  librosa.fft_frequencies = loudness_ref.fft_frequencies
  librosa.A_weighting = loudness_ref.A_weighting


def loudness():
  ddsp = ref_on_shim.load()
  _install_weighting(ddsp)
  so = ddsp.spectral_ops
  out = {}
  for i, (sr, n_fft, padding, _, _) in enumerate(LOUD):
    x = loud_input(i)
    out['loudness_%02d' % i] = wide(lambda: so.compute_loudness(
        x, sample_rate=sr, n_fft=n_fft, padding=padding))
  for i, (sr, frame, padding, _, _) in enumerate(POWER):
    x = power_input(i)
    out['power_%02d' % i] = wide(lambda: so.compute_power(
        x, sample_rate=sr, frame_size=frame, padding=padding))
  target, audio = loss_inputs()
  loss = ddsp.losses.SpectralLoss(mag_weight=1.0, logmag_weight=1.0, loudness_weight=1.0)
  out['spectral_loss'] = wide(lambda: loss(target, audio))
  return out


if __name__ == '__main__':
  got = loudness()
  if '--check' in sys.argv:
    compare('loudness', got, np.load(PATH))
    print('ok    loudness')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote loudness %.0f kB' % (os.path.getsize(PATH) / 1e3))
