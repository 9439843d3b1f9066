"""Writes tests/golden/harmonic_oscillator_bank.npz: outputs of the UNMODIFIED
REFERENCE's core.harmonic_oscillator_bank (core.py:966-1025) and
core.streaming_harmonic_synthesis (core.py:1114-1164) on seeded inputs, run on the NumPy
TensorFlow shim the way tests/golden/make_golden.py runs the decoder path (narrow float32
and wide float64).

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_harmonic_oscillator_bank_golden.py          # rewrite
  python tests/golden/make_harmonic_oscillator_bank_golden.py --check  # compare

tests/test_harmonic_oscillator_bank.py reads the fixture; the inputs come from the
seeded generators below.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests.golden.make_golden import _both, compare   # noqa: E402

PATH = os.path.join(HERE, 'harmonic_oscillator_bank.npz')

# (N, K, initial phase given, use_angular_cumsum)
BANK_CASES = [(1, 1, False, True), (63, 7, True, True), (63, 7, True, False),
              (500, 16, False, False), (2000, 3, True, True)]
# (F, N, K, amp_resample_method, initial phase given)
STREAM_CASES = [(5, 160, 4, 'linear', True), (5, 150, 4, 'nearest', False),
                (4, 130, 3, 'cubic', True), (4, 128, 1, 'window', False)]


def bank_inputs():
  """Seeded (frequency [2, N, 1], amplitudes [2, N, K], initial phase or None)."""
  rng = np.random.default_rng(966)
  out = []
  for n, k, init, _ in BANK_CASES:
    f = rng.uniform(50.0, 900.0, (2, n, 1)).astype(np.float32)
    a = rng.uniform(-1.0, 1.0, (2, n, k)).astype(np.float32)
    p = rng.uniform(-4.0, 4.0, (2, 1, 1)).astype(np.float32) if init else None
    out.append((f, a, p))
  return out


def stream_inputs():
  """Seeded (f0 [2, F, 1], amplitudes [2, F, 1], distribution [2, F, K], phase)."""
  rng = np.random.default_rng(1114)
  out = []
  for f, _, k, _, init in STREAM_CASES:
    f0 = rng.uniform(100.0, 3000.0, (2, f, 1)).astype(np.float32)
    amp = rng.uniform(0.1, 1.0, (2, f, 1)).astype(np.float32)
    hd = rng.uniform(0.0, 1.0, (2, f, k)).astype(np.float32)
    p = rng.uniform(0.0, 6.0, (2, 1, 1)).astype(np.float32) if init else None
    out.append((f0, amp, hd, p))
  return out


def harmonic_oscillator_bank():
  """The reference's harmonic_oscillator_bank and streaming_harmonic_synthesis, narrow
  and wide, on every case: audio and final phase."""
  ddsp = ref_on_shim.load()
  tf = ref_on_shim.tf()
  out = {}
  for i, ((_, _, _, mode), (f, a, p)) in enumerate(zip(BANK_CASES, bank_inputs())):
    for j, name in enumerate(('audio', 'phase')):
      n, w = _both(lambda: ddsp.core.harmonic_oscillator_bank(
          tf.convert_to_tensor(f), tf.convert_to_tensor(a),
          None if p is None else tf.convert_to_tensor(p), sample_rate=16000,
          use_angular_cumsum=mode)[j])
      out['bank_%s_f32_%d' % (name, i)] = n
      out['bank_%s_wide_%d' % (name, i)] = w.astype(np.float64)
  for i, ((_, n_samples, _, method, _), (f0, amp, hd, p)) in enumerate(
      zip(STREAM_CASES, stream_inputs())):
    for j, name in enumerate(('audio', 'phase')):
      n, w = _both(lambda: ddsp.core.streaming_harmonic_synthesis(
          tf.convert_to_tensor(f0), tf.convert_to_tensor(amp), tf.convert_to_tensor(hd),
          None if p is None else tf.convert_to_tensor(p), n_samples=n_samples,
          sample_rate=16000, amp_resample_method=method)[j])
      out['stream_%s_f32_%d' % (name, i)] = n
      out['stream_%s_wide_%d' % (name, i)] = w.astype(np.float64)
  return out


if __name__ == '__main__':
  got = harmonic_oscillator_bank()
  if '--check' in sys.argv:
    compare('harmonic_oscillator_bank', got, np.load(PATH))
    print('ok    harmonic_oscillator_bank')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote harmonic_oscillator_bank %.0f kB' % (os.path.getsize(PATH) / 1e3))
