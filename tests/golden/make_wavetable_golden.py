"""Writes tests/golden/wavetable.npz: outputs of the UNMODIFIED REFERENCE's
core.wavetable_synthesis (core.py:1238-1282), synths.Wavetable
(synths.py:199-257) and core.harmonic_distribution_to_wavetable
(core.py:1217-1235) on seeded inputs, run on the NumPy TensorFlow shim: float32
(narrow) for the processor's host composition, float64 (wide) for the references
of tests/wavetable_ref.py.

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_wavetable_golden.py          # rewrite the fixture
  python tests/golden/make_wavetable_golden.py --check  # regenerate in memory and compare

The reference builds [B, N, W + 1] tensors, so the cases are small.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests.golden.make_golden import _both, compare   # noqa: E402

PATH = os.path.join(HERE, 'wavetable.npz')

# core.wavetable_synthesis cases: (f0 frames, amplitude frames, N, table frames
# ('2d', 1 or a count), W, sample rate, f0 regime).  Hops 1 and 441 come from f0
# frame counts (the amplitudes' 'window' resample needs fewer frames than N).
SYNTH = [
    (64, 16, 64, '2d', 3, 16000, 'normal'),       # f0 hop 1
    (32, 32, 64, 1, 257, 16000, 'zero'),          # hop 2, [B, 1, W]
    (8, 8, 504, 7, 1, 44100, 'normal'),           # hop 63, W = 1
    (8, 8, 512, 8, 2, 48000, 'negative'),         # hop 64, Fw = F, W = 2
    (4, 4, 1764, 1764, 257, 44100, 'above'),      # hop 441, Fw = N, above Nyquist
    (3, 3, 1536, 7, 1024, 16000, 'normal'),       # hop 512, W = 1024
    (16, 16, 1024, 16, 1024, 48000, 'mixed'),     # hop 64, every regime in one item
    (7, 5, 100, '2d', 257, 16000, 'normal'),      # f0 frames not dividing N, Ff != Fa
    (250, 10, 1000, 3, 64, 16000, 'normal'),      # f0 hop 4 under 'window' amps at hop 100
]
B = 2
# synths.Wavetable cases: (scale_fn default?, table shape kind, F, Fw, W, N)
PROC = [(True, '3d', 10, 10, 64, 400), (False, '3d', 10, 10, 64, 400),
        (True, '2d', 10, None, 64, 400), (False, '3d1', 10, 1, 128, 400),
        (True, '3d', 10, 4, 32, 400), (False, '2d', 8, None, 16, 256)]
HD = [(3, 4, 2048), (1, 10, 64), (2, 3, 8)]   # (time, harmonics, n_wavetable)


def synth_inputs(i):
  ff, fa, N, fw, W, sr, regime = SYNTH[i]
  rng = np.random.default_rng(1000 + i)
  base = {'normal': (50.0, 0.3 * sr), 'zero': (0.0, 0.0), 'negative': (-0.3 * sr, -20.0),
          'above': (0.5 * sr, 1.2 * sr), 'mixed': (-0.2 * sr, 0.9 * sr)}[regime]
  f0 = rng.uniform(base[0], base[1], (B, ff, 1))
  if regime == 'mixed':
    f0[:, :4] = 0.0
  amps = rng.uniform(0.1, 1.0, (B, fa, 1))
  shape = (B, W) if fw == '2d' else (B, fw, W)
  tab = rng.standard_normal(shape)
  return f0.astype(np.float32), amps.astype(np.float32), tab.astype(np.float32)


def proc_inputs(i):
  _, kind, F, fw, W, _ = PROC[i]
  rng = np.random.default_rng(1100 + i)
  f0 = rng.uniform(100.0, 1000.0, (B, F, 1)).astype(np.float32)
  amps = rng.standard_normal((B, F, 1)).astype(np.float32)
  shape = (B, W) if kind == '2d' else (B, fw, W)
  return amps, rng.standard_normal(shape).astype(np.float32), f0


def hd_input(i):
  T, K, _ = HD[i]
  return np.random.default_rng(1200 + i).uniform(0.0, 1.0, (B, T, K)).astype(np.float32)


def wavetable():
  ddsp = ref_on_shim.load()
  tf = ref_on_shim.tf()
  out = {}
  for i, (_, _, N, _, _, sr, _) in enumerate(SYNTH):
    f0, amps, tab = synth_inputs(i)
    _, w = _both(lambda: ddsp.core.wavetable_synthesis(
        tf.convert_to_tensor(f0), tf.convert_to_tensor(amps), tf.convert_to_tensor(tab),
        n_samples=N, sample_rate=sr))
    out['synth_wide_%d' % i] = np.asarray(w, np.float64)
  for i, (default, _, _, _, _, N) in enumerate(PROC):
    amps, tab, f0 = proc_inputs(i)
    kw = {} if default else {'scale_fn': None}
    synth = ddsp.synths.Wavetable(n_samples=N, sample_rate=16000, **kw)
    n, _ = _both(lambda: synth(amps, tab, f0))
    out['proc_f32_%d' % i] = n
  for i, (_, _, W) in enumerate(HD):
    hd = hd_input(i)
    _, w = _both(lambda: ddsp.core.harmonic_distribution_to_wavetable(
        tf.convert_to_tensor(hd), n_wavetable=W))
    out['hd_wide_%d' % i] = np.asarray(w, np.float64)
  return out


if __name__ == '__main__':
  got = wavetable()
  if '--check' in sys.argv:
    compare('wavetable', got, np.load(PATH))
    print('ok    wavetable')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote wavetable %.0f kB' % (os.path.getsize(PATH) / 1e3))
