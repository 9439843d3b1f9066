"""Writes tests/golden/mod_delay.npz: outputs of the UNMODIFIED REFERENCE's
core.variable_length_delay (core.py:1285-1314) and effects.ModDelay
(effects.py:328-394) on seeded inputs, run on the NumPy TensorFlow shim the way
tests/golden/make_golden.py runs the decoder path (narrow float32 and wide float64).

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_mod_delay_golden.py          # rewrite the fixture
  python tests/golden/make_mod_delay_golden.py --check  # regenerate in memory and compare

tests/test_mod_delay.py reads the fixture (and regenerates it when the reference is
present); the inputs come from the seeded generators below.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests.golden.make_golden import _both, compare   # noqa: E402

PATH = os.path.join(HERE, 'mod_delay.npz')


MOD_DELAY_SIZES = [(1, 800), (10, 800), (400, 800), (1000, 1200), (400, 250)]  # (L, N)
MOD_DELAY_PHASES = ('const0', 'const05', 'const1', 'lfo', 'rough', 'wide_range')
# ModDelay cases: (sample_rate, add_dry, default scale fns, gain rank, phase rank, N)
MOD_DELAY_PROCESSOR = [(16000, True, True, 3, 3, 1000), (44100, True, True, 3, 3, 1500),
                       (16000, False, True, 2, 2, 1000), (16000, True, False, 3, 2, 1000),
                       (44100, False, False, 2, 3, 1500)]


def mod_delay_phase(kind, b, n, rng):
  """[b, n, 1] float32 phases: constants 0 / 0.5 / 1, a smooth LFO over ModDelay's
  default range (0.6, 1] that passes through the wrap region near 1, a rough
  uniform phase, and one that leaves [0, 1] on both sides."""
  if kind.startswith('const'):
    value = {'const0': 0.0, 'const05': 0.5, 'const1': 1.0}[kind]
    return np.full((b, n, 1), value, np.float32)
  if kind == 'lfo':
    t = np.arange(n)[None, :, None] / 16000.0
    rate = rng.uniform(2.0, 6.0, (b, 1, 1))
    return (0.8 + 0.2 * np.sin(2 * np.pi * rate * t + rng.uniform(0, 6.28, (b, 1, 1)))
            ).astype(np.float32)
  lo, hi = (0.0, 1.0) if kind == 'rough' else (-0.2, 1.2)
  return rng.uniform(lo, hi, (b, n, 1)).astype(np.float32)


def mod_delay_inputs():
  """Seeded (L, N, kind, phase [2, N, 1], audio [2, N]) of the delay fixture."""
  rng = np.random.default_rng(909)
  cases = []
  for L, n in MOD_DELAY_SIZES:
    audio = rng.standard_normal((2, n)).astype(np.float32)
    for kind in MOD_DELAY_PHASES:
      cases.append((L, n, kind, mod_delay_phase(kind, 2, n, rng), audio))
  return cases


def mod_delay_processor_inputs():
  """Seeded raw (audio, gain, phase) of each MOD_DELAY_PROCESSOR case: network-like
  raw controls for the default scale functions, a gain around 0.5 and a phase over
  [-0.2, 1.2] without them."""
  rng = np.random.default_rng(910)
  out = []
  for sr, _, scaled, g_rank, p_rank, n in MOD_DELAY_PROCESSOR:
    audio = rng.standard_normal((2, n)).astype(np.float32)
    if scaled:
      gain = rng.standard_normal((2, n, 1)).astype(np.float32)
      phase = (2.0 * rng.standard_normal((2, n, 1))).astype(np.float32)
    else:
      gain = rng.uniform(0.2, 0.8, (2, n, 1)).astype(np.float32)
      phase = rng.uniform(-0.2, 1.2, (2, n, 1)).astype(np.float32)
    out.append((audio, gain if g_rank == 3 else gain[..., 0],
                phase if p_rank == 3 else phase[..., 0]))
  return out


def mod_delay():
  """core.variable_length_delay (core.py:1285-1314) of the reference, narrow and
  wide, on every mod_delay_inputs() case, and effects.ModDelay (effects.py:328-394)
  end to end from raw controls, float32, on every MOD_DELAY_PROCESSOR case."""
  ddsp = ref_on_shim.load()
  tf = ref_on_shim.tf()
  out = {}
  for i, (L, _, _, phase, audio) in enumerate(mod_delay_inputs()):
    n, w = _both(lambda: ddsp.core.variable_length_delay(
        tf.convert_to_tensor(phase), tf.convert_to_tensor(audio), max_length=L))
    out['delay_f32_%02d' % i] = n
    out['delay_wide_%02d' % i] = w.astype(np.float64)
  for i, (case, (audio, gain, phase)) in enumerate(zip(MOD_DELAY_PROCESSOR,
                                                       mod_delay_processor_inputs())):
    sr, add_dry, scaled = case[:3]
    kw = {} if scaled else dict(gain_scale_fn=None, phase_scale_fn=None)
    md = ddsp.effects.ModDelay(sample_rate=sr, add_dry=add_dry, **kw)
    out['processor_f32_%d' % i] = ref_on_shim.to_numpy(md(audio, gain, phase))
  return out


if __name__ == '__main__':
  got = mod_delay()
  if '--check' in sys.argv:
    compare('mod_delay', got, np.load(PATH))
    print('ok    mod_delay')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote mod_delay %.0f kB' % (os.path.getsize(PATH) / 1e3))
