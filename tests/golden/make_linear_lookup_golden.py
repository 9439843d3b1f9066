"""Writes tests/golden/linear_lookup.npz: outputs of the UNMODIFIED REFERENCE's
core.linear_lookup (core.py:1168-1214) on seeded inputs, run on the NumPy TensorFlow
shim the way tests/golden/make_golden.py runs the decoder path (narrow float32 and wide
float64).

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_linear_lookup_golden.py          # rewrite the fixture
  python tests/golden/make_linear_lookup_golden.py --check  # regenerate in memory and compare

tests/test_linear_lookup.py reads the fixture; the inputs come from the seeded
generator below.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests.golden.make_golden import _both, compare   # noqa: E402

PATH = os.path.join(HERE, 'linear_lookup.npz')

# (W, table layout, phase kind): layout 'item' is [B, W], 'item3' [B, 1, W], 'sample'
# [B, N, W]; phases inside [0, 1], on the grid points, just outside on both sides, far
# outside, and a [B, N, 1] phase.
LOOKUP_CASES = [(w, layout, kind) for w in (1, 2, 7, 64)
                for layout in ('item', 'item3', 'sample')
                for kind in ('inside', 'grid', 'edges', 'far', 'rank3')]
N = 40


def lookup_phase(kind, b, n, w, rng):
  """[b, n] (or [b, n, 1] for 'rank3') float32 phases of one case."""
  if kind == 'grid':
    p = (rng.integers(0, w + 1, (b, n)) / np.float32(w)).astype(np.float32)
  elif kind == 'edges':
    lo = rng.uniform(-1.0 / w, 0.0, (b, n))
    hi = rng.uniform(1.0, 1.0 + 1.0 / w, (b, n))
    p = np.where(rng.random((b, n)) < 0.5, lo, hi).astype(np.float32)
  elif kind == 'far':
    p = rng.choice([-3.5, -1.0, 2.0, 7.25], (b, n)).astype(np.float32)
  else:
    p = rng.uniform(0.0, 1.0, (b, n)).astype(np.float32)
  return p[..., None] if kind == 'rank3' else p


def lookup_inputs():
  """Seeded (W, layout, kind, phase, wavetables) of every LOOKUP_CASES case."""
  rng = np.random.default_rng(1168)
  out = []
  for w, layout, kind in LOOKUP_CASES:
    phase = lookup_phase(kind, 2, N, w, rng)
    shape = {'item': (2, w), 'item3': (2, 1, w), 'sample': (2, N, w)}[layout]
    out.append((w, layout, kind, phase, rng.standard_normal(shape).astype(np.float32)))
  return out


def linear_lookup():
  """core.linear_lookup of the reference, narrow and wide, on every case."""
  ddsp = ref_on_shim.load()
  tf = ref_on_shim.tf()
  out = {}
  for i, (_, _, _, phase, tab) in enumerate(lookup_inputs()):
    n, w = _both(lambda: ddsp.core.linear_lookup(tf.convert_to_tensor(phase),
                                                 tf.convert_to_tensor(tab)))
    out['lookup_f32_%02d' % i] = n
    out['lookup_wide_%02d' % i] = w.astype(np.float64)
  return out


if __name__ == '__main__':
  got = linear_lookup()
  if '--check' in sys.argv:
    compare('linear_lookup', got, np.load(PATH))
    print('ok    linear_lookup')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote linear_lookup %.0f kB' % (os.path.getsize(PATH) / 1e3))
