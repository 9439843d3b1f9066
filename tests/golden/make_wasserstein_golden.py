"""Writes tests/golden/wasserstein.npz: outputs of the UNMODIFIED REFERENCE's
losses.wasserstein_distance and losses.WassersteinConsistencyLoss on seeded inputs, run
on the NumPy TensorFlow shim in its float64 (wide) mode.

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_wasserstein_golden.py          # rewrite the fixture
  python tests/golden/make_wasserstein_golden.py --check  # regenerate and compare

tests/test_wasserstein.py reads the fixture; the inputs come from the seeded generators
below.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests.golden.make_golden import _both, compare   # noqa: E402

PATH = os.path.join(HERE, 'wasserstein.npz')

# (name, batch shape, n_u, n_v, p, edge)
DISTANCE_CASES = [
    ('p1', (3,), 7, 7, 1.0, None),
    ('p2', (2, 3), 9, 5, 2.0, None),
    ('p_half', (2, 3), 6, 11, 0.5, None),
    ('one_d', (), 8, 3, 1.0, None),
    ('four_d', (2, 2, 2), 5, 6, 1.0, None),
    ('ties', (2, 3), 10, 8, 1.0, 'ties'),
    ('ties_p2', (4,), 12, 12, 2.0, 'ties'),
    ('zero_weights', (2, 3), 8, 6, 1.0, 'zeros'),
    ('totals_differ', (3,), 6, 9, 1.0, 'scaled'),
    ('one_each', (4,), 1, 1, 1.0, None),
    ('one_u', (2, 2), 1, 6, 2.0, None),
    ('one_v', (3,), 5, 1, 0.5, None),
]
# (name, B, T, n_a, n_b, weight, midi)
LOSS_CASES = [
    (f'loss_w{w}_midi{int(m)}', 2, 3, 6, 4, w, m)
    for w in (1.0, 0.3, 0.0) for m in (True, False)
]


def distance_inputs(i):
  """Values and weights of DISTANCE_CASES[i]: values over [-3, 3], weights in (0, 1];
  `edge` puts the values on a grid of 0.5 so that they tie within u and across u and v
  ('ties'), zeroes every third weight and a whole row of u's ('zeros'), or scales v's
  weights by 3 ('scaled')."""
  _, batch, nu, nv, _, edge = DISTANCE_CASES[i]
  rng = np.random.default_rng(2100 + i)
  u = rng.uniform(-3.0, 3.0, batch + (nu,))
  v = rng.uniform(-3.0, 3.0, batch + (nv,))
  wu = rng.uniform(0.05, 1.0, batch + (nu,))
  wv = rng.uniform(0.05, 1.0, batch + (nv,))
  if edge == 'ties':
    u = np.round(u * 2.0) / 2.0
    v = np.round(v * 2.0) / 2.0
  elif edge == 'zeros':
    wu[..., ::3] = 0.0
    wv[..., 1::3] = 0.0
    wu[0, 0, :] = 0.0
  elif edge == 'scaled':
    wv = wv * 3.0
  return tuple(x.astype(np.float32) for x in (u, v, wu, wv))


def loss_inputs(i):
  """Sinusoids of LOSS_CASES[i]: amplitudes in (0, 1], frequencies over 40 Hz .. 7 kHz,
  with a 0 Hz and a negative frequency (MIDI 0) and one exact zero amplitude."""
  _, b, t, na, nb, _, _ = LOSS_CASES[i]
  rng = np.random.default_rng(2200 + i)
  amps_a = rng.uniform(0.05, 1.0, (b, t, na))
  amps_b = rng.uniform(0.05, 1.0, (b, t, nb))
  freqs_a = np.exp(rng.uniform(np.log(40.0), np.log(7000.0), (b, t, na)))
  freqs_b = np.exp(rng.uniform(np.log(40.0), np.log(7000.0), (b, t, nb)))
  freqs_a[0, 0, 0] = 0.0
  freqs_b[-1, -1, 0] = -50.0
  amps_b[0, 1, 1] = 0.0
  return tuple(x.astype(np.float32) for x in (amps_a, freqs_a, amps_b, freqs_b))


def wasserstein():
  ddsp = ref_on_shim.load()
  wide = lambda fn: _both(fn)[1]
  losses = ddsp.losses
  out = {}
  for i, (name, *_, p, _) in enumerate(DISTANCE_CASES):
    x = distance_inputs(i)
    out[name] = wide(lambda: losses.wasserstein_distance(*x, p=p))
  for i, (name, *_, w, m) in enumerate(LOSS_CASES):
    x = loss_inputs(i)
    loss = losses.WassersteinConsistencyLoss(weight=w, midi=m)
    out[name] = wide(lambda: loss(*x))
  return {k: np.asarray(v, np.float64) for k, v in out.items()}


if __name__ == '__main__':
  got = wasserstein()
  if '--check' in sys.argv:
    compare('wasserstein', got, np.load(PATH))
    print('ok    wasserstein')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote wasserstein %.0f kB' % (os.path.getsize(PATH) / 1e3))
