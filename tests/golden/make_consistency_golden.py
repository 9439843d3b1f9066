"""Writes tests/golden/consistency.npz: outputs of the UNMODIFIED REFERENCE's
losses.KDEConsistencyLoss (call, nll), losses.TWMLoss (call, get_loss_tensors,
predict_f0), losses.HarmonicConsistencyLoss and core.harmonic_to_sinusoidal on seeded
inputs, run on the NumPy TensorFlow shim in its float64 (wide) mode.  The shim's
tensorflow_probability is a stub; `consistency()` installs tests/consistency_ref.py's
restatements of tfd.MixtureSameFamily, Categorical and Normal for the run and removes
them afterwards, so the shim itself is unchanged.

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_consistency_golden.py          # rewrite the fixture
  python tests/golden/make_consistency_golden.py --check  # regenerate and compare

tests/test_consistency_losses.py reads the fixture; the inputs come from the seeded
generators below.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests.golden.make_golden import _both, compare   # noqa: E402

PATH = os.path.join(HERE, 'consistency.npz')

# (name, B, T, Ka, Kb, edge, constructor keyword arguments)
KDE_CASES = [
    ('kde_default', 2, 3, 12, 12, None, {}),
    ('kde_args', 2, 2, 9, 5, 'zeros', dict(weight_a=0.7, weight_b=2.5, weight_mean_amp=0.3,
                                           scale_a=0.05, scale_b=0.4)),
    ('kde_k1', 3, 2, 1, 1, 'nonpositive', {}),
    ('kde_only_a', 1, 4, 6, 10, 'far', dict(weight_b=0.0, weight_mean_amp=0.0)),
]
# (name, B, T, C, P, edge, constructor keyword arguments); C = 0 means candidates =
# the sinusoid frequencies, as TWMEvaluator passes them
TWM_CASES = [
    ('twm_default', 2, 3, 0, 10, None, {}),
    ('twm_c1', 2, 3, 1, 8, 'zeros', {}),
    ('twm_args', 2, 2, 5, 7, 'edges', dict(sinusoids_weight=0.6, harmonics_weight=1.7,
                                           sinusoids_scale=0.3, harmonics_scale=0.1,
                                           n_harmonic_points=6, n_harmonic_gaussians=12,
                                           softmin_temperature=3.0, sample_rate=22050)),
    ('twm_wide', 1, 2, 4, 9, 'edges', dict(harmonics_scale=0.9, n_harmonic_gaussians=5,
                                           sample_rate=8000)),
]


def sinusoids(rng, b, t, k, edge=None):
  """Amplitudes in (0, 1] and frequencies over 40 Hz .. 7 kHz; `edge` adds exact zero
  amplitudes and an all-zero row ('zeros'), frequencies <= 0 ('nonpositive') or a
  row five octaves away from the rest ('far')."""
  amps = rng.uniform(0.05, 1.0, (b, t, k))
  freqs = np.exp(rng.uniform(np.log(40.0), np.log(7000.0), (b, t, k)))
  if edge == 'zeros':
    amps[0, 0, ::2] = 0.0
    amps[-1, -1, :] = 0.0
  elif edge == 'nonpositive':
    freqs[0, 0, 0] = 0.0
    freqs[-1, -1, 0] = -50.0
  elif edge == 'far':
    freqs[0, 0, :] = freqs[0, 0, :] / 32.0
  return amps.astype(np.float32), freqs.astype(np.float32)


def harmonic_sinusoids(rng, b, t, p):
  """Noisy harmonics of f0 in 80 .. 400 Hz: TWM's natural input."""
  f0 = np.exp(rng.uniform(np.log(80.0), np.log(400.0), (b, t, 1)))
  n = np.arange(1, p + 1)
  freqs = f0 * n * np.exp(rng.normal(0.0, 0.01, (b, t, p)))
  amps = rng.uniform(0.1, 1.0, (b, t, p)) / n
  return amps.astype(np.float32), freqs.astype(np.float32), f0


def kde_inputs(i):
  _, b, t, ka, kb, edge, _ = KDE_CASES[i]
  rng = np.random.default_rng(1700 + i)
  amps_a, freqs_a = sinusoids(rng, b, t, ka, edge)
  amps_b, freqs_b = sinusoids(rng, b, t, kb, edge if edge != 'far' else None)
  return amps_a, freqs_a, amps_b, freqs_b


def twm_inputs(i):
  _, b, t, c, p, edge, _ = TWM_CASES[i]
  rng = np.random.default_rng(1800 + i)
  amps, freqs, f0 = harmonic_sinusoids(rng, b, t, p)
  if c == 0:
    cands = freqs.copy()
  else:
    cands = (f0 * np.exp(rng.uniform(-0.7, 0.7, (b, t, c)))).astype(np.float32)
  if edge == 'zeros':
    amps[0, 0, ::2] = 0.0
    amps[-1, -1, :] = 0.0
  elif edge == 'edges':
    cands[0, 0, 0] = 0.0              # f0 = 0
    cands[-1, -1, -1] = 12000.0       # every harmonic above Nyquist
    freqs[0, -1, 0] = 0.0
    freqs[-1, 0, 1] = -30.0
  return cands, freqs, amps


def harmonic_inputs():
  rng = np.random.default_rng(1900)
  b, t, k = 2, 5, 6
  harm_amp = rng.uniform(0.0, 1.0, (b, t, 1)).astype(np.float32)
  harm_amp[0, 0, 0] = 5e-5                                    # below amp_threshold
  harm_dist = rng.uniform(0.0, 1.0, (b, t, k)).astype(np.float32)
  f0 = np.exp(rng.uniform(np.log(60.0), np.log(3000.0), (b, t, 1))).astype(np.float32)
  f0[1, 2, 0] = 9000.0                                        # all above Nyquist
  return harm_amp, harm_dist, f0


def _install(ddsp):
  """Restated tfd.MixtureSameFamily / Categorical / Normal; returns an undo."""
  from tests import consistency_ref as ref
  tfd = ddsp.losses.tfd
  names = {'MixtureSameFamily': ref.ShimMixtureSameFamily,
           'Categorical': ref.ShimCategorical, 'Normal': ref.ShimNormal}
  for k, v in names.items():
    setattr(tfd, k, v)

  def undo():
    for k in names:
      delattr(tfd, k)
  return undo


def consistency():
  ddsp = ref_on_shim.load()
  undo = _install(ddsp)
  wide = lambda fn: _both(fn)[1]
  try:
    losses = ddsp.losses
    out = {}
    for i, (name, *_, kw) in enumerate(KDE_CASES):
      x = kde_inputs(i)
      loss = losses.KDEConsistencyLoss(**kw)
      out[name + '_call'] = wide(lambda: loss(*x))
      out[name + '_nll'] = wide(lambda: loss.nll(x[0], x[1], x[2], x[3], loss.scale_b))
    for i, (name, *_, kw) in enumerate(TWM_CASES):
      x = twm_inputs(i)
      loss = losses.TWMLoss(**kw)
      out[name + '_call'] = wide(lambda: loss(*x))
      s, h = wide(lambda: loss.get_loss_tensors(*x))
      out[name + '_sinusoids'], out[name + '_harmonics'] = s, h
      out[name + '_f0'] = wide(lambda: loss.predict_f0(*x))
    harm_amp, harm_dist, f0 = harmonic_inputs()
    hc = losses.HarmonicConsistencyLoss(amp_weight=0.5, dist_weight=2.0, f0_weight=1.5)
    targets = harmonic_consistency_targets()
    got = wide(lambda: hc(harm_amp, targets[0], harm_dist, targets[1], f0, targets[2]))
    for k, v in got.items():
      out['harmonic_consistency_' + k] = v
    amps, freqs = wide(lambda: ddsp.core.harmonic_to_sinusoidal(harm_amp, harm_dist, f0))
    out['h2s_amps'], out['h2s_freqs'] = amps, freqs
    return {k: np.asarray(v, np.float64) for k, v in out.items()}
  finally:
    undo()


def harmonic_consistency_targets():
  harm_amp, harm_dist, f0 = harmonic_inputs()
  rng = np.random.default_rng(1901)
  return (harm_amp * rng.uniform(0.5, 1.5, harm_amp.shape).astype(np.float32),
          harm_dist[:, ::-1].copy(), f0 * np.float32(1.01))


if __name__ == '__main__':
  got = consistency()
  if '--check' in sys.argv:
    compare('consistency', got, np.load(PATH))
    print('ok    consistency')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote consistency %.0f kB' % (os.path.getsize(PATH) / 1e3))
