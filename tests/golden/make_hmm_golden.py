"""Writes tests/golden/hmm.npz: outputs of the UNMODIFIED REFERENCE's
losses.HmmTranscriber (log_prob, nll with and without per_example_loss, predict_midi) on
seeded note sequences, run on the NumPy TensorFlow shim in its float64 (wide) mode.

The shim's tensorflow_probability is a stub, and HmmTranscriber binds its base class
tfp.distributions.HiddenMarkovModel when losses.py is imported.  So `hmm()` installs
tests/hmm_ref.py's restatements of HiddenMarkovModel, Categorical and
MultivariateNormalDiag into the shim's tfp BEFORE the reference package is imported,
and this script must run in a process that has not imported it yet.  The shim itself is
unchanged.

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_hmm_golden.py          # rewrite the fixture
  python tests/golden/make_hmm_golden.py --check  # regenerate and compare

tests/test_hmm_transcriber.py reads the fixture; the inputs come from `inputs` below.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests.golden.make_golden import compare          # noqa: E402

PATH = os.path.join(HERE, 'hmm.npz')

# (name, B, constructor keyword arguments; n_timesteps is T)
CASES = [
    ('default', 2, {}),
    ('k2', 3, dict(n_pitches=2, n_timesteps=40)),
    ('k3', 3, dict(n_pitches=3, n_timesteps=40)),
    ('avg1', 2, dict(avg_length=1, n_pitches=16, n_timesteps=60)),
    ('avg2', 2, dict(avg_length=2, n_pitches=16, n_timesteps=60)),
    ('avg1e6', 2, dict(avg_length=1e6, n_timesteps=200)),
    ('off_centre', 2, dict(amps_on_center=0.7, amps_on_scale=0.3, amps_off_center=0.2,
                           amps_off_scale=0.05, midi_std=0.8, n_pitches=64,
                           n_timesteps=120, weight=5.0)),
    ('t1', 3, dict(n_timesteps=1)),
    ('t5', 2, dict(n_timesteps=5, avg_length=10)),
]

DEFAULTS = dict(avg_length=200, midi_std=0.5, amps_on_center=1.5, amps_on_scale=0.5,
                amps_off_center=0.0, amps_off_scale=0.1, n_timesteps=1000,
                n_pitches=128, weight=1.0)


def case_kwargs(i):
  return dict(DEFAULTS, **CASES[i][2])


def notes(rng, b, t, k=128, amps_on_center=1.5, amps_off_center=0.0, midi_std=0.5,
          **_):
  """Noisy note sequences (pitch [B, T, 1] in MIDI, amps [B, T, 1]): runs of random
  length, a quarter of them silent (amplitude near amps_off_center, pitch anywhere),
  the rest a pitch in 1 .. K - 1 with noise of midi_std / 2 and amplitude near
  amps_on_center."""
  pitch = np.empty((b, t, 1))
  amps = np.empty((b, t, 1))
  for i in range(b):
    s = 0
    while s < t:
      n = min(t - s, int(rng.integers(1, max(2, t // 4))))
      if rng.uniform() < 0.25:
        pitch[i, s:s + n, 0] = rng.uniform(0.0, k - 1.0, n)
        amps[i, s:s + n, 0] = amps_off_center + 0.05 * rng.normal(size=n)
      else:
        pitch[i, s:s + n, 0] = rng.integers(1, k) + 0.25 * midi_std * rng.normal(size=n)
        amps[i, s:s + n, 0] = amps_on_center + 0.2 * rng.normal(size=n)
      s += n
  return pitch.astype(np.float32), amps.astype(np.float32)


def inputs(i):
  name, b, _ = CASES[i]
  kw = case_kwargs(i)
  return notes(np.random.default_rng(2100 + i), b, kw['n_timesteps'], kw['n_pitches'],
               **kw)


def _install():
  """Restated tfd.HiddenMarkovModel / Categorical / MultivariateNormalDiag, before the
  reference's losses.py binds its base class."""
  assert 'ddsp.losses' not in sys.modules, (
      'the reference was imported before its tfp could be restated')
  sys.path.insert(0, ref_on_shim.SHIM_DIR)
  import tensorflow_probability as tfp    # the shim's
  from tests import hmm_ref as ref
  names = {'HiddenMarkovModel': ref.ShimHiddenMarkovModel,
           'Categorical': ref.ShimCategorical,
           'MultivariateNormalDiag': ref.ShimMultivariateNormalDiag}
  for k, v in names.items():
    setattr(tfp.distributions, k, v)


def hmm():
  _install()
  ddsp = ref_on_shim.load()
  tf = ref_on_shim.tf()
  tf.set_wide(True)
  try:
    out = {}
    for i, (name, _, kw) in enumerate(CASES):
      pitch, amps = inputs(i)
      hmm_ = ddsp.losses.HmmTranscriber(**kw)
      pa = tf.concat([pitch, amps], axis=-1)
      got = {'log_prob': hmm_.log_prob(pa), 'nll': hmm_.nll(pitch, amps),
             'nll_per_example': hmm_.nll(pitch, amps, per_example_loss=True),
             'predict_midi': hmm_.predict_midi(pitch, amps)}
      for k, v in got.items():
        out[name + '_' + k] = np.asarray(ref_on_shim.to_numpy(v), np.float64)
    return out
  finally:
    tf.set_wide(False)


if __name__ == '__main__':
  got = hmm()
  if '--check' in sys.argv:
    compare('hmm', got, np.load(PATH))
    print('ok    hmm')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote hmm %.0f kB' % (os.path.getsize(PATH) / 1e3))
