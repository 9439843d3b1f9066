"""Writes tests/golden/crepe.npz: outputs of the UNMODIFIED REFERENCE's spectral_ops.pad
and PretrainedCREPE's batch_frames, normalize_frames, activations_to_f0_and_confidence
and viterbi_decode on seeded inputs, run on the NumPy TensorFlow shim in its float64
(wide) mode.  tests/test_crepe.py pins tests/crepe_ref.py to it.

The shim's tensorflow_probability is a stub, so `_install` puts tests/hmm_ref.py's
Categorical and tests/crepe_ref.py's Multinomial and HiddenMarkovModel into it, and the
shim's tf.gather, whose batch_dims=1 takes along axis 0, is replaced for this run by
TensorFlow's batch_dims semantics.  PretrainedCREPE is built without its __init__,
which would load the crepe package's weights; these methods do not touch the network.
The shim itself is unchanged.

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_crepe_golden.py          # rewrite the fixture
  python tests/golden/make_crepe_golden.py --check  # regenerate and compare
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests.golden.make_golden import compare          # noqa: E402

PATH = os.path.join(HERE, 'crepe.npz')

# pad: (name, shape, frame_size, hop_size, padding, axis, mode)
PAD_CASES = [
    ('center', (2, 3000), 1024, 160, 'center', 1, 'CONSTANT'),
    ('same', (2, 3000), 1024, 160, 'same', 1, 'CONSTANT'),
    ('same_exact', (3, 1600), 1024, 160, 'same', 1, 'CONSTANT'),
    ('valid', (2, 3000), 1024, 2048, 'valid', 1, 'CONSTANT'),
    ('one_d', (700,), 64, 16, 'center', 1, 'CONSTANT'),
    ('axis0', (40, 3), 16, 4, 'same', 0, 'CONSTANT'),
    ('reflect', (2, 100), 64, 16, 'center', 1, 'REFLECT'),
    ('symmetric', (2, 100), 64, 16, 'center', 1, 'symmetric'),
]

# frames: (name, B, N, hop, padding)
FRAME_CASES = [
    ('center320', 1, 1800, 320, 'center'),
    ('same320', 1, 1800, 320, 'same'),
    ('valid480', 2, 2000, 480, 'valid'),
    ('center512', 1, 1100, 512, 'center'),
    ('same1024', 1, 3000, 1024, 'same'),
    ('exact1024', 2, 1024, 160, 'valid'),
    ('short_same', 2, 100, 160, 'same'),
]

# viterbi: (name, B, T)
VITERBI_CASES = [('t1', 2, 1), ('t2', 2, 2), ('t7', 3, 7), ('t60', 2, 60), ('t200', 1, 200)]


def pad_input(i):
  return np.random.default_rng(3100 + i).normal(size=PAD_CASES[i][1])


def frame_input(i):
  _, b, n, _, _ = FRAME_CASES[i]
  x = np.random.default_rng(3200 + i).normal(size=(b, n))
  x[:, n // 4:n // 4 + 1100] = 0.25     # a constant stretch: frames of zero variance
  return x


def activations(rng, b, t, noise=0.05):
  """Sigmoid-like activations [B, T, 360]: a wandering pitch track with a Gaussian bump
  around it, some jumps, and noise."""
  centre = np.clip(180 + np.cumsum(rng.normal(0, 3, (b, t)), -1), 0, 359)
  jumps = rng.uniform(size=(b, t)) < 0.05
  centre = np.where(jumps, rng.uniform(0, 359, (b, t)), centre)
  bins = np.arange(360)
  act = 0.9 * np.exp(-0.5 * ((bins - centre[..., None]) / 2.0) ** 2)
  return np.clip(act + noise * rng.uniform(size=act.shape), 0.0, 1.0)


def viterbi_input(i):
  _, b, t = VITERBI_CASES[i]
  return activations(np.random.default_rng(3300 + i), b, t)


def decode_input():
  """Rows [64, 360]: random ones, and peaks at every edge bin 0..5 and 354..359."""
  rng = np.random.default_rng(3400)
  acts = rng.uniform(size=(64, 360)) * 0.1
  for r, c in enumerate([0, 1, 2, 3, 4, 5, 354, 355, 356, 357, 358, 359, 100, 250]):
    acts[r, c] = 1.0
  centers = rng.integers(-10, 370, size=64)
  return acts, centers


def _install(ddsp):
  """The restated tfp classes, and tf.gather with batch_dims=1, in the namespaces the
  reference's spectral_ops reads."""
  from tests import crepe_ref
  from tests import hmm_ref
  tf, tfp = ddsp.spectral_ops.tf, ddsp.spectral_ops.tfp
  tfp.distributions.Categorical = hmm_ref.ShimCategorical
  tfp.distributions.Multinomial = crepe_ref.ShimMultinomial
  tfp.distributions.HiddenMarkovModel = crepe_ref.ShimHiddenMarkovModel
  shim_gather = tf.gather

  def gather(params, indices, axis=0, batch_dims=0, name=None):
    if batch_dims == 1 and axis == 0:      # TensorFlow's batch_dims: rows stay aligned
      a, i = np.asarray(params.numpy() if hasattr(params, 'numpy') else params), \
          np.asarray(indices.numpy() if hasattr(indices, 'numpy') else indices)
      return tf.constant(np.take_along_axis(a, i, axis=1))
    return shim_gather(params, indices, axis=axis, batch_dims=batch_dims, name=name)
  tf.gather = gather


def crepe():
  ddsp = ref_on_shim.load()
  _install(ddsp)
  tf = ref_on_shim.tf()
  tf.set_wide(True)
  try:
    out = {}
    so = ddsp.spectral_ops
    for i, (name, _, frame, hop, padding, axis, mode) in enumerate(PAD_CASES):
      out['pad_' + name] = so.pad(pad_input(i), frame, hop, padding=padding, axis=axis,
                                  mode=mode)
    for i, (name, _, _, hop, padding) in enumerate(FRAME_CASES):
      model = so.PretrainedCREPE.__new__(so.PretrainedCREPE)
      model.hop_size, model.frame_size = hop, 1024
      padded = so.pad(frame_input(i), 1024, hop, padding=padding)
      out['frames_' + name] = model.normalize_frames(model.batch_frames(padded))
    acts, centers = decode_input()
    f0, conf = so.PretrainedCREPE.activations_to_f0_and_confidence(acts)
    out['decode_f0'], out['decode_confidence'] = f0, conf
    f0, conf = so.PretrainedCREPE.activations_to_f0_and_confidence(acts, centers)
    out['decode_given_f0'], out['decode_given_confidence'] = f0, conf
    for i, (name, _, _) in enumerate(VITERBI_CASES):
      model = so.PretrainedCREPE.__new__(so.PretrainedCREPE)
      out['viterbi_' + name] = model.viterbi_decode(viterbi_input(i))
    return {k: np.asarray(ref_on_shim.to_numpy(v), np.float64) for k, v in out.items()}
  finally:
    tf.set_wide(False)


if __name__ == '__main__':
  got = crepe()
  if '--check' in sys.argv:
    compare('crepe', got, np.load(PATH))
    print('ok    crepe')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote crepe %.0f kB' % (os.path.getsize(PATH) / 1e3))
