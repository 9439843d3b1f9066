"""Writes tests/golden/embedding_loss.npz: outputs of the UNMODIFIED REFERENCE's
losses.PretrainedCREPE.frame_audio and call, EmbeddingLoss.call and the weights
PretrainedCREPEEmbeddingLoss derives, run on the NumPy TensorFlow shim in its float64
(wide) mode.  tests/test_embedding_loss.py pins tests/embedding_ref.py to it.

PretrainedCREPE is built with __new__, as in make_crepe_golden.py, because its
__init__ loads the crepe package's weights; its `_activation_model` is the stub network
of tests/embedding_ref.py.  For the weights, the loaded losses module's PretrainedCREPE
is replaced by a stand-in for this run.  mean_difference's COSINE calls
tf.losses.cosine_distance, which the shim lacks: tests/embedding_ref.cosine_distance
(TF1's function, on unit vectors 1 - the cosine similarity) is installed as the loaded
shim's for this run, and the COSINE case uses the stub scaled to unit length.  The
shim's files are not changed.

Frames of long cases are many: the fixture keeps the first and the last frame of each
(all frames are checked against the restatement on the GPU).

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_embedding_loss_golden.py          # rewrite the fixture
  python tests/golden/make_embedding_loss_golden.py --check  # regenerate and compare
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests import embedding_ref                       # noqa: E402
from tests.golden.make_golden import compare          # noqa: E402

PATH = os.path.join(HERE, 'embedding_loss.npz')

HOPS = (1, 160, 512, 1024, 2048)
LENGTHS = (0, 1000, 1024, 3000, 64000)
# (name, hop, center, N) for every combination that gives at least one frame
FRAME_CASES = [(f'h{hop}_{"c" if center else "v"}_n{n}', hop, center, n)
               for hop in HOPS for center in (True, False) for n in LENGTHS
               if embedding_ref.n_frames(n, hop, center) > 0]
LOSS_TYPES = ('L1', 'L2', 'COSINE')
LOSS_WEIGHT = 2.5
LAYERS = ('conv1-BN', 'conv1-maxpool', 'conv2-BN', 'conv2-maxpool', 'conv3-BN',
          'conv3-maxpool', 'conv4-BN', 'conv4-maxpool', 'conv5-BN', 'conv5-maxpool',
          'conv6-BN', 'conv6-maxpool', 'classifier')
LAYER_WEIGHT = 0.75


def frame_input(i):
  """Audio [1, N]; from 3000 samples on, a constant stretch gives frames of variance 0."""
  n = FRAME_CASES[i][3]
  x = np.random.default_rng(4200 + i).normal(size=(1, n)) * 0.3
  if n >= 3000:
    x[:, 1000:2100] = 0.25
  return x


def kept_rows(f):
  """The frames the fixture keeps of f: the first and the last."""
  return sorted({0, f - 1})


def call_input():
  return np.random.default_rng(4300).normal(size=(2, 3000)) * 0.5


def loss_inputs():
  rng = np.random.default_rng(4400)
  return rng.normal(size=(2, 4000)) * 0.5, rng.normal(size=(2, 4000)) * 0.5


def _stub_model(tf, activations):
  return lambda frames: tf.constant(activations(ref_on_shim.to_numpy(frames)))


def embedding():
  ddsp = ref_on_shim.load()
  tf = ref_on_shim.tf()
  losses = ddsp.losses
  tf.set_wide(True)
  shim_cosine, shim_crepe = tf.losses.cosine_distance, losses.PretrainedCREPE
  tf.losses.cosine_distance = lambda labels, predictions, weights=1.0, axis=-1: \
      tf.constant(embedding_ref.cosine_distance(ref_on_shim.to_numpy(labels),
                                                ref_on_shim.to_numpy(predictions), axis))
  try:
    out = {}

    def crepe(activations=embedding_ref.stub_activations):
      m = shim_crepe.__new__(shim_crepe)
      m.frame_length = 1024
      m._activation_model = _stub_model(tf, activations)
      m.built = True    # build() reads the crepe model's layers
      return m

    for i, (name, hop, center, n) in enumerate(FRAME_CASES):
      frames = ref_on_shim.to_numpy(crepe().frame_audio(frame_input(i), hop_length=hop,
                                                        center=center))
      out['frames_' + name] = np.asarray(frames)[:, kept_rows(frames.shape[1])]
    out['call'] = crepe().call(call_input())
    target, audio = loss_inputs()
    for loss_type in LOSS_TYPES:
      act = (embedding_ref.unit_stub_activations if loss_type == 'COSINE'
             else embedding_ref.stub_activations)
      loss = losses.EmbeddingLoss(weight=LOSS_WEIGHT, loss_type=loss_type,
                                  pretrained_model=crepe(act))
      out['loss_' + loss_type] = loss.call(target, audio)
    zero = losses.EmbeddingLoss(weight=0.0, pretrained_model=None).call(target, audio)
    assert isinstance(zero, float), type(zero)
    out['loss_weight0'] = zero
    losses.PretrainedCREPE = lambda **kwargs: None
    out['layer_weights'] = [
        losses.PretrainedCREPEEmbeddingLoss(weight=LAYER_WEIGHT, activation_layer=l).weight
        for l in LAYERS]
    return {k: np.asarray(ref_on_shim.to_numpy(v), np.float64) for k, v in out.items()}
  finally:
    tf.set_wide(False)
    tf.losses.cosine_distance, losses.PretrainedCREPE = shim_cosine, shim_crepe


if __name__ == '__main__':
  got = embedding()
  if '--check' in sys.argv:
    compare('embedding_loss', got, np.load(PATH))
    print('ok    embedding_loss')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote embedding_loss %.0f kB' % (os.path.getsize(PATH) / 1e3))
