"""Writes tests/golden/notes.npz: outputs of the UNMODIFIED REFERENCE's note functions
(training/nn.py:375-557: get_note_mask, get_note_mask_from_onset, get_note_moments,
pool_over_notes, get_note_lengths, get_short_note_loss_mask) on seeded inputs, run on
the NumPy TensorFlow shim in its float64 (wide) mode.

ddsp/training/__init__.py imports google.cloud, so nn.py is loaded by its file path
under a stub `ddsp.training` package.  Its module body subclasses keras classes the
shim does not build (tf.keras.Sequential, tf.keras.layers.Wrapper, Dense, ...); this
script gives them stand-in classes that raise when instantiated.  No layer is used.

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_notes_golden.py          # rewrite the fixture
  python tests/golden/make_notes_golden.py --check  # regenerate and compare
"""
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests.golden.make_golden import _both, compare   # noqa: E402

PATH = os.path.join(HERE, 'notes.npz')
NAN, INF = np.nan, np.inf

# (name, q_pitch rows, max_regions): get_note_mask, with note_on_only both ways
MASK_CASES = [
    ('last_frame', [[0, 0, 60, 60, 60, 62, 62, 0, 0, 64]], 5),
    ('t1', [[3.0], [-2.0], [0.0]], 3),
    ('t2', [[1, 2], [0, 5], [-1, -1]], 3),
    ('t3', [[1, 2, 3], [0, 0, -1], [4, 4, 4]], 4),
    ('over_max_regions', 'random_transitions', 6),
    ('c3', 'three_channels', 100),
    ('nonfinite', [[1, INF, INF, 2, NAN, 5, 5], [60, 60, -INF, -INF, 0, 7, 7],
                   [NAN, 3, 3, 3, 4, 4, 0], [5, 5, 6, 6, 6, 6, INF]], 6),
    ('finite_rows', [[1, 1, 2, 2, -3, -3, 0], [60, 60, 0, 0, 64, 64, 64]], 6),
    ('last_frame_sign', [[0, 0, 2, 2, 2, -7], [-1, -1, -1, 0, 3, 3], [5, 5, 5, 5, 5, -20]], 4),
]
# (name, q rows, onset rows, max_regions): get_note_mask_from_onset
ONSET_CASES = [
    ('onset_trunc', [[0, 0, 60, 60, 60, 62, 62, 0, 0, 64]],
     [[0, 1.7, -1, 2, 0, 0, 1, 0, 0, 0]], 4),
    ('onset_first_ignored', [[5, 5, 0, 7], [1, -1, 1, 1]], [[3, 0, 1, 0], [1, 1, 1, 1]], 3),
    ('onset_t1', [[2.0], [-1.0]], [[1.0], [0.0]], 2),
]
# (name, x shape, mask kind): get_note_moments and pool_over_notes
MOMENT_CASES = [
    ('x3_binary', (2, 12, 5), 'binary'),
    ('x2_binary', (3, 9), 'binary'),
    ('x3_soft', (2, 11, 4), 'soft'),
    ('x2_soft', (2, 8), 'soft'),
    ('x3_empty_const', (2, 10, 3), 'const'),
]


def mask_input(i):
  _, q, _ = MASK_CASES[i]
  rng = np.random.default_rng(3100 + i)
  if q == 'random_transitions':
    return rng.integers(0, 4, (3, 40)).astype(np.float32)
  if q == 'three_channels':
    q = rng.integers(0, 3, (2, 16, 3)).astype(np.float32)
    q[:, :, 1:] = rng.normal(size=(2, 16, 2)) * 100.0   # only channel 0 counts
    return q
  return np.asarray(q, np.float32)


def onset_inputs(i):
  _, q, on, _ = ONSET_CASES[i]
  return np.asarray(q, np.float32), np.asarray(on, np.float32)


def moment_inputs(i):
  """x over N(0, 1) plus an offset of 3 (a large mean), and the mask: 'binary' from the
  edges of integer pitches with 6 regions, 'soft' uniform on [0, 1) over 5 notes,
  'const' a binary mask with an empty note and x constant and integer-valued on a note."""
  _, shape, kind = MOMENT_CASES[i]
  rng = np.random.default_rng(3300 + i)
  x = (rng.normal(size=shape) + 3.0).astype(np.float32)
  b, t = shape[:2]
  if kind == 'soft':
    return x, rng.uniform(0.0, 1.0, (b, t, 5)).astype(np.float32)
  idx = np.sort(rng.integers(0, 4, (b, t)), axis=1)
  mask = (idx[..., None] == np.arange(6)).astype(np.float32)
  if kind == 'const':
    first = idx[:, :1] == idx
    x[first] = 2.0
  return x, mask


def _load_nn():
  ddsp = ref_on_shim.load()
  if 'ddsp.training.nn' in sys.modules:
    return ddsp, sys.modules['ddsp.training.nn']
  tf = ref_on_shim.tf()

  def unbuilt(name):
    def init(self, *args, **kwargs):
      raise NotImplementedError(f'tf.keras {name} is not on the shim')
    return type(name, (), {'__init__': init})

  type(tf.keras.layers).__getattr__ = lambda self, item: unbuilt(item)
  tf.keras.Sequential = unbuilt('Sequential')
  root = os.path.join(ref_on_shim.REFERENCE_ROOT, 'ddsp', 'training')
  pkg = types.ModuleType('ddsp.training')
  pkg.__path__ = [root]
  sys.modules['ddsp.training'] = pkg
  spec = importlib.util.spec_from_file_location('ddsp.training.nn',
                                                os.path.join(root, 'nn.py'))
  nn = importlib.util.module_from_spec(spec)
  sys.modules['ddsp.training.nn'] = nn
  spec.loader.exec_module(nn)
  return ddsp, nn


def notes():
  _, nn = _load_nn()
  tf = ref_on_shim.tf()
  c = tf.constant
  wide = lambda fn: _both(fn)[1]
  out = {}
  with np.errstate(invalid='ignore'):
    for i, (name, _, r) in enumerate(MASK_CASES):
      q = mask_input(i)
      for on in (True, False):
        out[f'{name}_on{int(on)}'] = wide(
            lambda: nn.get_note_mask(c(q), max_regions=r, note_on_only=on))
    for i, (name, _, _, r) in enumerate(ONSET_CASES):
      q, onset = onset_inputs(i)
      for on in (True, False):
        out[f'{name}_on{int(on)}'] = wide(
            lambda: nn.get_note_mask_from_onset(c(q), c(onset), max_regions=r,
                                                note_on_only=on))
    for i, (name, _, _) in enumerate(MOMENT_CASES):
      x, m = moment_inputs(i)
      mean, std = wide(lambda: nn.get_note_moments(c(x), c(m)))
      out[f'{name}_mean'], out[f'{name}_std'] = mean, std
      out[f'{name}_mean_only'] = wide(lambda: nn.get_note_moments(c(x), c(m), False))
      if x.ndim == 3:
        pm, ps = wide(lambda: nn.pool_over_notes(c(x), c(m)))
        out[f'{name}_pool_mean'], out[f'{name}_pool_std'] = pm, ps
      lengths = wide(lambda: nn.get_note_lengths(c(m)))
      out[f'{name}_lengths'] = lengths
      out[f'{name}_short'] = wide(lambda: nn.get_short_note_loss_mask(
          c(m), c(lengths), c(np.asarray(mean if mean.ndim == 2 else mean[..., 0])),
          min_length=4))
  return {k: np.asarray(v, np.float64) for k, v in out.items()}


if __name__ == '__main__':
  got = notes()
  if '--check' in sys.argv:
    compare('notes', got, np.load(PATH))
    print('ok    notes')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote notes %.0f kB' % (os.path.getsize(PATH) / 1e3))
