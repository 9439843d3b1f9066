"""Writes tests/golden/synthetic_data.npz: outputs of the UNMODIFIED REFERENCE's
training/data_preparation/synthetic_data.py (generate_notes_v2 and generate_notes) on
the NumPy TensorFlow shim, with numpy's global RandomState seeded per case.

ddsp/training/__init__.py imports google.cloud, so synthetic_data.py is loaded by its
file path under stub `ddsp.training` and `ddsp.training.data_preparation` packages.  To
store the reference's float64 arrays from before its TF steps, this script wraps (in
the loaded module's namespace, without changing what they return or draw)
`ddsp.core.exp_sigmoid`, `ddsp.core.midi_to_hz` and `tf.nn.softmax`, which record their
inputs, and `uniform_float`, whose last call in generate_notes_v2 is the harm_amp
divisor.

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_synthetic_data_golden.py          # rewrite the fixture
  python tests/golden/make_synthetic_data_golden.py --check  # regenerate and compare
"""
import hashlib
import importlib.util
import os
import sys
import types
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                   # noqa: E402

PATH = os.path.join(HERE, 'synthetic_data.npz')


def example_seeds(n, random_seed=42):
  np.random.seed(random_seed)
  return np.random.randint(2**32, size=n)


# (name, seed, kwargs) of seeded n_batch=1 calls of generate_notes_v2.  The edge
# configurations use few harmonics and noise bands: the behaviour they pin does not
# depend on K and M, and the file stays small.
SMALL = dict(n_harmonics=16, n_mags=8)
V2_CASES = (
    [('seed0', 0, {}), ('seed1', 1, {}), ('seedmax', 2**32 - 1, {})] +
    [(f'example{i}', int(s), {}) for i, s in enumerate(example_seeds(4))] +
    [('t1', 5, dict(n_timesteps=1, min_note_length=1, max_note_length=1)),
     ('k1m1', 6, dict(n_harmonics=1, n_mags=1)),
     ('silent', 7, dict(p_silent=1.0, **SMALL)),
     ('novibrato', 8, dict(p_vibrato=0.0, **SMALL)),
     ('vibrato', 9, dict(p_vibrato=1.0, **SMALL)),
     ('nocontrols', 10, dict(get_controls=False, **SMALL)),
     ('long', 11, dict(n_timesteps=1000, min_note_length=1, max_note_length=200,
                       n_harmonics=2, n_mags=2))])
# Paper-shape cases whose float64 arrays are stored as SHA-256 digests of their
# little-endian bytes (`digest`), with only the small float32 outputs in full: the
# restatement reproduces them bit for bit, and one full paper-shape case (seed0) is
# enough to hold the kernel to the values themselves.
DIGEST_CASES = ('seed1', 'seedmax', 'example0', 'example1', 'example2', 'example3')
# state-mode calls: (name, seed, draws before the call, kwargs) with n_batch = 3
STATE_CASES = (('state_a', 21, 0, dict(n_timesteps=60, **SMALL)),
               ('state_b', 22, 3, dict(n_timesteps=60, get_controls=False, **SMALL)))
# generate_notes calls: (name, seed, n_batch, n_timesteps, n_harmonics, n_mags)
V1_CASES = (('v1_b1', 31, 1, 125, 100, 65), ('v1_b4', 32, 4, 125, 16, 8))
# sin_freqs is f0_hz times 1..K and is not stored
OUTPUTS = ('harm_amp', 'harm_dist', 'f0_hz', 'sin_amps', 'noise_magnitudes')
SMALL_OUTPUTS = ('harm_amp', 'f0_hz')
RAW = ('harm_amp', 'harm_dist', 'f0_midi', 'mags')


def digest(a):
  """SHA-256 of a float64 array's little-endian C-order bytes, as a numpy bytes scalar."""
  return np.bytes_(hashlib.sha256(np.ascontiguousarray(a, '<f8').tobytes()).hexdigest())


def _load():
  ddsp = ref_on_shim.load()
  name = 'ddsp.training.data_preparation.synthetic_data'
  if name in sys.modules:
    return ddsp, sys.modules[name]
  root = os.path.join(ref_on_shim.REFERENCE_ROOT, 'ddsp', 'training')
  for pkg_name, path in (('ddsp.training', root),
                         ('ddsp.training.data_preparation',
                          os.path.join(root, 'data_preparation'))):
    if pkg_name not in sys.modules:
      pkg = types.ModuleType(pkg_name)
      pkg.__path__ = [path]
      sys.modules[pkg_name] = pkg
  spec = importlib.util.spec_from_file_location(
      name, os.path.join(root, 'data_preparation', 'synthetic_data.py'))
  m = importlib.util.module_from_spec(spec)
  sys.modules[name] = m
  with warnings.catch_warnings():
    warnings.simplefilter('ignore')
    spec.loader.exec_module(m)
  return ddsp, m


class _Recorder:
  """Records the inputs of exp_sigmoid, midi_to_hz and softmax and the last
  uniform_float of one call of the loaded module, and leaves their results alone."""

  def __init__(self, ddsp, m):
    self.ddsp, self.m = ddsp, m

  def __enter__(self):
    core, tf, m = self.ddsp.core, ref_on_shim.tf(), self.m
    self.saved = (core.exp_sigmoid, core.midi_to_hz, tf.nn.softmax, m.uniform_float)
    exp_sigmoid, midi_to_hz, softmax, uniform_float = self.saved
    self.sig, self.midi, self.soft, self.uniforms = [], [], [], []

    def rec(store, fn):
      def wrapped(x, *a, **k):
        store.append(np.array(ref_on_shim.to_numpy(x), copy=True))
        return fn(x, *a, **k)
      return wrapped

    def rec_uniform(*a, **k):
      v = uniform_float(*a, **k)
      self.uniforms.append(v)
      return v

    core.exp_sigmoid = rec(self.sig, exp_sigmoid)
    core.midi_to_hz = rec(self.midi, midi_to_hz)
    tf.nn.softmax = rec(self.soft, softmax)
    m.uniform_float = rec_uniform
    return self

  def __exit__(self, *exc):
    core, tf = self.ddsp.core, ref_on_shim.tf()
    core.exp_sigmoid, core.midi_to_hz, tf.nn.softmax, self.m.uniform_float = self.saved


def _state(prefix):
  _, key, pos, has_gauss, gauss = np.random.get_state()
  return {f'{prefix}_key': key.copy(), f'{prefix}_pos': np.int64(pos),
          f'{prefix}_has_gauss': np.int64(has_gauss), f'{prefix}_gauss': np.float64(gauss)}


def _v2(ddsp, m, name, kwargs, n_batch=1):
  out = {}
  get_controls = kwargs.get('get_controls', True)
  with _Recorder(ddsp, m) as r:
    c = m.generate_notes_v2(n_batch=n_batch, **kwargs)
  c = ref_on_shim.to_numpy(c)
  raw = {'f0_midi': r.midi[0][..., 0]}
  if get_controls:
    raw.update(harm_amp=r.sig[0][..., 0], mags=r.sig[1], harm_dist=r.soft[0])
    out[f'{name}_divisor'] = np.float64(r.uniforms[-1])
  else:
    raw.update(harm_amp=np.asarray(c['harm_amp'])[..., 0],
               mags=np.asarray(c['noise_magnitudes']), harm_dist=np.asarray(c['harm_dist']))
  small = name in DIGEST_CASES or name == 'long'
  for k in SMALL_OUTPUTS if small else OUTPUTS:
    if not get_controls and k in ('harm_amp', 'harm_dist', 'noise_magnitudes'):
      continue   # the float64 arrays themselves, stored as raw_*
    if k == 'sin_amps' and np.shape(c[k])[-1] > SMALL['n_harmonics']:
      continue   # harm_amp times the stored harm_dist, at paper shape
    out[f'{name}_{k}'] = np.asarray(c[k])
  for k in RAW:
    if name in DIGEST_CASES:
      out[f'{name}_raw_{k}_sha256'] = digest(raw[k])
    else:
      out[f'{name}_raw_{k}'] = raw[k]
  return out


def generate():
  ddsp, m = _load()
  out = {}
  with warnings.catch_warnings():
    warnings.simplefilter('ignore')
    for name, seed, kwargs in V2_CASES:
      np.random.seed(seed)
      out.update(_v2(ddsp, m, name, kwargs))
      out[f'{name}_seed'] = np.int64(seed)
    for name, seed, pre, kwargs in STATE_CASES:
      np.random.seed(seed)
      np.random.uniform(size=pre)
      if pre % 2:
        np.random.randn(1)   # leaves a cached Gaussian for the call
      out.update(_state(f'{name}_before'))
      out.update(_v2(ddsp, m, name, kwargs, n_batch=3))
      out.update(_state(f'{name}_after'))
      out[f'{name}_next'] = np.random.uniform(size=4)
    for name, seed, b, t, k, n_mags in V1_CASES:
      np.random.seed(seed)
      out.update(_state(f'{name}_before'))
      c = ref_on_shim.to_numpy(m.generate_notes(b, t, n_harmonics=k, n_mags=n_mags))
      for key in OUTPUTS:
        if not (key == 'sin_amps' and k > SMALL['n_harmonics']):
          out[f'{name}_{key}'] = np.asarray(c[key])
      out.update(_state(f'{name}_after'))
  return out


def main():
  got = generate()
  if '--check' in sys.argv:
    want = dict(np.load(PATH))
    assert sorted(got) == sorted(want), sorted(set(got) ^ set(want))
    for k in want:
      assert got[k].dtype == want[k].dtype and np.array_equal(got[k], want[k]), k
    print('synthetic_data.npz: %d arrays regenerate bit for bit' % len(want))
    return
  np.savez_compressed(PATH, **got)
  print('wrote %s (%d arrays, %d bytes)' % (PATH, len(got), os.path.getsize(PATH)))


if __name__ == '__main__':
  main()
