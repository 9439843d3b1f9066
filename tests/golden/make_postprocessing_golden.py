"""Writes tests/golden/postprocessing.npz and tests/golden/dataset_statistics.pkl: outputs
of the UNMODIFIED REFERENCE's training/postprocessing.py (smooth, detect_notes,
QuantileTransformer, fit_quantile_transform, compute_dataset_statistics) and of
colab/colab_utils.py's get_tuning_factor and auto_tune, run on the NumPy TensorFlow shim.

ddsp/training/__init__.py imports google.cloud, so postprocessing.py is loaded by its
file path under a stub `ddsp.training` package, and colab_utils.py under stub
`google.colab`, `IPython` and `note_seq` modules.  smooth needs tf.nn.conv1d, which the
shim lacks: this script installs tests/postprocessing_ref.conv1d (stride 1, float32) as
the loaded shim's tf.nn.conv1d.  The shim's files are not changed.  The numpy version is
recorded, since the quantiles follow its nanpercentile.

  python tests/golden/make_postprocessing_golden.py          # rewrite the fixtures
  python tests/golden/make_postprocessing_golden.py --check  # regenerate and compare
"""
import importlib.util
import io
import os
import pickle
import sys
import types
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                   # noqa: E402
from tests import postprocessing_ref             # noqa: E402

PATH = os.path.join(HERE, 'postprocessing.npz')
PKL_PATH = os.path.join(HERE, 'dataset_statistics.pkl')
NAN = np.nan


def _load_file(name, path):
  spec = importlib.util.spec_from_file_location(name, path)
  mod = importlib.util.module_from_spec(spec)
  sys.modules[name] = mod
  spec.loader.exec_module(mod)
  return mod


def _load():
  """(postprocessing, colab_utils) of the reference on the shim."""
  ddsp = ref_on_shim.load()
  tf = ref_on_shim.tf()
  tf.nn.conv1d = lambda *a, **k: tf.convert_to_tensor(postprocessing_ref.conv1d(*a, **k))
  if 'ddsp.training.postprocessing' in sys.modules:
    return sys.modules['ddsp.training.postprocessing'], sys.modules['ddsp.colab.colab_utils']
  root = os.path.join(ref_on_shim.REFERENCE_ROOT, 'ddsp')
  if 'ddsp.training' not in sys.modules:
    pkg = types.ModuleType('ddsp.training')
    pkg.__path__ = [os.path.join(root, 'training')]
    sys.modules['ddsp.training'] = pkg
  training = sys.modules['ddsp.training']
  training.plotting = types.SimpleNamespace(specplot=None, plot_impulse_responses=None,
                                            transfer_function=None)
  ddsp.training = training
  post = _load_file('ddsp.training.postprocessing',
                    os.path.join(root, 'training', 'postprocessing.py'))
  training.postprocessing = post
  colab = types.ModuleType('google.colab')
  colab.files = types.SimpleNamespace(download=None, upload=None)
  colab.output = types.SimpleNamespace(eval_js=None)
  google = types.ModuleType('google')
  google.colab = colab
  sys.modules.setdefault('google', google)
  sys.modules['google.colab'] = colab
  ipython = types.ModuleType('IPython')
  ipython.display = types.SimpleNamespace()
  sys.modules['IPython'] = ipython
  sys.modules.setdefault('note_seq', types.SimpleNamespace())
  cpkg = types.ModuleType('ddsp.colab')
  cpkg.__path__ = [os.path.join(root, 'colab')]
  sys.modules['ddsp.colab'] = cpkg
  cu = _load_file('ddsp.colab.colab_utils', os.path.join(root, 'colab', 'colab_utils.py'))
  return post, cu


def clip(t, seed, gaps=True):
  """Seeded loudness (dB, quantised to 0.25 dB so that quantiles repeat), f0 (Hz) and
  confidence [T] with held notes separated by quiet, unvoiced gaps."""
  rng = np.random.default_rng(seed)
  loud = np.full(t, -75.0)
  f0 = np.zeros(t)
  conf = rng.uniform(0.0, 0.3, t)
  i = int(rng.integers(0, 20))
  while i < t:
    n = int(rng.integers(20, 200))
    k = np.arange(min(n, t - i))
    loud[i:i + n] = rng.uniform(-40, -10) - k * rng.uniform(0, 0.05)
    f0[i:i + n] = 440 * 2**((rng.uniform(50, 72) + 0.1 * np.sin(0.3 * k) - 69) / 12)
    conf[i:i + n] = rng.uniform(0.75, 0.98, len(k))
    i += n + (int(rng.integers(5, 60)) if gaps else 0)
  loud = np.round((loud + rng.normal(0, 0.3, t)) * 4) / 4
  return loud.astype(np.float32), f0.astype(np.float32), conf.astype(np.float32)


class Provider:
  """The part of a ddsp DataProvider compute_dataset_statistics uses."""

  def __init__(self, batches):
    self.batches = batches

  def get_batch(self, batch_size, repeats=1):
    del batch_size, repeats
    return self.batches

  def __repr__(self):
    return 'Provider()'


def provider_batches(post_spectral_ops):
  """Two batches of two items: audio [2, N] and frame-rate controls with as many frames
  as compute_power(audio, frame_size=1024, frame_rate=50) gives; the second item of the
  second batch has no confident frame (no notes)."""
  rng = np.random.default_rng(7100)
  n = 16000
  batches = []
  for b in range(2):
    audio = (rng.normal(0, 0.1, (2, n)) * np.repeat(rng.uniform(0, 1, (2, 50)) > 0.3, 320,
                                                     axis=1)).astype(np.float32)
    frames = np.asarray(post_spectral_ops.compute_power(audio, frame_size=1024,
                                                        frame_rate=50)).shape[-1]
    rows = [clip(frames, 7200 + 2 * b + j) for j in range(2)]
    loud, f0, conf = (np.stack([r[i] for r in rows]) for i in range(3))
    if b == 1:
      conf[1] = 0.0
    batches.append({'audio': audio, 'loudness_db': loud, 'f0_hz': f0, 'f0_confidence': conf})
  return batches


def _qt_case(out, post, key, x, **kwargs):
  qt = post.QuantileTransformer(**kwargs)
  qt.fit(x)
  out[f'{key}_x'] = x
  out[f'{key}_references'] = qt.references_
  out[f'{key}_quantiles'] = qt.quantiles_
  probe = np.concatenate([x, np.asarray(qt.quantiles_, x.dtype)[:5],
                          np.full((2, x.shape[1]), 1e9, x.dtype),
                          np.full((2, x.shape[1]), -1e9, x.dtype)])
  out[f'{key}_probe'] = probe
  for dist in ('uniform', 'normal'):
    qt.output_distribution = dist
    fwd = qt.transform(probe)
    out[f'{key}_{dist}_forward'] = fwd
    out[f'{key}_{dist}_inverse'] = qt.inverse_transform(fwd)
  qt.output_distribution = 'uniform'
  return qt


def postprocessing():
  post, cu = _load()
  out = {'numpy_version': np.asarray(np.__version__)}
  warnings.simplefilter('ignore', RuntimeWarning)
  with np.errstate(all='ignore'):
    # smooth: odd and even filters, a filter longer than the signal, [B, T]
    x = np.random.default_rng(7000).uniform(0, 1, (2, 37)).astype(np.float32)
    out['smooth_x'] = x
    for k in (1, 3, 4, 40):
      out[f'smooth_k{k}'] = post.smooth(x, k)
    out['smooth_1d_k5'] = post.smooth(x[0], 5)
    # detect_notes on seeded clips: [T] and [B, T], float32 and float64
    loud, f0, conf = clip(1500, 7001)
    out['clip_loud'], out['clip_f0'], out['clip_conf'] = loud, f0, conf
    mask, ratio = post.detect_notes(loud, conf)
    out['detect_mask'], out['detect_ratio'] = mask, ratio
    mask64, ratio64 = post.detect_notes(loud.astype(np.float64), conf.astype(np.float64),
                                        note_threshold=0.8, exponent=3.0, smoothing=9)
    out['detect64_mask'], out['detect64_ratio'] = mask64, ratio64
    rows = [clip(600, 7010 + j) for j in range(3)]
    bl, bc = np.stack([r[0] for r in rows]), np.stack([r[2] for r in rows])
    out['batch_loud'], out['batch_conf'] = bl, bc
    out['batch_mask'], out['batch_ratio'] = post.detect_notes(bl, bc)
    # quantile fits: duplicates, NaN, an all-NaN column, n < n_quantiles, 1 and 2
    # quantiles, float32
    rng = np.random.default_rng(7300)
    xq = np.stack([np.round(rng.normal(-30, 8, 300)),                 # repeated values
                   np.where(rng.uniform(0, 1, 300) < 0.2, NAN, rng.normal(0, 1, 300)),
                   np.full(300, NAN)], axis=1)
    _qt_case(out, post, 'qt_dup', xq[:, :2])
    qt_nan = post.QuantileTransformer().fit(xq)
    out['qt_allnan_x'], out['qt_allnan_quantiles'] = xq, qt_nan.quantiles_
    xl = rng.normal(0, 3, (1500, 2))
    _qt_case(out, post, 'qt_large', xl)
    _qt_case(out, post, 'qt_nq1', xl[:40], n_quantiles=1)
    _qt_case(out, post, 'qt_nq2', xl[:40], n_quantiles=2)
    _qt_case(out, post, 'qt_f32', xl[:500].astype(np.float32), n_quantiles=100)
    np.random.seed(7400)
    _qt_case(out, post, 'qt_subsample', xl, n_quantiles=50, subsample=200)
    # fit_quantile_transform with an inverse transform
    mask_b = np.zeros_like(mask)
    mask_b[::3] = True
    inv = post.fit_quantile_transform(loud, mask_b)
    qt, norm = post.fit_quantile_transform(loud, mask, inv_quantile=inv)
    out['fit_mask_b'] = mask_b
    out['fit_quantiles'], out['fit_inv_quantiles'] = qt.quantiles_, inv.quantiles_
    out['fit_loudness_norm'] = norm
    # tuning: the clip, one note frame, none
    f0_midi = np.asarray(post.hz_to_midi(f0)).astype(np.float32)
    out['f0_midi'] = f0_midi
    out['tuning'] = cu.get_tuning_factor(f0_midi, conf, mask)
    one = np.zeros_like(mask)
    one[np.argmax(mask)] = True
    out['tuning_one'] = cu.get_tuning_factor(f0_midi, conf, one)
    out['tuning_none'] = cu.get_tuning_factor(f0_midi, conf, np.zeros_like(mask))
    for amount in (0.0, 0.6):
      out[f'autotune_scale_{amount}'] = cu.auto_tune(f0_midi, out['tuning'], mask,
                                                     amount=amount)
      out[f'autotune_chromatic_{amount}'] = cu.auto_tune(f0_midi, out['tuning'], mask,
                                                         amount=amount, chromatic=True)
    out['autotune_scale_none'] = cu.auto_tune(f0_midi, 0.0, np.zeros_like(mask), amount=1.0)
    # dataset statistics (one row without notes)
    batches = provider_batches(sys.modules['ddsp.spectral_ops'])
    for i, b in enumerate(batches):
      for k, v in b.items():
        out[f'stats_batch{i}_{k}'] = v
    stats = post.compute_dataset_statistics(Provider(batches), batch_size=2)
    for k, v in stats.items():
      if k != 'quantile_transform':
        out[f'stats_{k}'] = v
    out['stats_quantiles'] = stats['quantile_transform'].quantiles_
  got = {}
  for k, v in out.items():
    v = np.asarray(v)
    got[k] = v if v.dtype.kind in 'US' else v.astype(np.float64)
  return got, pickle.dumps(stats)


def _compare(got, want):
  assert set(want.files) == set(got), sorted(set(want.files) ^ set(got))
  for k in want.files:
    if want[k].dtype.kind in 'US':
      assert str(got[k]) == str(want[k]), (k, got[k], want[k])
    else:
      np.testing.assert_array_equal(got[k], want[k], err_msg=k)


if __name__ == '__main__':
  got, pkl = postprocessing()
  if '--check' in sys.argv:
    _compare(got, np.load(PATH))
    want = pickle.load(io.BytesIO(open(PKL_PATH, 'rb').read()))
    np.testing.assert_array_equal(pickle.loads(pkl)['quantile_transform'].quantiles_,
                                  want['quantile_transform'].quantiles_)
    print('ok    postprocessing')
  else:
    np.savez_compressed(PATH, **got)
    with open(PKL_PATH, 'wb') as f:
      f.write(pkl)
    print('wrote postprocessing %.0f kB, dataset_statistics %.0f kB' %
          (os.path.getsize(PATH) / 1e3, os.path.getsize(PKL_PATH) / 1e3))
