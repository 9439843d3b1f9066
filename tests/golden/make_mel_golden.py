"""Writes tests/golden/mel.npz: outputs of the UNMODIFIED REFERENCE's
spectral_ops.compute_mel, compute_logmel, compute_mfcc (spectral_ops.py:73-133) and
compute_logmag (spectral_ops.py:92-94) on seeded inputs, run on the NumPy TensorFlow
shim in its float64 (wide) mode.  The shim has tf.signal.linear_to_mel_weight_matrix
and mfccs_from_log_mel_spectrograms only as stubs, and its tensors lack set_shape and
TensorShape.concatenate, which compute_mel calls; `mel()` installs
tests/mel_ref.py's restatements and those two methods for the run and removes them
afterwards, so the shim itself is unchanged.

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_mel_golden.py          # rewrite the fixture
  python tests/golden/make_mel_golden.py --check  # regenerate in memory and compare

tests/test_mel.py reads the fixture; the inputs come from the seeded generator below.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests.golden.make_golden import _both, compare   # noqa: E402

PATH = os.path.join(HERE, 'mel.npz')
B = 3


def _c(fn, n, layout='2d', **kw):
  return (fn, n, layout, kw)


# (function, N, input layout, keyword arguments of the reference's function)
CASES = [
    _c('compute_mel', 8000),
    _c('compute_mel', 6000, fft_size=1000, overlap=0.5, pad_end=False, bins=128, lo_hz=20.0,
       hi_hz=11025.0, sample_rate=22050),
    _c('compute_mel', 5000, '3d', fft_size=1001, overlap=0.75, bins=229, sample_rate=44100),
    _c('compute_mel', 4000, '1d', fft_size=768, overlap=0.0, bins=1, lo_hz=100.0,
       hi_hz=24000.0, sample_rate=48000),
    _c('compute_mel', 2000, fft_size=64, overlap=-0.5, bins=128),
    _c('compute_mel', 800, fft_size=1024, overlap=0.5, pad_end=False),
    _c('compute_logmel', 8000),
    _c('compute_logmel', 9000, fft_size=2048, overlap=0.75, bins=229, lo_hz=0.0,
       hi_hz=8000.0),
    _c('compute_logmel', 5000, '1d', fft_size=1001, overlap=0.5, pad_end=False, lo_hz=0.0,
       hi_hz=11025.0, sample_rate=22050),
    _c('compute_logmel', 3000, '3d', fft_size=64, overlap=-0.5, pad_end=False, bins=1,
       sample_rate=48000),
    _c('compute_mfcc', 8000, fft_size=1024, overlap=0.5, mel_bins=128, mfcc_bins=30),
    _c('compute_mfcc', 6000, '3d'),
    _c('compute_mfcc', 5000, fft_size=768, overlap=0.0, pad_end=False, mel_bins=64,
       mfcc_bins=100, lo_hz=0.0, hi_hz=22050.0, sample_rate=44100),
    _c('compute_mfcc', 4000, '1d', fft_size=1000, overlap=0.75, mfcc_bins=-5,
       sample_rate=22050),
    _c('compute_mfcc', 9000, fft_size=2048, overlap=0.5, mel_bins=229, mfcc_bins=1,
       sample_rate=48000),
    _c('compute_mfcc', 500, fft_size=1024, overlap=0.5, pad_end=False, mfcc_bins=30),
    _c('compute_logmag', 2000, size=1024, overlap=0.75),
    _c('compute_logmag', 3000, '3d', size=1001, overlap=0.5, pad_end=False),
    _c('compute_logmag', 3000, '1d', size=64, overlap=0.0),
]


def mel_input(i):
  """Seeded noise rows at three levels (1, 0.03, 1e-4 of full scale), laid out as the
  case asks: [B, N], [N] (the first row) or [B, N, 1]."""
  _, n, layout, _ = CASES[i]
  rng = np.random.default_rng(1300 + i)
  x = (rng.uniform(-1.0, 1.0, (B, n)) * np.array([[1.0], [0.03], [1e-4]])).astype(np.float32)
  return {'1d': x[0], '2d': x, '3d': x[:, :, None]}[layout]


def _install(ddsp):
  """The shim pieces compute_mel and compute_mfcc call; returns an undo."""
  from tests import mel_ref
  tf = ddsp.spectral_ops.tf
  shape_cls = type(tf.constant(np.zeros(1)).shape)
  tensor_cls = type(tf.constant(np.zeros(1)))
  saved = {k: getattr(tf.signal, k) for k in ('linear_to_mel_weight_matrix',
                                               'mfccs_from_log_mel_spectrograms')}

  def getitem(self, i):
    r = tuple.__getitem__(self, i)
    return shape_cls(r) if isinstance(i, slice) else r

  def set_shape(self, shape):
    assert tuple(self.shape) == tuple(shape), (self.shape, shape)

  tf.signal.linear_to_mel_weight_matrix = (
      lambda *a, **k: tf.constant(mel_ref.linear_to_mel_weight_matrix(*a, **k)))
  tf.signal.mfccs_from_log_mel_spectrograms = (
      lambda x, name=None: tf.constant(mel_ref.mfccs_from_log_mel_spectrograms(x.numpy())))
  shape_cls.__getitem__ = getitem
  shape_cls.concatenate = lambda self, other: shape_cls(tuple(self) + tuple(other))
  tensor_cls.set_shape = set_shape

  def undo():
    for k, v in saved.items():
      setattr(tf.signal, k, v)
    del shape_cls.__getitem__, shape_cls.concatenate, tensor_cls.set_shape
  return undo


def mel():
  ddsp = ref_on_shim.load()
  undo = _install(ddsp)
  try:
    so = ddsp.spectral_ops
    out = {}
    for i, (fn, _, _, kw) in enumerate(CASES):
      x = mel_input(i)
      out['%s_%02d' % (fn, i)] = np.asarray(_both(lambda: getattr(so, fn)(x, **kw))[1],
                                            np.float64)
    return out
  finally:
    undo()


if __name__ == '__main__':
  got = mel()
  if '--check' in sys.argv:
    compare('mel', got, np.load(PATH))
    print('ok    mel')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote mel %.0f kB' % (os.path.getsize(PATH) / 1e3))
