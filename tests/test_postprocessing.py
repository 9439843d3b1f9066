"""postprocessing.py (training/postprocessing.py) and colab_utils' get_tuning_factor /
auto_tune on the CUDA kernels of csrc/postprocessing.cuh.

On the CPU: the shim's conv1d, the float64 restatement (tests/postprocessing_ref.py)
against the reference's fixture (tests/golden/postprocessing.npz), the reading of a
reference-written dataset_statistics.pkl and its refusal of other globals, and the C
ABI's refusals before any launch.  On the GPU: bit equality with the fixture or the
restatement where the kernels repeat numpy's arithmetic, stated tolerances elsewhere,
sizes up to 2^20 frames and a [1000, 1000] fit, reproducibility, side streams,
unaligned operands, and errors.
"""
import ctypes
import io
import os
import pickle

import numpy as np
import pytest
import torch
from scipy import special

from ddsp_b200 import _lib, colab_utils, postprocessing
from tests import postprocessing_ref as ref

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = np.load(os.path.join(HERE, 'golden', 'postprocessing.npz'))
PKL = os.path.join(HERE, 'golden', 'dataset_statistics.pkl')


def _np(x):
  return x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)


def _same_bits(got, want, what=''):
  got, want = _np(got), np.asarray(want)
  assert got.shape == want.shape, (what, got.shape, want.shape)
  np.testing.assert_array_equal(got.astype(np.float64), want.astype(np.float64), err_msg=what)


def _ulps32(got, want):
  g = np.asarray(_np(got), np.float32).view(np.int32).astype(np.int64)
  w = np.asarray(want, np.float32).view(np.int32).astype(np.int64)
  return np.abs(g - w)


# ---- CPU ---------------------------------------------------------------------------------
def test_conv1d_matches_np_convolve():
  rng = np.random.default_rng(1)
  for k in (1, 2, 3, 4, 9, 40):
    x = rng.uniform(-1, 1, (2, 50)).astype(np.float32)
    w = rng.uniform(-1, 1, k).astype(np.float32)
    same = ref.conv1d(x[:, :, None], w[:, None, None])[:, :, 0]
    valid = ref.conv1d(x[:, :, None], w[:, None, None], padding='VALID')[:, :, 0]
    for b in range(2):
      full = np.convolve(x[b].astype(np.float64), w[::-1].astype(np.float64))
      left = (k - 1) // 2
      np.testing.assert_allclose(same[b], full[k - 1 - left:k - 1 - left + 50], atol=1e-5)
      np.testing.assert_allclose(valid[b], full[k - 1:50], atol=1e-5)
    assert same.dtype == np.float32


def test_restated_smooth_and_detect_notes_match_the_reference():
  x = GOLD['smooth_x'].astype(np.float32)
  for k in (1, 3, 4, 40):
    _same_bits(ref.smooth(x, k), GOLD[f'smooth_k{k}'], k)
  _same_bits(ref.smooth(x[0], 5), GOLD['smooth_1d_k5'])
  loud, conf = GOLD['clip_loud'].astype(np.float32), GOLD['clip_conf'].astype(np.float32)
  mask, ratio = ref.detect_notes(loud, conf)
  # numpy's float32 pairwise mean may differ from the double sum in the last place
  assert _ulps32(ratio, GOLD['detect_ratio']).max() <= 2
  near = np.abs(GOLD['detect_ratio'] - 1.0) <= 1e-6
  assert np.array_equal(mask[~near], GOLD['detect_mask'][~near].astype(bool))


def test_restated_quantiles_match_the_reference():
  for key in ('qt_dup', 'qt_large', 'qt_nq1', 'qt_nq2', 'qt_f32'):
    x = GOLD[f'{key}_x']
    if key == 'qt_f32':
      x = x.astype(np.float32)
    nq = {'qt_nq1': 1, 'qt_nq2': 2, 'qt_f32': 100}.get(key, 1000)
    refs, q = ref.fit_quantiles(x, nq)
    _same_bits(refs, GOLD[f'{key}_references'], key)
    _same_bits(q, GOLD[f'{key}_quantiles'], key)
    probe = GOLD[f'{key}_probe']
    if key != 'qt_f32':
      for f in range(x.shape[1]):
        fwd = ref.transform_col(probe[:, f], q[:, f], refs, False)
        _same_bits(fwd, GOLD[f'{key}_uniform_forward'][:, f], (key, f))
        inv = ref.transform_col(fwd, q[:, f], refs, True)
        _same_bits(inv, GOLD[f'{key}_uniform_inverse'][:, f], (key, f))
  _, q = ref.fit_quantiles(GOLD['qt_allnan_x'])
  _same_bits(q, GOLD['qt_allnan_quantiles'])


def test_restated_tuning_matches_the_reference():
  f0, conf = GOLD['f0_midi'].astype(np.float32), GOLD['clip_conf'].astype(np.float32)
  mask = GOLD['detect_mask'].astype(bool)
  factors = np.linspace(-0.5, 0.5, 101)
  assert factors[ref.tuning_index(f0[mask], conf[mask])] == GOLD['tuning']
  one = np.zeros_like(mask)
  one[np.argmax(mask)] = True
  assert factors[ref.tuning_index(f0[one], conf[one])] == GOLD['tuning_one']
  assert factors[ref.tuning_index([], [])] == GOLD['tuning_none']
  for amount in (0.0, 0.6):
    _, got = ref.auto_tune(f0, GOLD['tuning'], mask, amount)
    _same_bits(got, GOLD[f'autotune_scale_{amount}'])
    _, got = ref.auto_tune(f0, GOLD['tuning'], mask, amount, chromatic=True)
    _same_bits(got, GOLD[f'autotune_chromatic_{amount}'])


def test_load_dataset_statistics_reads_the_reference_pickle():
  stats = postprocessing.load_dataset_statistics(PKL)
  qt = stats['quantile_transform']
  assert isinstance(qt, postprocessing.QuantileTransformer)
  _same_bits(qt.quantiles_, GOLD['stats_quantiles'])
  assert qt.n_quantiles == 1000 and qt.output_distribution == 'uniform'
  assert isinstance(qt.random_state, np.random.RandomState)
  for k, v in stats.items():
    if k != 'quantile_transform':
      assert isinstance(v, np.float32), k
      assert v == np.float32(GOLD[f'stats_{k}']), k
  # and from bytes / a file object, and after a round trip through this module's class
  with open(PKL, 'rb') as f:
    data = f.read()
  assert postprocessing.load_dataset_statistics(data).keys() == stats.keys()
  again = postprocessing.load_dataset_statistics(io.BytesIO(pickle.dumps(stats)))
  _same_bits(again['quantile_transform'].quantiles_, qt.quantiles_)


class _Evil:

  def __reduce__(self):
    return (os.system, ('true',))


@pytest.mark.parametrize('payload', [_Evil(), {'x': np.random.Generator(np.random.PCG64(1))},
                                     {'f': print}])
def test_load_dataset_statistics_refuses_other_globals(payload):
  with pytest.raises(pickle.UnpicklingError, match='refusing'):
    postprocessing.load_dataset_statistics(pickle.dumps(payload))


def test_abi_refuses_before_launching():
  lib = _lib.load()
  fake = ctypes.c_void_p(0x10000)
  ws = _lib.load().ddsp_b200_detect_notes_workspace_bytes(100)
  # bad shapes, filter size, flags, workspace
  assert lib.ddsp_b200_detect_notes(fake, fake, 0x20000, 0x30000, 0x40000, ws, 1, 0, 3, 2.0,
                                    0.49, -80.0, 1.0, 0, None) == _lib.E_INVALID
  assert lib.ddsp_b200_detect_notes(fake, fake, 0x20000, 0x30000, 0x40000, ws, 1, 100, 0, 2.0,
                                    0.49, -80.0, 1.0, 0, None) == _lib.E_INVALID
  assert lib.ddsp_b200_detect_notes(fake, fake, 0x20000, 0x30000, 0x40000, ws, 1, 100, 3, 2.0,
                                    0.49, -80.0, 1.0, 8, None) == _lib.E_INVALID
  assert lib.ddsp_b200_detect_notes(fake, fake, 0x20000, 0x30000, 0x40000, ws - 1, 1, 100, 3,
                                    2.0, 0.49, -80.0, 1.0, 0, None) == _lib.E_WORKSPACE
  # ratio overlapping the confidence, mask overlapping the ratio
  assert lib.ddsp_b200_detect_notes(0x80000, 0x10000, 0x10000 + 8, 0x30000, 0x40000, ws, 1,
                                    100, 3, 2.0, 0.49, -80.0, 1.0, 0, None) == _lib.E_INVALID
  assert b'ratio must not overlap conf' in lib.ddsp_b200_last_error()
  assert lib.ddsp_b200_detect_notes(0x80000, 0x10000, 0x20000, 0x20000 + 799, 0x40000, ws, 1,
                                    100, 3, 2.0, 0.49, -80.0, 1.0, 0, None) == _lib.E_INVALID
  # quantile fit / transform: shapes, modes, overlaps
  assert lib.ddsp_b200_quantile_fit(fake, fake, fake, 0x90000, 10, 2, 0, 0, None) == \
      _lib.E_INVALID
  assert lib.ddsp_b200_quantile_fit(fake, 0x20000, 0x30000, 0x10000 + 8, 10, 2, 5, 0,
                                    None) == _lib.E_INVALID
  assert lib.ddsp_b200_quantile_transform(0x10000, 0x20000, 0x30000, 0x40000, 10, 2, 5, 0, 2,
                                          0, None) == _lib.E_INVALID
  assert lib.ddsp_b200_quantile_transform(0x10000, 0x20000, 0x30000, 0x40000, 10, 2, 5, 2, 0,
                                          0, None) == _lib.E_INVALID
  assert lib.ddsp_b200_quantile_transform(0x10000, 0x20000, 0x30000, 0x10000 + 8, 10, 2, 5, 0,
                                          0, 0, None) == _lib.E_INVALID
  assert lib.ddsp_b200_quantile_transform(0x10000, 0x20000, 0x30000, 0x40000, 10, 2,
                                          _lib.QUANTILE_MAX_N + 1, 0, 0, 0, None) == \
      _lib.E_UNSUPPORTED
  # tuning and auto_tune
  assert lib.ddsp_b200_tuning_factor(fake, fake, fake, 0x90000, 0xA0000, 10, 0, None) == \
      _lib.E_INVALID
  assert lib.ddsp_b200_tuning_factor(0x10000, 0x20000, 0x30000, 0x10000, 0xA0000, 10, 101,
                                     None) == _lib.E_INVALID
  assert lib.ddsp_b200_auto_tune(0x10000, 0x20000, 0x30000, 0x40000, 0x10000, 10, 5, 0.0,
                                 0.5, 0, 0, None) == _lib.E_INVALID
  assert lib.ddsp_b200_auto_tune(0x10000, None, None, None, 0x50000, 10, 0, 0.0, 0.5, 2, 0,
                                 None) == _lib.E_INVALID
  assert lib.ddsp_b200_auto_tune(0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 10, 5, 0.0,
                                 0.5, 0, _lib.AUTO_TUNE_F32, None) == _lib.E_INVALID


# ---- GPU ---------------------------------------------------------------------------------
gpu = pytest.mark.gpu


def _cuda(x, dtype=None):
  t = torch.as_tensor(np.asarray(x))
  return t.to('cuda', dtype=dtype or t.dtype)


@gpu
def test_smooth_and_detect_notes_match_the_reference():
  x = GOLD['smooth_x'].astype(np.float32)
  for k in (1, 3, 4, 40):
    _same_bits(postprocessing.smooth(_cuda(x), k), GOLD[f'smooth_k{k}'], k)
  _same_bits(postprocessing.smooth(x[0], 5), GOLD['smooth_1d_k5'])
  loud, conf = GOLD['clip_loud'].astype(np.float32), GOLD['clip_conf'].astype(np.float32)
  mask, ratio = postprocessing.detect_notes(_cuda(loud), _cuda(conf))
  assert mask.dtype == torch.bool and ratio.dtype == torch.float32 and ratio.is_cuda
  want_mask, want_ratio = ref.detect_notes(loud, conf)
  _same_bits(ratio, want_ratio)
  assert _ulps32(ratio, GOLD['detect_ratio']).max() <= 2
  near = np.abs(GOLD['detect_ratio'] - 1.0) <= 1e-6
  assert np.array_equal(_np(mask)[~near], GOLD['detect_mask'][~near].astype(bool))
  assert np.array_equal(_np(mask), want_mask)
  # float64 inputs, another exponent and threshold
  m64, r64 = postprocessing.detect_notes(loud.astype(np.float64), conf.astype(np.float64),
                                         note_threshold=0.8, exponent=3.0, smoothing=9)
  assert r64.dtype == torch.float64
  np.testing.assert_allclose(_np(r64), GOLD['detect64_ratio'], rtol=1e-6)
  near = np.abs(GOLD['detect64_ratio'] - 0.8) <= 0.8e-6
  assert np.array_equal(_np(m64)[~near], GOLD['detect64_mask'][~near].astype(bool))
  # [B, T]: the mean over the whole input
  bl, bc = GOLD['batch_loud'].astype(np.float32), GOLD['batch_conf'].astype(np.float32)
  bm, br = postprocessing.detect_notes(bl, bc)
  assert _ulps32(br, GOLD['batch_ratio']).max() <= 2
  near = np.abs(GOLD['batch_ratio'] - 1.0) <= 1e-6
  assert np.array_equal(_np(bm)[~near], GOLD['batch_mask'][~near].astype(bool))


def _fit(key, nq, **kw):
  x = GOLD[f'{key}_x']
  if key == 'qt_f32':
    x = x.astype(np.float32)
  qt = postprocessing.QuantileTransformer(n_quantiles=nq, **kw)
  return qt.fit(_cuda(x)), x


@gpu
@pytest.mark.parametrize('key,nq', [('qt_dup', 1000), ('qt_large', 1000), ('qt_nq1', 1),
                                    ('qt_nq2', 2), ('qt_f32', 100)])
def test_quantile_transformer_matches_the_reference(key, nq):
  qt, x = _fit(key, nq)
  _same_bits(qt.references_, GOLD[f'{key}_references'])
  _same_bits(qt.quantiles_, GOLD[f'{key}_quantiles'])
  probe = GOLD[f'{key}_probe'].astype(x.dtype)
  fwd = qt.transform(_cuda(probe))
  inv = qt.inverse_transform(fwd)
  want_f, want_i = GOLD[f'{key}_uniform_forward'], GOLD[f'{key}_uniform_inverse']
  if x.dtype == np.float64:
    _same_bits(fwd, want_f)
    _same_bits(inv, want_i)
  else:
    assert fwd.dtype == torch.float32
    assert _ulps32(fwd, want_f).max() <= 1 and _ulps32(inv, want_i).max() <= 1
  qt.output_distribution = 'normal'
  fwd = qt.transform(_cuda(probe))
  want_f = GOLD[f'{key}_normal_forward']
  inside = np.isfinite(want_f)
  tol = 1e-13 if x.dtype == np.float64 else 1e-6 * np.maximum(1, np.abs(want_f))
  assert np.all(np.abs(_np(fwd).astype(np.float64) - want_f)[inside] <= np.broadcast_to(
      tol, want_f.shape)[inside])
  inv = qt.inverse_transform(fwd)
  want_i = GOLD[f'{key}_normal_inverse']
  scale = np.maximum(1.0, np.abs(want_i))
  assert np.nanmax(np.abs(_np(inv).astype(np.float64) - want_i) / scale) <= (
      1e-9 if x.dtype == np.float64 else 1e-6)
  assert np.array_equal(np.isnan(_np(inv)), np.isnan(want_i))


@gpu
def test_all_nan_column_and_subsample():
  qt = postprocessing.QuantileTransformer().fit(GOLD['qt_allnan_x'])
  _same_bits(qt.quantiles_, GOLD['qt_allnan_quantiles'])
  np.random.seed(7400)
  qt, _ = _fit('qt_subsample', 50, subsample=200)
  _same_bits(qt.quantiles_, GOLD['qt_subsample_quantiles'])
  fwd = qt.transform(GOLD['qt_subsample_probe'])
  _same_bits(fwd, GOLD['qt_subsample_uniform_forward'])


@gpu
def test_fit_quantile_transform_with_an_inverse():
  loud = GOLD['clip_loud'].astype(np.float32)
  inv = postprocessing.fit_quantile_transform(loud, GOLD['fit_mask_b'].astype(bool))
  _same_bits(inv.quantiles_, GOLD['fit_inv_quantiles'])
  qt, norm = postprocessing.fit_quantile_transform(_cuda(loud), GOLD['detect_mask'] != 0,
                                                   inv_quantile=inv)
  _same_bits(qt.quantiles_, GOLD['fit_quantiles'])
  assert tuple(norm.shape) == (len(loud), 1) and norm.dtype == torch.float32
  assert _ulps32(norm[:, 0], GOLD['fit_loudness_norm'][:, 0]).max() <= 1
  with pytest.raises(ValueError, match='inv_quantile'):
    postprocessing.fit_quantile_transform(np.stack([loud, loud]),
                                          np.ones((2, len(loud)), bool), inv_quantile=inv)


@gpu
def test_reference_pickle_inverse_transform_on_the_gpu():
  qt = postprocessing.load_dataset_statistics(PKL)['quantile_transform']
  x = np.linspace(-0.1, 1.1, 997)
  x[::50] = np.nan
  got = qt.inverse_transform(_cuda(x[:, None]))
  refs = np.asarray(qt.references_)
  want = ref.transform_col(x, qt.quantiles_[:, 0], refs, True)
  _same_bits(got[:, 0], want)


@gpu
def test_tuning_and_auto_tune_match_the_reference():
  f0, conf = GOLD['f0_midi'].astype(np.float32), GOLD['clip_conf'].astype(np.float32)
  mask = GOLD['detect_mask'].astype(bool)
  tuning = colab_utils.get_tuning_factor(_cuda(f0), _cuda(conf), _cuda(mask))
  assert isinstance(tuning, np.float64) and tuning == GOLD['tuning']
  one = np.zeros_like(mask)
  one[np.argmax(mask)] = True
  assert colab_utils.get_tuning_factor(f0, conf, one) == GOLD['tuning_one']
  assert colab_utils.get_tuning_factor(f0, conf, np.zeros_like(mask)) == GOLD['tuning_none']
  for amount in (0.0, 0.6):
    got = colab_utils.auto_tune(_cuda(f0), tuning, mask, amount=amount)
    assert got.dtype == torch.float64
    _same_bits(got, GOLD[f'autotune_scale_{amount}'])
    got = colab_utils.auto_tune(f0, tuning, mask, amount=amount, chromatic=True)
    _same_bits(got, GOLD[f'autotune_chromatic_{amount}'])
  _same_bits(colab_utils.auto_tune(f0, 0.0, np.zeros_like(mask), amount=1.0),
             GOLD['autotune_scale_none'])
  # float32 chromatic arithmetic where numpy keeps float32
  got = colab_utils.auto_tune(f0, 0.25, mask, amount=0.5, chromatic=True)
  assert got.dtype == torch.float32
  d = (f0 - np.float32(0.25)) % np.float32(1.0)
  d[d > 0.5] -= np.float32(1.0)
  _same_bits(got, f0 - 0.5 * d)


@gpu
def test_tuning_against_the_restatement_on_random_pitch():
  rng = np.random.default_rng(11)
  for n in (2, 3, 257, 3000):
    f0 = rng.uniform(40, 80, n)
    f0[rng.uniform(0, 1, n) < 0.5] = np.round(f0[:1])
    conf = rng.uniform(0, 1, n)
    mask = np.ones(n, bool)
    want = np.linspace(-0.5, 0.5, 101)[ref.tuning_index(f0, conf)]
    assert colab_utils.get_tuning_factor(f0, conf, mask) == want, n
    s, want = ref.auto_tune(f0, want, mask, 0.7)
    _same_bits(colab_utils.auto_tune(f0, want[0] * 0, mask, amount=0.7), want)


class _Provider:

  def __init__(self, batches):
    self.batches = batches

  def get_batch(self, batch_size, repeats=1):
    return self.batches


def _batches():
  return [{k: GOLD[f'stats_batch{i}_{k}'].astype(np.float32)
           for k in ('audio', 'loudness_db', 'f0_hz', 'f0_confidence')} for i in range(2)]


@gpu
def test_compute_dataset_statistics_matches_the_reference():
  stats = postprocessing.compute_dataset_statistics(_Provider(_batches()), batch_size=2)
  qt = stats.pop('quantile_transform')
  _same_bits(qt.quantiles_, GOLD['stats_quantiles'])
  for k, v in stats.items():
    want = GOLD[f'stats_{k}']
    assert isinstance(v, np.float32), k
    assert abs(float(v) - want) <= 1e-6 * max(1.0, abs(want)), (k, v, want)
  assert set(stats) == {
      k[len('stats_'):] for k in GOLD.files
      if k.startswith('stats_') and 'batch' not in k and k != 'stats_quantiles'}
  bad = _batches()
  for b in bad:
    for k in ('loudness_db', 'f0_hz', 'f0_confidence'):
      b[k] = b[k][:, :-1]
  with pytest.raises(ValueError, match='frames'):
    postprocessing.compute_dataset_statistics(_Provider(bad), batch_size=2)


@gpu
@pytest.mark.parametrize('t', [1, 2, 39, 40, 41, 4097, 2**20])
def test_sizes_streams_offsets_and_reproducibility(t):
  rng = np.random.default_rng(t)
  feats = 4 if t <= 4097 else 1
  loud = rng.uniform(-80, 0, (feats, t)).astype(np.float32)
  conf = rng.uniform(0, 1, (feats, t)).astype(np.float32)
  runs = []
  for side in (False, True):
    stream = torch.cuda.Stream() if side else torch.cuda.current_stream()
    with torch.cuda.stream(stream):
      # inputs one element past an aligned start
      lb = torch.zeros(loud.size + 1, device='cuda')
      cb = torch.zeros(conf.size + 1, device='cuda')
      lb[1:] = _cuda(loud).reshape(-1)
      cb[1:] = _cuda(conf).reshape(-1)
      m, r = postprocessing.detect_notes(lb[1:].view(feats, t), cb[1:].view(feats, t))
      np.random.seed(t)   # past 1e5 frames the fit draws a subsample
      qt = postprocessing.QuantileTransformer().fit(lb[1:].view(feats, t).t())
      y = qt.transform(lb[1:].view(feats, t).t())
    stream.synchronize()
    runs.append((m.clone(), r.clone(), qt.quantiles_.copy(), y.clone()))
  for a, b in zip(runs[0], runs[1]):
    _same_bits(_np(b), _np(a))
  if t <= 4097:
    want_mask, want_ratio = ref.detect_notes(loud, conf)
    _same_bits(runs[0][1], want_ratio)
    _, q = ref.fit_quantiles(loud.T.astype(np.float32))
    _same_bits(runs[0][2], q)


@gpu
def test_dataset_sized_fit():
  rng = np.random.default_rng(5)
  x = np.round(rng.normal(-30, 10, (1000, 1000)) * 4) / 4
  qt = postprocessing.QuantileTransformer().fit(_cuda(x))
  cols = rng.choice(1000, 8, replace=False)
  _, q = ref.fit_quantiles(x[:, cols])
  _same_bits(qt.quantiles_[:, cols], q)
  y = qt.transform(_cuda(x))
  for c in cols[:3]:
    _same_bits(y[:, c], ref.transform_col(x[:, c], qt.quantiles_[:, c], qt.references_, False))


@gpu
def test_errors_and_grad():
  x = torch.rand(50, device='cuda', requires_grad=True)
  for call in (lambda: postprocessing.smooth(x), lambda: postprocessing.detect_notes(x, x),
               lambda: postprocessing.QuantileTransformer().fit(x[:, None]),
               lambda: colab_utils.get_tuning_factor(x, x, x.detach() > 0),
               lambda: colab_utils.auto_tune(x, 0.0, x.detach() > 0)):
    with pytest.raises(RuntimeError, match='requires grad'):
      call()
  with pytest.raises(ValueError, match='same shape'):
    postprocessing.detect_notes(np.zeros(5), np.zeros(6))
  with pytest.raises(ValueError, match='n_quantiles'):
    postprocessing.QuantileTransformer(n_quantiles=0).fit(np.zeros((3, 1)))
  with pytest.raises(ValueError, match='features'):
    qt = postprocessing.QuantileTransformer().fit(np.zeros((3, 2)))
    qt.transform(np.zeros((3, 1)))
  with pytest.raises(ValueError, match='scale mode'):
    colab_utils.auto_tune(np.zeros((2, 3)), 0.0, np.ones((2, 3), bool))
  short = [{'audio': np.zeros((1, 1600), np.float32), 'loudness_db': np.zeros((1, 6)),
            'f0_hz': np.zeros((1, 6)), 'f0_confidence': np.zeros((1, 6))}]
  with pytest.raises(ValueError, match='frames'):
    postprocessing.compute_dataset_statistics(_Provider(short))
