"""Adjusting controls for tone transfer (`ddsp/training/postprocessing.py`): note
detection, quantile normalisation of loudness and the dataset statistics that the
tone-transfer notebook and exported models read.  Same names, arguments and defaults
as the reference.

Inputs are numpy arrays or torch tensors on any device; results are CUDA tensors.
detect_notes and smooth run on `ddsp_b200_detect_notes`, QuantileTransformer's fit and
transforms on `ddsp_b200_quantile_fit` / `ddsp_b200_quantile_transform`
(csrc/postprocessing.cuh, DESIGN.md section 3.29).  The kernels repeat numpy's and
scipy's operation order, so that float64 results are the reference's bits; float32
inputs keep the reference's float32 steps.

QuantileTransformer keeps its fitted state as host numpy arrays under the reference's
attribute names, so that it pickles as the reference's does; load_dataset_statistics
reads a `dataset_statistics.pkl` that the reference wrote.

Forward only: an input that requires grad raises.  Deviations from the reference: the
mean loudness of detect_notes is summed in double (numpy sums float32 input pairwise in
float32), fit_quantile_transform raises ValueError where the reference raises
IndexError (inv_quantile with 2-D loudness), and compute_dataset_statistics raises
ValueError where the reference fails on mismatched or too few frames.
"""
import io
import pickle

import numpy as np
import torch

from ddsp_b200 import _lib
from ddsp_b200 import core
from ddsp_b200 import spectral_ops


# ---- operands ----------------------------------------------------------------------------
def _is_f32(x):
  dt = x.dtype
  return dt == torch.float32 if torch.is_tensor(x) else np.dtype(dt) == np.float32


def _double(x, device=None):
  """x as a contiguous float64 CUDA tensor (float32 values widened exactly)."""
  if torch.is_tensor(x):
    return x.detach().to(device=device or (x.device if x.is_cuda else core._device()),
                         dtype=torch.float64).contiguous()
  return torch.as_tensor(np.asarray(x, np.float64), device=device or core._device())


def _operand(x, name):
  """(x as an array or tensor, its shape) after the grad check."""
  core._no_grad_path(name, x)
  if not torch.is_tensor(x):
    x = np.asarray(x)
  return x, tuple(x.shape)


def _device_of(*xs):
  for x in xs:
    if torch.is_tensor(x) and x.is_cuda:
      return x.device
  return core._device()


# ---- smooth and detect_notes -------------------------------------------------------------
def _detect(loudness, conf, shape, smoothing, exponent=2.0, weight=1.0, min_db=0.0,
            note_threshold=1.0, flags=0):
  """One ddsp_b200_detect_notes call: (ratio float64 [n], mask bool [n] or None)."""
  if len(shape) not in (1, 2) or 0 in shape:
    raise ValueError(f'expected [time] or [batch, time] with frames, got {shape}')
  b, t = (1, shape[0]) if len(shape) == 1 else shape
  smoothing = int(smoothing)
  device = _device_of(loudness, conf)
  c = _double(conf, device)
  ld = None if loudness is None else _double(loudness, device)
  ratio = torch.zeros(shape, dtype=torch.float64, device=device)
  mask = None if ld is None else torch.zeros(shape, dtype=torch.bool, device=device)
  core._launch('ddsp_b200_detect_notes', ld, c, ratio, mask,
               *core._workspace('ddsp_b200_detect_notes_workspace_bytes', device, b * t),
               b, t, smoothing, float(exponent), float(weight), float(min_db),
               float(note_threshold), flags)
  return ratio, mask


def smooth(x, filter_size=3):
  """postprocessing.smooth: the box filter of filter_size taps of float32(1 / k) with TF
  'SAME' zero padding over [T] or each row of [B, T], in float32 (the reference's
  tf.nn.conv1d); float32 result."""
  x, shape = _operand(x, 'smooth')
  y, _ = _detect(None, x if _is_f32(x) else _f32(x), shape, filter_size,
                 flags=_lib.DETECT_SMOOTH_ONLY)
  return y.to(torch.float32)


def _f32(x):
  """x rounded to float32, as tf.convert_to_tensor(x, tf.float32) does."""
  if torch.is_tensor(x):
    return x.to(torch.float32)
  return np.asarray(x, np.float32)


def detect_notes(loudness_db,
                 f0_confidence,
                 note_threshold=1.0,
                 exponent=2.0,
                 smoothing=40,
                 f0_confidence_threshold=0.7,
                 min_db=-spectral_ops.DB_RANGE):
  """postprocessing.detect_notes: (mask_on, note_on_ratio) of [T] or [B, T] controls.
  note_on_ratio = smooth(f0_confidence ** exponent, smoothing) (loudness_db - min_db) /
  ((mean_db - min_db) f0_confidence_threshold ** exponent), with mean_db the mean of the
  whole loudness input; mask_on = note_on_ratio >= note_threshold.  note_on_ratio is
  float32 for float32 loudness (computed in float32, as numpy does), else float64."""
  loudness_db, shape = _operand(loudness_db, 'detect_notes')
  f0_confidence, cshape = _operand(f0_confidence, 'detect_notes')
  if shape != cshape:
    raise ValueError(f'detect_notes: loudness_db {shape} and f0_confidence {cshape} must '
                     'have the same shape')
  loud_f32 = _is_f32(loudness_db)
  flags = ((_lib.DETECT_CONF_F32 if _is_f32(f0_confidence) else 0) |
           (_lib.DETECT_LOUD_F32 if loud_f32 else 0))
  weight = float(f0_confidence_threshold)**float(exponent)
  ratio, mask = _detect(loudness_db, f0_confidence, shape, smoothing, exponent, weight,
                        min_db, note_threshold, flags)
  return mask, ratio.to(torch.float32) if loud_f32 else ratio


# ---- QuantileTransformer -----------------------------------------------------------------
_DISTRIBUTIONS = {'uniform': _lib.QUANTILE_UNIFORM, 'normal': _lib.QUANTILE_NORMAL}


class QuantileTransformer:
  """postprocessing.QuantileTransformer (sklearn's, stripped down): per-feature quantiles
  of the fitted data, and the map to a uniform or normal distribution and back.

  The fitted state is host numpy under the reference's names (n_quantiles_,
  references_, quantiles_ [n_quantiles_, n_features]), and random_state is numpy's
  global RandomState, so that an instance pickles as the reference's does.  fit,
  transform and inverse_transform take [n_samples, n_features] arrays or tensors and
  return CUDA tensors of the input's float dtype (float64 for other dtypes)."""

  def __init__(self,
               n_quantiles=1000,
               output_distribution='uniform',
               subsample=int(1e5)):
    self.n_quantiles = n_quantiles
    self.output_distribution = output_distribution
    self.subsample = subsample
    self.random_state = np.random.mtrand._rand

  def __getstate__(self):
    state = dict(self.__dict__)
    state.pop('_device', None)
    return state

  def _dense_fit(self, x, random_state, flags=0):
    """quantiles_ of the [n, F] CUDA operand x: the columns (a subsample of
    `subsample` rows each, drawn on the host as the reference draws them) sorted on the
    device, then the percentile kernel."""
    n_samples, n_features = x.shape
    cols = x.t()
    if self.subsample < n_samples:
      idx = [random_state.choice(n_samples, size=self.subsample, replace=False)
             for _ in range(n_features)]
      idx = torch.as_tensor(np.stack(idx), device=x.device)
      cols = torch.gather(cols, 1, idx)
    cols = torch.sort(cols, dim=1).values.contiguous()   # NaN last
    counts = (~torch.isnan(cols)).sum(dim=1).to(torch.int64).contiguous()
    q = np.true_divide(self.references_ * 100, 100.0)
    qd = torch.as_tensor(q, dtype=torch.float64, device=x.device)
    out = torch.zeros((len(q), n_features), dtype=torch.float64, device=x.device)
    core._launch('ddsp_b200_quantile_fit', cols, counts, qd, out, cols.shape[1], n_features,
                 len(q), flags)
    self.quantiles_ = out.cpu().numpy()
    self._device = (x.device, self.quantiles_.copy(), self.references_.copy(), out,
                    torch.as_tensor(self.references_, device=x.device))

  def fit(self, x):
    """Computes quantiles_ of x [n_samples, n_features]."""
    if self.n_quantiles <= 0:
      raise ValueError("Invalid value for 'n_quantiles': %d. "
                       'The number of quantiles must be at least one.' %
                       self.n_quantiles)
    x, shape, flags, _ = self._operand(x, 'fit')
    n_samples = shape[0]
    self.n_quantiles_ = max(1, min(self.n_quantiles, n_samples))
    self.references_ = np.linspace(0, 1, self.n_quantiles_, endpoint=True)
    self._dense_fit(x, self.random_state, flags)
    return self

  @staticmethod
  def _operand(x, name):
    """(x as a float64 CUDA tensor, its shape, the kernels' flags, the result dtype)."""
    x, shape = _operand(x, f'QuantileTransformer.{name}')
    if len(shape) != 2:
      raise ValueError(f'QuantileTransformer.{name}: expected [n_samples, n_features], '
                       f'got {shape}')
    f32 = _is_f32(x)
    return (_double(x), shape, _lib.QUANTILE_F32 if f32 else 0,
            torch.float32 if f32 else torch.float64)

  def _device_quantiles(self, device):
    """(quantiles_, references_) on `device`, copied once and reused while the host
    arrays keep their values."""
    q = np.asarray(self.quantiles_, np.float64)
    r = np.asarray(self.references_, np.float64)
    cached = getattr(self, '_device', None)
    if (cached is not None and cached[0] == device and
        np.array_equal(cached[1], q, equal_nan=True) and np.array_equal(cached[2], r)):
      return cached[3], cached[4]
    qs = torch.as_tensor(np.ascontiguousarray(q), device=device)
    refs = torch.as_tensor(np.ascontiguousarray(r), device=device)
    self._device = (device, q.copy(), r.copy(), qs, refs)
    return qs, refs

  def _transform(self, x, inverse=False):
    if self.output_distribution not in _DISTRIBUTIONS:
      raise ValueError(f'QuantileTransformer: output_distribution must be uniform or '
                       f'normal, got {self.output_distribution!r}')
    name = 'inverse_transform' if inverse else 'transform'
    x, (n, f), flags, dtype = self._operand(x, name)
    qs, refs = self._device_quantiles(x.device)
    if qs.dim() != 2 or qs.shape[1] != f:
      raise ValueError(f'QuantileTransformer.{name}: {f} features, but fitted on '
                       f'{tuple(qs.shape)} quantiles')
    out = torch.zeros((n, f), dtype=torch.float64, device=x.device)
    core._launch('ddsp_b200_quantile_transform', x, qs, refs, out, n, f, qs.shape[0],
                 int(inverse), _DISTRIBUTIONS[self.output_distribution], flags)
    return out.to(dtype)

  def transform(self, x):
    """Feature-wise transformation of the data."""
    return self._transform(x, inverse=False)

  def inverse_transform(self, x):
    """Back-projection to the original space."""
    return self._transform(x, inverse=True)

  def fit_transform(self, x):
    """Fit and transform."""
    return self.fit(x).transform(x)


def _flat_masked(x, mask_on, name):
  """np.ravel(x[mask_on])[:, np.newaxis] on the device."""
  x, shape = _operand(x, name)
  mask_on, mshape = _operand(mask_on, name)
  if mshape != shape:
    raise ValueError(f'{name}: mask_on {mshape} must have the shape of {shape}')
  xt = x if torch.is_tensor(x) else torch.as_tensor(x)
  xt = xt.to(_device_of(xt))
  m = mask_on if torch.is_tensor(mask_on) else torch.as_tensor(mask_on)
  m = (m.to(xt.device) != 0)
  return xt, m, xt[m].reshape(-1, 1)


def fit_quantile_transform(loudness_db, mask_on, inv_quantile=None):
  """postprocessing.fit_quantile_transform: a QuantileTransformer fitted on the loudness
  of the note frames; with inv_quantile also the loudness [T, 1] with the note frames
  mapped through this transform and inv_quantile's inverse (the other frames
  unchanged).  inv_quantile takes [T] loudness only (ValueError for [B, T], where the
  reference raises IndexError)."""
  x, m, flat = _flat_masked(loudness_db, mask_on, 'fit_quantile_transform')
  quantile_transform = QuantileTransformer()
  flat_q = quantile_transform.fit_transform(flat)
  if inv_quantile is None:
    return quantile_transform
  if x.dim() != 1:
    raise ValueError('fit_quantile_transform: inv_quantile takes [time] loudness, got '
                     f'{tuple(x.shape)} (the reference fails to index it)')
  flat_norm = inv_quantile.inverse_transform(flat_q)
  loudness_norm = x.reshape(-1, 1).clone()
  loudness_norm[m] = flat_norm.to(loudness_norm.dtype)
  return quantile_transform, loudness_norm


# ---- dataset statistics ------------------------------------------------------------------
def _batch_tensor(v, device):
  if torch.is_tensor(v):
    return v.detach().to(device)
  return torch.as_tensor(np.asarray(v), device=device)


def _stat_rows(x, mask=None):
  """The six statistics of get_stats as one float64 tensor (mean, max, min, mean_max,
  mean_min, std)."""
  x = x.to(torch.float64)
  if mask is None:
    mean_max, mean_min = x.amax(-1).mean(), x.amin(-1).mean()
    v = x.reshape(-1)
  else:
    rows = mask.any(-1)
    inf = torch.full_like(x, float('inf'))
    mean_max = torch.where(mask, x, -inf).amax(-1)[rows].mean()
    mean_min = torch.where(mask, x, inf).amin(-1)[rows].mean()
    v = x[mask]
  return torch.stack([v.mean(), v.max(), v.min(), mean_max, mean_min,
                      v.std(unbiased=False)])


def compute_dataset_statistics(data_provider,
                               batch_size=1,
                               power_frame_size=1024,
                               power_frame_rate=50):
  """postprocessing.compute_dataset_statistics: pitch, power and loudness statistics of
  every batch of data_provider.get_batch(batch_size, repeats=1) ('audio_16k' or 'audio',
  'loudness_db', 'f0_hz', 'f0_confidence'), over all frames and over note frames, and
  the quantile transform of the note frames' loudness, under the reference's keys.  The
  statistics are numpy scalars of the inputs' dtype, reduced in float64 on the device.
  ValueError when the power and loudness frame counts differ or there are at most 20
  frames."""
  print('Calculating dataset statistics for', data_provider)
  ds = data_provider.get_batch(batch_size, repeats=1)
  batch = next(iter(ds))
  audio_key = 'audio_16k' if 'audio_16k' in batch.keys() else 'audio'
  device = core._device()
  loudness, power, f0, f0_conf = [], [], [], []
  i = 0
  for batch in iter(ds):
    audio = _batch_tensor(batch[audio_key], device)
    core._no_grad_path('compute_dataset_statistics', audio)
    loudness.append(_batch_tensor(batch['loudness_db'], device))
    power.append(spectral_ops.compute_power(audio, frame_size=power_frame_size,
                                            frame_rate=power_frame_rate))
    f0.append(_batch_tensor(batch['f0_hz'], device))
    f0_conf.append(_batch_tensor(batch['f0_confidence'], device))
    i += 1
  print(f'Computing statistics for {i * batch_size} examples.')

  loudness, power = torch.cat(loudness), torch.cat(power)
  f0, f0_conf = torch.cat(f0), torch.cat(f0_conf)
  trim_end = 20
  if power.shape[-1] != loudness.shape[-1]:
    raise ValueError(f'compute_dataset_statistics: {power.shape[-1]} power frames and '
                     f'{loudness.shape[-1]} loudness frames; they must match')
  if loudness.shape[-1] <= trim_end:
    raise ValueError(f'compute_dataset_statistics: {loudness.shape[-1]} frames; more than '
                     f'{trim_end} are needed')
  pitch_trimmed = core.hz_to_midi(f0[:, :-trim_end])
  power_trimmed = power[:, :-trim_end]
  loudness_trimmed = loudness[:, :-trim_end].contiguous()
  mask_on, _ = detect_notes(loudness_trimmed, f0_conf[:, :-trim_end])
  mask_on = mask_on | ~mask_on.any(dim=1, keepdim=True)
  quantile_transform = fit_quantile_transform(loudness_trimmed, mask_on)

  groups = [('pitch', pitch_trimmed, None), ('power', power_trimmed, None),
            ('loudness', loudness_trimmed, None), ('pitch_note', pitch_trimmed, mask_on),
            ('power_note', power_trimmed, mask_on),
            ('loudness_note', loudness_trimmed, mask_on)]
  values = torch.stack([_stat_rows(x, m) for _, x, m in groups]).cpu().numpy()
  ds_stats = {}
  for (prefix, x, _), row in zip(groups, values):
    kind = np.float32 if x.dtype == torch.float32 else np.float64
    for name, v in zip(('mean', 'max', 'min', 'mean_max', 'mean_min', 'std'), row):
      ds_stats[f'{name}_{prefix}'] = kind(v)
  ds_stats['quantile_transform'] = quantile_transform
  return ds_stats


# ---- reading the reference's pickle -------------------------------------------------------
_REFERENCE_CLASS = ('ddsp.training.postprocessing', 'QuantileTransformer')
_ALLOWED = {
    ('builtins', 'dict'), ('builtins', 'list'), ('builtins', 'tuple'), ('builtins', 'int'),
    ('builtins', 'float'), ('builtins', 'str'), ('builtins', 'bytes'),
    ('builtins', 'bytearray'), ('builtins', 'set'), ('builtins', 'frozenset'),
    ('builtins', 'complex'), ('builtins', 'bool'),
    ('numpy', 'ndarray'), ('numpy', 'dtype'),
    ('numpy.core.multiarray', '_reconstruct'), ('numpy.core.multiarray', 'scalar'),
    ('numpy._core.multiarray', '_reconstruct'), ('numpy._core.multiarray', 'scalar'),
    ('numpy.random._pickle', '__randomstate_ctor'),
    ('numpy.random._pickle', '__bit_generator_ctor'),
    ('numpy.random._pickle', '__generator_ctor'),
    ('numpy.random.mtrand', 'RandomState'),
    ('numpy.random._mt19937', 'MT19937'),
}


class _StatisticsUnpickler(pickle.Unpickler):
  """Resolves the reference's QuantileTransformer to this module's, and allows only
  builtins and numpy's array, scalar and RandomState reconstructors besides."""

  def find_class(self, module, name):
    if (module, name) == _REFERENCE_CLASS or (module, name) == (__name__,
                                                                 'QuantileTransformer'):
      return QuantileTransformer
    if (module, name) in _ALLOWED:
      return super().find_class(module, name)
    raise pickle.UnpicklingError(f'load_dataset_statistics: refusing the global '
                                 f'{module}.{name}')


def load_dataset_statistics(file):
  """The dict of a `dataset_statistics.pkl` (a path, bytes or a binary file), as
  colab_utils.save_dataset_statistics writes it, with its quantile_transform as this
  module's QuantileTransformer.  Any global other than that class, builtins and
  numpy's reconstructors raises pickle.UnpicklingError."""
  if isinstance(file, (bytes, bytearray)):
    return _StatisticsUnpickler(io.BytesIO(file)).load()
  if hasattr(file, 'read'):
    return _StatisticsUnpickler(file).load()
  with open(file, 'rb') as f:
    return _StatisticsUnpickler(f).load()
