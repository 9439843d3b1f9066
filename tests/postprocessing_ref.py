"""Independent host restatements of postprocessing.py and colab_utils' tuning helpers,
written from their numpy / scipy / TF semantics in the operation order the CUDA kernels
follow (csrc/postprocessing.cuh), and pinned to tests/golden/postprocessing.npz.

Also `conv1d`: tf.nn.conv1d at stride 1 ('SAME' or 'VALID', float32, taps summed in
order), which the NumPy TensorFlow shim lacks; make_postprocessing_golden.py installs it
as the shim's tf.nn.conv1d so that the reference's `smooth` runs there.
"""
import math

import numpy as np
from scipy import special

F32 = np.float32


# ---- tf.nn.conv1d ---------------------------------------------------------------------
def conv1d(x, filters, stride=1, padding='SAME', name=None):
  """tf.nn.conv1d of x [B, T, C_in] with filters [k, C_in, C_out] at stride 1, in
  float32: out[b, t, o] = sum over taps j (in order) and channels of x[t - pad + j] w[j];
  'SAME' pads (k - 1) // 2 zeros on the left and the rest on the right."""
  del name
  if stride != 1:
    raise NotImplementedError('conv1d: stride 1 only')
  x = np.asarray(getattr(x, 'numpy', lambda: x)(), F32)
  w = np.asarray(getattr(filters, 'numpy', lambda: filters)(), F32)
  k = w.shape[0]
  b, t, _ = x.shape
  if padding == 'SAME':
    left = (k - 1) // 2
    x = np.concatenate([np.zeros((b, left, x.shape[2]), F32), x,
                        np.zeros((b, k - 1 - left, x.shape[2]), F32)], axis=1)
    t_out = t
  elif padding == 'VALID':
    t_out = max(t - k + 1, 0)
  else:
    raise ValueError(f'conv1d: padding {padding!r}')
  out = np.zeros((b, t_out, w.shape[2]), F32)
  for j in range(k):
    for c in range(w.shape[1]):
      out = out + x[:, j:j + t_out, c, None] * w[j, c][None, None, :]
  return out


# ---- smooth / detect_notes ------------------------------------------------------------
def np_power(x, e):
  """numpy's array ** Python scalar for a float array, with its fast paths."""
  x = np.asarray(x)
  return x**e


def smooth(x, filter_size=3):
  x = np.asarray(x, F32)
  rows = x if x.ndim == 2 else x[None]
  y = conv1d(rows[:, :, None], (np.ones([filter_size], F32) / F32(filter_size))[:, None, None])
  return y[:, :, 0] if x.ndim == 2 else y[0, :, 0]


def detect_notes(loudness_db, f0_confidence, note_threshold=1.0, exponent=2.0, smoothing=40,
                 f0_confidence_threshold=0.7, min_db=-80.0):
  """The reference's arithmetic, with the mean of the loudness summed in double (as the
  kernel sums it) and rounded to the loudness dtype."""
  loud = np.asarray(loudness_db)
  mean_db = loud.dtype.type(math.fsum(loud.astype(np.float64).ravel()) / loud.size)
  db = smooth(np_power(np.asarray(f0_confidence), exponent), smoothing) * (loud - min_db)
  db_threshold = (mean_db - min_db) * f0_confidence_threshold**exponent
  ratio = db / db_threshold
  return ratio >= note_threshold, ratio


# ---- quantiles --------------------------------------------------------------------------
def nanpercentile(col, q):
  """np.nanpercentile(col, 100 q) by numpy 2.3's linear method, restated: (n - 1) q,
  floor / floor + 1 neighbours (both the last past the end, with gamma v + 1), b - a in
  the column's dtype, then a + d t or b - d (1 - t) in float64."""
  col = np.asarray(col)
  s = np.sort(col[~np.isnan(col)])
  n = len(s)
  out = np.empty(len(q))
  for i, qi in enumerate(q):
    if n == 0:
      out[i] = np.nan
      continue
    v = float(n - 1) * float(qi)
    if v >= n - 1:
      prev, ia, ib = -1.0, n - 1, n - 1
    else:
      prev = math.floor(v)
      ia, ib = int(prev), int(prev) + 1
    t = v - prev
    a, b = s[ia], s[ib]
    d = float(np.subtract(b, a))
    out[i] = float(b) - d * (1.0 - t) if t >= 0.5 else float(a) + d * t
  return out


def running_max(q):
  out = np.array(q, np.float64)
  for i in range(1, len(out)):
    m, x = out[i - 1], out[i]
    out[i] = m if (m > x or np.isnan(m)) else x
  return out


def fit_quantiles(x, n_quantiles=1000):
  """(references_, quantiles_) of x [n, F] without subsampling."""
  n = x.shape[0]
  nq = max(1, min(n_quantiles, n))
  refs = np.linspace(0, 1, nq)
  q = np.true_divide(refs * 100, 100.0)
  return refs, np.stack([running_max(nanpercentile(c, q)) for c in x.T], axis=1)


def interp(x, xp, fp):
  """np.interp of one non-NaN x (numpy's arr_interp rules)."""
  m = len(xp)
  if m == 1:
    return fp[0]
  if x > xp[-1]:
    return fp[-1]
  if x < xp[0]:
    return fp[0]
  j = max(int(np.searchsorted(xp, x, side='right')) - 1, 0)
  if j == m - 1 or xp[j] == x:
    return fp[j]
  slope = (fp[j + 1] - fp[j]) / (xp[j + 1] - xp[j])
  r = slope * (x - xp[j]) + fp[j]
  if np.isnan(r):
    r = slope * (x - xp[j + 1]) + fp[j + 1]
    if np.isnan(r) and fp[j] == fp[j + 1]:
      r = fp[j]
  return r


def transform_col(x, quantiles, refs, inverse, distribution='uniform'):
  """_transform_col of a float64 column, element by element (scipy's ndtr / ndtri)."""
  out = np.empty(len(x))
  q0, qn = quantiles[0], quantiles[-1]
  cmin = special.ndtri(1e-7 - np.spacing(1))
  cmax = special.ndtri(1 - (1e-7 - np.spacing(1)))
  for i, v in enumerate(np.asarray(x, np.float64)):
    if inverse and distribution == 'normal':
      v = special.ndtr(v)
    if distribution == 'normal':
      lo, hi = (v - 1e-7 < (0 if inverse else q0)), (v + 1e-7 > (1 if inverse else qn))
    else:
      lo, hi = v == (0 if inverse else q0), v == (1 if inverse else qn)
    y = v
    if not np.isnan(v):
      if inverse:
        y = interp(v, refs, quantiles)
      else:
        y = 0.5 * (interp(v, quantiles, refs) - interp(-v, -quantiles[::-1], -refs[::-1]))
    if hi:
      y = qn if inverse else 1.0
    if lo:
      y = q0 if inverse else 0.0
    if not inverse and distribution == 'normal':
      y = special.ndtri(y) if 0 <= y <= 1 else np.nan
      if not np.isnan(y):
        y = min(max(y, cmin), cmax)
    out[i] = y
  return out


# ---- tuning -----------------------------------------------------------------------------
def _mod1(a):
  m = math.fmod(a, 1.0)
  if m != 0.0:
    if m < 0.0:
      m += 1.0
  else:
    m = 0.0
  return m


def _midi_diff(f, factor):
  d = _mod1(f - factor)
  return d - 1.0 if d > 0.5 else d


def _pairwise(x):
  """numpy's pairwise sum of at most 128 doubles."""
  n = len(x)
  if n < 8:
    s = -0.0
    for v in x:
      s += v
    return s
  r = [float(v) for v in x[:8]]
  i = 8
  while i < n - n % 8:
    for j in range(8):
      r[j] += x[i + j]
    i += 8
  s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
  while i < n:
    s += x[i]
    i += 1
  return s


def _normalise(x):
  mean = _pairwise(x) / len(x)
  sd = math.sqrt(_pairwise([(v - mean) * (v - mean) for v in x]) / len(x))
  with np.errstate(all='ignore'):
    return [np.float64(v - mean) / np.float64(sd) for v in x]


def _argmin(x):
  best = 0
  for i, v in enumerate(x):
    if np.isnan(v):
      return i
    if v < x[best]:
      best = i
  return best


def tuning_index(f0_on, conf_on):
  """The index into np.linspace(-0.5, 0.5, 101) that get_tuning_factor picks."""
  factors = np.linspace(-0.5, 0.5, 101)
  f0_on = [float(v) for v in f0_on]
  conf_on = [float(v) for v in conf_on]
  n = len(f0_on)
  diffs, deltas = [], []
  for fac in factors:
    d = [_midi_diff(f, fac) for f in f0_on]
    sd = 0.0
    for w, di in zip(conf_on, d):
      sd += w * abs(di)
    sw = 0.0
    for i in range(n - 1):
      sw += conf_on[i] * (1.0 if (f0_on[i + 1] - d[i + 1]) - (f0_on[i] - d[i]) != 0.0
                          else 0.0)
    with np.errstate(all='ignore'):
      diffs.append(np.float64(sd) / np.float64(n))
      deltas.append(np.float64(sw) / np.float64(max(n - 1, 0)))
  a, b = _normalise(deltas), _normalise(diffs)
  return _argmin([x + y for x, y in zip(a, b)])


def scale_notes(s):
  return np.ravel([np.array([0, 2, 4, 5, 7, 9, 11]) + 12 * i for i in range(10)]) + s


def auto_tune(f0_midi, tuning_factor, mask_on, amount=0.0, chromatic=False):
  """float64 restatement (scale index, result) of colab_utils.auto_tune."""
  f0 = np.asarray(f0_midi, np.float64)
  if chromatic:
    d = np.array([_midi_diff(v, float(tuning_factor)) for v in f0.ravel()]).reshape(f0.shape)
    return None, f0 - amount * d
  on = f0[np.asarray(mask_on, bool)]
  costs = []
  for s in range(12):
    notes = scale_notes(s)
    total = 0.0
    for v in on:
      total += np.min(np.abs(v - notes))
    with np.errstate(all='ignore'):
      costs.append(np.float64(total) / np.float64(len(on)))
  s = _argmin(costs)
  notes = scale_notes(s)
  d = np.array([v - notes[int(np.argmin(np.abs(v - notes)))] for v in f0])
  return s, f0 - amount * d
