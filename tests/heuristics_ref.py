"""Float64 NumPy restatement of the reference's controls-to-notes heuristics
(training/heuristics.py), per item: the pooled-outlier tests, strided_freq_change,
remove_short, midi_heuristic(_power) and the note table of segment_notes.  Pinned to
the unmodified reference by tests/golden/heuristics.npz.

Float32 where the reference's values are float32 and the comparison depends on them:
log amplitudes, shifted power and hz_to_midi are float32 with correctly rounded logs
(as the kernel computes them); window statistics are float64 over deviations from the
frame's own value, so a constant window decides exactly False.  `margins` return, per
frame, the float64 distance of each decision from its threshold."""
import math

import numpy as np

F32 = np.float32
DB_RANGE = 80.0


class EdgeError(ValueError):
  """pad_for_frame's int() of a non-finite edge value."""


def log32(x):
  with np.errstate(divide='ignore', invalid='ignore'):
    return np.log(np.asarray(x, np.float32).astype(np.float64)).astype(np.float32)


def hz_to_midi32(f0):
  """core.hz_to_midi in float32, the reference's op order, correctly rounded logs."""
  f = np.asarray(f0, np.float32)
  ln2 = F32(math.log(2.0))
  c = F32(F32(math.log(440.0)) / ln2)
  with np.errstate(divide='ignore', invalid='ignore'):
    l = (log32(np.where(f <= 0, F32(1.0), f)) / ln2).astype(np.float32)
    m = (F32(12.0) * (l - c)).astype(np.float32) + F32(69.0)
  return np.where(f <= 0, F32(0.0), m).astype(np.float32)


def pad_before(mode, width):
  return {'front': width - 1, 'center': width // 2, 'end': 0}[mode]


def _padded(v, mode, width):
  if not (np.isfinite(v[0]) and np.isfinite(v[-1])):
    raise EdgeError('non-finite edge value')
  lo = pad_before(mode, width)
  hi = width - 1 - lo
  return np.concatenate([np.full(lo, np.trunc(v[0]), v.dtype), v,
                         np.full(hi, np.trunc(v[-1]), v.dtype)])


def pooled(v, width=80, num_devs=2.0, pad='center', positive=False):
  """(decision [T] bool, margin [T]) of the pooled-outlier test on the float32 values v."""
  v = np.asarray(v, np.float32)
  p = _padded(v, pad, width).astype(np.float64)
  t = len(v)
  w = np.lib.stride_tricks.sliding_window_view(p, width)[:t]
  with np.errstate(invalid='ignore'):
    d = w - v.astype(np.float64)[:, None]
    mean = d.sum(axis=1) / width
    std = np.sqrt(((d - mean[:, None]) ** 2).sum(axis=1) / width)
    score = mean - num_devs * std
  finite = np.isfinite(w).all(axis=1)
  on = finite & (score < 0.0)
  # a constant window is exact: 0 < 0 on every platform
  margin = np.where(finite & ((mean != 0) | (std != 0)), np.abs(score), np.inf)
  if positive:
    on &= v > 0
  return on, margin


def strided(f0, widths=(2, 4, 8, 16, 32), pad='front'):
  """(transitions & (f0 > 0) [T], margin [T]): margin is the smallest ||a - b| - 0.75|
  over the widths, in float64 of the float32 pitches."""
  f0 = np.asarray(f0, np.float32)
  m = hz_to_midi32(f0)
  t = len(f0)
  tr = np.ones(t, bool)
  margin = np.full(t, np.inf)
  for w in widths:
    pm = _padded(m, pad, w)
    first, last = pm[:t], pm[w - 1:w - 1 + t]
    diff = np.abs((first - last).astype(np.float32))
    with np.errstate(invalid='ignore'):
      change = diff > F32(0.75)
      margin = np.minimum(margin, np.where(np.isnan(diff), np.inf,
                                           np.abs(diff.astype(np.float64) - 0.75)))
    lo = pad_before(pad, w)
    ptr = np.concatenate([np.full(lo, tr[0]), tr, np.full(w - 1 - lo, tr[-1])])
    allon = np.lib.stride_tricks.sliding_window_view(ptr, w)[:t].all(axis=1)
    tr = tr & ~(allon & change)
  return tr & (f0 > 0), margin


def remove_short(on, min_samples=20, glue_back=False):
  """The reference's loop, on a copy."""
  on = np.array(on, bool)
  has_been_on = 0
  prev_note_end = 0
  for i in range(len(on)):
    if on[i]:
      has_been_on += 1
    else:
      if has_been_on < min_samples:
        if glue_back:
          on[prev_note_end:i] = True
        else:
          on[i - has_been_on:i] = False
      has_been_on = 0
      prev_note_end = i
  return on


def midi_heuristic(f0, amps):
  """(mask, margin) of remove_short(strided & amp_pooled, 10); margin per frame is the
  smaller of the two tests' (remove_short spreads a flip over its run: callers compare
  runs, see tests/test_heuristics.py)."""
  s, ms = strided(f0)
  a, ma = pooled(log32(np.asarray(amps, np.float32)), 80, 2.0, 'center')
  return remove_short(s & a, 10), np.minimum(ms, ma)


def midi_heuristic_power(f0, power):
  s, ms = strided(f0)
  shifted = (np.asarray(power, np.float32) + F32(DB_RANGE)).astype(np.float32)
  a, ma = pooled(shifted, 80, 2.5, 'center', positive=True)
  return remove_short(s & a, 10), np.minimum(ms, ma)


def median32(x):
  x = np.asarray(x, np.float32)
  if len(x) == 0 or np.isnan(x).any():
    return F32(np.nan)
  s = np.sort(x)
  n = len(s)
  return s[(n - 1) // 2] if n % 2 else F32((s[n // 2 - 1] + s[n // 2]) * F32(0.5))


def pitch(f):
  m = hz_to_midi32(np.asarray([f], np.float32))[0]
  return int(np.rint(m)) if np.isfinite(m) else -2**31


def note_table(mask, f0, median=False):
  """[(start, stop, f0 float32, pitch)] of the runs of truthy frames."""
  mask = np.asarray(mask, bool)
  f0 = np.asarray(f0, np.float32)
  notes = []
  t = 0
  while t < len(mask):
    if not mask[t]:
      t += 1
      continue
    s = t
    while t < len(mask) and mask[t]:
      t += 1
    run = f0[s:t]
    f = median32(run) if median else F32(run.astype(np.float64).sum() / len(run))
    notes.append((s, t, f, pitch(f)))
  return notes
