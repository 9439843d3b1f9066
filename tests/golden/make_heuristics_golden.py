"""Writes tests/golden/heuristics.npz: outputs of the UNMODIFIED REFERENCE's
training/heuristics.py (amp_pooled_outliers, strided_freq_change, remove_short,
midi_heuristic, midi_heuristic_power, segment_notes with mean_f0 and median_f0) on
seeded controls, run on the NumPy TensorFlow shim.

ddsp/training/__init__.py imports google.cloud, so heuristics.py is loaded by its file
path under a stub `ddsp.training` package.  It imports note_seq, which is not
installed: this script gives it a stub NoteSequence with `notes.add()` and
`total_time`.  power_pooled_outliers adds `ddsp.spectral_ops.LD_RANGE`, which the
reference does not define; this script sets it to DB_RANGE (80 dB) on the loaded module
so that midi_heuristic_power runs.  The shim itself is not changed.

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_heuristics_golden.py          # rewrite the fixture
  python tests/golden/make_heuristics_golden.py --check  # regenerate and compare
"""
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                   # noqa: E402
from tests.golden.make_golden import compare     # noqa: E402

PATH = os.path.join(HERE, 'heuristics.npz')
NAN = np.nan

TRACK_LENGTHS = (2, 3, 79, 80, 81, 1003)
PADS = ('front', 'center', 'end')
# remove_short inputs: (name, vector, min_samples)
SHORT_CASES = [
    ('issue', [1, 1, 0, 0, 1, 1, 1, 0, 1], 3),
    ('leading_off', [0, 0, 1, 0, 1, 1, 0, 0, 0, 1, 1], 2),
    ('all_on', [1, 1, 1, 1], 10),
    ('all_off', [0, 0, 0], 2),
    ('random', 'random', 4),
]


def track(t, seed):
  """Seeded f0 [T, 1] (Hz) and amplitudes [T, 1]: held notes with vibrato, separated by
  silences (f0 0 Hz, small amplitudes), amplitudes strictly positive."""
  rng = np.random.default_rng(seed)
  f0 = np.zeros(t, np.float64)
  amps = np.full(t, 1e-3)
  i = int(rng.integers(0, 6))
  while i < t:
    n = int(rng.integers(8, 90))
    midi = rng.uniform(45, 75)
    k = np.arange(min(n, t - i))
    f0[i:i + n] = 440.0 * 2 ** ((midi + 0.25 * np.sin(k * rng.uniform(0.1, 0.5)) - 69) / 12)
    amps[i:i + n] = rng.uniform(0.05, 0.8) * np.exp(-k / rng.uniform(20, 200))
    i += n + int(rng.integers(0, 12))
  amps *= np.exp(rng.normal(0, 0.05, t))
  return f0.astype(np.float32)[:, None], amps.astype(np.float32)[:, None]


def edge_amps(seed, t=60):
  """Amplitudes whose log edge values truncate (signs both ways), with an inner zero,
  an inner NaN and a constant stretch."""
  rng = np.random.default_rng(seed)
  la = rng.normal(0, 1.5, t)
  la[0], la[-1] = -3.7, 2.9
  la[20:32] = 0.0            # constant windows (amplitude exactly 1)
  amps = np.exp(la).astype(np.float32)
  amps[44] = 0.0             # log -inf
  amps[50] = NAN
  return amps[:, None]


def _stub_note_seq():
  class _Notes(list):

    def add(self):
      n = types.SimpleNamespace(pitch=0, start_time=0.0, end_time=0.0, velocity=0)
      self.append(n)
      return n

  class NoteSequence:

    def __init__(self):
      self.notes = _Notes()
      self.total_time = 0.0

  sys.modules['note_seq'] = types.SimpleNamespace(NoteSequence=NoteSequence)


def _load():
  ddsp = ref_on_shim.load()
  if 'ddsp.training.heuristics' in sys.modules:
    return ddsp, sys.modules['ddsp.training.heuristics']
  _stub_note_seq()
  ddsp.spectral_ops.LD_RANGE = ddsp.spectral_ops.DB_RANGE
  root = os.path.join(ref_on_shim.REFERENCE_ROOT, 'ddsp', 'training')
  if 'ddsp.training' not in sys.modules:
    pkg = types.ModuleType('ddsp.training')
    pkg.__path__ = [root]
    sys.modules['ddsp.training'] = pkg
  spec = importlib.util.spec_from_file_location('ddsp.training.heuristics',
                                                os.path.join(root, 'heuristics.py'))
  h = importlib.util.module_from_spec(spec)
  sys.modules['ddsp.training.heuristics'] = h
  spec.loader.exec_module(h)
  return ddsp, h


def short_input(i):
  _, v, _ = SHORT_CASES[i]
  if v == 'random':
    return np.random.default_rng(4100 + i).random(200) < 0.7
  return np.asarray(v, bool)


def _notes(seq):
  """[n, 4] float64 rows (pitch, start_time, end_time, velocity) and total_time."""
  rows = [(n.pitch, n.start_time, n.end_time, n.velocity) for n in seq.notes]
  return np.asarray(rows, np.float64).reshape(-1, 4), np.float64(seq.total_time)


def _error(fn):
  try:
    fn()
  except Exception as e:  # noqa: BLE001 - the reference's error class is the datum
    return np.asarray(type(e).__name__)
  return np.asarray('')


def heuristics():
  _, h = _load()
  tf = ref_on_shim.tf()

  def controls(f0, amps=None, audio=None):
    c = {'f0_hz': tf.constant(f0)}
    if amps is not None:
      c['harmonic'] = {'controls': {'amplitudes': amps}}
    if audio is not None:
      c['audio'] = audio
    return c

  out = {}
  with np.errstate(all='ignore'):
    for t in TRACK_LENGTHS:
      f0, amps = track(t, 4000 + t)
      c = controls(f0, amps)
      out[f'track{t}_f0'], out[f'track{t}_amps'] = f0, amps
      out[f'track{t}_midi_heuristic'] = h.midi_heuristic(c)
      out[f'track{t}_strided'] = h.strided_freq_change(c)
      out[f'track{t}_amp_pooled'] = h.amp_pooled_outliers(c)
      for pick in ('mean_f0', 'median_f0'):
        rows, total = _notes(h.segment_notes(h.midi_heuristic, getattr(h, pick),
                                             h.median_amps, c))
        out[f'track{t}_{pick}_notes'], out[f'track{t}_{pick}_total'] = rows, total
    # pad modes, truncated edges, inner zeros and NaN, constant windows
    for k, seed in enumerate((4200, 4201)):
      amps = edge_amps(seed)
      f0, _ = track(len(amps), seed)
      f0[0, 0], f0[-1, 0] = 100.0, 1200.0
      f0[30, 0] = NAN
      out[f'edge{k}_amps'], out[f'edge{k}_f0'] = amps, f0
      for pad in PADS:
        out[f'edge{k}_amp_pooled_{pad}'] = h.amp_pooled_outliers(
            controls(f0, amps), frame_width=9 + k, num_devs=1.5, pad_mode=pad)
        out[f'edge{k}_strided_{pad}'] = h.strided_freq_change(
            controls(f0), frame_widths=(3, 6, 2), pad_mode=pad)
    for i, (name, _, min_samples) in enumerate(SHORT_CASES):
      v = short_input(i)
      out[f'short_{name}_in'] = v
      for glue in (False, True):
        out[f'short_{name}_glue{int(glue)}'] = h.remove_short(v.copy(), min_samples, glue)
    # median_f0 on runs of even length
    f0, amps = track(40, 4300)
    mask = np.zeros(40, bool)
    mask[2:6] = mask[10:16] = mask[20:21] = mask[30:40] = True
    out['even_f0'], out['even_mask'] = f0, mask
    for pick in ('mean_f0', 'median_f0'):
      rows, total = _notes(h.segment_notes(lambda c: mask, getattr(h, pick), h.median_amps,
                                           controls(f0, amps)))
      out[f'even_{pick}_notes'], out[f'even_{pick}_total'] = rows, total
    # centre-framed power: T + 1 frames
    rng = np.random.default_rng(4400)
    frames = 200
    audio = (rng.normal(0, 0.1, 64 * frames) *
             np.repeat(rng.uniform(0, 1, frames) > 0.3, 64)).astype(np.float32)
    f0, _ = track(frames + 1, 4401)
    out['power_audio'], out['power_f0'] = audio, f0
    out['power_midi_heuristic'] = h.midi_heuristic_power(controls(f0, audio=audio))
    out['power_pooled'] = h.power_pooled_outliers(controls(f0, audio=audio))
    # the reference's errors
    f0, amps = track(50, 4500)
    zero_edge, nan_edge = amps.copy(), amps.copy()
    zero_edge[-1] = 0.0
    nan_edge[0] = NAN
    inf_f0 = f0.copy()
    inf_f0[0] = np.inf
    out['err_zero_edge'] = _error(lambda: h.midi_heuristic(controls(f0, zero_edge)))
    out['err_nan_edge'] = _error(lambda: h.amp_pooled_outliers(controls(f0, nan_edge)))
    out['err_inf_f0_edge'] = _error(lambda: h.strided_freq_change(controls(inf_f0)))
    out['err_t1'] = _error(lambda: h.midi_heuristic(controls(f0[:1], amps[:1])))
    out['err_power_length'] = _error(lambda: h.midi_heuristic_power(
        controls(f0[:49], audio=audio[:64 * 49])))
  return {k: np.asarray(v) if np.asarray(v).dtype.kind in 'US' else
          np.asarray(v, np.float64) for k, v in out.items()}


def _compare(got, want):
  assert set(want.files) == set(got), sorted(set(want.files) ^ set(got))
  for k in want.files:
    if want[k].dtype.kind in 'US':
      assert str(got[k]) == str(want[k]), (k, got[k], want[k])
    else:
      np.testing.assert_array_equal(got[k], want[k], err_msg=k)


if __name__ == '__main__':
  got = heuristics()
  if '--check' in sys.argv:
    _compare(got, np.load(PATH))
    print('ok    heuristics')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote heuristics %.0f kB' % (os.path.getsize(PATH) / 1e3))
