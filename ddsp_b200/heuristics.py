"""DDSP controls to notes (`ddsp/training/heuristics.py`): the binarizers that decide
when a note is on, and the segmentation of their masks into notes, as the MIDI
autoencoder's `MidiHeuristicEvaluator` uses them.  Same names, arguments and defaults
as the reference.

Every function takes the reference's per-item controls (`f0_hz` [T] or [T, 1],
amplitudes [T] or [T, 1], audio [N]) and batched controls ([B, T, 1], audio [B, N]),
and returns [T] or [B, T] to match.  amp_pooled_outliers, strided_freq_change,
power_pooled_outliers, remove_short, midi_heuristic and midi_heuristic_power run on the
`ddsp_b200_note_heuristic` kernel (csrc/heuristics.cuh, DESIGN.md section 3.28), and
note_table on `ddsp_b200_note_segments`.  segment_notes and segment_notes_batch are
built on them and return objects with the part of `note_seq.NoteSequence` the
reference fills.  mean_f0, median_f0, median_amps, pad_for_frame, window_array and
get_active_frame_indices are torch ops.

Forward only: an input that requires grad raises.  The reference's one deviation:
power_pooled_outliers shifts the power by spectral_ops.DB_RANGE (80 dB), because the
reference's `LD_RANGE` does not exist.
"""
import collections
import math

import numpy as np
import torch

from ddsp_b200 import _lib
from ddsp_b200 import core
from ddsp_b200 import spectral_ops

DDSP_DEFAULT_FRAME_RATE = 250

_PADS = {'front': _lib.HEURISTIC_PAD_FRONT, 'center': _lib.HEURISTIC_PAD_CENTER,
         'end': _lib.HEURISTIC_PAD_END}
_POOL, _STRIDED = _lib.HEURISTIC_POOL, _lib.HEURISTIC_STRIDED
_F0_POSITIVE, _REMOVE_SHORT = _lib.HEURISTIC_F0_POSITIVE, _lib.HEURISTIC_REMOVE_SHORT

NoteTable = collections.namedtuple('NoteTable', ['start', 'stop', 'f0', 'pitch', 'count'])


def note_heuristic_takes(t):
  """True where the heuristic kernels take T frames (1 <= T <= NOTE_HEURISTIC_MAX_T)."""
  return bool(_lib.load().ddsp_b200_note_heuristic_takes(int(t)))


# ---- the NoteSequence subset the reference fills -----------------------------------------
class Note:
  """A note of note_seq.NoteSequence: pitch, start_time, end_time, velocity."""
  __slots__ = ('pitch', 'start_time', 'end_time', 'velocity')

  def __init__(self, pitch=0, start_time=0.0, end_time=0.0, velocity=0):
    self.pitch, self.start_time = pitch, start_time
    self.end_time, self.velocity = end_time, velocity

  def __repr__(self):
    return (f'Note(pitch={self.pitch}, start_time={self.start_time}, '
            f'end_time={self.end_time}, velocity={self.velocity})')


class _Notes(list):

  def add(self):
    note = Note()
    self.append(note)
    return note


class NoteSequence:
  """The part of note_seq.NoteSequence that segment_notes fills: `notes` (with
  `notes.add()`) and `total_time`."""

  def __init__(self):
    self.notes = _Notes()
    self.total_time = 0.0


# ---- controls ----------------------------------------------------------------------------
def _rows(x, name):
  """([B, T] float32 CUDA tensor, batched) of per-item [T] / [T, 1] or batched [B, T, 1]
  controls.  T < 2 raises ValueError (the reference's np.squeeze leaves a 0-d array),
  T beyond the kernels' limit NotImplementedError, both before any device work."""
  shape = core._shape(x)
  if len(shape) == 1 or (len(shape) == 2 and shape[1] == 1):
    batched = False
  elif len(shape) == 3 and shape[2] == 1:
    batched = True
  else:
    raise ValueError(f'{name}: expected [time], [time, 1] or [batch, time, 1], got {shape}')
  t = shape[1] if batched else shape[0]
  if t < 2:
    raise ValueError(f'{name}: needs at least two frames, got shape {shape}')
  if not note_heuristic_takes(t):
    raise NotImplementedError(f'{name}: {t} frames exceed the '
                              f'{_lib.NOTE_HEURISTIC_MAX_T} the heuristic kernels take')
  core._no_grad_path(name, x)
  x = core.torch_float32(x)
  return x.reshape(shape[0] if batched else 1, t), batched


def _amplitudes(controls):
  return controls['harmonic']['controls']['amplitudes']


def _pad(pad_mode):
  if pad_mode not in _PADS:
    raise ValueError(f'Unrecognized pad mode {pad_mode}.')
  return _PADS[pad_mode]


def _width(frame_width, name):
  w = int(frame_width)
  if w != frame_width or w < 1:
    raise ValueError(f'{name}: frame widths must be positive integers, got {frame_width}')
  return w


class _Args:
  """The arguments of one ddsp_b200_note_heuristic launch beyond its operands."""

  def __init__(self, stages=0):
    self.stages = stages
    self.log_values, self.shift, self.positive = 1, 0.0, 0
    self.pool_width, self.pool_pad, self.num_devs = 1, _PADS['center'], 0.0
    self.widths, self.strided_pad = (), _PADS['front']
    self.min_samples, self.glue_back = 0, 0

  def pool(self, frame_width, num_devs, pad_mode, power):
    self.stages |= _POOL
    self.pool_width = _width(frame_width, 'pooled outliers')
    self.num_devs, self.pool_pad = float(num_devs), _pad(pad_mode)
    if math.isnan(self.num_devs):
      raise ValueError('pooled outliers: num_devs is NaN')
    if power:
      self.log_values, self.shift, self.positive = 0, float(spectral_ops.DB_RANGE), 1
    return self

  def strided(self, frame_widths, pad_mode):
    self.stages |= _STRIDED | _F0_POSITIVE
    self.widths = tuple(_width(w, 'strided_freq_change') for w in frame_widths)
    if len(self.widths) > _lib.HEURISTIC_MAX_WIDTHS:
      raise NotImplementedError(f'strided_freq_change: {len(self.widths)} frame widths, '
                                f'at most {_lib.HEURISTIC_MAX_WIDTHS}')
    if self.widths:
      self.strided_pad = _pad(pad_mode)
    return self

  def remove_short(self, min_samples, glue_back):
    self.stages |= _REMOVE_SHORT
    self.min_samples = int(min_samples)
    if self.min_samples != min_samples:
      raise ValueError(f'remove_short: min_samples must be an integer, got {min_samples}')
    self.min_samples = max(min(self.min_samples, 2**31 - 1), -2**31)
    self.glue_back = int(bool(glue_back))
    return self


def note_heuristic(args, x=None, f0=None, on=None, status=None):
  """One ddsp_b200_note_heuristic launch on [B, T] operands: (mask [B, T] bool, status
  [B] int32), without a host synchronisation.  status may be a preallocated int32 [B]."""
  return core.note_heuristic(x, f0, on, status, args.stages, args.log_values, args.shift,
                             args.pool_width, args.pool_pad, args.positive, args.num_devs,
                             args.widths, args.strided_pad, args.min_samples, args.glue_back)


def _raise_status(status, name):
  """The reference's error for a non-finite padded edge value, after one read of the
  per-item status.  Skipped while the stream is captured into a CUDA graph (the status
  then stays on the device, and the failed items' mask rows are all False)."""
  if torch.cuda.is_current_stream_capturing():
    return
  s = status.cpu() if status.is_cuda else status
  bad = torch.nonzero(s).flatten().tolist()
  if bad:
    what = ('f0_midi' if int(s[bad[0]]) == _lib.HEURISTIC_PITCH_EDGE
            else 'the pooled values')
    raise ValueError(f'{name}: item {bad[0]}: {what} has a non-finite first or last frame, '
                     'which pad_for_frame cannot pad (the reference converts it with int())')


def _binarize(name, args, batched, **operands):
  with core._on_device_of(*[v for v in operands.values() if v is not None]):
    mask, status = note_heuristic(args, **operands)
    _raise_status(status, name)
  return mask if batched else mask[0]


def _f0_rows(controls, name):
  return _rows(controls['f0_hz'], name)


def _power_rows(controls, name, device):
  """Shift-free power [B, F] of controls['audio'] ([N] or [B, N]), frame size 256."""
  audio = controls['audio']
  core._no_grad_path(name, audio)
  if not torch.is_tensor(audio) or not audio.is_cuda:
    audio = core.torch_float32(audio, device)
  power = spectral_ops.compute_power(audio, frame_size=256)
  return power.reshape(-1, power.shape[-1])


# ---- binarizers --------------------------------------------------------------------------
@core.on_operands_device
def remove_short(is_on_vec, min_samples=20, glue_back=False):
  """heuristics.remove_short: clears every run of truthy frames (NaN is truthy) that a
  falsy frame ends when it is shorter than min_samples; a trailing run no falsy frame
  ends is kept.  With glue_back every falsy frame i with a short (possibly empty) run
  before the next falsy frame j is set True instead, the reference's
  is_on_vec[prev_note_end:i] = True.  [T] or [B, T] in, bool of that shape out.  The
  reference also writes the result into is_on_vec; this returns a new tensor."""
  shape = core._shape(is_on_vec)
  if len(shape) not in (1, 2) or shape[-1] < 1:
    raise ValueError(f'remove_short: expected [time] or [batch, time], got {shape}')
  core._no_grad_path('remove_short', is_on_vec)
  v = is_on_vec if torch.is_tensor(is_on_vec) else torch.as_tensor(np.asarray(is_on_vec))
  on = (v != 0).to(torch.uint8)
  on = on.to(core._device()) if not on.is_cuda else on
  on = on.reshape(-1, shape[-1]).contiguous()
  if not note_heuristic_takes(shape[-1]):
    raise NotImplementedError(f'remove_short: {shape[-1]} frames exceed the '
                              f'{_lib.NOTE_HEURISTIC_MAX_T} the heuristic kernels take')
  mask = _binarize('remove_short', _Args().remove_short(min_samples, glue_back), True, on=on)
  return mask.reshape(shape)


@core.on_operands_device
def amp_pooled_outliers(controls, frame_width=80, num_devs=2, pad_mode='center'):
  """heuristics.amp_pooled_outliers: frames whose log amplitude is above the mean less
  num_devs population standard deviations of its padded window of frame_width log
  amplitudes.  A window with a non-finite value (an inner zero amplitude) is False, and
  so is a constant one.  A zero or non-finite first or last amplitude raises ValueError,
  as the reference's pad_for_frame does (OverflowError or ValueError there)."""
  args = _Args().pool(frame_width, num_devs, pad_mode, power=False)
  x, batched = _rows(_amplitudes(controls), 'amp_pooled_outliers')
  return _binarize('amp_pooled_outliers', args, batched, x=x)


@core.on_operands_device
def strided_freq_change(controls, frame_widths=(2, 4, 8, 16, 32), pad_mode='front'):
  """heuristics.strided_freq_change: starting all True, for each width in order, frames
  whose padded window of the transitions so far is all True and whose window's first
  and last float32 MIDI pitches differ by more than 0.75 are switched off; then & (f0 > 0).
  A non-finite first or last pitch (f0 +inf or NaN) raises ValueError."""
  args = _Args().strided(frame_widths, pad_mode)
  f0, batched = _f0_rows(controls, 'strided_freq_change')
  return _binarize('strided_freq_change', args, batched, f0=f0)


@core.on_operands_device
def power_pooled_outliers(controls, frame_width=80, num_devs=2.5, pad_mode='center'):
  """heuristics.power_pooled_outliers on the shifted power
  compute_power(audio, frame_size=256) + DB_RANGE (the reference's LD_RANGE does not
  exist): the pooled-outlier test, and shifted power > 0.  audio [N] gives [F], [B, N]
  [B, F]; F is n_samples / 64 + 1 under centre padding."""
  args = _Args().pool(frame_width, num_devs, pad_mode, power=True)
  batched = len(core._shape(controls['audio'])) == 2
  x = _power_rows(controls, 'power_pooled_outliers', None)
  if x.shape[1] < 2:
    raise ValueError(f'power_pooled_outliers: needs at least two frames, got {x.shape[1]}')
  return _binarize('power_pooled_outliers', args, batched, x=x)


def _fused(binarize_f, controls):
  """binarize_f (midi_heuristic or midi_heuristic_power) with the defaults, in one launch."""
  name = binarize_f.__name__
  f0, batched = _f0_rows(controls, name)
  with core._on_device_of(f0):
    mask, status = _fused_mask(binarize_f, controls, f0, None)
    _raise_status(status, name)
  return mask if batched else mask[0]


@core.on_operands_device
def midi_heuristic(controls):
  """heuristics.midi_heuristic: remove_short(strided_freq_change(controls) &
  amp_pooled_outliers(controls), min_samples=10) with the defaults, in one launch.
  Amplitudes and f0_hz must have the same frames."""
  return _fused(midi_heuristic, controls)


@core.on_operands_device
def midi_heuristic_power(controls):
  """heuristics.midi_heuristic_power: as midi_heuristic with power_pooled_outliers, after
  the compute_power launch.  The power has n_samples / 64 + 1 frames under centre
  padding; f0_hz must have as many (ValueError otherwise, the reference's broadcast
  error)."""
  return _fused(midi_heuristic_power, controls)


# ---- the note table ----------------------------------------------------------------------
def _table(mask, f0, median, buf=None):
  b, t = f0.shape
  if buf is None:
    buf = core.note_table_buffer(b, t, f0.device)
  _, _, count, notes = buf
  core.note_segments(mask, f0, notes, count, median)
  return NoteTable(notes[..., 0], notes[..., 1], notes[..., 3].view(torch.float32),
                   notes[..., 2], count)


@core.on_operands_device
def note_table(mask, f0_hz, pick='mean'):
  """The notes of the runs of truthy frames of mask ([T] or [B, T]; NaN is truthy), as
  fixed-capacity device tensors without a host synchronisation: start, stop (frames,
  int32), f0 (float32) and pitch (int32), each [B, (T+1)//2] with the first count [B]
  rows filled and the rest zero ([(T+1)//2] and a 0-d count for per-item input).  f0
  is the run's mean_f0 (summed in double, rounded once to float32) or median_f0
  (np.median's, exact); pitch is np.round(hz_to_midi(f0)) in float32, half to even,
  -2^31 for NaN."""
  if pick not in ('mean', 'median'):
    raise ValueError(f"note_table: pick must be 'mean' or 'median', got {pick!r}")
  f0, batched = _rows(f0_hz, 'note_table')
  ms = core._shape(mask)
  if ms != ((f0.shape[0], f0.shape[1]) if batched else (f0.shape[1],)):
    raise ValueError(f'note_table: mask {ms} and f0_hz {core._shape(f0_hz)} must share '
                     'their frames')
  core._no_grad_path('note_table', mask)
  m = mask if torch.is_tensor(mask) else torch.as_tensor(np.asarray(mask))
  m = (m.to(f0.device) != 0).to(torch.uint8).reshape(f0.shape).contiguous()
  table = _table(m, f0, pick == 'median')
  return table if batched else NoteTable(*(x[0] for x in table))


# ---- segmentation ------------------------------------------------------------------------
_BINARIZERS = {}   # this module's binarizers: their fused launch arguments
_PICKS = {}        # this module's f0 picks: median or not


def _unbatch(batch):
  """heuristics._unbatch: a dict of batched tensors (and dicts of them) as a list of
  per-item dicts; None values are dropped."""
  unbatched = []
  for key, val in batch.items():
    if isinstance(val, (torch.Tensor, np.ndarray)):
      if not unbatched:
        unbatched = [{} for _ in range(val.shape[0])]
      assert val.shape[0] == len(
          unbatched), f'batch size mismatch: {val.shape[0]} vs {len(unbatched)}'
      for i in range(val.shape[0]):
        unbatched[i][key] = val[i]
    elif isinstance(val, dict):
      sub_batch = _unbatch(val)
      if not unbatched:
        unbatched = [{} for _ in sub_batch]
      for i in range(len(sub_batch)):
        unbatched[i][key] = sub_batch[i]
    elif val is None:
      continue
    else:
      raise Exception(f'unsupported value at {key}:{val} of type {type(val)}')
  return unbatched


def _np_hz_to_midi(f0):
  """core.hz_to_midi of one float32 value in float32, the reference's op order, with
  correctly rounded logs (as the kernel computes it)."""
  f = np.float32(f0)
  if not f > 0:
    return np.float32(np.nan) if np.isnan(f) else np.float32(0.0)
  ln2 = np.float32(math.log(2.0))
  c = np.float32(np.float32(math.log(440.0)) / ln2)
  lf = np.float32(np.log(np.float64(f)))
  return np.float32(np.float32(12.0) * np.float32(np.float32(lf / ln2) - c)) + np.float32(69.0)


def _np_pitch(f0):
  m = _np_hz_to_midi(f0)
  return int(np.rint(m)) if np.isfinite(m) and abs(m) < 2**31 else -2**31


def _sequence(rows, n, t, frame_rate):
  """A NoteSequence from the host note records rows [cap, 4] (n filled)."""
  seq = NoteSequence()
  for start, stop, pitch, _ in rows[:n].tolist():
    note = seq.notes.add()
    note.pitch = pitch
    note.start_time = start / frame_rate
    note.end_time = stop / frame_rate
    note.velocity = 127
  seq.total_time = t / frame_rate
  return seq


def _foreign_notes(mask, pick_f0_f, pick_amps_f, controls, frame_rate):
  """segment_notes' per-note loop over the host mask [T], calling the caller's picks as
  the reference does."""
  seq = NoteSequence()

  def construct_note(curr_ind, duration):
    note_start = curr_ind - duration
    f0 = pick_f0_f(controls, start=note_start, stop=curr_ind)
    if pick_amps_f is not median_amps:
      pick_amps_f(controls, start=note_start, stop=curr_ind)   # unused, as there
    f0 = f0.item() if torch.is_tensor(f0) else f0
    note = seq.notes.add()
    note.pitch = _np_pitch(f0)
    note.start_time = note_start / frame_rate
    note.end_time = (note_start + duration) / frame_rate
    note.velocity = 127

  has_been_on = 0
  for i, sample_i in enumerate(mask.tolist()):
    if sample_i:
      has_been_on += 1
    elif has_been_on > 0:
      construct_note(i, has_been_on)
      has_been_on = 0
  if has_been_on > 0:
    construct_note(len(mask), has_been_on)
  seq.total_time = len(mask) / frame_rate
  return seq


def _batch_mask(binarize_f, controls_batch, items):
  """[B, T] device mask and status of binarize_f over the batch: one launch for this
  module's binarizers, else binarize_f per item on the unbatched dicts."""
  if binarize_f in _BINARIZERS:
    mask = binarize_f(controls_batch)
    return mask if mask.dim() == 2 else mask[None]
  masks = []
  for controls in items:
    m = binarize_f(controls)
    m = m if torch.is_tensor(m) else torch.as_tensor(np.asarray(m))
    masks.append(m.reshape(-1) != 0)
  return torch.stack(masks)


@core.on_operands_device
def segment_notes_batch(binarize_f, pick_f0_f, pick_amps_f, controls_batch,
                        frame_rate=DDSP_DEFAULT_FRAME_RATE):
  """heuristics.segment_notes_batch: a NoteSequence per item of controls_batch
  ([B, T, 1] controls).  With this module's binarizers the mask of the whole batch is
  one launch, and with mean_f0 or median_f0 the note table another; the notes then come
  to the host in one copy.  Any other callable is called as the reference calls it: per
  item on the unbatched dict, and picks per note.  median_amps, whose result the
  reference discards, is not evaluated."""
  items = None
  if binarize_f not in _BINARIZERS or pick_f0_f not in _PICKS:
    items = _unbatch(controls_batch)
  if pick_f0_f not in _PICKS:
    masks = _batch_mask(binarize_f, controls_batch, items).cpu()
    return [_foreign_notes(m, pick_f0_f, pick_amps_f, c, frame_rate)
            for m, c in zip(masks, items)]
  f0, _ = _rows(controls_batch['f0_hz'], 'segment_notes_batch')
  b, t = f0.shape
  with core._on_device_of(f0):
    buf = core.note_table_buffer(b, t, f0.device)
    if binarize_f in _BINARIZERS:
      mask, _ = _fused_mask(binarize_f, controls_batch, f0, buf[1])
    else:
      mask = _batch_mask(binarize_f, controls_batch, items).to(f0.device)
      buf[1].zero_()
    if mask.shape != f0.shape:
      raise ValueError(f'segment_notes_batch: the mask {tuple(mask.shape)} and f0_hz '
                       f'{tuple(f0.shape)} must share their frames')
    _table(mask.to(torch.uint8).contiguous(), f0, _PICKS[pick_f0_f], buf)
    host = buf[0].cpu()
  _raise_status(host[:b], binarize_f.__name__)
  count = host[b:2 * b].tolist()
  rows = host[buf[0].shape[0] - buf[3].numel():].view(b, -1, 4)
  if pick_amps_f is not median_amps:
    items = items or _unbatch(controls_batch)
    for i, c in enumerate(items):
      for start, stop in rows[i, :count[i], :2].tolist():
        pick_amps_f(c, start=start, stop=stop)
  return [_sequence(rows[i], count[i], t, frame_rate) for i in range(b)]


def _fused_mask(binarize_f, controls_batch, f0, status):
  """(mask [B, T], status [B]) of binarize_f over a batch in one launch; status may be a
  preallocated int32 [B]."""
  name = binarize_f.__name__
  args = _BINARIZERS[binarize_f]()
  x = None
  if args.stages & _POOL:
    if args.log_values:
      x, _ = _rows(_amplitudes(controls_batch), name)
      x = x.to(f0.device)
    else:
      x = _power_rows(controls_batch, name, f0.device)
    if x.shape != f0.shape:
      raise ValueError(f'{name}: the pooled values have {tuple(x.shape)} frames and '
                       f'f0_hz {tuple(f0.shape)}; they must match')
  return note_heuristic(args, x=x, f0=f0 if args.stages & _STRIDED else None, status=status)


def segment_notes(binarize_f, pick_f0_f, pick_amps_f, controls,
                  frame_rate=DDSP_DEFAULT_FRAME_RATE):
  """heuristics.segment_notes: a NoteSequence with one note per maximal run of truthy
  frames of binarize_f(controls): pitch np.round(hz_to_midi(pick_f0_f(...))) as int32,
  start_time start / frame_rate, end_time stop / frame_rate, velocity 127, and
  total_time T / frame_rate.  controls are one item's ([T, 1]); this module's own
  functions take the fused path of segment_notes_batch."""
  if binarize_f in _BINARIZERS and pick_f0_f in _PICKS:
    batch = _add_batch_axis(controls)
    return segment_notes_batch(binarize_f, pick_f0_f, pick_amps_f, batch, frame_rate)[0]
  mask = binarize_f(controls)
  mask = mask if torch.is_tensor(mask) else torch.as_tensor(np.asarray(mask))
  return _foreign_notes(mask.reshape(-1).cpu() != 0, pick_f0_f, pick_amps_f, controls,
                        frame_rate)


def _add_batch_axis(controls):
  out = {}
  for k, v in controls.items():
    if isinstance(v, dict):
      out[k] = _add_batch_axis(v)
    elif isinstance(v, (torch.Tensor, np.ndarray)):
      v = v if torch.is_tensor(v) else torch.as_tensor(np.asarray(v))
      out[k] = v[None] if v.dim() != 1 or k == 'audio' else v[None, :, None]
    else:
      out[k] = v
  return out


# ---- f0 and amplitude picks --------------------------------------------------------------
def _median(x):
  """np.median of the float32 values x: the middle value, or the float32 mean of the two
  middle values; NaN for a NaN among them or no values."""
  x = core._as_f32(x).reshape(-1)
  n = x.numel()
  if n == 0 or bool(torch.isnan(x).any()):
    return torch.tensor(float('nan'), dtype=torch.float32, device=x.device)
  s = torch.sort(x).values
  a, b = s[(n - 1) // 2], s[n // 2]
  return a if n % 2 else (a + b) / 2


def mean_f0(controls, start, stop):
  """heuristics.mean_f0: the float32 mean of f0_hz[start:stop]."""
  return torch.mean(core._as_f32(controls['f0_hz'])[start:stop])


def median_f0(controls, start, stop):
  """heuristics.median_f0: np.median of f0_hz[start:stop] (torch.median would return the
  lower of the two middle values)."""
  return _median(core._as_f32(controls['f0_hz'])[start:stop])


def median_amps(controls, start, stop):
  """heuristics.median_amps: np.median of the squeezed amplitudes[start:stop]."""
  return _median(torch.squeeze(core._as_f32(_amplitudes(controls)))[start:stop])


_PICKS.update({mean_f0: False, median_f0: True})
_BINARIZERS.update({
    midi_heuristic: lambda: _midi_heuristic_args(power=False),
    midi_heuristic_power: lambda: _midi_heuristic_args(power=True),
    amp_pooled_outliers: lambda: _Args().pool(80, 2, 'center', power=False),
    power_pooled_outliers: lambda: _Args().pool(80, 2.5, 'center', power=True),
    strided_freq_change: lambda: _Args().strided((2, 4, 8, 16, 32), 'front'),
})


def _midi_heuristic_args(power):
  args = _Args().strided((2, 4, 8, 16, 32), 'front').remove_short(10, False)
  return args.pool(80, 2.5 if power else 2, 'center', power=power)


# ---- helpers of the reference ------------------------------------------------------------
def _edge_int(v, name):
  """int() of a one-element value, as pad_for_frame converts its edges: truncation toward
  zero; a non-finite value raises ValueError (the reference: OverflowError for inf)."""
  v = torch.as_tensor(v)
  if v.numel() != 1:
    raise TypeError(f'{name}: only length-1 edge values can be converted to an integer')
  f = float(v.reshape(()).item())
  if not math.isfinite(f):
    raise ValueError(f'{name}: cannot convert the non-finite edge value {f} to an integer')
  return int(f)


def pad_for_frame(vec, mode, frame_width, axis=0):
  """heuristics.pad_for_frame: pads so that with frame step 1 every element is the
  centre ('center'), the end ('front') or the start ('end') of its frame of
  frame_width.  The pad values are int() of the first and last element along `axis`,
  truncated toward zero, and, as np.pad does, every axis is padded."""
  if mode == 'front':
    before, after = frame_width - 1, 0
  elif mode == 'center':
    before, after = int(frame_width / 2), frame_width - int(frame_width / 2) - 1
  elif mode == 'end':
    before, after = 0, frame_width - 1
  else:
    raise ValueError(f'Unrecognized pad mode {mode}.')
  v = vec if torch.is_tensor(vec) else torch.as_tensor(np.asarray(vec))
  lo = _edge_int(v.select(axis, 0), 'pad_for_frame')
  hi = _edge_int(v.select(axis, -1), 'pad_for_frame')
  for ax in range(v.dim()):
    shape = list(v.shape)
    shape[ax] = before
    front = torch.full(shape, lo, dtype=v.dtype, device=v.device)
    shape[ax] = after
    back = torch.full(shape, hi, dtype=v.dtype, device=v.device)
    v = torch.cat([front, v, back], dim=ax)
  return v


def window_array(array, sr, win_len, frame_step_ratio=0.75, ax=0):
  """heuristics.window_array: overlapping frames of int(sr * win_len) samples every
  int(sr * win_len * frame_step_ratio), after int(sr * win_len * (1 - ratio)) leading
  zeros, the last frame padded with zeros (tf.signal.frame with pad_end)."""
  frame_length = int(sr * win_len)
  frame_step = int(sr * win_len * frame_step_ratio)
  pad_front = int(sr * win_len * (1 - frame_step_ratio))
  a = array if torch.is_tensor(array) else torch.as_tensor(np.asarray(array))
  a = torch.movedim(a, ax, 0)
  a = torch.cat([torch.zeros_like(a)[:pad_front], a], dim=0)
  n = a.shape[0]
  n_frames = -(-n // frame_step)
  total = (n_frames - 1) * frame_step + frame_length
  if total > n:
    a = torch.cat([a, a.new_zeros((total - n,) + tuple(a.shape[1:]))], dim=0)
  frames = a.unfold(0, frame_length, frame_step)[:n_frames]   # [F, ..., frame_length]
  frames = torch.movedim(frames, -1, 1)                          # [F, frame_length, ...]
  return torch.movedim(torch.movedim(frames, 1, 0), 0, ax + 1) if ax else frames


def get_active_frame_indices(piano_roll):
  """heuristics.get_active_frame_indices: per frame and pitch, (previous + 1) * active,
  with row 0 zero: the frames since the onset.  A bool piano roll gives bool."""
  roll = piano_roll if torch.is_tensor(piano_roll) else torch.as_tensor(np.asarray(piano_roll))
  out = torch.zeros_like(roll)
  for i in range(1, roll.shape[0]):
    out[i] = (out[i - 1] + 1) * roll[i] if roll.dtype != torch.bool else roll[i]
  return out
