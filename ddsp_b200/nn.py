"""The masking functions of `ddsp/training/nn.py:359-557`: note segmentation, per-note
moments and pooling over notes, as the MIDI autoencoder uses them
(`models/midi_autoencoder.py`: `add_slowness_loss` and `ZMidiAutoencoder.z_note_encode`).
Same names, arguments and defaults as the reference; no network layers.

get_note_mask, get_note_mask_from_onset, get_note_moments and pool_over_notes run on the
CUDA kernels of `csrc/notes.cuh` (DESIGN.md section 3.25), which never build the
reference's [batch, time, notes, dims] products.  get_note_lengths,
get_short_note_loss_mask and straight_through_int_quantization are small torch
reductions and elementwise ops.
"""
import torch

from ddsp_b200 import autograd
from ddsp_b200 import core


def straight_through_int_quantization(x):
  """nn.straight_through_int_quantization: x rounded to the nearest integer (half to
  even, as TensorFlow's round), with the gradient of the identity."""
  x = x if torch.is_tensor(x) else core._as_f32(x)
  return x + (torch.round(x) - x).detach()


def _pitch(q, name):
  """[batch, time] float32 CUDA tensor of a [batch, time] or [batch, time, channels]
  value (channel 0, as the reference takes), detached: the mask comes from comparisons
  and carries no gradient."""
  shape = core._shape(q)
  if len(shape) not in (2, 3):
    raise ValueError(f'{name}: expected [batch, time] or [batch, time, channels], got '
                     f'{shape}')
  if shape[1] < 1:
    raise ValueError(f'{name}: needs at least one frame, got shape {shape}')
  q = q.detach() if torch.is_tensor(q) else q
  q = core.torch_float32(q)
  return q[:, :, 0].contiguous() if q.dim() == 3 else q


def _max_regions(max_regions, name):
  r = int(max_regions)
  if r != max_regions or r < 0:
    raise ValueError(f'{name}: max_regions must be a non-negative integer, got '
                     f'{max_regions}')
  return r


def _note_mask(name, q_pitch, onset, max_regions, note_on_only):
  r = _max_regions(max_regions, name)
  if onset is not None and core._shape(onset)[:2] != core._shape(q_pitch)[:2]:
    raise ValueError(f'{name}: onset {core._shape(onset)} and q_pitch '
                     f'{core._shape(q_pitch)} must share [batch, time]')
  q = _pitch(q_pitch, name)
  on = None if onset is None else _pitch(onset, name)
  if on is not None and on.device != q.device:
    raise ValueError(f'{name}: q_pitch on {q.device} and onset on {on.device}')
  return core.note_mask(q, on, r, note_on_only)


@core.on_operands_device
def get_note_mask(q_pitch, max_regions=100, note_on_only=True):
  """nn.get_note_mask (nn.py:375-425): the binary mask [batch, time, max_regions] of the
  regions of constant q_pitch ([batch, time], or [batch, time, channels] read at channel
  0).  Frame 0 opens region 0; frame t in 1 .. T-2 opens a new one iff
  |q_t - q_{t-1}| > 0, so NaN never does; the last frame joins the region before it.
  Frames of regions max_regions and later get zero rows.  With note_on_only a region is
  kept iff the reference's mask-weighted sum of q over the item is > 0 (decided in
  float64; a non-finite frame anywhere else makes it NaN, so the region is dropped).  As
  in the reference, one frame gives two rows.  The mask never requires grad, whatever
  q_pitch does."""
  return _note_mask('get_note_mask', q_pitch, None, max_regions, note_on_only)


@core.on_operands_device
def get_note_mask_from_onset(q_pitch, onset, max_regions=100, note_on_only=True):
  """nn.get_note_mask_from_onset (nn.py:428-476): regions opened by onset
  ([batch, time] or [batch, time, 1]): frame 0 always, frame t >= 1 by int(onset_t),
  truncated toward zero, so 1.7 counts as 1 and -1 closes one.  Region indices below 0
  or from max_regions on give zero rows.  With note_on_only a frame is kept iff
  q_t > 0.  Non-finite onsets and onsets of magnitude 2^31 or more are outside the
  contract (TensorFlow's cast is undefined there)."""
  return _note_mask('get_note_mask_from_onset', q_pitch, onset, max_regions, note_on_only)


def get_note_lengths(note_mask):
  """nn.get_note_lengths (nn.py:479-481): frames per note, [batch, notes]."""
  return torch.sum(core._as_f32(note_mask), dim=1)


def _moments(name, x, note_mask, pool, return_std):
  sx, sm = core._shape(x), core._shape(note_mask)
  if len(sx) not in (2, 3):
    raise ValueError(f'{name}: x must be [batch, time] or [batch, time, dims], got {sx}')
  if len(sm) != 3:
    raise ValueError(f'{name}: note_mask must be [batch, time, notes], got {sm}')
  if sx[:2] != sm[:2]:
    raise ValueError(f'{name}: x {sx} and note_mask {sm} must share [batch, time] (the '
                     'reference would broadcast a length-1 axis; this does not)')
  if sx[1] < 1:
    raise ValueError(f'{name}: needs at least one frame, got x {sx}')
  core._no_grad_path(name, note_mask)
  x = x if torch.is_tensor(x) and x.is_cuda else core.torch_float32(x)
  is_2d = x.dim() == 2
  x3 = (x[:, :, None] if is_2d else x).to(torch.float32).contiguous()
  mask = core.torch_float32(note_mask, x3.device)
  out = autograd.NoteMomentsFn.apply(x3, mask, pool, bool(return_std))
  outs = out if return_std else (out,)
  if is_2d:
    outs = tuple(o[:, :, 0] for o in outs)
  return outs if return_std else outs[0]


@core.on_operands_device
def get_note_moments(x, note_mask, return_std=True):
  """nn.get_note_moments (nn.py:484-520): the mean and standard deviation of x
  ([batch, time, dims] or [batch, time]) over each note of note_mask
  ([batch, time, notes], any float values), [batch, notes, dims] or [batch, notes]:
  mean = sum_t m x / L and std = (sum_t ((x - mean) m)^2 / L)^0.5 with L = sum_t m, or
  1e-7 where that is 0.  The mean only when return_std is false.

  Differentiable in x; a note_mask that requires grad raises RuntimeError.  x and
  note_mask must share [batch, time] (ValueError otherwise; the reference would broadcast
  a length-1 axis).  Gradients put NaN exactly where float64 autograd of the reference
  does: a note whose variance is 0 (an empty note, or one of constant x with an exact
  mean) makes every gradient through its std NaN for the whole (batch, dim), and
  max_regions = 100 almost always leaves empty notes.  Gradients through the mean alone
  are finite, also when the std is returned and unused."""
  return _moments('get_note_moments', x, note_mask, False, return_std)


@core.on_operands_device
def pool_over_notes(x, note_mask, return_std=True):
  """nn.pool_over_notes (nn.py:523-547): each frame's note mean and std spread back over
  the frames, [batch, time, dims]: sum_n m_tn mean_nd and sum_n m_tn std_nd.  The mean
  only when return_std is false.  Arguments, errors and the NaN convention of
  get_note_moments."""
  return _moments('pool_over_notes', x, note_mask, True, return_std)


def get_short_note_loss_mask(note_mask, note_lengths, note_pitches, min_length=40):
  """nn.get_short_note_loss_mask (nn.py:550-557): per frame [batch, time], the sum of the
  mask over the notes shorter than min_length with a pitch above 0."""
  note_mask = core._as_f32(note_mask)
  short = ((core._as_f32(note_lengths).to(note_mask.device) < min_length) &
           (core._as_f32(note_pitches).to(note_mask.device) > 0.0))
  return torch.sum(note_mask * short.to(torch.float32)[:, None, :], dim=-1)
