"""The layers of `ddsp/training/nn.py` that decoders.RnnFcDecoder builds from (Fc,
FcStack, Rnn, split_to_dict), and its masking functions (nn.py:359-557): note
segmentation, per-note moments and pooling over notes, as the MIDI autoencoder uses them
(`models/midi_autoencoder.py`: `add_slowness_loss` and `ZMidiAutoencoder.z_note_encode`).
Same names, arguments and defaults as the reference.

The layers are torch modules with Keras semantics: parameters keep the Keras names,
layouts and initialisers (Dense `kernel` [in, out] glorot-uniform and `bias` zeros,
LayerNormalization `gamma` ones and `beta` zeros, GRU `kernel` [in, 3H] glorot-uniform,
`recurrent_kernel` [H, 3H] orthogonal and `bias` [2, 3H] zeros), so a reference
checkpoint's arrays assign one to one.  As Keras builds a layer at its first call, the
input width is fixed then and the parameters are created on the input's device.
Dense and LayerNormalization are torch ops (cuBLAS); the GRU's recurrence runs on the
CUDA kernels of `csrc/gru.cuh` (DESIGN.md section 3.32).

get_note_mask, get_note_mask_from_onset, get_note_moments and pool_over_notes run on the
CUDA kernels of `csrc/notes.cuh` (DESIGN.md section 3.25), which never build the
reference's [batch, time, notes, dims] products.  get_note_lengths,
get_short_note_loss_mask and straight_through_int_quantization are small torch
reductions and elementwise ops.
"""
import math

import torch

from ddsp_b200 import _lib
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


# ------------------ Utilities ---------------------------------------------------
def split_to_dict(tensor, tensor_splits):
  """nn.split_to_dict (nn.py:324-329): the last axis of tensor cut into
  {label: [..., size]} for the (label, size) pairs of tensor_splits, in order.  The sizes
  must add up to the axis (ValueError otherwise, as tf.split raises)."""
  labels = [v[0] for v in tensor_splits]
  sizes = [int(v[1]) for v in tensor_splits]
  if sum(sizes) != tensor.shape[-1]:
    raise ValueError(f'split_to_dict: sizes {sizes} add up to {sum(sizes)}, but the last '
                     f'axis of the tensor has {tensor.shape[-1]}')
  return dict(zip(labels, torch.split(tensor, sizes, dim=-1)))


# ------------------ Shapes ------------------------------------------------------
def ensure_4d(x):
  """nn.ensure_4d (nn.py:302-309): [B, C] -> [B, 1, 1, C] and [B, T, C] -> [B, T, 1, C];
  any other rank is returned as it is."""
  if x.dim() == 2:
    return x[:, None, None, :]
  if x.dim() == 3:
    return x[:, :, None, :]
  return x


def inv_ensure_4d(x, n_dims):
  """nn.inv_ensure_4d (nn.py:312-319): the inverse of ensure_4d for an input of rank
  n_dims."""
  if n_dims == 2:
    return x[:, 0, 0, :]
  if n_dims == 3:
    return x[:, :, 0, :]
  return x


# ------------------ Normalization -----------------------------------------------
def normalize_op(x, norm_type='layer', eps=1e-5):
  """nn.normalize_op (nn.py:561-575): group, instance or layer normalization of x
  [B, H, W, C], or x itself for norm_type None.  The C channels form
  {'instance': C, 'layer': 1, 'group': 32}[norm_type] groups (KeyError for any other
  name); each item's group is normalized over H, W and its channels by its mean and
  population variance, (x - mean) / sqrt(var + eps).  'group' needs C to be a multiple
  of 32 (ValueError otherwise, where TensorFlow fails in its reshape).  Torch ops,
  differentiable, on any device."""
  if norm_type is None:
    return x
  if x.dim() != 4:
    raise ValueError(f'normalize_op: expected x [batch, height, width, channels], got '
                     f'shape {tuple(x.shape)}')
  shape = x.shape
  channels = int(shape[-1])
  n_groups = {'instance': channels, 'layer': 1, 'group': 32}[norm_type]
  if channels % n_groups:
    raise ValueError(f'normalize_op: norm_type={norm_type!r} splits the channels into '
                     f'{n_groups} groups; {channels} channels do not divide evenly')
  x = x.reshape(*shape[:-1], n_groups, channels // n_groups)
  var, mean = torch.var_mean(x, dim=(1, 2, 4), correction=0, keepdim=True)
  return ((x - mean) / torch.sqrt(var + eps)).reshape(shape)


def _leaky_relu(x):
  """get_nonlinearity('leaky_relu') (nn.py:332-339): tf.nn.leaky_relu, slope 0.2."""
  return torch.nn.functional.leaky_relu(x, 0.2)


def _glorot_uniform(shape, device):
  """tf.keras.initializers.GlorotUniform for a [fan_in, fan_out] kernel."""
  limit = math.sqrt(6.0 / (shape[0] + shape[1]))
  return torch.nn.init.uniform_(torch.zeros(shape, device=device), -limit, limit)


def _width(x, name):
  if not torch.is_tensor(x):
    raise TypeError(f'{name}: expected a torch tensor, got {type(x).__name__}')
  if x.dim() < 2:
    raise ValueError(f'{name}: expected [..., features], got shape {tuple(x.shape)}')
  return int(x.shape[-1])


class _Lazy(torch.nn.Module):
  """A layer whose parameters are created at its first call (Keras build): the input
  width is fixed then, and a later call with another width raises ValueError."""

  def __init__(self, name):
    super().__init__()
    self._name = name
    self.input_width = None

  def _built(self, x):
    width = _width(x, self._name)
    if self.input_width is None:
      self.input_width = width
      self.build(width, x.device)
    elif width != self.input_width:
      raise ValueError(f'{self._name}: built for inputs of width {self.input_width}, '
                       f'called with width {width}')


class Dense(_Lazy):
  """tf.keras.layers.Dense(units) without activation: x kernel + bias."""

  def __init__(self, units):
    super().__init__('Dense')
    self.units = int(units)

  def build(self, width, device):
    self.kernel = torch.nn.Parameter(_glorot_uniform((width, self.units), device))
    self.bias = torch.nn.Parameter(torch.zeros(self.units, device=device))

  def forward(self, x):
    self._built(x)
    return torch.matmul(x, self.kernel) + self.bias


class LayerNormalization(_Lazy):
  """tf.keras.layers.LayerNormalization() over the last axis: epsilon 1e-3, gamma ones,
  beta zeros."""

  def __init__(self, epsilon=1e-3):
    super().__init__('LayerNormalization')
    self.epsilon = float(epsilon)

  def build(self, width, device):
    self.gamma = torch.nn.Parameter(torch.ones(width, device=device))
    self.beta = torch.nn.Parameter(torch.zeros(width, device=device))

  def forward(self, x):
    self._built(x)
    return torch.nn.functional.layer_norm(x, (self.input_width,), self.gamma, self.beta,
                                          self.epsilon)


class Normalize(_Lazy):
  """nn.Normalize (nn.py:578-603): normalize_op(x, norm_type) with epsilon 1e-5, then a
  learned per-channel `scale` (ones) and `shift` (zeros), both [1, 1, 1, C].  x is
  [B, C], [B, T, C] or [B, H, W, C] (made 4-D by ensure_4d) and the result has x's
  rank."""

  def __init__(self, norm_type='layer'):
    super().__init__('Normalize')
    self.norm_type = norm_type

  def build(self, width, device):
    self.scale = torch.nn.Parameter(torch.ones((1, 1, 1, width), device=device))
    self.shift = torch.nn.Parameter(torch.zeros((1, 1, 1, width), device=device))

  def forward(self, x):
    if not torch.is_tensor(x) or x.dim() not in (2, 3, 4):
      raise ValueError('Normalize: expected x of rank 2, 3 or 4, got '
                       f'{tuple(x.shape) if torch.is_tensor(x) else type(x).__name__}')
    n_dims = x.dim()
    x = normalize_op(ensure_4d(x), self.norm_type)
    self._built(x)
    return inv_ensure_4d(x * self.scale + self.shift, n_dims)


class Fc(torch.nn.Sequential):
  """nn.Fc (nn.py:843-852): Dense(ch) -> LayerNormalization -> leaky ReLU."""

  def __init__(self, ch=128, nonlinearity='leaky_relu'):
    if nonlinearity != 'leaky_relu':
      raise NotImplementedError(f'Fc: nonlinearity {nonlinearity!r}; only '
                                "'leaky_relu' is supported")
    super().__init__(Dense(ch), LayerNormalization())

  def forward(self, x):
    return _leaky_relu(super().forward(x))


class FcStack(torch.nn.Sequential):
  """nn.FcStack (nn.py:855-862): `layers` Fc(ch) layers."""

  def __init__(self, ch=256, layers=2, nonlinearity='leaky_relu'):
    super().__init__(*[Fc(ch, nonlinearity) for _ in range(layers)])


class Gru(_Lazy):
  """tf.keras.layers.GRU(units, return_sequences) with TF2's defaults: reset_after=True,
  gate columns z | r | h, h0 = 0.  x [B, T, in] (float32 CUDA) -> [B, T, units], or the
  last state [B, units] without return_sequences.  units must be a multiple of 32 from 32
  to 512 (NotImplementedError at construction otherwise).  One handle per device
  holds the packed recurrent weights; it is created at the first call on that device
  and freed with the layer.  copy.deepcopy and pickling (torch.save) leave the handles
  behind, so a copy never shares or frees the original's."""

  def __init__(self, units, return_sequences=True):
    super().__init__('GRU')
    self.units = int(units)
    if not _lib.load().ddsp_b200_gru_takes(self.units):
      raise NotImplementedError(f'GRU: units={units}; the CUDA recurrence takes '
                                'multiples of 32 from 32 to 512')
    self.return_sequences = bool(return_sequences)
    self._handles = {}

  def __getstate__(self):
    """Copies and pickles leave the handles behind: they own device memory, and the copy
    creates its own at its first call on each device."""
    state = dict(super().__getstate__())
    state['_handles'] = {}
    return state

  def build(self, width, device):
    self.kernel = torch.nn.Parameter(_glorot_uniform((width, 3 * self.units), device))
    self.recurrent_kernel = torch.nn.Parameter(torch.nn.init.orthogonal_(
        torch.zeros((self.units, 3 * self.units), device=device)))
    self.bias = torch.nn.Parameter(torch.zeros((2, 3 * self.units), device=device))

  def forward(self, x):
    if not torch.is_tensor(x) or x.dim() != 3:
      raise ValueError('GRU: expected x [batch, time, features], got '
                       f'{tuple(x.shape) if torch.is_tensor(x) else type(x).__name__}')
    if not x.is_cuda:
      raise ValueError(f'GRU: x is on {x.device}; the recurrence runs on CUDA devices only')
    self._built(x)
    params = (self.kernel, self.recurrent_kernel, self.bias)
    if any(p.device != x.device for p in params):
      raise ValueError(f'GRU: x is on {x.device}, the parameters on {self.kernel.device}')
    handle = self._handles.get(x.device)
    if handle is None:
      handle = self._handles[x.device] = autograd.GruHandle(self.units, x.device)
    save = torch.is_grad_enabled() and any(t.requires_grad for t in (x,) + params)
    with torch.cuda.device(x.device):
      out = autograd.GruFn.apply(x.to(torch.float32).contiguous(),
                                 *[p.contiguous() for p in params], handle, save)
    return out if self.return_sequences else out[:, -1]


class Rnn(torch.nn.Module):
  """nn.Rnn (nn.py:866-879): one RNN layer, `dims` units.  rnn_type 'gru' only;
  'lstm' and bidir=True raise NotImplementedError."""

  def __init__(self, dims, rnn_type, return_sequences=True, bidir=False):
    super().__init__()
    if rnn_type not in ('gru', 'lstm'):
      raise KeyError(rnn_type)
    if rnn_type != 'gru' or bidir:
      raise NotImplementedError(
          f'Rnn: rnn_type={rnn_type!r}, bidir={bidir}; only the unidirectional '
          "rnn_type='gru' is supported")
    self.rnn = Gru(dims, return_sequences=return_sequences)

  def forward(self, x):
    return self.rnn(x)
