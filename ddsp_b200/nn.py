"""The layers of `ddsp/training/nn.py` that decoders.RnnFcDecoder builds from (Fc,
FcStack, Rnn, split_to_dict), the ResNet and RnnSandwich of the inverse-synthesis
encoders (Conv2D, MaxPool2D, NormReluConv, ResidualLayer, ResidualStack, ResNet), the
MIDI autoencoders' DilatedConvStack with ConditionalNorm, FcStackOut and get_embedding, and
its masking functions (nn.py:359-557): note
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
CUDA kernels of `csrc/gru.cuh` (DESIGN.md section 3.32).  The ResNet's convolutions are
torch ops (cuDNN) on channels-last views, with TensorFlow's 'same' padding; every one of
its Normalize -> ReLU pairs runs on the fused kernel of `csrc/norm.cuh` (normalize_relu,
DESIGN.md section 3.34), and every residual site of DilatedConvStack on the same header's
norm_residual kernel (DESIGN.md section 3.35).

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


_N_GROUPS = {'layer': lambda channels: 1, 'group': lambda channels: 32,
             'instance': lambda channels: channels}


def normalize_relu(x, scale, shift, norm_type='layer'):
  """relu(normalize_op(x, norm_type) * scale + shift) for x [B, H, W, C] (a CUDA tensor)
  and scale, shift of C elements ([1, 1, 1, C] as Normalize holds them), on the fused
  kernel of csrc/norm.cuh: one launch forward, two backward, with gradients to x, scale
  and shift.  Only each (item, group)'s mean and rstd are saved besides x.

  The numerics are normalize_op's (eps 1e-5, population variance); the gradient at a
  ReLU input of exactly 0 is 0.  An unknown norm_type raises KeyError and a channel
  count that the groups do not divide ValueError, as normalize_op does; channel counts
  the kernel does not take (ddsp_b200_norm_relu_takes: C a multiple of 4 up to 2048)
  raise NotImplementedError.  A CPU tensor raises ValueError: there is no CPU path."""
  if not torch.is_tensor(x) or x.dim() != 4:
    raise ValueError('normalize_relu: expected x [batch, height, width, channels], got '
                     f'{tuple(x.shape) if torch.is_tensor(x) else type(x).__name__}')
  if not x.is_cuda:
    raise ValueError(f'normalize_relu: x is on {x.device}; the kernel runs on CUDA '
                     'devices only')
  b, h, w, c = (int(v) for v in x.shape)
  groups = _N_GROUPS[norm_type](c)
  if c % groups:
    raise ValueError(f'normalize_relu: norm_type={norm_type!r} splits the channels into '
                     f'{groups} groups; {c} channels do not divide evenly')
  if not _lib.load().ddsp_b200_norm_relu_takes(c, groups):
    raise NotImplementedError(f'normalize_relu: {c} channels in {groups} groups; the '
                              'kernel takes multiples of 4 from 4 to 2048')
  if scale.numel() != c or shift.numel() != c:
    raise ValueError(f'normalize_relu: scale and shift need {c} elements, got '
                     f'{scale.numel()} and {shift.numel()}')
  if scale.device != x.device or shift.device != x.device:
    raise ValueError(f'normalize_relu: x is on {x.device}, scale on {scale.device} and '
                     f'shift on {shift.device}')
  x = x.to(torch.float32).contiguous()
  if x.data_ptr() % 16:   # the kernel reads rows of four channels
    x = x.clone()
  return autograd.NormReluFn.apply(x, scale.to(torch.float32).reshape(c).contiguous(),
                                   shift.to(torch.float32).reshape(c).contiguous(), groups)


class NormRelu(Normalize):
  """A Normalize layer (`scale` and `shift`, [1, 1, 1, C]) whose output goes through a
  ReLU, both on the fused normalize_relu: the Normalize -> ReLU pair of every ResNet
  site, with the parameters the reference's Normalize holds there."""

  def __init__(self, norm_type='layer'):
    super().__init__(norm_type)
    self._name = 'NormRelu'

  def forward(self, x):
    if not torch.is_tensor(x) or x.dim() not in (2, 3, 4):
      raise ValueError('NormRelu: expected x of rank 2, 3 or 4, got '
                       f'{tuple(x.shape) if torch.is_tensor(x) else type(x).__name__}')
    n_dims = x.dim()
    x = ensure_4d(x)
    self._built(x)
    return inv_ensure_4d(normalize_relu(x, self.scale, self.shift, self.norm_type), n_dims)


def norm_residual(y, x, norm_type=None, scale=None, shift=None, film=None,
                  shift_only=False, relu=True):
  """One residual site of DilatedConvStack on the fused kernel of csrc/norm.cuh:
  x_next = x + normalize_op(y, norm_type) s + h, and r = relu(x_next), the next layer's
  convolution input.  Returns (x_next, r), or x_next alone with relu=False (the stack's
  last layer).  y and x are [B, T, C] CUDA tensors.

  s and h are Normalize's scale and shift (C elements each), or, with film, read in place
  from the FiLM Dense output film [B, T, ld] of ConditionalNorm: scale in columns
  [0, C) and shift in [C, 2C), or the shift alone in [0, C) with shift_only (s = 1).
  One launch forward; the backward gives y, x and the parameters or film their
  gradients (ReLU gradient 0 at exactly 0).  The numerics are normalize_op's (eps 1e-5,
  population variance); norm_type None normalizes nothing.  An unknown norm_type raises
  KeyError and channels the groups do not divide ValueError, as normalize_op does;
  channel counts the kernel does not take (multiples of 4 up to 2048) raise
  NotImplementedError.  A CPU tensor raises ValueError: there is no CPU path."""
  for name, t in (('y', y), ('x', x)):
    if not torch.is_tensor(t) or t.dim() != 3:
      raise ValueError(f'norm_residual: expected {name} [batch, time, channels], got '
                       f'{tuple(t.shape) if torch.is_tensor(t) else type(t).__name__}')
  if y.shape != x.shape:
    raise ValueError(f'norm_residual: y {tuple(y.shape)} and x {tuple(x.shape)} differ')
  if not y.is_cuda:
    raise ValueError(f'norm_residual: y is on {y.device}; the kernel runs on CUDA devices '
                     'only')
  b, t, c = (int(v) for v in y.shape)
  groups = 0 if norm_type is None else _N_GROUPS[norm_type](c)
  if groups and c % groups:
    raise ValueError(f'norm_residual: norm_type={norm_type!r} splits the channels into '
                     f'{groups} groups; {c} channels do not divide evenly')
  if not _lib.load().ddsp_b200_norm_residual_takes(c, groups):
    raise NotImplementedError(f'norm_residual: {c} channels in {groups} groups; the '
                              'kernel takes multiples of 4 from 4 to 2048')
  params = [film] if film is not None else [scale, shift]
  if any(p is None for p in params) or (film is not None and (scale, shift) != (None, None)):
    raise ValueError('norm_residual: give scale and shift, or film alone')
  if any(p.device != y.device for p in params + [x]):
    raise ValueError(f'norm_residual: y is on {y.device}, and x or the parameters are not')

  def rows(v):
    v = v.to(torch.float32).contiguous()
    return v.clone() if v.data_ptr() % 16 else v   # the kernel reads rows of four channels

  if film is not None:
    width = c if shift_only else 2 * c
    if film.dim() != 3 or tuple(film.shape[:2]) != (b, t) or film.shape[-1] != width:
      raise ValueError(f'norm_residual: film must be [{b}, {t}, {width}], got '
                       f'{tuple(film.shape)}')
    return autograd.NormResidualFn.apply(rows(y), rows(x), None, None, rows(film), groups,
                                         bool(shift_only), bool(relu))
  if scale.numel() != c or shift.numel() != c:
    raise ValueError(f'norm_residual: scale and shift need {c} elements, got '
                     f'{scale.numel()} and {shift.numel()}')
  return autograd.NormResidualFn.apply(
      rows(y), rows(x), scale.to(torch.float32).reshape(c).contiguous(),
      shift.to(torch.float32).reshape(c).contiguous(), None, groups, False, bool(relu))


# ------------------ Convolutions -------------------------------------------------
def same_padding(size, kernel, stride):
  """TensorFlow's 'same' padding of one axis of `size` for a window of `kernel` at
  `stride`: (before, after).  The output has ceil(size / stride) elements; the padding
  is max((out - 1) stride + kernel - size, 0), with the odd element after."""
  out = -(-int(size) // int(stride))
  total = max((out - 1) * int(stride) + int(kernel) - int(size), 0)
  return total // 2, total - total // 2


def _pair(v):
  return (int(v), int(v)) if isinstance(v, int) else tuple(int(u) for u in v)


def _check_nhwc(x, name):
  if not torch.is_tensor(x) or x.dim() != 4:
    raise ValueError(f'{name}: expected x [batch, height, width, channels], got '
                     f'{tuple(x.shape) if torch.is_tensor(x) else type(x).__name__}')


class Conv2D(_Lazy):
  """tf.keras.layers.Conv2D(filters, kernel_size, strides, padding='same', dilation_rate,
  kernel_initializer) on NHWC x: `kernel` [kh, kw, in, filters], glorot-uniform (fans
  kh kw in and kh kw filters) or 'orthogonal' (Keras's: the kernel as a
  [kh kw in, filters] matrix with orthonormal columns or rows, gain 1), and `bias`
  [filters] zeros.  Runs as torch's conv2d (cuDNN) on x's channels-last NCHW view with
  the kernel viewed as OIHW, so neither is copied to another layout; the output is
  contiguous NHWC.  'same' padding is TensorFlow's for the dilated extent (k - 1) d + 1;
  its symmetric part goes to the convolution and the odd element after (stride 2, or an
  even dilated extent) is padded explicitly.  Keras refuses strides and dilations both
  above 1, and so does this layer (ValueError)."""

  def __init__(self, filters, kernel_size, strides=(1, 1), padding='same',
               dilation_rate=(1, 1), kernel_initializer='glorot_uniform'):
    super().__init__('Conv2D')
    if padding != 'same':
      raise NotImplementedError(f"Conv2D: padding={padding!r}; only 'same' is supported")
    if kernel_initializer not in ('glorot_uniform', 'orthogonal'):
      raise NotImplementedError(f'Conv2D: kernel_initializer={kernel_initializer!r}; only '
                                "'glorot_uniform' and 'orthogonal' are supported")
    self.filters = int(filters)
    self.kernel_size = _pair(kernel_size)
    self.strides = _pair(strides)
    self.dilation_rate = _pair(dilation_rate)
    self.kernel_initializer = kernel_initializer
    if max(self.strides) > 1 and max(self.dilation_rate) > 1:
      raise ValueError(f'Conv2D: strides {self.strides} and dilation_rate '
                       f'{self.dilation_rate} cannot both exceed 1')

  def build(self, width, device):
    kh, kw = self.kernel_size
    kernel = torch.zeros((kh, kw, width, self.filters), device=device)
    if self.kernel_initializer == 'orthogonal':
      kernel = torch.nn.init.orthogonal_(kernel.view(kh * kw * width, self.filters)).view(
          kernel.shape)
    else:
      limit = math.sqrt(6.0 / (kh * kw * width + kh * kw * self.filters))
      torch.nn.init.uniform_(kernel, -limit, limit)
    self.kernel = torch.nn.Parameter(kernel)
    self.bias = torch.nn.Parameter(torch.zeros(self.filters, device=device))

  def forward(self, x):
    _check_nhwc(x, 'Conv2D')
    self._built(x)
    (kh, kw), (sh, sw), (dh, dw) = self.kernel_size, self.strides, self.dilation_rate
    top, bottom = same_padding(x.shape[1], (kh - 1) * dh + 1, sh)
    left, right = same_padding(x.shape[2], (kw - 1) * dw + 1, sw)
    ph, pw = min(top, bottom), min(left, right)
    if (top, bottom, left, right) != (ph, ph, pw, pw):
      x = torch.nn.functional.pad(x, (0, 0, left - pw, right - pw, top - ph, bottom - ph))
    y = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2), self.kernel.permute(3, 2, 0, 1),
                                   self.bias, self.strides, (ph, pw), self.dilation_rate)
    return y.permute(0, 2, 3, 1).contiguous()


class MaxPool2D(torch.nn.Module):
  """tf.keras.layers.MaxPool2D(pool_size, strides, padding='same') on NHWC x: the
  'same' padding is -inf, so padded positions never win."""

  def __init__(self, pool_size=(2, 2), strides=None, padding='same'):
    super().__init__()
    if padding != 'same':
      raise NotImplementedError(f"MaxPool2D: padding={padding!r}; only 'same' is "
                                'supported')
    self.pool_size = _pair(pool_size)
    self.strides = _pair(strides if strides is not None else pool_size)

  def forward(self, x):
    _check_nhwc(x, 'MaxPool2D')
    (kh, kw), (sh, sw) = self.pool_size, self.strides
    top, bottom = same_padding(x.shape[1], kh, sh)
    left, right = same_padding(x.shape[2], kw, sw)
    if top or bottom or left or right:
      x = torch.nn.functional.pad(x, (0, 0, left, right, top, bottom), value=-math.inf)
    y = torch.nn.functional.max_pool2d(x.permute(0, 3, 1, 2), self.pool_size, self.strides)
    return y.permute(0, 2, 3, 1).contiguous()


# ------------------ ResNet ------------------------------------------------------
def _unconditional(name, conditional):
  if conditional:
    raise NotImplementedError(f'{name}: conditional=True needs ConditionalNorm, which '
                              'this library does not have')


class NormReluConv(torch.nn.Module):
  """nn.NormReluConv (nn.py:699-709): Normalize -> ReLU (fused, `norm`) -> Conv2D(ch,
  (k, k), (1, s)) (`conv`)."""

  def __init__(self, ch, k, s, norm_type):
    super().__init__()
    self.norm = NormRelu(norm_type)
    self.conv = Conv2D(ch, (k, k), (1, s))

  def forward(self, x):
    return self.conv(self.norm(x))


class ResidualLayer(torch.nn.Module):
  """nn.ResidualLayer (nn.py:712-756): a bottleneck layer with 4 ch output channels,
  downsampling the frequency axis by `stride`.  norm_input -> ReLU (fused), then
  `bottleneck` (Conv2D(ch, 1x1), NormReluConv(ch, 3, stride), NormReluConv(4 ch, 1, 1))
  plus the shortcut: `conv_proj` (Conv2D(4 ch, 1x1, (1, stride))) of the normalized
  input when `shortcut`, else the input itself.  conditional=True raises
  NotImplementedError."""

  def __init__(self, ch, stride, shortcut, norm_type, conditional=False, shift_only=False):
    super().__init__()
    _unconditional('ResidualLayer', conditional)
    self.shortcut = bool(shortcut)
    self.conditional = False
    self.norm_input = NormRelu(norm_type)
    if self.shortcut:
      self.conv_proj = Conv2D(4 * ch, (1, 1), (1, stride))
    self.bottleneck = torch.nn.Sequential(
        Conv2D(ch, (1, 1), (1, 1)),
        NormReluConv(ch, 3, stride, norm_type),
        NormReluConv(4 * ch, 1, 1, norm_type))

  def forward(self, x):
    r = x
    x = self.norm_input(ensure_4d(x))
    r = self.conv_proj(x) if self.shortcut else r
    return self.bottleneck(x) + r


class ResidualStack(torch.nn.Module):
  """nn.ResidualStack (nn.py:759-802): for each (ch, n_layers, stride), a
  ResidualLayer with the shortcut and the stride, then n_layers - 1 without; then
  Normalize -> ReLU (fused, the last of `layers`).  nonlinearity 'relu' only (another
  raises NotImplementedError, as does conditional=True)."""

  def __init__(self, filters, block_sizes, strides, norm_type, conditional=False,
               shift_only=False, nonlinearity='relu'):
    super().__init__()
    _unconditional('ResidualStack', conditional)
    if nonlinearity != 'relu':
      raise NotImplementedError(f'ResidualStack: nonlinearity {nonlinearity!r}; only '
                                "'relu' is supported")
    self.conditional = False
    layers = []
    for ch, n_layers, stride in zip(filters, block_sizes, strides):
      layers.append(ResidualLayer(ch, stride, True, norm_type))
      for _ in range(1, n_layers):
        layers.append(ResidualLayer(ch, 1, False, norm_type))
    layers.append(NormRelu(norm_type))
    self.layers = torch.nn.ModuleList(layers)

  def forward(self, x):
    for layer in self.layers:
      x = layer(x)
    return x


class ResNet(torch.nn.Module):
  """nn.ResNet (nn.py:805-839) on x [B, T, F, channels]: Conv2D(64, 7x7, (1, 2)),
  MaxPool2D((1, 3), (1, 2)), ResidualStack([ch, 2 ch, 4 ch], blocks, [1, 2, 2]) and
  ResidualStack([8 ch], [3], [2]), with (ch, blocks) = (32, [2, 3, 4]) 'small',
  (32, [3, 4, 6]) 'medium' and (64, [3, 4, 6]) 'large' (another size raises KeyError,
  as the reference's lookup does).  The frequency axis shrinks by 16 and the output has
  32 ch channels: log-mel [B, 125, 229, 1] -> [B, 125, 8, 1024] at 'small'.
  conditional=True raises NotImplementedError."""

  def __init__(self, size='large', norm_type='layer', conditional=False, shift_only=False):
    super().__init__()
    _unconditional('ResNet', conditional)
    self.conditional = False
    size_dict = {
        'small': (32, [2, 3, 4]),
        'medium': (32, [3, 4, 6]),
        'large': (64, [3, 4, 6]),
    }
    ch, blocks = size_dict[size]
    self.layers = torch.nn.ModuleList([
        Conv2D(64, (7, 7), (1, 2)),
        MaxPool2D((1, 3), (1, 2)),
        ResidualStack([ch, 2 * ch, 4 * ch], blocks, [1, 2, 2], norm_type),
        ResidualStack([8 * ch], [3], [2], norm_type),
    ])

  def forward(self, x):
    for layer in self.layers:
      x = layer(x)
    return x


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


class RnnSandwich(torch.nn.Sequential):
  """nn.RnnSandwich (nn.py:919-934): FcStack(fc_stack_ch, fc_stack_layers) ->
  Rnn(rnn_ch, rnn_type) -> FcStack(fc_stack_ch, fc_stack_layers)."""

  def __init__(self, fc_stack_ch=256, fc_stack_layers=2, rnn_ch=512, rnn_type='gru'):
    super().__init__(FcStack(fc_stack_ch, fc_stack_layers), Rnn(rnn_ch, rnn_type),
                     FcStack(fc_stack_ch, fc_stack_layers))


# ------------------ Embeddings --------------------------------------------------
class Embedding(torch.nn.Module):
  """tf.keras.layers.Embedding(input_dim, output_dim): `embeddings` [input_dim,
  output_dim], uniform(-0.05, 0.05), created on the ids' device at the first call.  Ids
  of any shape (float ids are truncated to integers, as Keras casts them) give
  [*ids.shape, output_dim]; an id outside [0, input_dim) raises IndexError."""

  def __init__(self, input_dim, output_dim):
    super().__init__()
    self.input_dim = int(input_dim)
    self.output_dim = int(output_dim)
    self.embeddings = None

  def forward(self, ids):
    if not torch.is_tensor(ids):
      raise TypeError(f'Embedding: expected a torch tensor, got {type(ids).__name__}')
    if self.embeddings is None:
      self.embeddings = torch.nn.Parameter(torch.nn.init.uniform_(
          torch.zeros((self.input_dim, self.output_dim), device=ids.device), -0.05, 0.05))
    return torch.nn.functional.embedding(ids.to(torch.int64), self.embeddings)


def get_embedding(vocab_size=1024, n_dims=256):
  """nn.get_embedding (nn.py:1066-1071): a real-valued embedding of integer ids."""
  return Embedding(vocab_size, n_dims)


# ------------------ Conditional normalization -------------------------------------
class ConditionalScaleAndShift(torch.nn.Module):
  """nn.ConditionalScaleAndShift (nn.py:1075-1099): x * scale + shift with (scale,
  shift) = `dense`(z) split at x's channel count C, or x + `dense`(z) with shift_only.
  The Dense (2 C units, or C) is created at the first call, when C is known.  Torch ops;
  x and z broadcast as TensorFlow's would."""

  def __init__(self, shift_only=False):
    super().__init__()
    self.shift_only = bool(shift_only)
    self.x_ch = None
    self.dense = None

  def film(self, x_ch, z):
    """The Dense output for x of x_ch channels: [..., 2 x_ch], or [..., x_ch] with
    shift_only.  DilatedConvStack's fused sites read it in place."""
    if self.dense is None:
      self.x_ch = int(x_ch)
      self.dense = Dense(self.x_ch if self.shift_only else 2 * self.x_ch)
    elif int(x_ch) != self.x_ch:
      raise ValueError(f'ConditionalScaleAndShift: built for {self.x_ch} channels, called '
                       f'with {x_ch}')
    return self.dense(z)

  def forward(self, inputs):
    x, z = inputs
    out = self.film(int(x.shape[-1]), z)
    if self.shift_only:
      return x + out
    return x * out[..., :self.x_ch] + out[..., self.x_ch:]


class ConditionalNorm(torch.nn.Module):
  """nn.ConditionalNorm (nn.py:1102-1136): normalize_op(x, norm_type) then
  ConditionalScaleAndShift(shift_only) with z (`conditional_scale_and_shift`).  x is
  [B, H, W, C].  Torch ops; inside DilatedConvStack the Dense feeds the fused site
  instead."""

  def __init__(self, norm_type='instance', shift_only=False):
    super().__init__()
    self.norm_type = norm_type
    self.conditional_scale_and_shift = ConditionalScaleAndShift(shift_only=shift_only)

  def forward(self, inputs):
    x, z = inputs
    return self.conditional_scale_and_shift([normalize_op(x, self.norm_type), z])


# ------------------ Stacks ------------------------------------------------------
class DilatedConvStack(torch.nn.Module):
  """nn.DilatedConvStack (nn.py:1152-1323): `conv_in` (Conv2D(ch, (kernel_size, 1))),
  then stacks x layers_per_stack residual layers
    x <- x + norm(conv_i(relu(x)))
  with conv_i (`layers`) a Conv2D(ch, (kernel_size, 1)) of dilation dilation^j at depth j
  of its stack (or (-dilation)^(layers_per_stack - 1 - j) for a negative dilation) and
  norm (`norms`) Normalize(norm_type), or ConditionalNorm(norm_type, shift_only) on the
  conditioning z when conditional.  Kernels are orthogonal with ortho_init, else
  glorot-uniform.

  Takes x [B, T, C_in], or [x, z] when conditional, with z [B, T, C_z] or of one frame
  ([B, C_z] or [B, 1, C_z]), broadcast over time as TensorFlow broadcasts it.  Returns
  [B, T, ch].  The convolutions run on cuDNN (Conv2D) and every residual site on the fused
  kernel of csrc/norm.cuh (norm_residual), which also writes the ReLU the next
  convolution reads; a conditional site reads its ConditionalNorm's Dense output in
  place.  The first ReLU, of conv_in's output, is a torch op.  CUDA tensors only
  (ValueError otherwise).  The kernel takes ch a multiple of 4 from 4 to 2048, which
  the reference does not require: another ch raises NotImplementedError at construction
  ('group' norm also needs ch a multiple of 32, ValueError).  Resampling (resample_type
  other than None, or a resample_stride other than 1) and spectral_norm=True raise
  NotImplementedError."""

  def __init__(self, ch=256, layers_per_stack=5, stacks=2, kernel_size=3, dilation=2,
               norm_type=None, resample_type=None, resample_stride=1,
               stacks_per_resample=1, resample_after_convolve=True, spectral_norm=False,
               ortho_init=False, shift_only=False, conditional=False):
    super().__init__()
    if resample_type is not None or resample_stride != 1:
      raise NotImplementedError(f'DilatedConvStack: resample_type={resample_type!r}, '
                                f'resample_stride={resample_stride}; resampling inside the '
                                'stack is not supported')
    if spectral_norm:
      raise NotImplementedError('DilatedConvStack: spectral_norm=True '
                                '(SpectralNormalization) is not supported')
    groups = 0 if norm_type is None else _N_GROUPS[norm_type](ch)   # KeyError if unknown
    if groups and ch % groups:
      raise ValueError(f'DilatedConvStack: norm_type={norm_type!r} splits the channels into '
                       f'{groups} groups; ch={ch} does not divide evenly')
    if not _lib.load().ddsp_b200_norm_residual_takes(ch, groups):
      raise NotImplementedError(f'DilatedConvStack: ch={ch}; the residual-site kernel takes '
                                'multiples of 4 from 4 to 2048')
    self.conditional = bool(conditional)
    self.norm_type = norm_type
    self.shift_only = bool(shift_only)
    self.resample_after_convolve = resample_after_convolve
    init = 'orthogonal' if ortho_init else 'glorot_uniform'

    def conv(dilation_rate=1):
      return Conv2D(ch, (kernel_size, 1), (1, 1), dilation_rate=(dilation_rate, 1),
                    kernel_initializer=init)

    def rate(i):
      if dilation > 0:
        return int(dilation**i)
      return int((-dilation)**(layers_per_stack - i - 1))

    self.conv_in = conv()
    self.layers = torch.nn.ModuleList(
        [conv(rate(j)) for _ in range(stacks) for j in range(layers_per_stack)])
    self.norms = torch.nn.ModuleList([
        ConditionalNorm(norm_type, shift_only) if self.conditional else Normalize(norm_type)
        for _ in range(stacks * layers_per_stack)])

  def forward(self, inputs):
    if self.conditional:
      x, z = inputs
    else:
      x, z = inputs, None
    if not torch.is_tensor(x) or x.dim() != 3:
      raise ValueError('DilatedConvStack: expected x [batch, time, channels], got '
                       f'{tuple(x.shape) if torch.is_tensor(x) else type(x).__name__}')
    x = self.conv_in(ensure_4d(x))[:, :, 0, :]
    b, t, ch = (int(v) for v in x.shape)
    r = torch.relu(x)
    if z is not None:
      if z.dim() == 2:
        z = z[:, None, :]
      if z.dim() != 3 or int(z.shape[0]) != b or int(z.shape[1]) not in (1, t):
        raise ValueError(f'DilatedConvStack: z {tuple(z.shape)} does not broadcast to '
                         f'[{b}, {t}, channels]')
    n = len(self.layers)
    for i, (layer, norm) in enumerate(zip(self.layers, self.norms)):
      y = layer(r[:, :, None, :])[:, :, 0, :]
      relu = i < n - 1
      if self.conditional:
        film = norm.conditional_scale_and_shift.film(ch, z)
        if int(film.shape[1]) != t:
          film = film.expand(b, t, int(film.shape[-1]))
        out = norm_residual(y, x, self.norm_type, film=film, shift_only=self.shift_only,
                            relu=relu)
      else:
        norm._built(y)
        out = norm_residual(y, x, self.norm_type, norm.scale, norm.shift, relu=relu)
      x, r = out if relu else (out, None)
    return x


class FcStackOut(torch.nn.Module):
  """nn.FcStackOut (nn.py:1326-1337): FcStack(ch, layers) (`stack`) then Dense(n_out)
  (`dense_out`)."""

  def __init__(self, ch, layers, n_out):
    super().__init__()
    self.stack = FcStack(ch, layers)
    self.dense_out = Dense(n_out)

  def forward(self, x):
    return self.dense_out(self.stack(x))
