"""Host-side mirror of the hot-path functions of `ddsp/core.py`.

Same names, argument meaning and error behaviour as the reference (file:line
cited per function); the arithmetic happens in libddsp_b200.so (hand-written
sm_90a kernels) through the ctypes C ABI in `_lib.py`.  torch is plumbing:
device memory and streams.  There is no CPU fallback.
"""
import ctypes
import functools
import math
from collections import abc
from typing import Any, Dict, Optional, Sequence, Text

import numpy as np
import torch

from ddsp_b200 import _lib

AMP_METHODS = {'window': _lib.AMP_WINDOW, 'linear': _lib.AMP_LINEAR}
DB_RANGE = 80.0  # dB (core.py:27)


# ----------------------------------------------------------------------------
# Utility functions (core.py:30-129)
# ----------------------------------------------------------------------------
def _device():
  if not torch.cuda.is_available():
    raise RuntimeError(
        'ddsp_b200 needs a CUDA device (H100, sm_90a); there is no CPU '
        'fallback.')
  return torch.device('cuda', torch.cuda.current_device())


def torch_float32(x, device=None):
  """`tf_float32` (core.py:31-36): a contiguous float32 CUDA tensor."""
  if isinstance(x, torch.Tensor):
    if x.is_cuda and device is None:
      return x.to(torch.float32).contiguous()
    return x.to(device=device or _device(), dtype=torch.float32).contiguous()
  return torch.as_tensor(np.asarray(x, dtype=np.float32),
                         device=device or _device()).contiguous()


tf_float32 = torch_float32  # the reference's name for the same coercion


def make_iterable(x):
  """core.py:39-47."""
  if x is None:
    return []
  elif isinstance(x, (np.ndarray, torch.Tensor)):
    return [x]
  else:
    return x if isinstance(x, abc.Iterable) else [x]


def to_dict(x, keys):
  """core.py:50-61."""
  if isinstance(x, dict):
    return x
  else:
    x = make_iterable(x)
    if len(keys) != len(x):
      raise ValueError(f'Keys: {keys} must be the same length as {x}')
    return dict(zip(keys, x))


def nested_keys(nested_dict: Dict[Text, Any], delimiter: Text = '/',
                prefix: Text = '') -> Sequence[Text]:
  """core.py:78-102."""
  keys = []
  for k, v in nested_dict.items():
    key = k if not prefix else f'{prefix}{delimiter}{k}'
    if not isinstance(v, dict):
      keys.append(key)
    else:
      keys += nested_keys(v, prefix=key)
  return keys


def nested_lookup(nested_key: Text, nested_dict: Dict[Text, Any],
                  delimiter: Text = '/'):
  """core.py:105-129."""
  keys = nested_key.split(delimiter)
  value = nested_dict
  for key in keys:
    try:
      value = value[key]
    except KeyError:
      raise KeyError(f'Key \'{key}\' as a part of nested key \'{nested_key}\' '
                     'not found during nested dictionary lookup, out of '
                     f'available keys: {nested_keys(nested_dict)}')
  return value


def copy_if_tf_function(x):
  """core.copy_if_tf_function (core.py:64-75): returns x unchanged.  The reference
  copies x only inside a tf.function, so that a later change to a traced input cannot
  reach the function; torch always runs eagerly, where the reference returns x too."""
  return x


def leaf_key(nested_key: Text, delimiter: Text = '/'):
  """core.leaf_key (core.py:132-144): the last key of "key/key/key..."."""
  return nested_key.split(delimiter)[-1]


def map_shape(x):
  """core.map_shape (core.py:147-149): the shape of every tensor or array of a nested
  dict / list / tuple as a list of ints, in the same structure."""
  if isinstance(x, dict):
    return {k: map_shape(v) for k, v in x.items()}
  if isinstance(x, (list, tuple)):
    return type(x)(map_shape(v) for v in x)
  return [int(d) for d in _shape(x)]


def pad_axis(x, padding=(0, 0), axis=0, **pad_kwargs):
  """core.pad_axis (core.py:152-168): pads only `axis` of x by (before, after) with
  torch.nn.functional.pad.  tf.pad's keywords map to torch's: `mode` in any case
  ('CONSTANT' -> 'constant') and `constant_values` -> `value`."""
  x = x if torch.is_tensor(x) else _as_f32(x)
  if 'constant_values' in pad_kwargs:
    pad_kwargs['value'] = pad_kwargs.pop('constant_values')
  if 'mode' in pad_kwargs:
    pad_kwargs['mode'] = pad_kwargs['mode'].lower()
  n_end_dims = x.dim() - axis % x.dim() - 1
  return torch.nn.functional.pad(x, (0, 0) * n_end_dims + tuple(padding), **pad_kwargs)


def _shape(x):
  """Static shape of a tensor / array / nested list, without touching a GPU."""
  return tuple(x.shape) if hasattr(x, 'shape') else tuple(np.shape(x))


def _workspace(query, device, *shape):
  """The scratch space of one launch as the (buffer, bytes) pair its parameters take,
  for `_launch(..., *_workspace(...))`.  `query` is the name of the entry point's
  workspace query, called with `shape`, or the byte count itself where the header
  states it.  A launch that needs none gets (None, 0): NULL and 0."""
  nbytes = query if isinstance(query, int) else getattr(_lib.load(), query)(*shape)
  return (torch.empty((nbytes,), dtype=torch.uint8, device=device) if nbytes else None,
          nbytes)


def _launch(symbol, *args):
  """Calls the launching entry point `symbol` (its full C name) of the library with
  `args` and the current stream of the operands' device as its last argument, with
  that device current, and raises its status.  A tensor argument goes as its
  data_ptr() and must be a contiguous CUDA tensor, all of them on one device; None
  goes as NULL; anything else as it is.  Every check raises ValueError before the
  launch."""
  tensors, c_args = [], []
  for i, a in enumerate(args):
    if isinstance(a, torch.Tensor):
      if not a.is_contiguous():
        raise ValueError(f'{symbol}: argument {i} is not contiguous (shape '
                         f'{tuple(a.shape)}, strides {a.stride()}).')
      if not a.is_cuda:
        raise ValueError(f'{symbol}: argument {i} is on {a.device}, not a CUDA device.')
      tensors.append(a)
      a = a.data_ptr()
    c_args.append(0 if a is None else a)
  with _on_device_of(*tensors):
    _lib.check(getattr(_lib.load(), symbol)(
        *c_args, torch.cuda.current_stream().cuda_stream))


class _on_device_of:
  """Context: make the device of the operands current (so the launch goes to
  THAT device's current stream), after checking they all live on one device."""

  def __init__(self, *tensors):
    devs = {t.device for t in tensors if isinstance(t, torch.Tensor)}
    if len(devs) > 1:
      raise ValueError('ddsp_b200: operands live on different devices: %s'
                       % sorted(str(d) for d in devs))
    dev = devs.pop() if devs else _device()
    if dev.type != 'cuda':
      raise ValueError('ddsp_b200: operands must be CUDA tensors, got %s' % dev)
    self._ctx = torch.cuda.device(dev)

  def __enter__(self):
    return self._ctx.__enter__()

  def __exit__(self, *exc):
    return self._ctx.__exit__(*exc)


def _cuda_tensors(xs):
  for x in xs:
    if isinstance(x, torch.Tensor):
      if x.is_cuda:
        yield x
    elif isinstance(x, dict):
      yield from _cuda_tensors(x.values())
    elif isinstance(x, (list, tuple)):
      yield from _cuda_tensors(x)


def on_operands_device(fn):
  """Runs `fn` with the device of its CUDA tensor arguments current (those inside
  dicts, lists and tuples included), after checking that they share one device: its
  host arithmetic, allocations and launches then go to that device and its current
  stream, and operands on two devices raise ValueError before any device work.
  Without CUDA tensor arguments (numpy arrays, CPU tensors) it changes nothing."""
  @functools.wraps(fn)
  def wrapper(*args, **kwargs):
    tensors = list(_cuda_tensors(args)) + list(_cuda_tensors(kwargs.values()))
    if not tensors:
      return fn(*args, **kwargs)
    with _on_device_of(*tensors):
      return fn(*args, **kwargs)
  return wrapper


def _byte_range(t):
  """[first, last + 1) byte of the contiguous tensor t in its device memory."""
  return t.data_ptr(), t.data_ptr() + t.numel() * t.element_size()


def _overlaps(a, b):
  """Whether the contiguous tensors a and b share a byte of memory."""
  if a.numel() == 0 or b.numel() == 0 or a.device != b.device:
    return False
  a0, a1 = _byte_range(a)
  b0, b1 = _byte_range(b)
  return a0 < b1 and b0 < a1


def _check_out(out, shape, like, inputs=(), exact_alias_ok=False, name='out'):
  """`out=` of the synthesizers is written by a kernel: B*N contiguous floats.

  Returns `inputs` (tensors or None) with every one that overlaps `out` cloned, so
  that no kernel reads memory it is writing: `out=` never changes the result.  With
  exact_alias_ok the kernel is elementwise, and an input that IS `out` (same first
  byte and extent) is passed as it is.  Inputs the kernel reads only in launches
  before the one that writes `out` need not be passed.  Un-aliased calls copy
  nothing.  Under grad mode an `out` that requires grad is refused, as torch's own
  out= ops refuse it; call _wrote(out) after the write."""
  if (not isinstance(out, torch.Tensor) or not out.is_cuda or
      out.dtype != torch.float32 or not out.is_contiguous() or
      tuple(out.shape) != tuple(shape) or out.device != like.device):
    raise ValueError(
        f'{name} must be a contiguous float32 CUDA tensor of shape {tuple(shape)} '
        f'on {like.device}; got {type(out).__name__}'
        + (f' {tuple(out.shape)} {out.dtype} {out.device}' if isinstance(out, torch.Tensor) else ''))
  if torch.is_grad_enabled() and out.requires_grad:
    raise RuntimeError(
        f'ddsp_b200: functions with {name}= arguments do not support automatic '
        f'differentiation, but {name} requires grad.  Call without {name}= to get a '
        'differentiable result, or pass an output that does not require grad.')
  return [x.clone() if x is not None and _overlaps(x, out) and not (
      exact_alias_ok and _byte_range(x) == _byte_range(out)) else x for x in inputs]


def _wrote(out):
  """Records a kernel's write to `out` in its autograd version counter, so that a
  backward pass that saved `out` before the write raises instead of using the new
  values.  Returns out."""
  torch.autograd.graph.increment_version(out)
  return out


def _no_grad_path(name, *tensors):
  """Refuses to return detached audio.  The calls that end here record no autograd
  graph: the fused signal-only `ProcessorGroup` call (`decoder_forward`), the
  synthesizers writing through `out=` / `accumulate=`, and the shapes no backward
  kernel takes.  A training loop gets gradients from the Processor API
  (`group(features, return_outputs_dict=True)`, or `get_controls` + `get_signal`),
  whose `core.*` ops route to ddsp_b200.autograd under grad, or from
  `autograd.decoder_train`; silently returning detached audio would train nothing."""
  if torch.is_grad_enabled() and any(
      isinstance(t, torch.Tensor) and t.requires_grad for t in tensors):
    raise RuntimeError(
        f'ddsp_b200.core.{name}: an input requires grad, but this call is the '
        'inference path and returns detached audio.  Train through the Processor '
        'API - group(features, return_outputs_dict=True), or get_controls + '
        'get_signal - or ddsp_b200.autograd.decoder_train / HarmonicSynthesisFn / '
        'FilteredNoiseFn (CUDA backward kernels), or wrap the call in '
        'torch.no_grad().')


# ----------------------------------------------------------------------------
# Scaling (core.py:386-404) - used by callers that want the bare function; the
# processors call the fused controls kernels instead.
# ----------------------------------------------------------------------------
def exp_sigmoid(x, exponent=10.0, max_value=2.0, threshold=1e-7):
  """core.py:386-404.  Default arguments run the CUDA controls kernel."""
  x = torch_float32(x)
  if (exponent, max_value, threshold) == (10.0, 2.0, 1e-7) and not (
      torch.is_grad_enabled() and x.requires_grad):
    out = torch.empty_like(x)
    _launch('ddsp_b200_noise_controls', x, out, x.numel(), 0.0, 1)
    return out
  return max_value * torch.sigmoid(x)**float(np.log(exponent)) + threshold


def sym_exp_sigmoid(x, width=8.0):
  """core.sym_exp_sigmoid (core.py:407-411): exp_sigmoid(width * (|x| / 2 - 1)),
  symmetric about x = 0.  exp_sigmoid's CUDA kernel runs it outside grad."""
  x = torch_float32(x)
  return exp_sigmoid(width * (torch.abs(x) / 2.0 - 1.0))


# ----------------------------------------------------------------------------
# Frequency scaling of network outputs (core.py:207-348, 414-508) - frame-rate
# torch ops (a few thousand elements per item), device-agnostic.
# ----------------------------------------------------------------------------
def _as_f32(x):
  if torch.is_tensor(x):
    return x.to(torch.float32)
  return torch.as_tensor(np.asarray(x, dtype=np.float32))


def diff(x, axis=-1):
  """core.diff (core.py:171-198): the finite difference x[1:] - x[:-1] along `axis`,
  one shorter there.  ValueError for axis >= x.ndim."""
  x = x if torch.is_tensor(x) else _as_f32(x)
  ndim = x.dim()
  if axis >= ndim:
    raise ValueError('Invalid axis index: %d for tensor with only %d axes.' % (axis, ndim))
  n = x.shape[axis] - 1
  return x.narrow(axis, 1, n) - x.narrow(axis, 0, n)


def safe_log(x, eps=1e-5):
  """core.safe_log (core.py:213-216)."""
  x = _as_f32(x)
  return torch.log(torch.where(x <= 0.0, torch.full_like(x, eps), x))


def logb(x, base=2.0, eps=1e-5):
  """core.logb (core.py:219-221): safe_divide(safe_log(x), safe_log(base))."""
  den = safe_log(base, eps)
  den = torch.where(den == 0.0, torch.full_like(den, eps), den)
  return safe_log(x, eps) / den


def log10(x, eps=1e-5):
  """core.log10 (core.py:224-226)."""
  return logb(x, base=10, eps=eps)


# The math helpers and scalers below take a tensor as it is (float64 stays float64) and
# anything else as a float32 CPU tensor.
def nan_to_num(x, value=0.0):
  """core.nan_to_num (core.py:202-204): NaN -> value.  +-inf stay, unlike the
  defaults of torch.nan_to_num."""
  x = x if torch.is_tensor(x) else _as_f32(x)
  return torch.where(torch.isnan(x), torch.full_like(x, value), x)


def log_scale(x, min_x, max_x):
  """core.log_scale (core.py:229-233): [-1, 1] to [min_x, max_x], logarithmically."""
  x = x if torch.is_tensor(x) else _as_f32(x)
  x = (x + 1.0) / 2.0
  log_min, log_max = (torch.log(torch.as_tensor(v, dtype=x.dtype, device=x.device))
                      for v in (min_x, max_x))
  return torch.exp((1.0 - x) * log_min + x * log_max)


def soft_limit(x, x_min=0.0, x_max=1.0):
  """core.soft_limit (core.py:236-238): softly limits x to [x_min, x_max]."""
  x = x if torch.is_tensor(x) else _as_f32(x)
  softplus = torch.nn.functional.softplus
  return softplus(x) + x_min - softplus(x - (x_max - x_min))


def gradient_reversal(x):
  """core.gradient_reversal (core.py:241-243): the identity forward, -grad backward,
  as the reference writes it: stop_gradient(2 x) - x."""
  x = x if torch.is_tensor(x) else _as_f32(x)
  return (2.0 * x).detach() - x


def amplitude_to_db(amplitude, ref_db=0.0, range_db=DB_RANGE, use_tf=True):
  """core.amplitude_to_db (core.py:247-250): power_to_db(amplitude**2)."""
  return power_to_db(amplitude**2.0, ref_db=ref_db, range_db=range_db, use_tf=use_tf)


def power_to_db(power, ref_db=0.0, range_db=DB_RANGE, use_tf=True):
  """core.power_to_db (core.py:253-268): 10 log10(max(10^(-range_db / 10), power))
  - ref_db, floored at -range_db.  use_tf=True is torch with core.log10 (safe_log,
  float32) on the input's device; use_tf=False is NumPy with np.log10."""
  pmin = 10**-(range_db / 10.0)
  if not use_tf:
    db = 10.0 * np.log10(np.maximum(pmin, power))
    return np.maximum(db - ref_db, -range_db)
  db = 10.0 * log10(torch.clamp(_as_f32(power), min=pmin))
  return torch.clamp(db - ref_db, min=-range_db)


def db_to_amplitude(db):
  """core.db_to_amplitude (core.py:271-273)."""
  return db_to_power(db / 2.0)


def db_to_power(db):
  """core.db_to_power (core.py:276-278)."""
  return 10.0**(db / 10.0)


def midi_to_hz(notes, midi_zero_silence: bool = False):
  """core.midi_to_hz (core.py:280-297)."""
  notes = _as_f32(notes)
  hz = 440.0 * (2.0 ** ((notes - 69.0) / 12.0))
  if midi_zero_silence:
    hz = torch.where(notes == 0.0, torch.zeros_like(hz), hz)
  return hz


def hz_to_midi(frequencies):
  """core.hz_to_midi (core.py:300-306): 0 Hz maps to MIDI 0."""
  frequencies = _as_f32(frequencies)
  notes = 12.0 * (logb(frequencies, 2.0) - logb(440.0, 2.0)) + 69.0
  return torch.where(frequencies <= 0.0, torch.zeros_like(notes), notes)


def unit_to_midi(unit, midi_min=20.0, midi_max=90.0, clip: bool = False):
  """core.unit_to_midi (core.py:309-315)."""
  unit = _as_f32(unit)
  unit = torch.clamp(unit, 0.0, 1.0) if clip else unit
  return midi_min + (midi_max - midi_min) * unit


def midi_to_unit(midi, midi_min=20.0, midi_max=90.0, clip: bool = False):
  """core.midi_to_unit (core.py:318-324)."""
  unit = (_as_f32(midi) - midi_min) / (midi_max - midi_min)
  return torch.clamp(unit, 0.0, 1.0) if clip else unit


def unit_to_hz(unit, hz_min, hz_max, clip: bool = False):
  """core.unit_to_hz (core.py:327-336): logarithmic map of [0, 1]."""
  midi = unit_to_midi(unit, midi_min=hz_to_midi(hz_min), midi_max=hz_to_midi(hz_max),
                      clip=clip)
  return midi_to_hz(midi)


def hz_to_unit(hz, hz_min, hz_max, clip: bool = False):
  """core.hz_to_unit (core.py:339-348)."""
  return midi_to_unit(hz_to_midi(hz), midi_min=hz_to_midi(hz_min),
                      midi_max=hz_to_midi(hz_max), clip=clip)


# Perceptual scales (core.py:351-383): NumPy stays NumPy, as frequencies_critical_bands
# needs for its float64 band centres, and tensors stay tensors.
def hz_to_bark(hz):
  """core.hz_to_bark (core.py:351-353): Traunmüller (1990)."""
  return 26.81 / (1.0 + (1960.0 / hz)) - 0.53


def bark_to_hz(bark):
  """core.bark_to_hz (core.py:356-358): Traunmüller (1990)."""
  return 1960.0 / (26.81 / (bark + 0.53) - 1.0)


def hz_to_mel(hz):
  """core.hz_to_mel (core.py:361-363): HTK's 2595 log10(1 + hz / 700) with core.logb's
  safe log.  A tensor gives float32 through core.logb; NumPy and numbers give float64
  NumPy."""
  if torch.is_tensor(hz):
    return 2595.0 * logb(1.0 + hz / 700.0, 10.0)
  x = 1.0 + np.asarray(hz, np.float64) / 700.0
  return 2595.0 * (np.log(np.where(x <= 0.0, 1e-5, x)) / np.log(10.0))


def mel_to_hz(mel):
  """core.mel_to_hz (core.py:366-368): HTK."""
  return 700.0 * (10.0**(mel / 2595.0) - 1.0)


def hz_to_erb(hz):
  """core.hz_to_erb (core.py:371-383): the equivalent rectangular bandwidth in Hz,
  Moore & Glasberg (1996)."""
  return 0.108 * hz + 24.7


def _add_depth_axis(freqs, depth: int = 1):
  """core._add_depth_axis (core.py:414-420): [B, T, N*D] -> [B, T, N, D]."""
  b, t, combined = freqs.shape
  return freqs.reshape(b, t, int(combined) // depth, depth)


def frequencies_softmax(freqs, depth: int = 1, hz_min: float = 20.0,
                        hz_max: float = 8000.0):
  """core.frequencies_softmax (core.py:424-457)."""
  freqs = torch_float32(freqs, device=freqs.device if torch.is_tensor(freqs) else 'cpu')
  if freqs.dim() == 3:
    freqs = _add_depth_axis(freqs, depth)
  else:
    depth = int(freqs.shape[-1])
  f_probs = torch.softmax(freqs, dim=-1)
  unit_bins = torch.linspace(0.0, 1.0, depth, device=freqs.device)
  unit_bins = unit_bins[None, None, None, :]
  f_unit = torch.sum(unit_bins * f_probs, dim=-1)
  return unit_to_hz(f_unit, hz_min=hz_min, hz_max=hz_max)


def frequencies_sigmoid(freqs, depth: int = 1, hz_min: float = 0.0,
                        hz_max: float = 8000.0):
  """core.frequencies_sigmoid (core.py:460-507): a sum of `depth` sigmoids, each
  mapped logarithmically onto a slice of [hz_min, hz_max]."""
  freqs = torch_float32(freqs, device=freqs.device if torch.is_tensor(freqs) else 'cpu')
  if freqs.dim() == 3:
    freqs = _add_depth_axis(freqs, depth)
  else:
    depth = int(freqs.shape[-1])
  f_probs = torch.sigmoid(freqs)
  hz_scales = []
  hz_min_copy = hz_min
  remainder = hz_max - hz_min
  scale_factor = remainder**(1.0 / depth)
  for i in range(depth):
    if i == (depth - 1):
      hz_max = remainder
      hz_min = hz_min_copy
    else:
      hz_max = remainder * (1.0 - 1.0 / scale_factor)
      hz_min = 0
      remainder -= hz_max
    hz_scales.append(unit_to_hz(f_probs[..., i], hz_min=hz_min, hz_max=hz_max))
  return torch.sum(torch.stack(hz_scales, dim=-1), dim=-1)


def frequencies_critical_bands(freqs, depth=1, depth_scale=10.0, bandwidth_scale=1.0,
                               hz_min=20.0, hz_max=8000.0, scale='bark'):
  """core.frequencies_critical_bands (core.py:511-569): sinusoid k sits at the k-th of
  centres spaced evenly on the bark scale (any other `scale`: mel) over [hz_min, hz_max]
  and moves by up to bandwidth_scale ERBs of its centre: soft_limit(centre +
  bandwidth_scale * erb * sum_d tanh(freqs_d) depth_scale^-d, hz_min, hz_max).
  freqs [B, T, N * depth] or [B, T, N, depth] -> Hz [B, T, N].  The centres are float64
  NumPy, as in the reference, used as float32 on the input's device."""
  freqs = freqs if torch.is_tensor(freqs) else _as_f32(freqs)
  if freqs.dim() == 3:
    freqs = _add_depth_axis(freqs, depth)
  else:
    depth = int(freqs.shape[-1])
  n_sinusoids = freqs.shape[-2]
  if scale == 'bark':
    f_center = bark_to_hz(np.linspace(hz_to_bark(hz_min), hz_to_bark(hz_max), n_sinusoids))
  else:
    f_center = mel_to_hz(np.linspace(hz_to_mel(hz_min), hz_to_mel(hz_max), n_sinusoids))
  bw = torch.as_tensor(hz_to_erb(f_center), dtype=torch.float32, device=freqs.device)
  f_center = torch.as_tensor(f_center, dtype=torch.float32, device=freqs.device)
  depth_modifier = depth_scale**-torch.arange(depth, dtype=torch.float32, device=freqs.device)
  modifier = torch.sum(torch.tanh(freqs) * depth_modifier, dim=-1)
  return soft_limit(f_center + bandwidth_scale * bw * modifier, hz_min, hz_max)


# ----------------------------------------------------------------------------
# Resampling (core.py:573-714) - stand-alone ops (the synthesizers fuse them)
# ----------------------------------------------------------------------------
_RESAMPLE_METHODS = {'window': 0, 'linear': 1, 'nearest': 2, 'cubic': 3}


def _resample_3d(inputs, n_timesteps, method, add_endpoint):
  """[B, F, C] -> [B, N, C]; routes to `autograd.ResampleFn` when grad is enabled
  and the input requires it."""
  inputs = torch_float32(inputs)
  if torch.is_grad_enabled() and inputs.requires_grad:
    from ddsp_b200 import autograd as _ag
    return _ag.ResampleFn.apply(inputs, int(n_timesteps), method, bool(add_endpoint))
  return resample_forward(inputs, n_timesteps, method, add_endpoint)


def resample_forward(inputs, n_timesteps, method, add_endpoint):
  """The resample kernel on a [B, F, C] float32 CUDA tensor."""
  b, f, c = inputs.shape
  out = torch.empty((b, int(n_timesteps), c), dtype=torch.float32,
                    device=inputs.device)
  _launch('ddsp_b200_resample', inputs, out, b, f, c, int(n_timesteps),
          _RESAMPLE_METHODS[method], int(bool(add_endpoint)))
  return out


def upsample_with_windows(inputs, n_timesteps: int, add_endpoint: bool = True):
  """core.upsample_with_windows (core.py:645-714)."""
  _check_window_upsample(_shape(inputs), n_timesteps, add_endpoint)
  return _resample_3d(inputs, n_timesteps, 'window', add_endpoint)


def _check_window_upsample(shape, n_timesteps, add_endpoint):
  """The ValueErrors of core.upsample_with_windows (core.py:670-693)."""
  if len(shape) != 3:
    raise ValueError('Upsample_with_windows() only supports 3 dimensions, '
                     'not {}.'.format(list(shape)))
  n_frames = shape[1] + (1 if add_endpoint else 0)
  n_intervals = n_frames - 1
  if n_frames >= n_timesteps:
    raise ValueError('Upsample with windows cannot be used for downsampling'
                     'More input frames ({}) than output timesteps ({})'.format(
                         n_frames, n_timesteps))
  if n_intervals <= 0 or n_timesteps % n_intervals != 0.0:
    minus_one = '' if add_endpoint else ' - 1'
    raise ValueError(
        'For upsampling, the target the number of timesteps must be divisible '
        'by the number of input frames{}. (timesteps:{}, frames:{}, '
        'add_endpoint={}).'.format(minus_one, n_timesteps, n_frames, add_endpoint))


def resample(inputs, n_timesteps: int, method: Text = 'linear',
             add_endpoint: bool = True):
  """core.resample (core.py:573-642) for 1-D / 2-D / 3-D / 4-D inputs, methods
  'nearest', 'linear', 'cubic' (tf.compat.v1 image kernels) and 'window'."""
  shape = _shape(inputs)
  if method not in ('nearest', 'linear', 'cubic', 'window'):
    raise ValueError('Method ({}) is invalid. Must be one of {}.'.format(
        method, "['nearest', 'linear', 'cubic', 'window']"))
  if len(shape) not in (1, 2, 3, 4):
    raise ValueError(f'resample takes 1-D to 4-D inputs, got shape {list(shape)}.')
  x = torch_float32(inputs)
  if len(shape) == 1:
    x = x[None, :, None]
  elif len(shape) == 2:
    x = x[:, :, None]
  elif len(shape) == 4:
    if method == 'window':
      # upsample_with_windows only takes 3-D (core.py:670-672)
      raise ValueError('Upsample_with_windows() only supports 3 dimensions, '
                       'not {}.'.format(list(shape)))
    # core.py:616-621 resizes [n_frames, n_freq] to [n_timesteps, n_freq]: the
    # n_freq axis maps onto itself, so this is the 3-D case over n_freq*channels.
    x = x.reshape(shape[0], shape[1], shape[2] * shape[3])
  if method == 'window':
    out = upsample_with_windows(x, n_timesteps, add_endpoint)
  else:
    out = _resample_3d(x, n_timesteps, method, add_endpoint)
  if len(shape) == 1:
    out = out[0, :, 0]
  elif len(shape) == 2:
    out = out[:, :, 0]
  elif len(shape) == 4:
    out = out.reshape(shape[0], int(n_timesteps), shape[2], shape[3])
  return out


def center_crop(audio, frame_size):
  """core.center_crop (core.py:717-730): removes the frame_size // 2 samples that
  centred framing pads at each end of axis 1."""
  pad_amount = int(frame_size // 2)
  return audio[:, pad_amount:-pad_amount]


# ----------------------------------------------------------------------------
# Harmonic synthesis (core.py:1048-1111)
# ----------------------------------------------------------------------------
@on_operands_device
def harmonic_controls(amplitudes, harmonic_distribution, f0_hz, sample_rate,
                      scale=True, normalize_below_nyquist=True):
  """synths.Harmonic.get_controls arithmetic (synths.py:94-121): exp_sigmoid,
  core.normalize_harmonics (core.py:894-907).  Routes to
  `autograd.HarmonicControlsFn` when grad is enabled and the amplitudes or the
  distribution require it; f0_hz gets no gradient through the mask (tf.where)."""
  sa, sh, sf = _shape(amplitudes), _shape(harmonic_distribution), _shape(f0_hz)
  if len(sh) != 3 or len(sa) != 3 or len(sf) != 3:
    raise ValueError('Harmonic controls must be 3-D [batch, frames, channels]; '
                     f'got {sa}, {sh}, {sf}.')
  b, f, k = sh
  if sa != (b, f, 1) or sf != (b, f, 1):
    raise ValueError(
        f'amplitudes {sa} and f0_hz {sf} must be [{b}, {f}, 1] to match '
        f'harmonic_distribution {sh}.')
  amplitudes = torch_float32(amplitudes)
  hd = torch_float32(harmonic_distribution)
  f0_hz = torch_float32(f0_hz)
  if _requires_grad(amplitudes, hd):
    from ddsp_b200 import autograd as _ag
    return _ag.HarmonicControlsFn.apply(amplitudes, hd, f0_hz, float(sample_rate),
                                        bool(scale), bool(normalize_below_nyquist))
  amps_out = torch.empty_like(amplitudes)
  hd_out = torch.empty_like(hd)
  flags = ((_lib.CTL_SCALE if scale else 0) |
           (_lib.CTL_NYQUIST if normalize_below_nyquist else 0))
  _launch('ddsp_b200_harmonic_controls', amplitudes, hd, f0_hz, amps_out, hd_out, b, f, k,
          float(sample_rate), flags)
  return amps_out, hd_out


def note_mask(q, onset, max_regions, note_on_only):
  """The launch behind nn.get_note_mask (onset None) and nn.get_note_mask_from_onset:
  the float32 mask [B, T_out, max_regions] of the contiguous float32 CUDA pitches q
  [B, T] (and onsets [B, T]); T_out = T, or 2 for one frame under the edge rule."""
  b, t = q.shape
  t_out = t if onset is not None or t > 1 else 2
  mask = torch.empty((b, t_out, max_regions), dtype=torch.float32, device=q.device)
  flag = int(bool(note_on_only))
  # the edge rule's per-region decisions: a byte per region that can hold a frame
  nbytes = b * min(max_regions, t) if onset is None and flag else 0
  _launch('ddsp_b200_note_mask', q, onset, mask, *_workspace(nbytes, q.device),
          b, t, max_regions, flag)
  return mask


def note_heuristic(x, f0, on, status, stages, log_values, shift, pool_width, pool_pad,
                   positive, num_devs, widths, strided_pad, min_samples, glue_back):
  """The launch behind the binarizers of ddsp_b200.heuristics: (mask [B, T] bool, status
  [B] int32) of the contiguous [B, T] CUDA operands x (float32 amplitudes or power), f0
  (float32 Hz) and on (uint8), any of them None where the stages do not read it.  status
  may be a preallocated int32 [B]; nothing is synchronised."""
  like = next(v for v in (x, f0, on) if v is not None)
  b, t = like.shape
  mask = torch.empty((b, t), dtype=torch.bool, device=like.device)
  if status is None:
    status = torch.empty((b,), dtype=torch.int32, device=like.device)
  host_widths = (ctypes.c_int * max(1, len(widths)))(*widths)   # read before the launch
  _launch('ddsp_b200_note_heuristic', x, f0, on, mask, status,
          *_workspace('ddsp_b200_note_heuristic_workspace_bytes', like.device, b, t),
          b, t, stages, log_values, shift, pool_width, pool_pad, positive, num_devs,
          ctypes.addressof(host_widths), len(widths), strided_pad, min_samples, glue_back)
  return mask, status


def note_table_buffer(b, t, device):
  """One int32 buffer and its views (buffer, status [B], count [B], note records
  [B, (T+1)//2, 4]), so that a whole batch comes to the host in one copy; the records
  start 16-byte aligned."""
  cap = (t + 1) // 2
  head = (2 * b + 3) // 4 * 4
  buf = torch.empty((head + b * cap * 4,), dtype=torch.int32, device=device)
  return buf, buf[:b], buf[b:2 * b], buf[head:].view(b, cap, 4)


def note_segments(mask, f0, notes, count, median):
  """The launch behind heuristics.note_table: the records {start, stop, pitch, f0 bits}
  of the runs of nonzero bytes of mask [B, T] into notes [B, (T+1)//2, 4] and count [B]."""
  b, t = f0.shape
  _launch('ddsp_b200_note_segments', mask, f0, notes, count, b, t, int(bool(median)))


def safe_divide(numerator, denominator, eps=1e-7):
  """core.safe_divide (core.py:207-210)."""
  safe = torch.where(denominator == 0.0, torch.full_like(denominator, eps),
                     denominator)
  return numerator / safe


def get_harmonic_frequencies(frequencies, n_harmonics: int):
  """core.get_harmonic_frequencies (core.py:1028-1045): f0 * [1..K]."""
  frequencies = torch_float32(frequencies)
  ratios = torch.linspace(1.0, float(n_harmonics), int(n_harmonics),
                          device=frequencies.device)
  return frequencies * ratios[None, None, :]


@on_operands_device
def remove_above_nyquist(frequency_envelopes, amplitude_envelopes,
                         sample_rate: int = 16000):
  """core.remove_above_nyquist (core.py:869-891)."""
  frequency_envelopes = torch_float32(frequency_envelopes)
  amplitude_envelopes = torch_float32(amplitude_envelopes)
  return torch.where(frequency_envelopes >= sample_rate / 2.0,
                     torch.zeros_like(amplitude_envelopes), amplitude_envelopes)


def harmonic_to_sinusoidal(harm_amp, harm_dist, f0_hz, sample_rate=16000):
  """core.harmonic_to_sinusoidal (core.py:784-794): the harmonic synthesizer's
  controls as sinusoids, amps [B, T, K] and freqs f0 * [1..K], with the harmonics
  at or above Nyquist dropped and the rest renormalised.  Frame-rate differentiable
  torch ops on the inputs' device, like hz_to_midi."""
  harm_amp, harm_dist, f0_hz = _as_f32(harm_amp), _as_f32(harm_dist), _as_f32(f0_hz)
  k = int(harm_dist.shape[-1])
  freqs = f0_hz * torch.linspace(1.0, float(k), k, device=f0_hz.device)[None, None, :]
  harm_dist = torch.where(freqs >= sample_rate / 2.0, torch.zeros_like(harm_dist),
                          harm_dist)
  harm_dist = safe_divide(harm_dist, torch.sum(harm_dist, dim=-1, keepdim=True))
  return harm_amp * harm_dist, freqs


def _sinusoidal_to_harmonic_shapes(sin_amps, sin_freqs, f0_hz, harmonic_width, n_harmonics):
  """(B, T, S, K) of sinusoidal_to_harmonic from static shapes, or the error."""
  sa, sf, s0 = _shape(sin_amps), _shape(sin_freqs), _shape(f0_hz)
  if len(sa) != 3 or sf != sa or s0 != sa[:2] + (1,):
    raise ValueError(f'sin_amps {sa} and sin_freqs {sf} must both be [batch, time, '
                     f'n_sinusoids] and f0_hz {s0} [batch, time, 1].')
  if isinstance(n_harmonics, bool) or int(n_harmonics) != n_harmonics or n_harmonics < 0:
    raise ValueError(f'n_harmonics must be a non-negative integer, got {n_harmonics}.')
  if np.float32(harmonic_width) == 0.0:
    raise ValueError('harmonic_width must be nonzero (the reference divides by it), got '
                     f'{harmonic_width}.')
  if sa[2] > _lib.CONSISTENCY_MAX_STAGED:
    raise NotImplementedError(
        f'sinusoidal_to_harmonic: {sa[2]} sinusoids per frame exceed the '
        f'{_lib.CONSISTENCY_MAX_STAGED} the kernels stage.')
  return sa + (int(n_harmonics),)


def sinusoidal_to_harmonic_forward(sin_amps, sin_freqs, f0_hz, n_harmonics, harmonic_width,
                                   sample_rate, normalize):
  """`ddsp_b200_sinusoidal_to_harmonic` on float32 CUDA operands -> (harm_amp [B, T, 1],
  harm_dist [B, T, K])."""
  b, t, s = sin_amps.shape
  harm_amp = torch.empty((b, t, 1), dtype=torch.float32, device=sin_amps.device)
  harm_dist = torch.empty((b, t, n_harmonics), dtype=torch.float32, device=sin_amps.device)
  _launch('ddsp_b200_sinusoidal_to_harmonic', sin_amps, sin_freqs, f0_hz, harm_amp,
          harm_dist, b, t, s, n_harmonics, harmonic_width, sample_rate, int(normalize))
  return harm_amp, harm_dist


@on_operands_device
def sinusoidal_to_harmonic(sin_amps, sin_freqs, f0_hz, harmonic_width=0.1,
                           n_harmonics=100, sample_rate=16000, normalize=False):
  """core.sinusoidal_to_harmonic (core.py:733-781): the amplitude and distribution of K
  harmonics of f0 that sinusoids [B, T, S] weighted by a Gaussian in their frequency
  distance relative to f0 amount to, (harm_amp [B, T, 1], harm_dist [B, T, K]).  Each
  frame is evaluated on chip (csrc/consistency.cuh, mode C); the reference's
  [B, T, K, S] tensors are never formed.  Routes to `autograd.SinusoidalToHarmonicFn`
  when grad is enabled and an input requires it.

  The inputs must have exactly these shapes (the reference would broadcast size-1
  axes); other shapes, a zero harmonic_width and more than 4096 sinusoids raise before
  any device work."""
  b, t, s, k = _sinusoidal_to_harmonic_shapes(sin_amps, sin_freqs, f0_hz, harmonic_width,
                                              n_harmonics)
  a, f, f0 = torch_float32(sin_amps), torch_float32(sin_freqs), torch_float32(f0_hz)
  cfg = (k, float(harmonic_width), float(sample_rate), bool(normalize))
  if _requires_grad(a, f, f0):
    from ddsp_b200 import autograd as _ag
    return _ag.SinusoidalToHarmonicFn.apply(a, f, f0, *cfg)
  return sinusoidal_to_harmonic_forward(a, f, f0, *cfg)


# ----------------------------------------------------------------------------
# The HMM of losses.HmmTranscriber (losses.py:247-345): csrc/hmm.cuh
# ----------------------------------------------------------------------------
def _hmm_shapes(observations, loc, scale):
  """(B, T, K) of an HMM call from static shapes, or the error."""
  so, sl, ss = _shape(observations), _shape(loc), _shape(scale)
  if len(so) != 3 or so[2] != 2 or so[1] < 1:
    raise ValueError(f'observations {so} must be [batch, time >= 1, 2] (pitch, amps).')
  if len(sl) != 2 or sl[1] != 2 or ss != sl:
    raise ValueError(f'loc {sl} and scale {ss} must both be [n_states, 2].')
  if sl[0] < 2:
    raise ValueError(f'the HMM needs at least 2 states, got {sl[0]}.')
  if sl[0] > _lib.HMM_MAX_STATES:
    raise NotImplementedError(f'HMM: {sl[0]} states exceed the {_lib.HMM_MAX_STATES} the '
                              'kernels run.')
  return so[0], so[1], sl[0]


def _hmm_transition(hold, other):
  hold, other = float(hold), float(other)
  if not (np.isfinite(hold) and np.isfinite(other) and hold >= 0.0 and other >= 0.0
          and hold + other > 0.0):
    raise ValueError(f'hold={hold} and other={other} must be finite, non-negative and '
                     'not both 0.')
  return hold, other


def hmm_segment(t, k):
  """Steps per checkpoint of the log-likelihood backward: about sqrt(T), so that the
  checkpoints ([B, ceil(T / seg), K] floats) and the segment buffer (seg x K floats
  of shared memory) are both O(K sqrt(T)); at most HMM_SEGMENT_FLOATS / K."""
  return min(math.isqrt(t - 1) + 1, _lib.HMM_SEGMENT_FLOATS // k)


def hmm_viterbi_takes(t, k):
  """True where `ddsp_b200_hmm_viterbi` keeps T steps of K states' back pointers in
  shared memory: 4 T (ceil(K / 32) + 1) <= HMM_VITERBI_BYTES."""
  return bool(_lib.load().ddsp_b200_hmm_viterbi_takes(t, k))


def _hmm_operands(observations, loc, scale):
  x = torch_float32(observations)
  return x, torch_float32(loc, device=x.device), torch_float32(scale, device=x.device)


def hmm_log_prob_forward(x, loc, scale, hold, other):
  """`ddsp_b200_hmm_log_prob` on float32 CUDA operands -> log_prob [B]."""
  b, t, _ = x.shape
  out = torch.empty((b,), dtype=torch.float32, device=x.device)
  _launch('ddsp_b200_hmm_log_prob', x, loc, scale, out, b, t, loc.shape[0], hold, other)
  return out


@on_operands_device
def hmm_log_prob(observations, loc, scale, hold, other):
  """log p(observations) [B] under the HMM of losses.HmmTranscriber: K states, a
  uniform initial distribution, transitions `hold` on the diagonal and `other`
  elsewhere, observations [B, T, 2] under MultivariateNormalDiag(loc_j, scale_j) with
  loc and scale [K, 2] (tfp's HiddenMarkovModel.log_prob).  The forward algorithm
  runs in O(K) per step in one launch (csrc/hmm.cuh).  Routes to
  `autograd.HmmLogProbFn` when grad is enabled and the observations require it;
  loc and scale are constants.

  Shapes, K < 2 and invalid hold / other raise ValueError, K > 1024
  NotImplementedError, before any device work."""
  _hmm_shapes(observations, loc, scale)
  hold, other = _hmm_transition(hold, other)
  if _requires_grad(loc, scale):
    raise NotImplementedError('hmm_log_prob: gradients reach the observations only; '
                              'loc and scale are constants.')
  x, loc, scale = _hmm_operands(observations, loc, scale)
  if _requires_grad(x):
    from ddsp_b200 import autograd as _ag
    return _ag.HmmLogProbFn.apply(x, loc, scale, hold, other)
  return hmm_log_prob_forward(x, loc, scale, hold, other)


@on_operands_device
def hmm_posterior_mode(observations, loc, scale, hold, other):
  """The most likely state sequence [B, T] (int64) of the HMM of `hmm_log_prob`
  (tfp's HiddenMarkovModel.posterior_mode), by Viterbi in one launch with its back
  pointers in shared memory.  Ties go to the lowest state index.  Besides the errors
  of `hmm_log_prob`, T steps of K states beyond `hmm_viterbi_takes` raise
  NotImplementedError before any device work."""
  b, t, k = _hmm_shapes(observations, loc, scale)
  hold, other = _hmm_transition(hold, other)
  if not hmm_viterbi_takes(t, k):
    raise NotImplementedError(
        f'hmm_posterior_mode: {t} steps of {k} states exceed the back pointers the '
        f'kernel keeps (4 T (ceil(K / 32) + 1) <= {_lib.HMM_VITERBI_BYTES} bytes).')
  x, loc, scale = _hmm_operands(observations, loc, scale)
  path = torch.empty((b, t), dtype=torch.int64, device=x.device)
  _launch('ddsp_b200_hmm_viterbi', x.detach(), loc.detach(), scale.detach(), path, b, t,
          k, hold, other)
  return path


@on_operands_device
def normalize_harmonics(harmonic_distribution, f0_hz=None, sample_rate=None):
  """core.normalize_harmonics (core.py:894-907) on the controls kernel."""
  sh = _shape(harmonic_distribution)
  if len(sh) != 3:
    raise ValueError(f'harmonic_distribution must be 3-D, got {sh}.')
  b, f, _ = sh
  mask = sample_rate is not None and f0_hz is not None
  if f0_hz is None:
    f0_hz = torch.zeros((b, f, 1), dtype=torch.float32, device=_device())
  amps = torch.zeros((b, f, 1), dtype=torch.float32, device=_device())
  _, hd = harmonic_controls(amps, harmonic_distribution, f0_hz,
                            sample_rate if mask else 2.0, scale=False,
                            normalize_below_nyquist=mask)
  return hd


def angular_cumsum(angular_frequency, chunk_size: int = 1000,
                   tf_sequential: bool = False):
  """core.angular_cumsum (core.py:799-866): accumulated phase in [0, 2 pi] of an
  angular frequency [batch, time, ...] in radians per sample.

  Default: the wrapped running sum computed EXACTLY (64-bit fixed-point turns,
  three-pass scan) - the quantity the reference's chunked float32 cumsum
  approximates; `chunk_size` does not matter then.  The exact phase lies in
  [0, 2 pi); rounding it to float32 takes a phase within about 6e-8 rad below
  2 pi up to float32(2 pi), so the result lies in [0, float32(2 pi)], the
  [0, 2 pi] the reference documents.  tf_sequential=True reproduces
  the reference's own float32 arithmetic in its own order (chunks of
  `chunk_size`, mod-2pi stitching) - a debug mode for comparing against
  TensorFlow, one thread per (batch, channel).

  Routes to `autograd.AngularCumsumFn` when grad is enabled and the input
  requires it; tf_sequential=True is forward-only and raises NotImplementedError
  there."""
  x = torch_float32(angular_frequency)
  if len(x.shape) < 2:
    raise ValueError(f'angular_frequency must be [batch, time, ...], got {list(x.shape)}.')
  if _requires_grad(x):
    if tf_sequential:
      raise NotImplementedError('angular_cumsum: tf_sequential=True is a forward-only '
                                'debug mode; it has no backward.')
    from ddsp_b200 import autograd as _ag
    return _ag.AngularCumsumFn.apply(x)
  return angular_cumsum_forward(x, chunk_size, tf_sequential)


def _bnc(shape):
  """(B, N, C) of a [batch, time, ...] shape, C the product of the trailing axes
  (at least 1)."""
  c = 1
  for d in shape[2:]:
    c *= int(d)
  return shape[0], shape[1], max(c, 1)


def angular_cumsum_forward(x, chunk_size=1000, tf_sequential=False):
  """`ddsp_b200_angular_cumsum` on a float32 CUDA tensor [batch, time, ...]."""
  shape = tuple(x.shape)
  b, n, c = _bnc(shape)
  x3 = x.reshape(b, n, c)
  out = torch.empty_like(x3)
  if tf_sequential:
    _launch('ddsp_b200_angular_cumsum', x3, out, b, n, c, int(chunk_size), 2, None, 0)
  else:
    _launch('ddsp_b200_angular_cumsum', x3, out, b, n, c, int(chunk_size), 0,
            *_workspace('ddsp_b200_oscillator_bank_workspace', x3.device, b, n, c))
  return out.reshape(shape)


@on_operands_device
def oscillator_bank(frequency_envelopes, amplitude_envelopes,
                    sample_rate: int = 16000, sum_sinusoids: bool = True,
                    use_angular_cumsum: bool = False,
                    phase_mode: Text = 'exact'):
  """core.oscillator_bank (core.py:911-962) on audio-rate envelopes
  [batch, n_samples, n_sinusoids].

  phase_mode='exact' (default): phase is accumulated wrapped and exactly (64-bit
  fixed point) whatever `use_angular_cumsum` says - both reference modes
  approximate this.  phase_mode='tf_sequential': the reference's own float32
  arithmetic in its own order - tf.cumsum, or angular_cumsum (chunks of 1000)
  when use_angular_cumsum - reproducing TensorFlow's phase error (debug).

  Routes to `autograd.OscillatorBankFn` when grad is enabled and an input
  requires it (both `sum_sinusoids` values); phase_mode='tf_sequential' is
  forward-only and raises NotImplementedError there."""
  if phase_mode not in ('exact', 'tf_sequential'):
    raise ValueError(f"phase_mode must be 'exact' or 'tf_sequential', got {phase_mode!r}.")
  sf, sa = _shape(frequency_envelopes), _shape(amplitude_envelopes)
  if len(sf) != 3 or sf != sa:
    raise ValueError(f'frequency_envelopes {sf} and amplitude_envelopes {sa} must '
                     'both be [batch, n_samples, n_sinusoids].')
  b, n, k = sf
  f = torch_float32(frequency_envelopes)
  a = torch_float32(amplitude_envelopes)
  if _requires_grad(f, a):
    if phase_mode == 'tf_sequential':
      raise NotImplementedError("oscillator_bank: phase_mode='tf_sequential' is a "
                                'forward-only debug mode; it has no backward.')
    from ddsp_b200 import autograd as _ag
    return _ag.OscillatorBankFn.apply(f, a, float(sample_rate), bool(sum_sinusoids))
  if phase_mode == 'tf_sequential':
    wavs = torch.empty((b, n, k), dtype=torch.float32, device=f.device)
    _launch('ddsp_b200_oscillator_bank_tf_sequential', f, a, wavs, b, n, k,
            float(sample_rate), int(bool(use_angular_cumsum)), 1000)
    return wavs.sum(-1) if sum_sinusoids else wavs
  return oscillator_bank_forward(f, a, sample_rate, sum_sinusoids)


def oscillator_bank_forward(f, a, sample_rate, sum_sinusoids):
  """`ddsp_b200_oscillator_bank` (exact phase) on float32 CUDA envelopes [B, N, K]."""
  b, n, k = f.shape
  out = torch.empty((b, n) if sum_sinusoids else (b, n, k), dtype=torch.float32,
                    device=f.device)
  _launch('ddsp_b200_oscillator_bank', f, a, out, b, n, k, float(sample_rate),
          int(bool(sum_sinusoids)),
          *_workspace('ddsp_b200_oscillator_bank_workspace', f.device, b, n, k))
  return out


@on_operands_device
def sinusoidal_synthesis(frequencies, amplitudes, n_samples: int = 64000,
                         sample_rate: int = 16000,
                         amp_resample_method: Text = 'window', out=None,
                         accumulate: bool = False):
  """Frame-rate bank of sinusoids with per-sinusoid frequencies
  [batch, n_frames, n_sinusoids] -> audio [batch, n_samples]: the fused form of
  resample + resample + core.oscillator_bank (synths.py:305-323) - the
  [batch, n_samples, n_sinusoids] envelopes are never materialised.  Routes to
  `autograd.SinusoidalSynthesisFn` when grad is enabled and an input requires
  it; `out=` / `accumulate=` are refused there."""
  sf, sa = _shape(frequencies), _shape(amplitudes)
  if len(sf) != 3 or sf != sa:
    raise ValueError(f'frequencies {sf} and amplitudes {sa} must both be '
                     '[batch, n_frames, n_sinusoids].')
  b, f, k = sf
  n_samples = int(n_samples)
  if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad
                                     for t in (frequencies, amplitudes)):
    if out is not None or accumulate:
      raise ValueError('sinusoidal_synthesis: out= and accumulate= write audio that '
                       'autograd cannot track; they are not available when an input '
                       'requires grad.')
    from ddsp_b200 import autograd as _ag
    return _ag.SinusoidalSynthesisFn.apply(frequencies, amplitudes, n_samples,
                                           sample_rate, amp_resample_method)
  freqs = torch_float32(frequencies)
  amps = torch_float32(amplitudes)
  if out is None:
    out = torch.empty((b, n_samples), dtype=torch.float32, device=freqs.device)
    accumulate = False
  else:
    freqs, amps = _check_out(out, (b, n_samples), freqs, (freqs, amps))
  _launch('ddsp_b200_sinusoidal_forward', freqs, amps, out, b, f, k, n_samples,
          float(sample_rate), AMP_METHODS[amp_resample_method], int(bool(accumulate)),
          *_workspace('ddsp_b200_sinusoidal_workspace', freqs.device, b, f, k))
  return _wrote(out)


@on_operands_device
def harmonic_synthesis(frequencies,
                       amplitudes,
                       harmonic_shifts=None,
                       harmonic_distribution=None,
                       n_samples: int = 64000,
                       sample_rate: int = 16000,
                       amp_resample_method: Text = 'window',
                       use_angular_cumsum: bool = False,
                       out: Optional[torch.Tensor] = None,
                       accumulate: bool = False,
                       phase_mode: Text = 'recurrence'):
  """core.harmonic_synthesis (core.py:1048-1111).

  The common case (no harmonic_shifts, 'window' / 'linear' amplitudes, n_samples
  a multiple of the frame count) is ONE fused kernel.  With `harmonic_shifts`
  (core.py:1084-1093) the harmonics are no longer integer multiples of one
  phase: f0 * k * (1 + shift) and amp * hd are formed at frame rate, as the
  reference does, and the frame-rate oscillator bank with per-sinusoid phases
  (`sinusoidal_synthesis`) takes over.  'nearest' / 'cubic' amplitudes and
  non-integer hops take the reference's own decomposition on our kernels:
  `resample` + `resample` + `oscillator_bank` (audio-rate envelopes exist then).

  Phase is accumulated wrapped and exactly (64-bit fixed point) whatever
  `use_angular_cumsum` says - that is what angular_cumsum approximates
  (core.py:803-817; DESIGN.md "phase").  phase_mode: 'recurrence' (default) /
  'direct' choose how sin(k phi) is evaluated in the fused kernel;
  'tf_sequential' reproduces TensorFlow's float32 phase arithmetic in its own
  order (tf.cumsum, or angular_cumsum if use_angular_cumsum) - a debug mode for
  small shapes that materialises the envelopes.

  When grad is enabled and an input requires it (DESIGN.md section 3.15): the fused
  case at hops the harmonic backward kernel takes (a multiple of 64, at most 8192)
  is `autograd.HarmonicSynthesisFn`; `harmonic_shifts`, or any other integer hop,
  goes through `sinusoidal_synthesis` and its backward; 'nearest' / 'cubic' and
  non-integer hops through `resample` and `oscillator_bank` and theirs.  `out=` is
  refused there (RuntimeError), and phase_mode='tf_sequential' has no backward
  (NotImplementedError).
  """
  if amp_resample_method not in ('nearest', 'linear', 'cubic', 'window'):
    # core.py:632-634
    raise ValueError('Method ({}) is invalid. Must be one of {}.'.format(
        amp_resample_method, "['nearest', 'linear', 'cubic', 'window']"))
  if phase_mode not in ('recurrence', 'direct', 'tf_sequential'):
    raise ValueError("phase_mode must be 'recurrence', 'direct' or "
                     f"'tf_sequential', got {phase_mode!r}.")
  sf, sa = _shape(frequencies), _shape(amplitudes)
  if len(sf) != 3 or len(sa) != 3:
    # core.py:670-672 (the window upsampler only takes 3-D inputs)
    raise ValueError('Upsample_with_windows() only supports 3 dimensions, '
                     'not {}.'.format(list(sa)))
  b, f, _ = sf
  if sa != (b, f, 1) or sf != (b, f, 1):
    raise ValueError(f'frequencies {sf} and amplitudes {sa} must both be '
                     f'[batch, n_frames, 1].')
  k = 1
  if harmonic_distribution is not None:
    sh = _shape(harmonic_distribution)
    if len(sh) != 3 or sh[:2] != (b, f):
      raise ValueError(f'harmonic_distribution {sh} must be [{b}, {f}, '
                       'n_harmonics].')
    k = int(sh[-1])
  if harmonic_shifts is not None:
    ss = _shape(harmonic_shifts)
    if len(ss) != 3 or ss[:2] != (b, f) or (harmonic_distribution is not None
                                             and ss[-1] != k):
      raise ValueError(f'harmonic_shifts {ss} must be [{b}, {f}, n_harmonics'
                       f'{"=" + str(k) if harmonic_distribution is not None else ""}].')
    k = int(ss[-1])
  n_samples = int(n_samples)
  grad = _requires_grad(frequencies, amplitudes, harmonic_distribution, harmonic_shifts)
  if grad and out is not None:
    _no_grad_path('harmonic_synthesis', frequencies, amplitudes, harmonic_distribution,
                  harmonic_shifts)
  if grad and phase_mode == 'tf_sequential':
    raise NotImplementedError("harmonic_synthesis: phase_mode='tf_sequential' is a "
                              'forward-only debug mode; it has no backward.')
  if amp_resample_method == 'window':
    if f >= n_samples:
      # core.py:682-685
      raise ValueError('Upsample with windows cannot be used for downsampling'
                       'More input frames ({}) than output timesteps ({})'.format(
                           f + 1, n_samples))
    if n_samples % f != 0:
      # core.py:687-693
      raise ValueError(
          'For upsampling, the target the number of timesteps must be divisible '
          'by the number of input frames{}. (timesteps:{}, frames:{}, '
          'add_endpoint={}).'.format('', n_samples, f + 1, True))
  frequencies = torch_float32(frequencies)
  amplitudes = torch_float32(amplitudes)
  if harmonic_distribution is not None:
    harmonic_distribution = torch_float32(harmonic_distribution)
  if harmonic_shifts is not None:
    harmonic_shifts = torch_float32(harmonic_shifts)
  if out is not None:
    frequencies, amplitudes, harmonic_distribution, harmonic_shifts = _check_out(
        out, (b, n_samples), frequencies,
        (frequencies, amplitudes, harmonic_distribution, harmonic_shifts))
  else:
    accumulate = False

  fused_ok = (amp_resample_method in AMP_METHODS and n_samples % f == 0 and
              phase_mode != 'tf_sequential')
  if grad and harmonic_shifts is None and fused_ok and _harmonic_backward_takes(
      b, f, n_samples):
    from ddsp_b200 import autograd as _ag
    if harmonic_distribution is None:
      harmonic_distribution = torch.ones_like(amplitudes)
    return _ag.HarmonicSynthesisFn.apply(frequencies, amplitudes, harmonic_distribution,
                                         n_samples, sample_rate, amp_resample_method)
  if harmonic_shifts is None and fused_ok and not grad:
    mode = {'recurrence': _lib.PHASE_RECURRENCE, 'direct': _lib.PHASE_DIRECT}[
        phase_mode]
    if out is None:
      out = torch.empty((b, n_samples), dtype=torch.float32,
                        device=frequencies.device)
    _launch('ddsp_b200_harmonic_forward', frequencies, amplitudes, harmonic_distribution,
            out, b, f, k, n_samples, float(sample_rate), AMP_METHODS[amp_resample_method],
            mode, int(bool(accumulate)))
    return _wrote(out)

  # frame-rate harmonic frequencies / amplitudes, float32 op for op as the
  # reference (core.py:1091-1099): (f0 * k) * (1 + shifts), amplitudes * hd
  harmonic_frequencies = get_harmonic_frequencies(frequencies, k)
  if harmonic_shifts is not None:
    harmonic_frequencies = harmonic_frequencies * (1.0 + harmonic_shifts)
  harmonic_amplitudes = (amplitudes * harmonic_distribution
                         if harmonic_distribution is not None
                         else amplitudes.expand(b, f, k).contiguous())
  if fused_ok:
    return sinusoidal_synthesis(harmonic_frequencies, harmonic_amplitudes,
                                n_samples=n_samples, sample_rate=sample_rate,
                                amp_resample_method=amp_resample_method, out=out,
                                accumulate=accumulate)
  # core.py:1101-1110 on the stand-alone kernels (audio-rate envelopes exist)
  frequency_envelopes = resample(harmonic_frequencies, n_samples)
  amplitude_envelopes = resample(harmonic_amplitudes, n_samples,
                                 method=amp_resample_method)
  audio = oscillator_bank(
      frequency_envelopes, amplitude_envelopes, sample_rate=sample_rate,
      use_angular_cumsum=use_angular_cumsum,
      phase_mode='tf_sequential' if phase_mode == 'tf_sequential' else 'exact')
  if out is None:
    return audio
  if accumulate:
    out += audio
  else:
    out.copy_(audio)
  return out


def _harmonic_backward_takes(b, f, n_samples):
  """Whether `ddsp_b200_harmonic_backward` takes an integer-hop shape: a hop that is a
  multiple of 64 and at most 8192, a batch within the grid limit."""
  return bool(_lib.load().ddsp_b200_harmonic_backward_takes(b, f, n_samples))


def _hob_shapes(frequency, amplitude_envelopes, initial_phase):
  """(B, N, K) of harmonic_oscillator_bank's operands; ValueError otherwise."""
  sf, sa = _shape(frequency), _shape(amplitude_envelopes)
  if len(sf) != 3 or len(sa) != 3 or sf[2] != 1 or sa[:2] != sf[:2] or sf[1] < 1 or sa[2] < 1:
    raise ValueError(f'frequency {sf} must be [batch, n_samples, 1] and amplitude_envelopes '
                     f'{sa} [batch, n_samples, n_harmonics], with n_samples >= 1 and '
                     'n_harmonics >= 1.')
  if initial_phase is not None and _shape(initial_phase) != (sf[0], 1, 1):
    raise ValueError(f'initial_phase {_shape(initial_phase)} must be [{sf[0]}, 1, 1].')
  return sf[0], sf[1], sa[2]


def _hob_backward_takes(b, n, k):
  """Whether `ddsp_b200_harmonic_oscillator_bank_backward` takes the shape."""
  return bool(_lib.load().ddsp_b200_harmonic_oscillator_bank_backward_takes(b, n, k))


@on_operands_device
def harmonic_oscillator_bank(frequency, amplitude_envelopes, initial_phase=None,
                             sample_rate: int = 16000, use_angular_cumsum: bool = True):
  """core.harmonic_oscillator_bank (core.py:966-1025): one audio-rate f0 [B, N, 1] drives
  the harmonics k = 1..K of amplitude_envelopes [B, N, K] from initial_phase [B, 1, 1]
  (None: 0).  Returns (audio [B, N], final_phase [B, 1, 1]); feed final_phase back as the
  next call's initial_phase.

  The phase is accumulated exactly in 64-bit fixed-point turns, and harmonic k's phase is
  k times it, wrapping exactly; there is no Nyquist mask, as in the reference.
  final_phase is the wrapped sum in [0, 2 pi) plus initial_phase with
  use_angular_cumsum=True, else the unwrapped sum plus initial_phase; the audio is the same
  in both modes.  Routes to `autograd.HarmonicOscillatorBankFn` when grad is enabled and an
  input requires it."""
  b, n, k = _hob_shapes(frequency, amplitude_envelopes, initial_phase)
  grad = _requires_grad(frequency, amplitude_envelopes, initial_phase)
  if grad and not _hob_backward_takes(b, n, k):
    _no_grad_path('harmonic_oscillator_bank', frequency, amplitude_envelopes, initial_phase)
  f = torch_float32(frequency)
  a = torch_float32(amplitude_envelopes)
  init = None if initial_phase is None else torch_float32(initial_phase, f.device)
  if grad:
    from ddsp_b200 import autograd as _ag
    return _ag.HarmonicOscillatorBankFn.apply(f, a, init, float(sample_rate),
                                              bool(use_angular_cumsum))
  return harmonic_oscillator_bank_forward(f, a, init, sample_rate, use_angular_cumsum)


def harmonic_oscillator_bank_forward(f, a, init, sample_rate, use_angular_cumsum):
  """`ddsp_b200_harmonic_oscillator_bank` on float32 CUDA operands f [B, N, 1],
  a [B, N, K] and init [B, 1, 1] or None."""
  b, n, k = a.shape
  audio = torch.empty((b, n), dtype=torch.float32, device=f.device)
  final_phase = torch.empty((b, 1, 1), dtype=torch.float32, device=f.device)
  if b == 0:
    return audio, final_phase
  _launch('ddsp_b200_harmonic_oscillator_bank', f, a, init, audio, final_phase, b, n, k,
          float(sample_rate), int(bool(use_angular_cumsum)))
  return audio, final_phase


@on_operands_device
def streaming_harmonic_synthesis(frequencies,
                                 amplitudes,
                                 harmonic_distribution=None,
                                 initial_phase=None,
                                 n_samples: int = 64000,
                                 sample_rate: int = 16000,
                                 amp_resample_method: Text = 'linear'):
  """core.streaming_harmonic_synthesis (core.py:1114-1164): single-f0 harmonic
  bank with a carried phase.  Returns (audio [B, n_samples], final_phase
  [B, 1, 1]) - feed final_phase back as initial_phase for the next hop
  (training/inference.py:463-478).

  Without grad, 'window' / 'linear' amplitudes at an integer hop run one fused kernel.
  Other hops, 'nearest' / 'cubic' amplitudes, and every call under grad run the
  reference's composition on our kernels: normalize_harmonics, resample and
  harmonic_oscillator_bank, each with its backward, so gradients reach frequencies,
  amplitudes, harmonic_distribution and initial_phase."""
  sf, sa = _shape(frequencies), _shape(amplitudes)
  if len(sf) != 3 or len(sa) != 3 or sa != sf or sf[2] != 1:
    raise ValueError(f'frequencies {sf} and amplitudes {sa} must both be '
                     '[batch, n_frames, 1].')
  if amp_resample_method not in ('nearest', 'linear', 'cubic', 'window'):
    raise ValueError('Method ({}) is invalid. Must be one of {}.'.format(
        amp_resample_method, "['nearest', 'linear', 'cubic', 'window']"))
  b, f, _ = sf
  n_samples = int(n_samples)
  k = 1
  if harmonic_distribution is not None:
    sh = _shape(harmonic_distribution)
    if len(sh) != 3 or sh[:2] != (b, f):
      raise ValueError(f'harmonic_distribution {sh} must be [{b}, {f}, n_harmonics].')
    k = int(sh[-1])
  if _requires_grad(frequencies, amplitudes, harmonic_distribution, initial_phase):
    if not _hob_backward_takes(b, n_samples, k):
      _no_grad_path('streaming_harmonic_synthesis', frequencies, amplitudes,
                    harmonic_distribution, initial_phase)
    return _streaming_composition(frequencies, amplitudes, harmonic_distribution,
                                  initial_phase, n_samples, sample_rate, amp_resample_method)
  if amp_resample_method not in AMP_METHODS or n_samples % f != 0:
    return _streaming_composition(frequencies, amplitudes, harmonic_distribution,
                                  initial_phase, n_samples, sample_rate, amp_resample_method)
  frequencies = torch_float32(frequencies)
  amplitudes = torch_float32(amplitudes)
  hd = None
  if harmonic_distribution is not None:
    hd = torch_float32(harmonic_distribution)
    # normalize_harmonics (core.py:1143-1146): Nyquist mask + row normalisation
    hd_n = torch.empty_like(hd)
    amp_copy = torch.empty_like(amplitudes)
    _launch('ddsp_b200_harmonic_controls', amplitudes, hd, frequencies, amp_copy, hd_n,
            b, f, k, float(sample_rate), _lib.CTL_NYQUIST)
    hd = hd_n
  init = None
  if initial_phase is not None:
    init = torch_float32(initial_phase).reshape(b).contiguous()
  audio = torch.empty((b, n_samples), dtype=torch.float32, device=frequencies.device)
  final_phase = torch.empty((b,), dtype=torch.float32, device=frequencies.device)
  _launch('ddsp_b200_streaming_harmonic_forward', frequencies, amplitudes, hd, init, audio,
          final_phase, b, f, k, n_samples, float(sample_rate),
          AMP_METHODS[amp_resample_method])
  return audio, final_phase.reshape(b, 1, 1)


def _streaming_composition(frequencies, amplitudes, harmonic_distribution, initial_phase,
                           n_samples, sample_rate, amp_resample_method):
  """core.py:1140-1164 op for op: normalize_harmonics, amplitudes * distribution,
  resample and harmonic_oscillator_bank, each differentiable."""
  frequencies = torch_float32(frequencies)
  amplitudes = torch_float32(amplitudes)
  if harmonic_distribution is not None:
    hd = normalize_harmonics(torch_float32(harmonic_distribution), frequencies, sample_rate)
    harmonic_amplitudes = amplitudes * hd
  else:
    harmonic_amplitudes = amplitudes
  frequency_envelopes = resample(frequencies, n_samples)
  amplitude_envelopes = resample(harmonic_amplitudes, n_samples, method=amp_resample_method)
  return harmonic_oscillator_bank(frequency_envelopes, amplitude_envelopes, initial_phase,
                                  sample_rate=sample_rate)


# ----------------------------------------------------------------------------
# Time-varying FIR / filtered noise (core.py:1316-1655)
# ----------------------------------------------------------------------------
def get_fft_size(frame_size: int, ir_size: int, power_of_2: bool = True) -> int:
  """core.py:1317-1335 (kept for API parity; the CUDA path is time-domain)."""
  convolved_frame_size = ir_size + frame_size - 1
  if power_of_2:
    return int(2**np.ceil(np.log2(convolved_frame_size)))
  raise NotImplementedError('power_of_2=False needs scipy.fftpack.')


def _ir_size(nb, window_size):
  """Taps of the windowed impulse response of nb bins: `ddsp_b200_ir_size`."""
  return _lib.load().ddsp_b200_ir_size(nb, window_size)


def _check_n_frequencies(nb):
  if nb < 2:
    raise ValueError(f'frequency_impulse_response needs >= 2 frequencies, got {nb}.')


def _requires_grad(*tensors):
  return torch.is_grad_enabled() and any(
      isinstance(t, torch.Tensor) and t.requires_grad for t in tensors)


def frequency_impulse_response(magnitudes, window_size: int = 0):
  """core.frequency_impulse_response (core.py:1534-1565).  Routes to
  `autograd.FrequencyImpulseResponseFn` when grad is enabled and the magnitudes
  require it."""
  nb = int(_shape(magnitudes)[-1])
  _check_n_frequencies(nb)
  if _requires_grad(magnitudes):
    from ddsp_b200 import autograd as _ag
    return _ag.FrequencyImpulseResponseFn.apply(magnitudes, int(window_size))
  s = _ir_size(nb, int(window_size))
  magnitudes = torch_float32(magnitudes)
  ir = torch.empty(tuple(magnitudes.shape[:-1]) + (s,), dtype=torch.float32,
                   device=magnitudes.device)
  _launch('ddsp_b200_frequency_impulse_response', magnitudes, ir, magnitudes.numel() // nb,
          nb, int(window_size))
  return ir


def apply_window_to_impulse_response(impulse_response, window_size: int = 0,
                                     causal: bool = False):
  """core.apply_window_to_impulse_response (core.py:1477-1531) for callers of the
  reference function: zero-phase (or `causal`) impulse responses [..., ir_size] ->
  Hann-windowed, causal form, cropped to `window_size` (made odd) when that is
  shorter.  Frame-rate torch ops on whatever device the input lives on; the
  synthesis path never calls it - `frequency_impulse_response` and the fused noise
  kernels build the windowed taps straight from the magnitudes."""
  ir = _as_f32(impulse_response)
  if causal:
    ir = torch.fft.fftshift(ir, dim=-1)
  ir_size = int(ir.shape[-1])
  if window_size <= 0 or window_size > ir_size:
    window_size = ir_size
  # tf.signal.hann_window: periodic for even lengths, symmetric for odd ones
  window = torch.hann_window(window_size, periodic=(window_size % 2 == 0),
                             dtype=torch.float32, device=ir.device)
  padding = ir_size - window_size
  if padding > 0:
    half_idx = (window_size + 1) // 2
    window = torch.cat([window[half_idx:],
                        torch.zeros(padding, dtype=torch.float32, device=ir.device),
                        window[:half_idx]], dim=0)
  else:
    window = torch.fft.fftshift(window, dim=-1)
  ir = window * ir
  if padding > 0:
    first_half_start = (ir_size - (half_idx - 1)) + 1
    second_half_end = half_idx + 1
    ir = torch.cat([ir[..., first_half_start:], ir[..., :second_half_end]], dim=-1)
  else:
    ir = torch.fft.fftshift(ir, dim=-1)
  return ir


def crop_and_compensate_delay(audio, audio_size: int, ir_size: int, padding: Text,
                              delay_compensation: int):
  """core.crop_and_compensate_delay (core.py:1338-1379): the slice
  `audio[:, start:-end]` of a convolution output, with the reference's ValueError and
  its Python slice semantics (an `end` of 0 gives an empty result).  A view - no
  kernel; `fft_convolve` applies the same index arithmetic (`_crop_range`) inside its
  kernels instead of materialising the uncropped signal."""
  if not isinstance(audio, torch.Tensor):
    audio = torch.as_tensor(np.asarray(audio, dtype=np.float32))
  start, _, _ = _crop_range(int(audio.shape[-1]), audio_size, ir_size, padding,
                            delay_compensation)
  crop_size = ir_size + audio_size - 1 if padding == 'valid' else audio_size
  end = (int(audio.shape[-1]) - crop_size) - start
  return audio[:, start:-end]


def _crop_range(total_size, audio_size, ir_size, padding, delay_compensation):
  """Index arithmetic of crop_and_compensate_delay (core.py:1338-1379),
  including Python's slice semantics of `audio[:, start:-end]`."""
  if padding == 'valid':
    crop_size = ir_size + audio_size - 1
  elif padding == 'same':
    crop_size = audio_size
  else:
    raise ValueError('Padding must be \'valid\' or \'same\', instead '
                     'of {}.'.format(padding))
  crop = total_size - crop_size
  start = ((ir_size - 1) // 2 - 1 if delay_compensation < 0
           else delay_compensation)
  end = crop - start
  rng = range(total_size)[start:-end]
  return start, len(rng), crop_size


# Impulse responses longer than this take a frequency-domain formulation instead of
# the direct-form FIR kernel: the direct form costs audio_size * ir_size MACs per
# item - the cross-over is a few thousand taps.  One long IR per item (the Reverb
# case: 48000 taps, effects.py:28-117; SURVEY 8f-3) runs the hand-written
# partitioned overlap-save convolution `ddsp_b200_fft_convolve_lti`.
FFT_CONVOLVE_MIN_IR = 2048


def _fft_convolve_cufft(audio, impulse_response, n_ir_frames, frame_size, fft_size,
                        start, crop_size):
  """The reference's own algorithm (core.py:1445-1473) on torch.fft: frame (hop =
  frame_size, zero padded), rfft both, multiply, irfft, overlap-add, crop."""
  b, n = audio.shape
  pad = n_ir_frames * frame_size - n
  frames = torch.nn.functional.pad(audio, (0, pad)).reshape(b, n_ir_frames, frame_size)
  audio_fft = torch.fft.rfft(frames, n=fft_size, dim=-1)
  ir_fft = torch.fft.rfft(impulse_response, n=fft_size, dim=-1)   # broadcasts batch 1
  frames_out = torch.fft.irfft(audio_fft * ir_fft, n=fft_size, dim=-1)
  if n_ir_frames == 1:
    total = frames_out[:, 0, :]
  else:
    total_size = (n_ir_frames - 1) * frame_size + fft_size
    total = torch.nn.functional.fold(
        frames_out.transpose(1, 2), output_size=(total_size, 1),
        kernel_size=(fft_size, 1), stride=(frame_size, 1))[:, 0, :, 0]
  return total[:, start:start + crop_size].contiguous()


@on_operands_device
def fft_convolve_lti(audio, impulse_response, start, out_len, out=None,
                     accumulate=False, reverse_audio=False, reverse_ir=False):
  """Full linear convolution of audio [B, N] with ONE impulse response per item
  [1 or B, S], cropped to [start, start + out_len): `ddsp_b200_fft_convolve_lti`
  (partitioned overlap-save, hand-written FFTs).  reverse_*: read that operand back
  to front (what the backward pass needs)."""
  audio = torch_float32(audio)
  impulse_response = torch_float32(impulse_response)
  b, n = audio.shape
  ir_batch, s_len = impulse_response.shape
  if out is None:
    out = torch.empty((b, out_len), dtype=torch.float32, device=audio.device)
    accumulate = False
  else:
    # the kernel reads both operands into its workspace before it writes out
    _check_out(out, (b, out_len), audio)
  flags = ((_lib.LTI_REVERSE_AUDIO if reverse_audio else 0) |
           (_lib.LTI_REVERSE_IR if reverse_ir else 0))
  _launch('ddsp_b200_fft_convolve_lti', audio, impulse_response, out, b, n, s_len, ir_batch,
          int(start), int(out_len), int(bool(accumulate)), flags,
          *_workspace('ddsp_b200_fft_convolve_lti_workspace', audio.device, b, n, s_len,
                      ir_batch))
  return _wrote(out)


def _fft_convolve_geometry(sa, si, padding, delay_compensation):
  """The shape checks of core.fft_convolve (core.py:1382-1473) on the static shapes
  of audio and impulse response, and what follows from them: (batch, audio size,
  [ir_batch, n_ir_frames, ir_size], frame size, FFT size, crop start, crop length,
  crop size)."""
  if len(sa) != 2 or len(si) not in (2, 3):
    raise ValueError(f'audio must be [batch, time] and impulse_response 2-D or '
                     f'3-D; got {sa} and {si}.')
  batch_size, audio_size = sa
  if len(si) == 2:
    si = (si[0], 1, si[1])
  ir_batch, n_ir_frames, ir_size = si
  if not (ir_batch == 1 and batch_size > 1) and batch_size != ir_batch:
    # core.py:1441-1443
    raise ValueError('Batch size of audio ({}) and impulse response ({}) must '
                     'be the same.'.format(batch_size, ir_batch))
  frame_size = int(np.ceil(audio_size / n_ir_frames))
  n_audio_frames = -(-audio_size // frame_size)
  if n_audio_frames != n_ir_frames:
    # core.py:1452-1457
    raise ValueError(
        'Number of Audio frames ({}) and impulse response frames ({}) do not '
        'match. For small hop size = ceil(audio_size / n_ir_frames), '
        'number of impulse response frames must be a multiple of the audio '
        'size.'.format(n_audio_frames, n_ir_frames))
  fft_size = get_fft_size(frame_size, ir_size, power_of_2=True)
  total_size = (n_ir_frames - 1) * frame_size + fft_size
  start, out_len, crop_size = _crop_range(total_size, audio_size, ir_size,
                                          padding, delay_compensation)
  return (batch_size, audio_size, si, frame_size, fft_size, start, out_len,
          crop_size)


@on_operands_device
def fft_convolve(audio, impulse_response, padding: Text = 'same',
                 delay_compensation: int = -1, out=None, accumulate=False):
  """core.fft_convolve (core.py:1382-1473).

  Computed as the mathematically identical direct-form time-varying FIR
  (frame / rfft / multiply / irfft / overlap_and_add / crop folded into index
  math; SURVEY.md A.6) - the name is kept for drop-in compatibility.
  """
  sa, si = _shape(audio), _shape(impulse_response)
  (batch_size, audio_size, si, frame_size, fft_size, start, out_len,
   crop_size) = _fft_convolve_geometry(sa, si, padding, delay_compensation)
  ir_batch, n_ir_frames, ir_size = si
  if out_len != crop_size:
    # The reference's `audio[:, start:-end]` degenerates when end <= 0 (e.g.
    # end == 0 yields an empty tensor).  Reproduce the empty case; refuse the
    # rest rather than guess.
    if out_len == 0:
      return torch.empty((batch_size, 0), dtype=torch.float32, device=_device())
    raise NotImplementedError(
        'crop_and_compensate_delay slice is degenerate for this shape '
        f'(start={start}, total={total_size}, crop={crop_size}).')
  audio = torch_float32(audio)
  impulse_response = torch_float32(impulse_response).reshape(si)
  if ir_size >= FFT_CONVOLVE_MIN_IR and n_ir_frames == 1:
    # one long impulse response per item (effects.Reverb): hand-written
    # partitioned overlap-save convolution (csrc/longconv.cuh)
    ir2 = impulse_response.reshape(ir_batch, ir_size).contiguous()
    if torch.is_grad_enabled() and (audio.requires_grad or ir2.requires_grad):
      # trainable reverb (effects.py:70-79): forward and backward are the same
      # kernels (the backward on time-reversed operands)
      from ddsp_b200 import autograd as _ag
      if out is not None:
        # the backward reads the operands it saved: not the ones out= overwrites
        audio, ir2 = _check_out(out, (batch_size, crop_size), audio, (audio, ir2))
      wet = _ag.FftConvolveLtiFn.apply(audio, ir2, int(start), int(crop_size))
      if out is None:
        return wet
      if accumulate:
        out += wet
      else:
        out.copy_(wet)
      return out
    return fft_convolve_lti(audio, ir2, int(start), int(crop_size), out=out,
                            accumulate=accumulate)
  if ir_size >= FFT_CONVOLVE_MIN_IR:
    # time-varying filter with long impulse responses (several IR frames of >= 2048
    # taps): no reference configuration does this; the reference's own framed
    # algorithm on cuFFT
    if out is not None:
      # the result is a fresh tensor: out is written only after every read
      _check_out(out, (batch_size, crop_size), audio)
    wet = _fft_convolve_cufft(audio, impulse_response, n_ir_frames, frame_size,
                              fft_size, int(start), int(crop_size))
    if out is None:
      return wet
    if accumulate:
      out += wet
    else:
      out.copy_(wet)
    return out
  if _requires_grad(audio, impulse_response):
    # time-varying FIR under training (FIRFilter, short reverbs): CUDA backward
    # kernels for both operands (csrc/fir_backward.cuh)
    if out is not None:
      # the backward reads the operands it saved: not the ones out= overwrites
      audio, impulse_response = _check_out(out, (batch_size, crop_size), audio,
                                           (audio, impulse_response))
    from ddsp_b200 import autograd as _ag
    wet = _ag.FirTimeVaryingFn.apply(audio, impulse_response, padding, int(start))
    if out is None:
      return wet
    if accumulate:
      out += wet
    else:
      out.copy_(wet)
    return out
  if out is None:
    out = torch.empty((batch_size, crop_size), dtype=torch.float32,
                      device=audio.device)
    accumulate = False
  else:
    audio, impulse_response = _check_out(out, (batch_size, crop_size), audio,
                                         (audio, impulse_response))
  impulse_response = impulse_response.contiguous()
  _launch('ddsp_b200_fir_time_varying', audio, impulse_response, out, batch_size,
          audio_size, n_ir_frames, ir_size, ir_batch, _lib.PADDING[padding], int(start),
          int(bool(accumulate)))
  return _wrote(out)


@on_operands_device
def frequency_filter(audio, magnitudes, window_size: int = 0,
                     padding: Text = 'same'):
  """core.frequency_filter (core.py:1628-1655).  When grad is enabled and an input
  requires it, impulse responses under FFT_CONVOLVE_MIN_IR taps route to
  `autograd.FrequencyFilterFn` (one backward call for both gradients); longer ones
  compose `FrequencyImpulseResponseFn` with fft_convolve's long-IR route."""
  if _requires_grad(audio, magnitudes):
    sm = _shape(magnitudes)
    nb = int(sm[-1])
    _check_n_frequencies(nb)
    # the shape checks do not depend on the taps: they raise before the library is asked
    _fft_convolve_geometry(_shape(audio), tuple(sm[:-1]) + (1,), padding, -1)
    s = _ir_size(nb, int(window_size))
    _, _, _, _, _, _, out_len, crop_size = _fft_convolve_geometry(
        _shape(audio), tuple(sm[:-1]) + (s,), padding, -1)
    if s < FFT_CONVOLVE_MIN_IR and out_len == crop_size:
      from ddsp_b200 import autograd as _ag
      return _ag.FrequencyFilterFn.apply(audio, magnitudes, int(window_size), padding)
  impulse_response = frequency_impulse_response(magnitudes,
                                                window_size=window_size)
  return fft_convolve(audio, impulse_response, padding=padding)


# ----------------------------------------------------------------------------
# Windowed-sinc filters (core.py:1568-1625, 1658-1690)
# ----------------------------------------------------------------------------
def sinc(x, threshold=1e-20):
  """core.sinc (core.py:1568-1573): sin(pi x) / (pi x), with |x| < threshold
  replaced by threshold.  Elementwise torch on whatever device x lives on."""
  x = _as_f32(x)
  x = torch.where(torch.abs(x) < threshold, torch.full_like(x, threshold), x)
  x = np.pi * x
  return torch.sin(x) / x


def _sinc_geometry(cutoff_shape, window_size, sample_rate):
  """Taps, impulse-response shape and cutoff scale of sinc_impulse_response
  (core.py:1576-1625), from static shapes only.  The response has the broadcast
  shape of cutoff [..., 1] and [1, 1, S]: a scalar gives [1, 1, S], [B, F, 1] gives
  [B, F, S] and [F, 1] gives one shared response of F frames, [1, F, S]."""
  if isinstance(window_size, bool) or int(window_size) != window_size or window_size < 0:
    raise ValueError(f'window_size must be a non-negative integer, got {window_size}.')
  if len(cutoff_shape) and cutoff_shape[-1] != 1:
    raise ValueError('cutoff_frequency must have a last axis of size 1 ([batch, '
                     f'n_frames, 1]); got shape {tuple(cutoff_shape)}.')
  s = 2 * (int(window_size) // 2) + 1
  lead = tuple(cutoff_shape[:-1]) if len(cutoff_shape) else ()
  shape = (1,) * max(0, 2 - len(lead)) + lead + (s,)
  # the reference scales with `*=` in float32; here the caller's array is left alone.
  # As there, a rate of 0 raises ZeroDivisionError and a negative one is accepted
  # (sinc is even, so it gives the positive rate's response and gradient).
  scale = 1.0 if sample_rate is None else float(np.float32(2.0 / float(sample_rate)))
  return s, shape, scale


def sinc_impulse_response_forward(cutoff, s, shape, scale, high_pass):
  """`ddsp_b200_sinc_impulse_response` on a float32 CUDA cutoff -> [shape] taps."""
  ir = torch.empty(shape, dtype=torch.float32, device=cutoff.device)
  _launch('ddsp_b200_sinc_impulse_response', cutoff, ir, cutoff.numel(), s, scale,
          int(bool(high_pass)))
  return ir


def sinc_impulse_response(cutoff_frequency, window_size: int = 512,
                          sample_rate: Optional[int] = None, high_pass: bool = False):
  """core.sinc_impulse_response (core.py:1576-1625): Hamming-windowed sinc low-pass
  (or, with high_pass, its complement) of 2 (window_size // 2) + 1 taps, normalised to
  unit DC gain.  Routes to `autograd.SincImpulseResponseFn` when grad is enabled and the
  cutoff requires it."""
  s, shape, scale = _sinc_geometry(_shape(cutoff_frequency), window_size, sample_rate)
  cutoff = torch_float32(cutoff_frequency)
  if _requires_grad(cutoff):
    from ddsp_b200 import autograd as _ag
    return _ag.SincImpulseResponseFn.apply(cutoff, s, shape, scale, bool(high_pass))
  return sinc_impulse_response_forward(cutoff, s, shape, scale, high_pass)


def sinc_filter_forward(audio, cutoff, s, scale, high_pass, padding, cutoff_batch, n_frames):
  """`ddsp_b200_sinc_filter` on float32 CUDA audio [B, N] and cutoff
  [cutoff_batch * n_frames] -> [B, N] ('same') or [B, N + S - 1] ('valid')."""
  b, n = audio.shape
  out_len = n if padding == 'same' else n + s - 1
  out = torch.empty((b, out_len), dtype=torch.float32, device=audio.device)
  _launch('ddsp_b200_sinc_filter', audio, cutoff, out, b, n, n_frames, s, cutoff_batch,
          scale, int(bool(high_pass)), _lib.PADDING[padding], 0)
  return out


@on_operands_device
def sinc_filter(audio, cutoff_frequency, window_size: int = 512,
                sample_rate: Optional[int] = None, padding: Text = 'same',
                high_pass: bool = False):
  """core.sinc_filter (core.py:1658-1690): audio [B, N] through the sinc filters of
  cutoff_frequency [B or 1, F, 1] (or a scalar, or [F, 1]), with fft_convolve's framing
  and delay compensation.  Under FFT_CONVOLVE_MIN_IR taps, and where the reference's
  crop is not empty, the fused kernels build the taps on chip (under grad through
  `autograd.SincFilterFn`); otherwise sinc_impulse_response feeds fft_convolve."""
  s, ir_shape, scale = _sinc_geometry(_shape(cutoff_frequency), window_size, sample_rate)
  _, _, si, _, _, _, out_len, crop_size = _fft_convolve_geometry(
      _shape(audio), ir_shape, padding, -1)
  if s < FFT_CONVOLVE_MIN_IR and out_len == crop_size:
    cutoff_batch, n_frames = si[0], si[1]
    audio = torch_float32(audio)
    cutoff = torch_float32(cutoff_frequency)
    if _requires_grad(audio, cutoff):
      from ddsp_b200 import autograd as _ag
      return _ag.SincFilterFn.apply(audio, cutoff, s, scale, bool(high_pass), padding,
                                    cutoff_batch, n_frames)
    return sinc_filter_forward(audio, cutoff, s, scale, high_pass, padding, cutoff_batch,
                               n_frames)
  impulse_response = sinc_impulse_response(cutoff_frequency, window_size=window_size,
                                            sample_rate=sample_rate, high_pass=high_pass)
  return fft_convolve(audio, impulse_response, padding=padding)


# ----------------------------------------------------------------------------
# Modulated delay (core.py:1168-1214, 1285-1314; effects.py:328-394)
# ----------------------------------------------------------------------------
def _per_sample_shape(x, batch_size, n_samples, name):
  """The [B, N] or [B, 1] shape of a [B, N, 1] / [B, N] control or of the
  per-item [B, 1, 1] / [B, 1] that TensorFlow broadcasts (static shape only)."""
  shape = _shape(x)
  if len(shape) == 3 and shape[2] == 1:
    shape = shape[:2]
  if len(shape) != 2 or shape[0] != batch_size or shape[1] not in (1, n_samples):
    raise ValueError(f'{name} must be [batch, n_samples(, 1)] or [batch, 1(, 1)] '
                     f'for audio of shape ({batch_size}, {n_samples}); got '
                     f'{_shape(x)}.')
  return shape


def _per_sample(x, shape, batch_size, n_samples):
  return torch_float32(x).reshape(shape).expand(batch_size, n_samples).contiguous()


@on_operands_device
def mod_delay(audio, gain, phase, max_length, scale=1.0, offset=0.0, add_dry=False):
  """`[add_dry] audio + gain * variable_length_delay(phase * scale + offset, audio,
  max_length)` in one kernel (csrc/mod_delay.cuh); `phase * scale + offset` is two
  float32 roundings, as ModDelay's host arithmetic.  gain None means 1.  Routes to
  `autograd.ModDelayFn` when grad is enabled and an input requires it."""
  sa = _shape(audio)
  if len(sa) != 2:
    raise ValueError(f'audio must be [batch, n_samples]; got {sa}.')
  batch_size, n_samples = sa
  if int(max_length) != max_length or max_length < 1:
    raise ValueError(f'max_length must be a positive integer; got {max_length}.')
  if n_samples < 1:
    raise ValueError(f'audio must have at least one sample; got {sa}.')
  phase_shape = _per_sample_shape(phase, batch_size, n_samples, 'phase')
  if gain is not None:
    gain = _per_sample(gain, _per_sample_shape(gain, batch_size, n_samples, 'gain'),
                       batch_size, n_samples)
  phase = _per_sample(phase, phase_shape, batch_size, n_samples)
  audio = torch_float32(audio)
  args = (int(max_length), float(np.float32(scale)), float(np.float32(offset)),
          bool(add_dry))
  if torch.is_grad_enabled() and any(t is not None and t.requires_grad
                                     for t in (audio, gain, phase)):
    from ddsp_b200 import autograd as _ag
    return _ag.ModDelayFn.apply(audio, gain, phase, *args)
  return mod_delay_forward(audio, gain, phase, *args)


def mod_delay_forward(audio, gain, phase, max_length, scale, offset, add_dry):
  """The forward kernel on [B, N] float32 CUDA tensors (gain may be None)."""
  out = torch.empty_like(audio)
  _launch('ddsp_b200_mod_delay_forward', audio, phase, gain, out, audio.shape[0],
          audio.shape[1], max_length, scale, offset, int(add_dry))
  return out


@on_operands_device
def variable_length_delay(phase, audio, max_length: int = 512):
  """core.variable_length_delay (core.py:1285-1314): audio delayed by
  phase * max_length samples with linear interpolation, the reference's wrap
  included (phase in ((L-1)/L, 1] blends the oldest sample with the current one;
  phase 1 is no delay)."""
  return mod_delay(audio, None, phase, max_length)


# ----------------------------------------------------------------------------
# Wavetable synthesis (core.py:1217-1282)
# ----------------------------------------------------------------------------
def _linear_lookup_shapes(phase, wavetables):
  """(B, N, W, per_sample) of linear_lookup's operands; ValueError otherwise."""
  sp, sw = _shape(phase), _shape(wavetables)
  if len(sp) not in (2, 3) or (len(sp) == 3 and sp[2] != 1) or sp[1] < 1:
    raise ValueError(f'phase {sp} must be [batch, n_samples] or [batch, n_samples, 1].')
  b, n = sp[:2]
  ok = (len(sw) == 2 and sw[0] == b) or (len(sw) == 3 and sw[0] == b and sw[1] in (1, n))
  if not ok or sw[-1] < 1:
    raise ValueError(f'wavetables {sw} must be [{b}, n_wavetable], [{b}, 1, n_wavetable] or '
                     f'[{b}, {n}, n_wavetable] for phase {sp}.')
  return b, n, sw[-1], len(sw) == 3 and sw[1] == n and n > 1


@on_operands_device
def linear_lookup(phase, wavetables):
  """core.linear_lookup (core.py:1168-1214): phase [B, N] or [B, N, 1] reads
  wavetables [B, W], [B, 1, W] (one table per item) or [B, N, W] (one per sample) with
  linear interpolation, column W being column 0 again -> [B, N].

  The weights are the reference's own, relu(1 - |phase - lin_j| W) with lin the float32
  linspace(0, 1, W + 1), evaluated in float32 at the few columns that can carry weight: a
  phase outside [0, 1] is not wrapped, it gets partial weights or none.  Routes to
  `autograd.LinearLookupFn` when grad is enabled and an input requires it (TensorFlow's
  subgradients: d phase is 0 on a grid point)."""
  b, n, w, per_sample = _linear_lookup_shapes(phase, wavetables)
  if w > _lib.LOOKUP_MAX_W:
    raise NotImplementedError(f'linear_lookup: {w} wavetable columns; at most '
                              f'{_lib.LOOKUP_MAX_W} are supported.')
  p = torch_float32(phase)
  tab = torch_float32(wavetables, p.device)
  if _requires_grad(p, tab):
    from ddsp_b200 import autograd as _ag
    return _ag.LinearLookupFn.apply(p, tab, per_sample)
  return linear_lookup_forward(p, tab, per_sample)


def linear_lookup_forward(p, tab, per_sample):
  """`ddsp_b200_linear_lookup_forward` on float32 CUDA operands."""
  b, n = p.shape[:2]
  out = torch.empty((b, n), dtype=torch.float32, device=p.device)
  if b == 0:
    return out
  _launch('ddsp_b200_linear_lookup_forward', p, tab, out, b, n, tab.shape[-1],
          int(per_sample))
  return out


def harmonic_distribution_to_wavetable(harmonic_distribution, n_wavetable=2048):
  """core.harmonic_distribution_to_wavetable (core.py:1217-1235): one period of
  the harmonic series [batch, time, n_harmonics] as [batch, time, n_wavetable]
  samples, irfft of the distribution padded with DC in front, times W / 2.  A
  differentiable torch op on the input's device and floating dtype."""
  hd = (harmonic_distribution if torch.is_tensor(harmonic_distribution)
        else torch.as_tensor(np.asarray(harmonic_distribution, np.float32)))
  n_pad = int(n_wavetable / 2 - hd.shape[-1])
  fft_in = torch.nn.functional.pad(hd, (1, n_pad))
  return torch.fft.irfft(fft_in) * (n_wavetable / 2)


def _frame_rows(x, name):
  """(B, F) of a [B, F, 1] or [B, F] control (static shape only)."""
  shape = _shape(x)
  if len(shape) == 3 and shape[2] == 1:
    shape = shape[:2]
  if len(shape) != 2:
    raise ValueError(f'{name} must be [batch, n_frames, 1]; got {_shape(x)}.')
  return shape


@on_operands_device
def wavetable_synthesis(frequencies, amplitudes, wavetables, n_samples: int = 64000,
                        sample_rate: int = 16000):
  """core.wavetable_synthesis (core.py:1238-1282) on one fused kernel
  (csrc/wavetable.cuh): the phase is exact and the tables are read at frame rate.

  frequencies, amplitudes: [batch, n_frames, 1]; wavetables: [batch, n_wavetable]
  or [batch, 1, n_wavetable] (static) or [batch, n_frames_w, n_wavetable], which
  is interpolated in time with core.resample's 'linear' taps.  When f0 and the
  amplitudes have one frame count that divides n_samples, the kernel reads them
  at frame rate; otherwise both are first resampled to n_samples (f0 'linear',
  amplitudes 'window') and the same kernel runs at hop 1.  Routes to
  `autograd.WavetableSynthesisFn` when grad is enabled and an input requires it."""
  n = int(n_samples)
  bf, ff = _frame_rows(frequencies, 'frequencies')
  ba, fa = _frame_rows(amplitudes, 'amplitudes')
  sw = _shape(wavetables)
  if len(sw) == 2:
    sw = (sw[0], 1, sw[1])
  if len(sw) != 3 or not bf == ba == sw[0]:
    raise ValueError(f'frequencies {_shape(frequencies)}, amplitudes '
                     f'{_shape(amplitudes)} and wavetables {_shape(wavetables)} must '
                     'share the batch size; wavetables are [batch, n_wavetable] or '
                     '[batch, n_frames, n_wavetable].')
  _check_window_upsample((ba, fa, 1), n, True)
  f0 = torch_float32(frequencies).reshape(bf, ff)
  amps = torch_float32(amplitudes).reshape(ba, fa)
  tab = torch_float32(wavetables).reshape(sw)
  if ff == fa and n % ff == 0:
    method = 'window'
  else:
    f0 = resample(f0[:, :, None], n)[:, :, 0].contiguous()
    amps = resample(amps[:, :, None], n, method='window')[:, :, 0].contiguous()
    method = 'linear'
  if torch.is_grad_enabled() and any(t.requires_grad for t in (f0, amps, tab)):
    from ddsp_b200 import autograd as _ag
    return _ag.WavetableSynthesisFn.apply(f0, amps, tab, n, float(sample_rate), method)
  return wavetable_forward(f0, amps, tab, n, float(sample_rate), method)


def wavetable_forward(f0, amps, tab, n_samples, sample_rate, method):
  """The wavetable kernel: f0, amps [B, F] and tables [B, Fw, W], float32 CUDA."""
  b, f = amps.shape
  _, fw, w = tab.shape
  out = torch.empty((b, n_samples), dtype=torch.float32, device=amps.device)
  _launch('ddsp_b200_wavetable_forward', f0, amps, tab, out, b, f, n_samples, fw, w,
          sample_rate, AMP_METHODS[method],
          *_workspace('ddsp_b200_wavetable_workspace', amps.device, b, f))
  return out


# ----------------------------------------------------------------------------
# Mix (processors.py:179-233) and the exponential-decay impulse response
# (effects.py:121-199)
# ----------------------------------------------------------------------------
def _mix_shapes(signal_one, signal_two, mix_level=None):
  """Static checks of Mix: two [B, N, C] signals of one shape and a [B, N, 1] mix
  level.  Returns (B, N, C)."""
  s1, s2 = _shape(signal_one), _shape(signal_two)
  if len(s1) != 3 or len(s2) != 3:
    raise ValueError(
        f'Mix takes 3-D signals [batch, n_samples, n_channels]; got {s1} and {s2}. '
        'The mix level is [batch, n_samples, 1], and broadcasting it against a 2-D '
        'signal [batch, n_samples] gives no crossfade of the two signals.')
  if s1 != s2:
    raise ValueError(f'Mix signals must have one shape; got {s1} and {s2}.')
  if mix_level is not None and _shape(mix_level) != (s1[0], s1[1], 1):
    raise ValueError(f'mix_level must be [{s1[0]}, {s1[1]}, 1]; got {_shape(mix_level)}.')
  return s1


@on_operands_device
def mix(signal_one, signal_two, mix_level):
  """processors.Mix.get_signal (processors.py:217-233): the constant-power crossfade
  sqrt(|m|) s1 + (1 - sqrt(|m - 1|)) s2 in one kernel (csrc/routing.cuh).  Routes to
  `autograd.MixFn` when grad is enabled and an input requires it."""
  _mix_shapes(signal_one, signal_two, mix_level)
  s1, s2, m = (torch_float32(x) for x in (signal_one, signal_two, mix_level))
  if torch.is_grad_enabled() and any(t.requires_grad for t in (s1, s2, m)):
    from ddsp_b200 import autograd as _ag
    return _ag.MixFn.apply(s1, s2, m)
  return mix_forward(s1, s2, m)


def mix_forward(signal_one, signal_two, mix_level):
  """The mix kernel on [B, N, C] / [B, N, 1] float32 CUDA tensors."""
  b, n, c = signal_one.shape
  out = torch.empty_like(signal_one)
  _launch('ddsp_b200_mix_forward', signal_one, signal_two, mix_level, out, b, n, c)
  return out


def _ir_rows(x, name):
  """[rows, 1] or [rows] (the reference's [batch, 1] gain and decay) -> rows."""
  shape = _shape(x)
  if len(shape) not in (1, 2) or (len(shape) == 2 and shape[1] != 1):
    raise ValueError(f'{name} must be [batch, 1]; got {shape}.')
  return shape[0]


@on_operands_device
def exp_decay_ir(gain, decay, reverb_length, noise=None, seed=0, offset=0):
  """ExpDecayReverb._get_ir (effects.py:144-151) on the SCALED gain:
  `(gain * exp(-(2 + exp(decay)) * linspace(0, 1, L))) * noise`, [rows, L], one
  kernel (csrc/routing.cuh).  gain and decay are [rows, 1] (or [1, 1], broadcast);
  the noise is one [1, L] row for every item, `noise` when given, else the Philox
  stream's row 0 at (seed, offset) - `uniform_noise(1, L, seed, offset)`.  Routes to
  `autograd.ExpDecayIrFn` when grad is enabled and gain or decay requires it."""
  rows_g, rows_d = _ir_rows(gain, 'gain'), _ir_rows(decay, 'decay')
  if rows_g != rows_d and 1 not in (rows_g, rows_d):
    raise ValueError(f'gain ({_shape(gain)}) and decay ({_shape(decay)}) do not '
                     'broadcast.')
  length = int(reverb_length)
  if length != reverb_length or length < 1:
    raise ValueError(f'reverb_length must be a positive integer; got {reverb_length}.')
  if noise is not None and _shape(noise) not in ((1, length), (length,)):
    raise ValueError(f'noise must be [1, {length}]; got {_shape(noise)}.')
  rows = max(rows_g, rows_d)
  gain = torch_float32(gain).reshape(-1).expand(rows).contiguous()
  decay = torch_float32(decay).reshape(-1).expand(rows).contiguous()
  if noise is not None:
    noise = torch_float32(noise).reshape(length)
  args = (length, noise, int(seed), int(offset))
  if torch.is_grad_enabled() and (gain.requires_grad or decay.requires_grad):
    from ddsp_b200 import autograd as _ag
    return _ag.ExpDecayIrFn.apply(gain, decay, *args)
  return exp_decay_ir_forward(gain, decay, *args)


def exp_decay_ir_forward(gain, decay, reverb_length, noise, seed, offset):
  """The impulse-response kernel on [rows] float32 CUDA gain and decay."""
  rows = gain.shape[0]
  ir = torch.empty((rows, reverb_length), dtype=torch.float32, device=gain.device)
  _launch('ddsp_b200_exp_decay_ir', gain, decay, noise, seed, offset, ir, rows,
          reverb_length)
  return ir


def uniform_noise(batch_size, n_samples, seed=0, offset=0, device=None):
  """Stand-in for tf.random.uniform([B, N], -1, 1) (synths.py:192-193):
  Philox4x32-10 keyed by `seed`, counter (sample/4, batch, offset)."""
  out = torch.empty((batch_size, n_samples), dtype=torch.float32,
                    device=device or _device())
  _launch('ddsp_b200_uniform_noise', out, batch_size, n_samples, int(seed), int(offset))
  return out


def _noise_backward_takes(f, nb, n_samples, window_size):
  """Whether `ddsp_b200_filtered_noise_backward` takes a shape: an impulse response of
  at least three taps, and 32 frames of noise, gradient and taps within one CTA's
  shared memory."""
  return bool(_lib.load().ddsp_b200_filtered_noise_backward_takes(f, nb, n_samples,
                                                                  window_size))


@on_operands_device
def filtered_noise(magnitudes, n_samples, window_size=257, noise=None, seed=0,
                   offset=0, out=None, accumulate=False):
  """FilteredNoise.get_signal arithmetic (synths.py:181-196): uniform noise ->
  core.frequency_filter (core.py:1628-1655), fused where the shape allows.  Routes to
  `autograd.FilteredNoiseFn` when grad is enabled and the magnitudes require it,
  for the shapes `ddsp_b200_filtered_noise_backward` takes; `out=` and the other
  shapes are refused there (RuntimeError)."""
  sm = _shape(magnitudes)
  if len(sm) != 3:
    raise ValueError('magnitudes must be [batch, n_frames, n_filter_banks], got '
                     f'{sm}.')
  b, f, nb = sm
  n_samples = int(n_samples)
  if noise is not None and _shape(noise) != (b, n_samples):
    raise ValueError(f'noise must be [{b}, {n_samples}], got {_shape(noise)}.')
  frame_size = int(np.ceil(n_samples / f))
  n_audio_frames = -(-n_samples // frame_size)
  if n_audio_frames != f:
    # core.py:1452-1457
    raise ValueError(
        'Number of Audio frames ({}) and impulse response frames ({}) do not '
        'match. For small hop size = ceil(audio_size / n_ir_frames), '
        'number of impulse response frames must be a multiple of the audio '
        'size.'.format(n_audio_frames, f))
  if _requires_grad(magnitudes):
    if out is not None or not _noise_backward_takes(f, nb, n_samples, int(window_size)):
      _no_grad_path('filtered_noise', magnitudes)
    from ddsp_b200 import autograd as _ag
    return _ag.FilteredNoiseFn.apply(magnitudes, n_samples, int(window_size), noise,
                                     int(seed), int(offset))
  magnitudes = torch_float32(magnitudes)
  if noise is not None:
    noise = torch_float32(noise)
  if out is None:
    out = torch.empty((b, n_samples), dtype=torch.float32,
                      device=magnitudes.device)
    accumulate = False
  else:
    magnitudes, noise = _check_out(out, (b, n_samples), magnitudes, (magnitudes, noise))
  _launch('ddsp_b200_filtered_noise_forward', magnitudes, noise, int(seed), int(offset),
          out, b, f, nb, n_samples, int(window_size), int(bool(accumulate)),
          *_workspace('ddsp_b200_filtered_noise_workspace', magnitudes.device, b, f, nb,
                      n_samples, int(window_size)))
  return _wrote(out)


@on_operands_device
def decoder_forward(amps, harmonic_distribution, f0_hz, noise_magnitudes,
                    n_samples, sample_rate=16000, amp_resample_method='window',
                    normalize_below_nyquist=True, window_size=0,
                    initial_bias=-5.0, noise=None, seed=0, offset=0):
  """The `ae.gin` DAG (ae.gin:47-72) from RAW network outputs, two launches:
  Harmonic (exp_sigmoid scaling + Nyquist normalisation fused into the tile
  staging) then FilteredNoise (exp_sigmoid fused likewise) accumulating into the
  same audio buffer (= processors.Add).  Raises NotImplementedError outside the
  fused regime; ProcessorGroup then runs the per-processor path."""
  sh = _shape(harmonic_distribution)
  sm = _shape(noise_magnitudes)
  if len(sh) != 3 or len(sm) != 3:
    raise ValueError(f'decoder inputs must be 3-D, got {sh} and {sm}.')
  b, f, k = sh
  if _shape(amps) != (b, f, 1) or _shape(f0_hz) != (b, f, 1) or sm[:2] != (b, f):
    raise ValueError(
        f'decoder inputs disagree: amps {_shape(amps)}, f0_hz {_shape(f0_hz)}, '
        f'harmonic_distribution {sh}, noise_magnitudes {sm}.')
  if amp_resample_method not in AMP_METHODS:
    raise NotImplementedError(amp_resample_method)
  n_samples = int(n_samples)
  if noise is not None and _shape(noise) != (b, n_samples):
    raise ValueError(f'noise must be [{b}, {n_samples}], got {_shape(noise)}.')
  amps = torch_float32(amps)
  hd = torch_float32(harmonic_distribution)
  f0_hz = torch_float32(f0_hz)
  mags = torch_float32(noise_magnitudes)
  if noise is not None:
    noise = torch_float32(noise)
  _no_grad_path('decoder_forward', amps, hd, f0_hz, mags)
  out = torch.empty((b, n_samples), dtype=torch.float32, device=hd.device)
  flags = _lib.CTL_SCALE | (_lib.CTL_NYQUIST if normalize_below_nyquist else 0)
  _launch('ddsp_b200_decoder_forward', amps, hd, f0_hz, mags, noise, int(seed),
          int(offset), out, b, f, k, sm[2], n_samples, float(sample_rate),
          AMP_METHODS[amp_resample_method], flags, int(window_size), float(initial_bias))
  return out


def noise_controls(magnitudes, initial_bias=-5.0, scale=True):
  """FilteredNoise.get_controls arithmetic (synths.py:165-179).  Routes to
  `autograd.NoiseControlsFn` when grad is enabled and the magnitudes require it."""
  magnitudes = torch_float32(magnitudes)
  if _requires_grad(magnitudes):
    from ddsp_b200 import autograd as _ag
    return _ag.NoiseControlsFn.apply(magnitudes, float(initial_bias), bool(scale))
  out = torch.empty_like(magnitudes)
  _launch('ddsp_b200_noise_controls', magnitudes, out, magnitudes.numel(),
          float(initial_bias), int(bool(scale)))
  return out


@on_operands_device
def add(signal_one, signal_two, out=None):
  """processors.Add.get_signal (processors.py:174-176).  Routes to
  `autograd.AddFn` when grad is enabled, an input requires it and no `out` is
  given."""
  a = torch_float32(signal_one)
  b = torch_float32(signal_two)
  if out is None and torch.is_grad_enabled() and (a.requires_grad or b.requires_grad):
    from ddsp_b200 import autograd as _ag
    return _ag.AddFn.apply(a, b)
  return add_forward(a, b, out)


def add_forward(a, b, out=None):
  """The add kernel on float32 CUDA tensors that broadcast against each other."""
  if a.shape != b.shape:
    a, b = torch.broadcast_tensors(a, b)
    a, b = a.contiguous(), b.contiguous()
  if out is None:
    out = torch.empty_like(a)
  else:
    a, b = _check_out(out, tuple(a.shape), a, (a, b), exact_alias_ok=True)
  _launch('ddsp_b200_add', a, b, out, a.numel())
  return _wrote(out)
