"""Float64 restatement of the inverse-synthesis networks from the reference's semantics
(ddsp/training/nn.py:561-934, encoders.py:129-251, core.py): nn.ResNet and its
layers, encoders.ResnetSinusoidalEncoder after its spectral function, and
encoders.SinusoidalToHarmonicEncoder over nn.RnnSandwich.  Differentiable by torch
autograd.  Parameters are read by name from a dict {parameter name: tensor}, named as
the library's modules name them; the structure (sizes, strides, shortcuts) is restated
here from the reference.

Every 'same' padding is applied in full before a valid convolution or pooling, as
TensorFlow defines it: out = ceil(n / s), total = max((out - 1) s + k - n, 0), the odd
element after."""
import math

import torch
import torch.nn.functional as F

from tests import gru_ref

SIZES = {'small': (32, [2, 3, 4]), 'medium': (32, [3, 4, 6]), 'large': (64, [3, 4, 6])}


def tf_same(n, k, s):
  out = math.ceil(n / s)
  total = max((out - 1) * s + k - n, 0)
  return total // 2, total - total // 2


def conv2d(x, kernel, bias, strides):
  """tf.nn.conv2d(x, kernel, strides, 'SAME') + bias on NHWC x, kernel [kh, kw, in, out]."""
  kh, kw = kernel.shape[:2]
  top, bottom = tf_same(x.shape[1], kh, strides[0])
  left, right = tf_same(x.shape[2], kw, strides[1])
  xp = F.pad(x, (0, 0, left, right, top, bottom))
  y = F.conv2d(xp.permute(0, 3, 1, 2), kernel.permute(3, 2, 0, 1), bias, strides)
  return y.permute(0, 2, 3, 1)


def max_pool(x, pool, strides):
  top, bottom = tf_same(x.shape[1], pool[0], strides[0])
  left, right = tf_same(x.shape[2], pool[1], strides[1])
  xp = F.pad(x, (0, 0, left, right, top, bottom), value=-math.inf)
  return F.max_pool2d(xp.permute(0, 3, 1, 2), pool, strides).permute(0, 2, 3, 1)


def normalize(x, norm_type, eps=1e-5):
  """normalize_op (nn.py:561-575)."""
  b, h, w, c = x.shape
  g = {'instance': c, 'layer': 1, 'group': 32}[norm_type]
  xg = x.reshape(b, h, w, g, c // g)
  mean = xg.mean(dim=(1, 2, 4), keepdim=True)
  var = ((xg - mean)**2).mean(dim=(1, 2, 4), keepdim=True)
  return ((xg - mean) / torch.sqrt(var + eps)).reshape(b, h, w, c)


def norm_relu(x, scale, shift, norm_type):
  return torch.relu(normalize(x, norm_type) * scale.reshape(-1) + shift.reshape(-1))


def _nr(p, prefix, x, norm_type):
  return norm_relu(x, p[prefix + 'scale'], p[prefix + 'shift'], norm_type)


def _conv(p, prefix, x, strides):
  return conv2d(x, p[prefix + 'kernel'], p[prefix + 'bias'], strides)


def residual_layer(p, prefix, x, stride, shortcut, norm_type):
  """nn.ResidualLayer (nn.py:712-756)."""
  r = x
  x = _nr(p, prefix + 'norm_input.', x, norm_type)
  if shortcut:
    r = _conv(p, prefix + 'conv_proj.', x, (1, stride))
  y = _conv(p, prefix + 'bottleneck.0.', x, (1, 1))
  y = _conv(p, prefix + 'bottleneck.1.conv.', _nr(p, prefix + 'bottleneck.1.norm.', y,
                                                  norm_type), (1, stride))
  y = _conv(p, prefix + 'bottleneck.2.conv.', _nr(p, prefix + 'bottleneck.2.norm.', y,
                                                  norm_type), (1, 1))
  return y + r


def residual_stack(p, prefix, x, filters, blocks, strides, norm_type):
  """nn.ResidualStack (nn.py:759-802)."""
  i = 0
  for _, n_layers, stride in zip(filters, blocks, strides):
    x = residual_layer(p, f'{prefix}layers.{i}.', x, stride, True, norm_type)
    i += 1
    for _ in range(1, n_layers):
      x = residual_layer(p, f'{prefix}layers.{i}.', x, 1, False, norm_type)
      i += 1
  return _nr(p, f'{prefix}layers.{i}.', x, norm_type)


def resnet(p, prefix, x, size, norm_type='layer'):
  """nn.ResNet (nn.py:805-839)."""
  ch, blocks = SIZES[size]
  x = _conv(p, prefix + 'layers.0.', x, (1, 2))
  x = max_pool(x, (1, 3), (1, 2))
  x = residual_stack(p, prefix + 'layers.2.', x, [ch, 2 * ch, 4 * ch], blocks, [1, 2, 2],
                     norm_type)
  return residual_stack(p, prefix + 'layers.3.', x, [8 * ch], [3], [2], norm_type)


def resnet_sinusoidal(p, mag, size, keys):
  """ResnetSinusoidalEncoder.call (encoders.py:154-173) after spectral_fn."""
  x = resnet(p, 'resnet.', mag[..., None], size)
  x = x.reshape(x.shape[0], x.shape[1], -1)
  return {k: x @ p[f'dense_outs.{i}.kernel'] + p[f'dense_outs.{i}.bias']
          for i, k in enumerate(keys)}


# ---- SinusoidalToHarmonicEncoder ---------------------------------------------------
def hz_to_midi(hz):
  notes = 12.0 * (torch.log2(hz) - math.log2(440.0)) + 69.0
  return torch.where(hz <= 0.0, torch.zeros_like(notes), notes)


def _hz_to_midi_scalar(hz):
  return 0.0 if hz <= 0.0 else 12.0 * (math.log2(hz) - math.log2(440.0)) + 69.0


def hz_to_unit(hz, hz_min, hz_max):
  lo, hi = _hz_to_midi_scalar(hz_min), _hz_to_midi_scalar(hz_max)
  return (hz_to_midi(hz) - lo) / (hi - lo)


def unit_to_hz(unit, hz_min, hz_max):
  lo, hi = _hz_to_midi_scalar(hz_min), _hz_to_midi_scalar(hz_max)
  midi = lo + (hi - lo) * unit
  return 440.0 * 2.0**((midi - 69.0) / 12.0)


def exp_sigmoid(x):
  return 2.0 * torch.sigmoid(x)**math.log(10.0) + 1e-7


def frequencies_softmax(x, depth, hz_min, hz_max):
  """core.frequencies_softmax on [B, T, n depth] (or [B, T, depth] for n = 1)."""
  x = x.reshape(*x.shape[:-1], -1, depth)
  probs = torch.softmax(x, dim=-1)
  unit = (torch.linspace(0.0, 1.0, depth, dtype=x.dtype) * probs).sum(-1)
  return unit_to_hz(unit, hz_min, hz_max)


def fc(p, prefix, x):
  """nn.Fc: Dense -> LayerNormalization (epsilon 1e-3) -> leaky ReLU 0.2."""
  x = x @ p[prefix + '0.kernel'] + p[prefix + '0.bias']
  x = F.layer_norm(x, (x.shape[-1],), p[prefix + '1.gamma'], p[prefix + '1.beta'], 1e-3)
  return F.leaky_relu(x, 0.2)


def rnn_sandwich(p, prefix, x, layers=2):
  for i in range(layers):
    x = fc(p, f'{prefix}0.{i}.', x)
  x = gru_ref.gru(x, p[prefix + '1.rnn.kernel'], p[prefix + '1.rnn.recurrent_kernel'],
                  p[prefix + '1.rnn.bias'])
  for i in range(layers):
    x = fc(p, f'{prefix}2.{i}.', x)
  return x


def sinusoidal_to_harmonic(p, sin_freqs, sin_amps, n_harmonics=100, sample_rate=16000):
  """SinusoidalToHarmonicEncoder.call (encoders.py:207-251) with net = RnnSandwich."""
  x = torch.cat([hz_to_unit(sin_freqs, 0.0, sample_rate / 2.0), sin_amps], dim=-1)
  x = rnn_sandwich(p, 'net.', x)
  harm_amp = exp_sigmoid(x @ p['amp_out.kernel'] + p['amp_out.bias'])
  harm_dist = exp_sigmoid(x @ p['hd_out.kernel'] + p['hd_out.bias'])
  f0_hz = frequencies_softmax(x @ p['f0_out.kernel'] + p['f0_out.bias'], 64, 20.0, 1200.0)
  harm_freqs = f0_hz * torch.arange(1, n_harmonics + 1, dtype=f0_hz.dtype)
  harm_dist = torch.where(harm_freqs >= sample_rate / 2.0, torch.zeros_like(harm_dist),
                          harm_dist)
  total = harm_dist.sum(-1, keepdim=True)
  harm_dist = harm_dist / torch.where(total == 0.0, torch.full_like(total, 1e-7), total)
  return {'harm_amp': harm_amp, 'harm_dist': harm_dist, 'f0_hz': f0_hz}
