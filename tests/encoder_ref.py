"""Float64 restatements of nn.normalize_op and nn.Normalize (nn.py:302-320, 561-603) and
of encoders.MfccTimeDistributedRnnEncoder.compute_z and expand_z
(encoders.py:27-127).  normalize_op and normalize take NumPy arrays or torch tensors
(differentiable by autograd); the encoder composes tests/mel_ref.py's MFCC, this
normalization, tests/gru_ref.py's GRU, a Dense layer and tests/routing_ref.py's linear
resample, all in float64."""
from tests import gru_ref
from tests import mel_ref
from tests import routing_ref

Z_AUDIO_SPEC = {63: (2048, 0.5), 125: (1024, 0.5), 250: (1024, 0.75), 500: (512, 0.75),
                1000: (256, 0.75)}


def normalize_op(x, norm_type='layer', eps=1e-5):
  """x [B, H, W, C]: each item's channel groups ({'instance': C, 'layer': 1,
  'group': 32}) minus their mean over H, W and the group's channels, over the square
  root of their population variance plus eps."""
  if norm_type is None:
    return x
  shape = tuple(x.shape)
  groups = {'instance': shape[-1], 'layer': 1, 'group': 32}[norm_type]
  g = x.reshape(shape[:-1] + (groups, shape[-1] // groups))
  mean = g.mean(axis=(1, 2, 4), keepdims=True)
  var = ((g - mean)**2).mean(axis=(1, 2, 4), keepdims=True)
  return ((g - mean) / (var + eps)**0.5).reshape(shape)


def normalize(x, norm_type, scale, shift):
  """nn.Normalize with weights scale and shift ([1, 1, 1, C]), on x of rank 2, 3 or 4."""
  n_dims = len(x.shape)
  x4 = x[:, None, None, :] if n_dims == 2 else x[:, :, None, :] if n_dims == 3 else x
  y = normalize_op(x4, norm_type) * scale + shift
  return y[:, 0, 0, :] if n_dims == 2 else y[:, :, 0, :] if n_dims == 3 else y


def encoder_z(audio, params, z_time_steps, time_steps):
  """z [B, time_steps, z_dims] of MfccTimeDistributedRnnEncoder from audio [B, N]
  (float64 torch), with params {named_parameters() name: float64 tensor}."""
  fft_size, overlap = Z_AUDIO_SPEC[z_time_steps]
  mfccs = mel_ref.compute_mfcc(audio, 20.0, 8000.0, fft_size, 128, 30, overlap, True)
  z = normalize(mfccs, 'instance', params['z_norm.scale'], params['z_norm.shift'])
  z = gru_ref.gru(z, params['rnn.rnn.kernel'], params['rnn.rnn.recurrent_kernel'],
                  params['rnn.rnn.bias'])
  z = z @ params['dense_out.kernel'] + params['dense_out.bias']
  return z if z.shape[1] == time_steps else routing_ref.resample(z, time_steps)
