"""encoders.ZEncoder and encoders.MfccTimeDistributedRnnEncoder
(ddsp/training/encoders.py:27-127), the encoder of ae.gin and of the z branch of
z_midiae.gin: MFCCs of the audio, instance-normalized, through a GRU and a Dense layer
to a latent z, resampled to the frame rate of the other conditioning.  The MFCCs
(`csrc/mel.cuh`), the GRU's recurrence (`csrc/gru.cuh`) and the resample run on the
library's CUDA kernels; the normalization and the Dense layer are torch ops.

encoders.ResnetSinusoidalEncoder and encoders.SinusoidalToHarmonicEncoder
(encoders.py:129-251) are the two networks of models.InverseSynthesis: audio -> log-mel
-> ResNet -> sinusoid controls, and sinusoids -> harmonic controls.  The log-mel
(`csrc/mel.cuh`), the ResNet's normalize-ReLU sites (`csrc/norm.cuh`) and the GRU of
nn.RnnSandwich run on the library's CUDA kernels; convolutions, Dense layers and the
output scalings are torch ops.

encoders.OneHotEncoder, encoders.HarmonicToMidiEncoder and encoders.ExpressionEncoder
(encoders.py:254-284, 419-517) are the MIDI autoencoders' encoders; the last two run a
network such as nn.DilatedConvStack, whose residual sites run on `csrc/norm.cuh`."""
import inspect

import torch

from ddsp_b200 import core
from ddsp_b200 import nn
from ddsp_b200 import spectral_ops


class ZEncoder(torch.nn.Module):
  """Base class of the encoders that make a latent z: subclasses define compute_z().

  The input keys are compute_z()'s argument names, then 'f0_scaled', which is read only
  for its time axis.  Called with a features dict it reads the input keys from it (a
  missing one raises KeyError); called with tensors it takes them in that order.
  Returns {'z': [B, time_steps, z_dims]}."""

  def __init__(self, input_keys=None):
    super().__init__()
    if not input_keys:
      input_keys = [name for name, p in inspect.signature(self.compute_z).parameters.items()
                    if p.kind == inspect.Parameter.POSITIONAL_OR_KEYWORD]
    self.input_keys = list(input_keys) + ['f0_scaled']

  def forward(self, *inputs):
    if len(inputs) == 1 and isinstance(inputs[0], dict):
      missing = [k for k in self.input_keys if k not in inputs[0]]
      if missing:
        raise KeyError(f'{type(self).__name__}: the features lack {missing}')
      inputs = [inputs[0][k] for k in self.input_keys]
    if len(inputs) != len(self.input_keys):
      raise ValueError(f'{type(self).__name__}: {len(inputs)} inputs for the input keys '
                       f'{self.input_keys}')
    time_steps = int(inputs[-1].shape[1])
    return {'z': self.expand_z(self.compute_z(*inputs[:-1]), time_steps)}

  def expand_z(self, z, time_steps):
    """z with a time axis ([B, z_dims] -> [B, 1, z_dims]), linearly resampled
    (core.resample, add_endpoint=True) to time_steps frames when it has another
    count."""
    if z.dim() == 2:
      z = z[:, None, :]
    if int(z.shape[1]) != time_steps:
      z = core.resample(z, time_steps)
    return z

  def compute_z(self, *inputs):
    """Takes in input tensors and returns a latent tensor z."""
    raise NotImplementedError


class MfccTimeDistributedRnnEncoder(ZEncoder):
  """MFCCs as latent variables, distributed across time steps: z from 'audio'
  ([B, n_samples] at 16 kHz).  z_time_steps (63, 125, 250, 500 or 1000 MFCC frames
  for 4 s of audio) picks the FFT size and overlap.  rnn_type 'lstm' raises
  NotImplementedError, as nn.Rnn does.  Parameters are created at the first call, as
  Keras builds its layers."""

  def __init__(self, rnn_channels=512, rnn_type='gru', z_dims=32, z_time_steps=250,
               input_keys=None):
    super().__init__(input_keys)
    if z_time_steps not in [63, 125, 250, 500, 1000]:
      raise ValueError('`z_time_steps` currently limited to 63,125,250,500 and 1000')
    self.z_audio_spec = {
        '63': {'fft_size': 2048, 'overlap': 0.5},
        '125': {'fft_size': 1024, 'overlap': 0.5},
        '250': {'fft_size': 1024, 'overlap': 0.75},
        '500': {'fft_size': 512, 'overlap': 0.75},
        '1000': {'fft_size': 256, 'overlap': 0.75},
    }
    self.fft_size = self.z_audio_spec[str(z_time_steps)]['fft_size']
    self.overlap = self.z_audio_spec[str(z_time_steps)]['overlap']
    self.z_norm = nn.Normalize('instance')
    self.rnn = nn.Rnn(rnn_channels, rnn_type)
    self.dense_out = nn.Dense(z_dims)

  def compute_z(self, audio):
    mfccs = spectral_ops.compute_mfcc(audio, lo_hz=20.0, hi_hz=8000.0,
                                      fft_size=self.fft_size, mel_bins=128, mfcc_bins=30,
                                      overlap=self.overlap, pad_end=True)
    z = self.z_norm(mfccs[:, :, None, :])[:, :, 0, :]
    z = self.rnn(z)
    return self.dense_out(z)


def _audio(features, name):
  if isinstance(features, dict):
    if 'audio' not in features:
      raise KeyError(f'{name}: the features lack [\'audio\']')
    return features['audio']
  return features


class ResnetSinusoidalEncoder(torch.nn.Module):
  """Audio [B, n_samples] (or a features dict's 'audio') straight to synthesizer
  controls: spectral_fn (log-mel) -> nn.ResNet(size) -> the frequency and channel axes
  flattened -> one Dense per (key, width) of output_splits.  Returns {key: [B, T, width]}.

  The defaults are the reference's, including size='tiny', which nn.ResNet does not
  have (KeyError at construction, as in the reference): pretrain_model.gin sets 'small'
  and a log-mel of 229 bins (fft_size 2048, overlap 0.75), for which 64000 samples give
  a ResNet output [B, 125, 8, 1024] and Dense inputs of 8192."""

  def __init__(self, output_splits=(('frequencies', 100 * 64), ('amplitudes', 100),
                                    ('noise_magnitudes', 60)),
               spectral_fn=spectral_ops.compute_logmel, size='tiny'):
    super().__init__()
    self.output_splits = tuple((k, int(v)) for k, v in output_splits)
    self.output_keys = [k for k, _ in self.output_splits]
    self.spectral_fn = spectral_fn
    self.resnet = nn.ResNet(size=size)
    self.dense_outs = torch.nn.ModuleList([nn.Dense(v) for _, v in self.output_splits])

  def forward(self, features, training=True):
    mag = self.spectral_fn(_audio(features, 'ResnetSinusoidalEncoder'))
    x = self.resnet(mag[:, :, :, None])
    x = x.reshape(int(x.shape[0]), int(x.shape[1]), -1)
    return {key: layer(x) for layer, key in zip(self.dense_outs, self.output_keys)}


def _f0_softmax(x):
  return core.frequencies_softmax(x, depth=64, hz_min=20.0, hz_max=1200.0)


class SinusoidalToHarmonicEncoder(torch.nn.Module):
  """Harmonic controls from sinusoidal ones: sin_freqs (Hz) mapped by hz_to_unit over
  [0, Nyquist] and concatenated with sin_amps, through `net` (e.g. nn.RnnSandwich; a
  dict output's 'out' is taken), then three Dense heads: harm_amp [.., 1] and harm_dist
  [.., n_harmonics] through amp_scale_fn (exp_sigmoid), f0_hz [.., 1] through
  freq_scale_fn (frequencies_softmax, depth 64, 20-1200 Hz).  Harmonics at or above
  Nyquist are zeroed and the distribution renormalized with safe_divide.  Returns
  {'harm_amp', 'harm_dist', 'f0_hz'}."""

  def __init__(self, net=None, n_harmonics=100, f0_depth=64, amp_scale_fn=core.exp_sigmoid,
               freq_scale_fn=_f0_softmax, sample_rate=16000):
    super().__init__()
    self.n_harmonics = int(n_harmonics)
    self.amp_scale_fn = amp_scale_fn
    self.freq_scale_fn = freq_scale_fn
    self.sample_rate = sample_rate
    self.net = net
    self.amp_out = nn.Dense(1)
    self.hd_out = nn.Dense(n_harmonics)
    self.f0_out = nn.Dense(f0_depth)

  def forward(self, sin_freqs, sin_amps):
    nyquist = self.sample_rate / 2.0
    sin_freqs_unit = core.hz_to_unit(sin_freqs, hz_min=0.0, hz_max=nyquist)
    x = torch.cat([sin_freqs_unit, sin_amps], dim=-1)
    x = self.net(x)
    x = x['out'] if isinstance(x, dict) else x
    harm_amp = self.amp_scale_fn(self.amp_out(x))
    harm_dist = self.amp_scale_fn(self.hd_out(x))
    f0_hz = self.freq_scale_fn(self.f0_out(x))
    harm_freqs = core.get_harmonic_frequencies(f0_hz, self.n_harmonics)
    harm_dist = core.remove_above_nyquist(harm_freqs, harm_dist, self.sample_rate)
    harm_dist = core.safe_divide(harm_dist, torch.sum(harm_dist, dim=-1, keepdim=True))
    return {'harm_amp': harm_amp, 'harm_dist': harm_dist, 'f0_hz': f0_hz}


class OneHotEncoder(ZEncoder):
  """An embedding (nn.get_embedding: `embedding`) of an integer id such as an instrument,
  read from one_hot_key ([B] or [B, 1]): z [B, n_dims] or [B, 1, n_dims].  Unless
  skip_expand, z is given a time axis and repeated over the frames of 'f0_scaled', as
  ZEncoder.expand_z does; with skip_expand it is returned as it is, for broadcasting."""

  def __init__(self, one_hot_key='instrument', vocab_size=1024, n_dims=256,
               skip_expand=True):
    super().__init__(input_keys=[one_hot_key])
    self.one_hot_key = one_hot_key
    self.vocab_size = vocab_size
    self.n_dims = n_dims
    self.skip_expand = skip_expand
    self.embedding = nn.get_embedding(vocab_size=vocab_size, n_dims=n_dims)

  def compute_z(self, one_hot):
    return self.embedding(one_hot)

  def expand_z(self, z, time_steps):
    return z if self.skip_expand else super().expand_z(z, time_steps)


class HarmonicToMidiEncoder(torch.nn.Module):
  """Harmonic synthesizer controls to a MIDI-like encoding: f0_midi, amps, hd and noise
  ([B, T, .] each) concatenated, through `net`, Normalize('layer') (`norm`) and
  Dense(2) (`dense_out`).  Returns {'z_pitch', 'z_vel'} ([B, T, 1] each), with f0_midi
  added to z_pitch when f0_residual."""

  def __init__(self, net=None, f0_residual=True):
    super().__init__()
    self.net = net
    self.f0_residual = f0_residual
    self.dense_out = nn.Dense(2)
    self.norm = nn.Normalize('layer')

  def forward(self, f0_midi, amps, hd, noise):
    x = torch.cat([f0_midi, amps, hd, noise], dim=-1)
    x = self.dense_out(self.norm(self.net(x)))
    z_pitch = x[..., 0:1]
    z_vel = x[..., 1:2]
    if self.f0_residual:
      z_pitch = z_pitch + f0_midi
    return {'z_pitch': z_pitch, 'z_vel': z_vel}


class ExpressionEncoder(ZEncoder):
  """A latent from frame-rate features: the input_keys ([B, T, .] each) concatenated,
  through `net`, Normalize('layer') (`norm`) and Dense(z_dims) (`dense_out`), averaged
  over time when pool_time, then expanded to the frames of 'f0_scaled'.  The reference's
  'audio' input (MFCCs) cannot run there (it pops from a tuple), so 'audio' in
  input_keys raises NotImplementedError."""

  def __init__(self, net=None, z_dims=128, input_keys=('f0_scaled', 'ld_scaled'),
               mfcc_bins=60, fft_size=1024, mel_bins=128, pool_time=True):
    if 'audio' in input_keys:
      raise NotImplementedError("ExpressionEncoder: 'audio' in input_keys (MFCC inputs) "
                                'is not supported')
    super().__init__(list(input_keys))
    self.compute_mfccs = False
    self.mfcc_bins = mfcc_bins
    self.fft_size = fft_size
    self.mel_bins = mel_bins
    self.pool_time = pool_time
    self.net = net
    self.norm = nn.Normalize('layer')
    self.dense_out = nn.Dense(z_dims)

  def compute_z(self, *inputs):
    z = self.dense_out(self.norm(self.net(torch.cat(inputs, dim=-1))))
    if self.pool_time:
      z = torch.mean(z, dim=1, keepdim=True)
    return z
