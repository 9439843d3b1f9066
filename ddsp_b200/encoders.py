"""encoders.ZEncoder and encoders.MfccTimeDistributedRnnEncoder
(ddsp/training/encoders.py:27-127), the encoder of ae.gin and of the z branch of
z_midiae.gin: MFCCs of the audio, instance-normalized, through a GRU and a Dense layer
to a latent z, resampled to the frame rate of the other conditioning.  The MFCCs
(`csrc/mel.cuh`), the GRU's recurrence (`csrc/gru.cuh`) and the resample run on the
library's CUDA kernels; the normalization and the Dense layer are torch ops."""
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
