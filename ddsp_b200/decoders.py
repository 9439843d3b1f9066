"""decoders.RnnFcDecoder (ddsp/training/decoders.py:26-109), the network every published
audio model of the reference decodes with (ae.gin, solo_instrument.gin, vst*.gin): one
FcStack per input, their concatenation through a GRU, the inputs again beside the GRU's
output, an output FcStack and a Dense layer split into the output dict.  The GRU's
recurrence runs on the CUDA kernels of `csrc/gru.cuh`; the rest are torch ops.

decoders.MidiToHarmonicDecoder and decoders.DilatedConvDecoder (decoders.py:163-285) are
the MIDI autoencoders' decoders, on nn.DilatedConvStack: cuDNN convolutions, and residual
sites on the fused kernel of `csrc/norm.cuh`."""
import torch

from ddsp_b200 import core
from ddsp_b200 import nn


class RnnFcDecoder(torch.nn.Module):
  """RNN and FC stacks for f0 and loudness, with the reference's arguments and defaults.

  Called with a features dict it reads `input_keys` from it; called with tensors it
  takes them in `input_keys` order.  Returns {key: [B, T, size]} for `output_splits`.
  stateless=True (nn.StatelessRnn, streaming) and rnn_type='lstm' raise
  NotImplementedError.  Parameters are created at the first call (the input widths are
  fixed then), as Keras builds its layers."""

  def __init__(self,
               rnn_channels=512,
               rnn_type='gru',
               ch=512,
               layers_per_stack=3,
               stateless=False,
               input_keys=('ld_scaled', 'f0_scaled', 'z'),
               output_splits=(('amps', 1), ('harmonic_distribution', 40))):
    super().__init__()
    if stateless:
      raise NotImplementedError('RnnFcDecoder: stateless=True (nn.StatelessRnn) is not '
                                'supported; the stateful decoder is')
    self.stateless = False
    self.input_keys = tuple(input_keys)
    self.output_splits = tuple((k, int(n)) for k, n in output_splits)
    self.output_keys = tuple(k for k, _ in self.output_splits)
    self.input_stacks = torch.nn.ModuleList(
        [nn.FcStack(ch, layers_per_stack) for _ in self.input_keys])
    self.rnn = nn.Rnn(rnn_channels, rnn_type)
    self.out_stack = nn.FcStack(ch, layers_per_stack)
    self.dense_out = nn.Dense(sum(n for _, n in self.output_splits))

  def forward(self, *inputs):
    if len(inputs) == 1 and isinstance(inputs[0], dict):
      missing = [k for k in self.input_keys if k not in inputs[0]]
      if missing:
        raise KeyError(f'RnnFcDecoder: the features lack {missing}')
      inputs = [inputs[0][k] for k in self.input_keys]
    if len(inputs) != len(self.input_keys):
      raise ValueError(f'RnnFcDecoder: {len(inputs)} inputs for the input keys '
                       f'{self.input_keys}')
    inputs = [stack(x) for stack, x in zip(self.input_stacks, inputs)]
    x = self.rnn(torch.cat(inputs, dim=-1))
    x = self.out_stack(torch.cat(inputs + [x], dim=-1))
    return nn.split_to_dict(self.dense_out(x), self.output_splits)


def _inputs(name, keys, inputs):
  """The tensors of `keys` from a features dict, or the positional tensors in that
  order."""
  if len(inputs) == 1 and isinstance(inputs[0], dict):
    missing = [k for k in keys if k not in inputs[0]]
    if missing:
      raise KeyError(f'{name}: the features lack {missing}')
    inputs = [inputs[0][k] for k in keys]
  if len(inputs) != len(keys):
    raise ValueError(f'{name}: {len(inputs)} inputs for the input keys {keys}')
  return list(inputs)


class MidiToHarmonicDecoder(torch.nn.Module):
  """MIDI pitch (and a latent z) to synthesizer controls: z_pitch [B, T, 1] through `net`
  (with [z_pitch, z] when z is given), Normalize('layer') (`norm`, when norm), Dense
  (`dense_out`) and split_to_dict(output_splits).  z_pitch is added to 'f0_midi' when
  f0_residual, and 'f0_hz' = midi_to_hz(f0_midi, midi_zero_silence) joins the outputs.
  z_vel is unused, as in the reference."""

  def __init__(self, net=None, f0_residual=True, norm=True,
               output_splits=(('f0_midi', 1), ('amplitudes', 1),
                              ('harmonic_distribution', 60), ('magnitudes', 65)),
               midi_zero_silence=True):
    super().__init__()
    self.output_splits = tuple((k, int(n)) for k, n in output_splits)
    self.n_out = sum(n for _, n in self.output_splits)
    self.output_keys = [k for k, _ in self.output_splits] + ['f0_hz']
    self.net = net
    self.f0_residual = f0_residual
    self.dense_out = nn.Dense(self.n_out)
    self.norm = nn.Normalize('layer') if norm else None
    self.midi_zero_silence = midi_zero_silence

  def forward(self, z_pitch, z_vel=None, z=None):
    x = self.net(z_pitch) if z is None else self.net([z_pitch, z])
    if self.norm is not None:
      x = self.norm(x)
    outputs = nn.split_to_dict(self.dense_out(x), self.output_splits)
    if self.f0_residual:
      outputs['f0_midi'] = outputs['f0_midi'] + z_pitch
    outputs['f0_hz'] = core.midi_to_hz(outputs['f0_midi'],
                                       midi_zero_silence=self.midi_zero_silence)
    return outputs


class DilatedConvDecoder(torch.nn.Module):
  """WaveNet-style decoder: the input_keys concatenated through nn.DilatedConvStack
  (`dilated_conv_stack`), conditioned on the conditioning_keys (concatenated, and
  through precondition_stack if given) when there are any, then Dense (`dense_out`) and
  split_to_dict(output_splits).  Called with a features dict it reads the input keys and
  then the conditioning keys; called with tensors it takes them in that order.  A
  precondition_stack without conditioning keys raises ValueError, as in the reference;
  resample_stride > 1 (upsampling) and spectral_norm=True raise NotImplementedError."""

  def __init__(self, ch=256, kernel_size=3, layers_per_stack=5, stacks=2, dilation=2,
               norm_type='layer', resample_stride=1, stacks_per_resample=1,
               resample_after_convolve=True, input_keys=('ld_scaled', 'f0_scaled'),
               output_splits=(('amps', 1), ('harmonic_distribution', 60)),
               conditioning_keys=('z'), precondition_stack=None, spectral_norm=False,
               ortho_init=False):
    super().__init__()
    self.conditioning_keys = [] if conditioning_keys is None else list(conditioning_keys)
    self.input_keys = list(input_keys) + self.conditioning_keys
    self.output_splits = tuple((k, int(n)) for k, n in output_splits)
    self.output_keys = [k for k, _ in self.output_splits]
    self.n_conditioning = len(self.conditioning_keys)
    self.conditional = bool(self.conditioning_keys)
    if not self.conditional and precondition_stack is not None:
      raise ValueError('You must specify conditioning keys if you specify'
                       'a precondition stack.')
    self.precondition_stack = precondition_stack
    self.dilated_conv_stack = nn.DilatedConvStack(
        ch=ch, kernel_size=kernel_size, layers_per_stack=layers_per_stack, stacks=stacks,
        dilation=dilation, norm_type=norm_type,
        resample_type='upsample' if resample_stride > 1 else None,
        resample_stride=resample_stride, stacks_per_resample=stacks_per_resample,
        resample_after_convolve=resample_after_convolve, conditional=self.conditional,
        spectral_norm=spectral_norm, ortho_init=ortho_init)
    self.dense_out = nn.Dense(sum(n for _, n in self.output_splits))

  def _parse_inputs(self, inputs):
    if self.conditional:
      x = torch.cat(inputs[:-self.n_conditioning], dim=-1)
      z = torch.cat(inputs[-self.n_conditioning:], dim=-1)
      if self.precondition_stack is not None:
        z = self.precondition_stack(z)
      return [x, z]
    return torch.cat(inputs, dim=-1)

  def forward(self, *inputs, training=None):
    inputs = _inputs('DilatedConvDecoder', self.input_keys, inputs)
    x = self.dilated_conv_stack(self._parse_inputs(inputs))
    return nn.split_to_dict(self.dense_out(x), self.output_splits)
