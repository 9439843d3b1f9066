"""decoders.RnnFcDecoder (ddsp/training/decoders.py:26-109), the network every published
audio model of the reference decodes with (ae.gin, solo_instrument.gin, vst*.gin): one
FcStack per input, their concatenation through a GRU, the inputs again beside the GRU's
output, an output FcStack and a Dense layer split into the output dict.  The GRU's
recurrence runs on the CUDA kernels of `csrc/gru.cuh`; the rest are torch ops."""
import torch

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
