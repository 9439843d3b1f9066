"""Processor / ProcessorGroup / Add / Mix / Crop with the reference's protocol
(`ddsp/processors.py:37-263`) - the drop-in boundary of this library.

Tensors are torch CUDA float32; the arithmetic runs in libddsp_b200.so.
"""
from typing import Dict, Text, Any

import torch

from ddsp_b200 import core
from ddsp_b200 import dags

TensorDict = Dict[Text, Any]


class Processor:
  """Abstract base class for signal processors (processors.py:37-76)."""

  def __init__(self, name: Text, trainable: bool = False):
    self.name = name
    self.trainable = trainable

  @core.on_operands_device
  def __call__(self, *args, return_outputs_dict: bool = False, **kwargs):
    return self.call(*args, return_outputs_dict=return_outputs_dict, **kwargs)

  def call(self, *args, return_outputs_dict: bool = False, **kwargs):
    """processors.py:53-68."""
    for k in ['training', 'mask']:
      if k in kwargs:
        _ = kwargs.pop(k)
    controls = self.get_controls(*args, **kwargs)
    signal = self.get_signal(**controls)
    if return_outputs_dict:
      return dict(signal=signal, controls=controls)
    else:
      return signal

  def get_controls(self, *args, **kwargs) -> TensorDict:
    raise NotImplementedError

  def get_signal(self, *args, **kwargs):
    raise NotImplementedError


class ProcessorGroup(dags.DAGLayer):
  """String Processor() objects together (processors.py:79-158)."""

  def __init__(self, dag: dags.DAG, **kwarg_processors):
    super().__init__(dag, **kwarg_processors)
    self.processor_names = self.module_names
    self._pattern_cache = None    # (dag identity, result of _decoder_pattern)

  @property
  def processors(self):
    return [getattr(self, name) for name in self.processor_names]

  @core.on_operands_device
  def __call__(self, inputs: TensorDict, return_outputs_dict: bool = False,
               **kwargs):
    return self.call(inputs, return_outputs_dict=return_outputs_dict, **kwargs)

  def call(self, inputs: TensorDict, return_outputs_dict: bool = False,
           **kwargs):
    """processors.py:121-131.

    When only the signal is asked for and the DAG is the `ae.gin` decoder
    (Harmonic, FilteredNoise, Add of their two signals), the three nodes run as
    the fused pipeline (noise accumulates into the harmonic buffer: one audio
    tensor instead of three).  With return_outputs_dict=True every node's signal
    and controls are materialised, as the reference's contract requires.
    """
    if not return_outputs_dict:
      fused = self._try_fused_decoder(inputs, **kwargs)
      if fused is not None:
        return fused
    controls = self.get_controls(inputs, **kwargs)
    signal = self.get_signal(controls)
    if return_outputs_dict:
      return dict(signal=signal, controls=controls)
    else:
      return signal

  def get_controls(self, inputs: TensorDict, **kwargs) -> TensorDict:
    """processors.py:133-146 - run the DAG, return the nested outputs dict."""
    return super().call(inputs, **kwargs)

  def get_signal(self, outputs: TensorDict):
    """processors.py:148-158."""
    return outputs['out']['signal']

  # -- fused fast path ---------------------------------------------------------
  def _decoder_pattern(self):
    """Returns (harmonic, noise, harmonic_keys, noise_keys) if the DAG is
    exactly [Harmonic(a,b,c), FilteredNoise(m), Add(two signals)], else None."""
    key = (id(self.dag), len(self.dag))
    if self._pattern_cache is not None and self._pattern_cache[0] == key:
      mods = self._pattern_cache[1]
      # the DAG is fixed at construction; only re-check what attribute
      # assignment could have changed since (the modules themselves)
      if all(getattr(self, n, None) is m for n, m in mods):
        return self._pattern_cache[2]
    pat = self._decoder_pattern_uncached()
    self._pattern_cache = (key, [(node[0], getattr(self, node[0], None))
                                 for node in self.dag], pat)
    return pat

  def _decoder_pattern_uncached(self):
    from ddsp_b200 import synths  # local import: synths imports this module
    if len(self.dag) != 3:
      return None
    mods = [getattr(self, node[0], None) for node in self.dag]
    kinds = [type(m) for m in mods]
    if kinds[2] is not Add:
      return None
    if kinds[:2] == [synths.Harmonic, synths.FilteredNoise]:
      h_i, n_i = 0, 1
    elif kinds[:2] == [synths.FilteredNoise, synths.Harmonic]:
      h_i, n_i = 1, 0
    else:
      return None
    harm, noise = mods[h_i], mods[n_i]
    want = {f'{harm.name}/signal', f'{noise.name}/signal'}
    if set(self.dag[2][1]) != want or len(self.dag[2][1]) != 2:
      return None
    if harm.n_samples != noise.n_samples:
      return None
    return harm, noise, list(self.dag[h_i][1]), list(self.dag[n_i][1])

  def _try_fused_decoder(self, inputs, **kwargs):
    pat = self._decoder_pattern()
    if pat is None:
      return None
    harm, noise, h_keys, n_keys = pat
    outputs = {'inputs': inputs}
    outputs.update(inputs)
    h_in = [core.nested_lookup(k, outputs) for k in h_keys]
    n_in = [core.nested_lookup(k, outputs) for k in n_keys]
    for k in ['training', 'mask']:
      kwargs.pop(k, None)
    # one Philox offset per call, whichever route runs (so the noise stream of
    # call i does not depend on whether the shape was inside the fused regime)
    offset = noise.next_offset()
    if (harm.scale_fn is core.exp_sigmoid and noise.scale_fn is core.exp_sigmoid
        and not kwargs and len(h_in) == 3 and len(n_in) == 1):
      # raw network outputs -> audio in two launches, controls never hit HBM
      try:
        return core.decoder_forward(
            h_in[0], h_in[1], h_in[2], n_in[0], n_samples=harm.n_samples,
            sample_rate=harm.sample_rate,
            amp_resample_method=harm.amp_resample_method,
            normalize_below_nyquist=harm.normalize_below_nyquist,
            window_size=noise.window_size, initial_bias=noise.initial_bias,
            noise=noise.injected_noise, seed=noise.seed, offset=offset)
      except NotImplementedError:
        pass   # outside the fused regime: per-processor path below
    audio = harm.get_signal(**harm.get_controls(*h_in, **kwargs))
    # the noise is added into the harmonic buffer through out=, which autograd does
    # not differentiate: a harmonic signal that carries a graph is refused here, with
    # the way to train, rather than by the out= check below
    core._no_grad_path('ProcessorGroup', audio)
    return noise.get_signal(out=audio, accumulate=True, offset=offset,
                            **noise.get_controls(*n_in, **kwargs))


class Add(Processor):
  """Sum two signals (processors.py:162-176)."""

  def __init__(self, name: Text = 'add'):
    super().__init__(name=name)

  def get_controls(self, signal_one, signal_two) -> TensorDict:
    return {'signal_one': signal_one, 'signal_two': signal_two}

  def get_signal(self, signal_one, signal_two):
    return core.add(signal_one, signal_two)


class Mix(Processor):
  """Constant-power crossfade between two signals (processors.py:179-233).

  The signals are [batch, n_samples, n_channels] and the mix level
  [batch, n_samples, 1], the shapes the reference's own test uses: broadcasting the
  mix level against 2-D signals gives no crossfade, so those are refused."""

  def __init__(self, name: Text = 'mix'):
    super().__init__(name=name)

  def get_controls(self, signal_one, signal_two, nn_out_mix_level) -> TensorDict:
    """processors.py:192-215: sigmoid of the mix logits at frame rate, resampled
    ('linear') to the signals' length - differentiable under grad."""
    n_time_one = int(core._shape(signal_one)[1])   # pylint: disable=protected-access
    n_time_two = int(core._shape(signal_two)[1])   # pylint: disable=protected-access
    if n_time_one != n_time_two:
      raise ValueError('The two signals must have the same length instead of'
                       '{} and {}'.format(n_time_one, n_time_two))
    core._mix_shapes(signal_one, signal_two)       # pylint: disable=protected-access
    mix_level = torch.sigmoid(core.torch_float32(nn_out_mix_level))
    mix_level = core.resample(mix_level, n_time_one)
    return {'signal_one': signal_one, 'signal_two': signal_two,
            'mix_level': mix_level}

  def get_signal(self, signal_one, signal_two, mix_level):
    """processors.py:217-233."""
    return core.mix(signal_one, signal_two, mix_level)


class Crop(Processor):
  """Remove audio generated from padding frames (processors.py:236-263): torch
  slicing of the time axis of 2-D or 3-D audio, a view."""

  def __init__(self, frame_size: int, crop_location: Text = 'back',
               name: Text = 'crop'):
    super().__init__(name=name)
    self.frame_size = frame_size
    self.crop_location = crop_location

  def get_controls(self, audio) -> TensorDict:
    return {'audio': audio}

  def get_signal(self, audio):
    half_pad_amount = int(self.frame_size // 2)  # Symmetric even.
    pad_amount = 2 * half_pad_amount
    if self.crop_location == 'front':
      return audio[:, pad_amount:]
    elif self.crop_location == 'center':
      return audio[:, half_pad_amount:-half_pad_amount]
    elif self.crop_location == 'back':
      return audio[:, :-pad_amount]
    else:
      raise ValueError(f'Crop_location: ({self.crop_location}), must be '
                       '"front", "center", or "back".')
