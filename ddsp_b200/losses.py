"""Losses with the reference's constructors and semantics (`ddsp/losses.py`): the
multi-scale spectral loss (`losses.py:102-243`, torch with cuFFT on the GPU) and the
consistency losses of the self-supervised pitch model (`losses.py:489-1076`).  The
Gaussian mixtures of `KDEConsistencyLoss` and `TWMLoss` are evaluated per frame by
the CUDA kernels of `csrc/consistency.cuh` (`autograd.MixtureNLLFn`, `CombNLLFn`);
the [B, T, K]-sized elementwise work around them is torch autograd.  The HMM of
`HmmTranscriber` (`losses.py:247-345`) runs on the kernels of `csrc/hmm.cuh`, and
`wasserstein_distance` (`losses.py:641-686`) on those of `csrc/wasserstein.cuh`.
The perceptual losses (`EmbeddingLoss`, `PretrainedCREPEEmbeddingLoss` and
`PretrainedCREPE`, `losses.py:353-486`) frame and normalise the audio on the kernels
of `csrc/crepe.cuh`, with their backward, around a CREPE network the caller supplies.
`LossGroup` (`losses.py:50-98`) runs a DAG of losses."""
import functools
import math
import re

import numpy as np
import torch

from ddsp_b200 import _lib
from ddsp_b200 import autograd
from ddsp_b200 import core
from ddsp_b200 import dags
from ddsp_b200 import spectral_ops
from ddsp_b200.core import hz_to_midi, safe_divide


def mean_difference(target, value, loss_type='L1', weights=None):
  """losses.mean_difference (losses.py:102-127)."""
  difference = target - value
  weights = 1.0 if weights is None else weights
  loss_type = loss_type.upper()
  if loss_type == 'L1':
    return torch.mean(torch.abs(difference * weights))
  elif loss_type == 'L2':
    return torch.mean(difference**2 * weights)
  elif loss_type == 'COSINE':
    cos = torch.nn.functional.cosine_similarity(target, value, dim=-1)
    return torch.mean((1.0 - cos) * weights)   # weights is 1.0 when none were given
  else:
    raise ValueError('Loss type ({}), must be '
                     '"L1", "L2", or "COSINE"'.format(loss_type))


def _snake_case(name):
  """A Keras layer's default name: its class name in snake case."""
  name = re.sub(r'(.)([A-Z][a-z]+)', r'\1_\2', name)
  return re.sub(r'([a-z])([A-Z])', r'\1_\2', name).lower()


class Loss:
  """losses.Loss (losses.py:41-47): a callable with a `name`; `get_losses_dict`
  returns {name: call(...)}."""

  def __init__(self, name=None):
    self.name = name if name is not None else _snake_case(type(self).__name__)

  @core.on_operands_device
  def __call__(self, *args, **kwargs):
    return self.call(*args, **kwargs)

  def get_losses_dict(self, *args, **kwargs):
    return {self.name: self(*args, **kwargs)}


class LossGroup(dags.DAGLayer):
  """losses.LossGroup (losses.py:50-98): the losses of a DAG, each node a loss (or its
  keyword name) and the nested keys of its inputs, e.g.
  [['f0_loss', ['f0_midi', 'f0_midi_pred', 'f0_loss_weights']], ...].  Keyword losses
  become attributes of the group; `name=` is split off as the group's own name.  Called
  on a dict of outputs, it returns the flat {loss.name: value} of every loss, in
  `loss_names` order; a keyword loss that no node runs raises KeyError there."""

  def __init__(self, dag, **kwarg_losses):
    super().__init__(dag, **kwarg_losses)
    if kwarg_losses.get('name') is None:
      self.name = 'loss_group'
    self.loss_names = self.module_names

  @property
  def losses(self):
    return [getattr(self, name) for name in self.loss_names]

  def call(self, outputs, **kwargs):
    dag_outputs = super().call(outputs, **kwargs)
    loss_outputs = {}
    for k in self.loss_names:
      loss_outputs.update(dag_outputs[k])
    return loss_outputs

  def get_losses_dict(self, outputs, **kwargs):
    """The same dict as calling the group."""
    return self(outputs, **kwargs)


class SpectralLoss:
  """Multi-scale spectrogram loss (losses.py:130-243)."""

  def __init__(self,
               fft_sizes=(2048, 1024, 512, 256, 128, 64),
               loss_type='L1',
               mag_weight=1.0,
               delta_time_weight=0.0,
               delta_freq_weight=0.0,
               cumsum_freq_weight=0.0,
               logmag_weight=0.0,
               loudness_weight=0.0,
               name='spectral_loss'):
    self.name = name
    self.fft_sizes = fft_sizes
    self.loss_type = loss_type
    self.mag_weight = mag_weight
    self.delta_time_weight = delta_time_weight
    self.delta_freq_weight = delta_freq_weight
    self.cumsum_freq_weight = cumsum_freq_weight
    self.logmag_weight = logmag_weight
    self.loudness_weight = loudness_weight
    self.spectrogram_ops = [
        functools.partial(spectral_ops.compute_mag, size=size)
        for size in self.fft_sizes]

  @core.on_operands_device
  def __call__(self, target_audio, audio, weights=None):
    return self.call(target_audio, audio, weights=weights)

  def get_losses_dict(self, target_audio, audio, **kwargs):
    """losses.Loss.get_losses_dict (losses.py:60-66)."""
    return {self.name: self.call(target_audio, audio, **kwargs)}

  def _fusable(self, target_audio, audio, weights):
    """The ae.gin configuration (L1 on magnitudes and log-magnitudes,
    ae.gin:39-41) on CUDA tensors runs through three hand-written kernels per FFT
    size around cuFFT instead of ~70 elementwise launches.  So does any
    configuration with a delta_time, delta_freq or cumsum_freq term, 'L1' or 'L2',
    at FFT sizes up to 8192 (spectral_terms)."""
    if not (torch.is_tensor(audio) and audio.is_cuda and torch.is_tensor(target_audio)
            and target_audio.is_cuda and weights is None
            and audio.dim() == 2 and target_audio.shape == audio.shape
            and all(int(sz) >= 16 and (int(sz) & (int(sz) - 1)) == 0
                    for sz in self.fft_sizes)):
      return False
    loss_type = self.loss_type.upper()
    if max(self.delta_time_weight, self.delta_freq_weight, self.cumsum_freq_weight) > 0:
      return (loss_type in ('L1', 'L2') and
              all(int(sz) // 2 + 1 <= _lib.SPECTRAL_TERMS_MAX_BINS for sz in self.fft_sizes))
    return loss_type == 'L1' and (self.mag_weight > 0 or self.logmag_weight > 0)

  def _call_fused(self, target_audio, audio):
    return spectral_ops.SpectralLossFn.apply(
        target_audio.detach(), audio, tuple(int(s) for s in self.fft_sizes),
        max(self.mag_weight, 0.0), max(self.logmag_weight, 0.0),
        max(self.delta_time_weight, 0.0), max(self.delta_freq_weight, 0.0),
        max(self.cumsum_freq_weight, 0.0), self.loss_type)

  def call(self, target_audio, audio, weights=None):
    if self._fusable(target_audio, audio, weights):
      loss = self._call_fused(target_audio, audio)
    else:
      loss = self._call_spectrograms(target_audio, audio, weights)
    if self.loudness_weight > 0:
      # losses.py:236-241: n_fft = 2048 and every other argument at its default,
      # whatever the audio's sample rate
      target = spectral_ops.compute_loudness(target_audio, n_fft=2048)
      value = spectral_ops.compute_loudness(audio, n_fft=2048)
      loss = loss + self.loudness_weight * mean_difference(
          target, value, self.loss_type, weights=weights)
    return loss

  def _call_spectrograms(self, target_audio, audio, weights):
    loss = 0.0
    diff = core.diff
    for loss_op in self.spectrogram_ops:
      target_mag = loss_op(target_audio)
      value_mag = loss_op(audio)
      if self.mag_weight > 0:
        loss = loss + self.mag_weight * mean_difference(
            target_mag, value_mag, self.loss_type, weights=weights)
      if self.delta_time_weight > 0:
        loss = loss + self.delta_time_weight * mean_difference(
            diff(target_mag, 1), diff(value_mag, 1), self.loss_type,
            weights=weights)
      if self.delta_freq_weight > 0:
        loss = loss + self.delta_freq_weight * mean_difference(
            diff(target_mag, 2), diff(value_mag, 2), self.loss_type,
            weights=weights)
      if self.cumsum_freq_weight > 0:
        loss = loss + self.cumsum_freq_weight * mean_difference(
            torch.cumsum(target_mag, 2), torch.cumsum(value_mag, 2),
            self.loss_type, weights=weights)
      if self.logmag_weight > 0:
        loss = loss + self.logmag_weight * mean_difference(
            spectral_ops.safe_log(target_mag), spectral_ops.safe_log(value_mag),
            self.loss_type, weights=weights)
    return loss


# ------------------------------------------------------------------------------
# Perceptual losses (losses.py:353-486)
# ------------------------------------------------------------------------------
class EmbeddingLoss(Loss):
  """losses.EmbeddingLoss (losses.py:356-388): weight * mean_difference of the
  embeddings `pretrained_model` gives the target audio and the audio, so that the
  synthesizer learns to match what a pretrained network hears.  pretrained_model is
  any callable on float32 audio tensors: a `PretrainedCREPE`, or a TorchScript module
  or plain function.  With weight <= 0 it returns the Python float 0.0 and does not
  call the model."""

  def __init__(self, weight=1.0, loss_type='L1', pretrained_model=None,
               name='embedding_loss'):
    super().__init__(name)
    self.weight = weight
    self.loss_type = loss_type
    self.pretrained_model = pretrained_model

  def call(self, target_audio, audio):
    loss = 0.0
    if self.weight > 0.0:
      audio = core.torch_float32(audio)
      target_audio = core.torch_float32(target_audio, audio.device)
      target_emb = self.pretrained_model(target_audio)
      synth_emb = self.pretrained_model(audio)
      loss = self.weight * mean_difference(target_emb, synth_emb, self.loss_type)
    return loss


# Scales that bring each layer's embedding loss to comparable sizes (losses.py:400-414).
CREPE_LAYER_SCALE = {
    'conv1-BN': 1.3,
    'conv1-maxpool': 1.0,
    'conv2-BN': 1.4,
    'conv2-maxpool': 1.1,
    'conv3-BN': 1.9,
    'conv3-maxpool': 1.6,
    'conv4-BN': 1.5,
    'conv4-maxpool': 1.4,
    'conv5-BN': 1.9,
    'conv5-maxpool': 1.7,
    'conv6-BN': 30,
    'conv6-maxpool': 25,
    'classifier': 130,
}


class PretrainedCREPEEmbeddingLoss(EmbeddingLoss):
  """losses.PretrainedCREPEEmbeddingLoss (losses.py:391-421): an EmbeddingLoss on the
  activations of `activation_layer` of a CREPE network (`PretrainedCREPE`), weighted by
  20 * CREPE_LAYER_SCALE[activation_layer] * weight.  model_capacity is the network, a
  torch.nn.Module (see PretrainedCREPE).  An unknown activation_layer raises KeyError
  before the network is looked at."""

  def __init__(self, weight=1.0, loss_type='L1', model_capacity='tiny',
               activation_layer='classifier', name='pretrained_crepe_embedding_loss'):
    scale = CREPE_LAYER_SCALE[activation_layer]
    super().__init__(
        weight=20.0 * scale * weight,
        loss_type=loss_type,
        name=name,
        pretrained_model=PretrainedCREPE(model_capacity=model_capacity,
                                         activation_layer=activation_layer))


class _Captured(Exception):
  """Stops a network's forward once the activation layer has run."""


class PretrainedCREPE:
  """losses.PretrainedCREPE (losses.py:424-486): the activations of one layer of a CREPE
  network on normalised frames of the audio, [batch, n_frames, -1].

  model_capacity is the network, a torch.nn.Module mapping frames [M, 1024] to its
  output; activation_layer names one of its submodules (`named_modules()`), whose
  output is taken by a forward hook, removed after each call, and the forward stops
  there.  The crepe package's size names ('tiny', 'small', 'medium', 'large', 'full')
  name weights that are not shipped here and raise NotImplementedError; anything but a
  torch.nn.Module raises TypeError, and so do TorchScript modules, which cannot take
  submodule hooks (pass such a network, or any callable on audio, to
  EmbeddingLoss(pretrained_model=...) instead).  An unknown activation_layer raises
  ValueError.

  The frames come from `autograd.CrepeLossFramesFn`, so gradients flow from the
  activations back to the audio.  With trainable=False the network runs on detached
  copies of its parameters (torch.func.functional_call): no gradient reaches them and
  their .grad stays None, while the caller's requires_grad flags and the module's
  train/eval mode are left as they are.  With trainable=True the module is called
  directly.

  The activation [M, ...] is reshaped to [batch, n_frames, -1] in the network's own
  memory order: a torch conv net's [M, C, T, 1] flattens channel-major where Keras's
  [M, T, 1, C] flattens time-major.  The L1, L2 and COSINE embedding losses compare the
  two embeddings element by element (COSINE along the last axis, where both share the
  order), so they do not depend on it."""

  def __init__(self, model_capacity='tiny', activation_layer='conv5-maxpool',
               name='pretrained_crepe', trainable=False):
    if isinstance(model_capacity, str) and model_capacity in _CREPE_CAPACITIES:
      raise NotImplementedError(
          f"losses.PretrainedCREPE: the '{model_capacity}' weights come with the crepe "
          'package and are not available here; pass the network as a torch.nn.Module.')
    if isinstance(model_capacity, torch.jit.ScriptModule):
      raise TypeError('losses.PretrainedCREPE: TorchScript modules cannot take the '
                      'forward hook that reads activation_layer; pass a callable on '
                      'audio to EmbeddingLoss(pretrained_model=...) instead.')
    if not isinstance(model_capacity, torch.nn.Module):
      raise TypeError('losses.PretrainedCREPE: model_capacity must be a torch.nn.Module, '
                      f'got {type(model_capacity).__name__}')
    self.layer_names = [n for n, _ in model_capacity.named_modules() if n]
    if activation_layer not in self.layer_names:
      raise ValueError('activation layer {} not found, valid names are {}'.format(
          activation_layer, self.layer_names))
    self.name = name
    self.trainable = trainable
    self._model_capacity = model_capacity
    self._activation_layer = activation_layer
    self._model = model_capacity
    self.frame_length = spectral_ops.CREPE_FRAME_SIZE

  def frame_audio(self, audio, hop_length=1024, center=True):
    """Frames [batch, n_frames, 1024] of audio [batch, length]: 512 zeros on both sides
    when `center`, frames of 1024 every hop_length (1 + (padded - 1024) // hop_length of
    them, or none when the padded audio is shorter than a frame), each normalised to
    (x - mean) / (sqrt(var) + 1e-5) with tf.nn.moments' mean and population variance.
    Differentiable in the audio."""
    shape = core._shape(audio)
    if len(shape) != 2:
      raise ValueError(f'audio must be [batch, length], got shape {tuple(shape)}')
    if int(hop_length) != hop_length or hop_length < 1:
      raise ValueError(f'hop_length must be a positive integer, got {hop_length}')
    return autograd.CrepeLossFramesFn.apply(core.torch_float32(audio), int(hop_length),
                                            bool(center))

  @core.on_operands_device
  def __call__(self, audio):
    return self.call(audio)

  def call(self, audio):
    """The activations of activation_layer, [batch, n_frames, -1], for audio
    [batch, length] framed every 1024 samples with centring."""
    frames = self.frame_audio(audio)
    batch_size, n_frames = frames.shape[:2]
    outputs = self._activations(frames.reshape(-1, self.frame_length))
    return outputs.reshape(batch_size, n_frames, -1)

  def _activations(self, frames):
    captured = []

    def hook(module, inputs, output):
      captured.append(output)
      raise _Captured

    layer = self._model.get_submodule(self._activation_layer)
    handle = layer.register_forward_hook(hook)
    try:
      if self.trainable:
        self._model(frames)
      else:
        state = {k: v.detach() for k, v in self._model.named_parameters()}
        state.update(self._model.named_buffers())
        torch.func.functional_call(self._model, state, (frames,))
    except _Captured:
      pass
    finally:
      handle.remove()
    if not captured:
      raise RuntimeError(f'losses.PretrainedCREPE: the network did not run '
                         f'{self._activation_layer!r}')
    return captured[0]


_CREPE_CAPACITIES = ('tiny', 'small', 'medium', 'large', 'full')


# ------------------------------------------------------------------------------
# Consistency losses (losses.py:489-578, 689-1076)
# ------------------------------------------------------------------------------
def amp_loss(amp, amp_target, loss_type='L1', weights=None, log=False, amin=1e-5):
  """losses.amp_loss (losses.py:492-504): optionally on a log10 scale."""
  amp = core.torch_float32(amp)
  amp_target = core.torch_float32(amp_target)
  if log:
    amp = core.log10(torch.clamp(amp, min=amin))
    amp_target = core.log10(torch.clamp(amp_target, min=amin))
  return mean_difference(amp, amp_target, loss_type, weights)


def freq_loss(f_hz, f_hz_target, loss_type='L1', weights=None):
  """losses.freq_loss (losses.py:507-513): compared in MIDI."""
  f_midi = hz_to_midi(core.torch_float32(f_hz))
  f_midi_target = hz_to_midi(core.torch_float32(f_hz_target))
  return mean_difference(f_midi, f_midi_target, loss_type, weights)


class FilteredNoiseConsistencyLoss(Loss):
  """losses.FilteredNoiseConsistencyLoss (losses.py:516-530)."""

  def __init__(self, weight=1.0, name=None):
    super().__init__(name)
    self.weight = weight

  def call(self, noise_magnitudes, noise_magnitudes_target):
    return self.weight * amp_loss(noise_magnitudes, noise_magnitudes_target)


class HarmonicConsistencyLoss(Loss):
  """losses.HarmonicConsistencyLoss (losses.py:533-578): a dict of three losses,
  the distribution and f0 terms masked where the target amplitude is below
  `amp_threshold`."""

  def __init__(self, amp_weight=1.0, dist_weight=1.0, f0_weight=1.0, amp_threshold=1e-4,
               name=None):
    super().__init__(name)
    self.amp_weight = amp_weight
    self.dist_weight = dist_weight
    self.f0_weight = f0_weight
    self.amp_threshold = amp_threshold

  def call(self, harm_amp, harm_amp_target, harm_dist, harm_dist_target, f0_hz,
           f0_hz_target):
    harm_amp_target = core.torch_float32(harm_amp_target)
    weights = (harm_amp_target >= self.amp_threshold).to(torch.float32)
    return {
        'harm_amp_loss': self.amp_weight * amp_loss(harm_amp, harm_amp_target),
        'harm_dist_loss': self.dist_weight * amp_loss(harm_dist, harm_dist_target,
                                                      weights=weights),
        'f0_hz_loss': self.f0_weight * freq_loss(f0_hz, f0_hz_target, weights=weights),
    }


class ParamLoss(Loss):
  """losses.ParamLoss (losses.py:1064-1076)."""

  def __init__(self, weight=1.0, loss_type='L1', name=None):
    super().__init__(name)
    self.weight = weight
    self.loss_type = loss_type

  def call(self, pred, target, weights=None):
    loss = mean_difference(core.torch_float32(pred), core.torch_float32(target),
                           self.loss_type, weights)
    return self.weight * loss


def _check_sinusoids(name, pairs):
  """Shape checks made before any device work: each (label, amps, freqs) pair is
  [batch, time, n] with amps and freqs alike, and all share batch and time."""
  frames = None
  for label, a, f in pairs:
    sa, sf = core._shape(a), core._shape(f)
    if len(sa) != 3 or sa != sf:
      raise ValueError(f'{name}: {label} must be two [batch, time, n] arrays of one '
                       f'shape, got {sa} and {sf}')
    if frames is not None and sa[:2] != frames:
      raise ValueError(f'{name}: {label} has [batch, time] {sa[:2]}, the other inputs '
                       f'{frames}')
    frames = sa[:2]


def _check_scale(name, label, scale):
  if not (scale > 0.0 and math.isfinite(scale)):
    raise ValueError(f'{name}: {label} must be positive and finite, got {scale}')


def _log_weights(amps):
  """The mixture weights of `Categorical(probs=amps_norm)` as MixtureSameFamily uses
  them, log_softmax(log p), with exact zeros raised to 1e-7 before normalising
  (losses.py:807-813, 1044-1051)."""
  amps = torch.where(amps == 0.0, torch.full_like(amps, 1e-7), amps)
  probs = safe_divide(amps, torch.sum(amps, dim=-1, keepdim=True))
  return torch.log_softmax(torch.log(probs), dim=-1)


class KDEConsistencyLoss(Loss):
  """losses.KDEConsistencyLoss (losses.py:689-813): -log p(a | b) and -log p(b | a)
  under Gaussian kernel density estimates in MIDI, plus the mean-amplitude match.
  Each direction is one `autograd.MixtureNLLFn` launch forward and one backward;
  gradients reach all four inputs."""

  def __init__(self, weight_a=1.0, weight_b=1.0, weight_mean_amp=1.0, scale_a=0.1,
               scale_b=0.1, name=None):
    super().__init__(name)
    self.weight_a = weight_a
    self.weight_b = weight_b
    self.weight_mean_amp = weight_mean_amp
    self.scale_a = scale_a
    self.scale_b = scale_b

  def call(self, amps_a, freqs_a, amps_b, freqs_b):
    """Scalar: weighted -log p(a|b) - log p(b|a) + the mean-amplitude L1."""
    _check_sinusoids('KDEConsistencyLoss', [('amps_a, freqs_a', amps_a, freqs_a),
                                            ('amps_b, freqs_b', amps_b, freqs_b)])
    if self.weight_a > 0.0:
      _check_scale('KDEConsistencyLoss', 'scale_b', self.scale_b)
    if self.weight_b > 0.0:
      _check_scale('KDEConsistencyLoss', 'scale_a', self.scale_a)
    amps_a, freqs_a, amps_b, freqs_b = (
        core.torch_float32(x) for x in (amps_a, freqs_a, amps_b, freqs_b))
    loss = 0.0
    if self.weight_a > 0.0:
      loss_a = self.nll(amps_a, freqs_a, amps_b, freqs_b, self.scale_b)
      loss = loss + torch.mean(self.weight_a * loss_a)
    if self.weight_b > 0.0:
      loss_b = self.nll(amps_b, freqs_b, amps_a, freqs_a, self.scale_a)
      loss = loss + torch.mean(self.weight_b * loss_b)
    if self.weight_mean_amp > 0.0:
      mean_amp_a = torch.mean(amps_a, dim=-1)
      mean_amp_b = torch.mean(amps_b, dim=-1)
      loss = loss + self.weight_mean_amp * torch.mean(torch.abs(mean_amp_a - mean_amp_b))
    return loss

  def nll(self, amps, freqs, amps_target, freqs_target, scale_target):
    """-log p(source | target), the amplitude-weighted mean over the source
    sinusoids, [batch, time]."""
    _check_sinusoids('KDEConsistencyLoss.nll',
                     [('amps, freqs', amps, freqs),
                      ('amps_target, freqs_target', amps_target, freqs_target)])
    _check_scale('KDEConsistencyLoss.nll', 'scale_target', scale_target)
    amps, freqs, amps_target, freqs_target = (
        core.torch_float32(x) for x in (amps, freqs, amps_target, freqs_target))
    nll = autograd.MixtureNLLFn.apply(hz_to_midi(freqs), hz_to_midi(freqs_target),
                                      _log_weights(amps_target), scale_target)
    amps_norm = safe_divide(amps, torch.sum(amps, dim=-1, keepdim=True))
    return torch.mean(nll * amps_norm, dim=-1)


class TWMLoss(Loss):
  """losses.TWMLoss (losses.py:819-1061), the differentiable two-way mismatch.

  -log p(sinusoids | harmonics) is the comb of `n_harmonic_gaussians` Gaussians of
  width `harmonics_scale` at the harmonic numbers, on f / f0 (`autograd.CombNLLFn`);
  -log p(harmonics | sinusoids) is the kernel density estimate of width
  `sinusoids_scale` around the sinusoids in MIDI, at each candidate's first
  `n_harmonic_points` harmonics (`autograd.MixtureNLLFn`).  (The reference's
  constructor comments pair the scales the other way round; its code, followed
  here, pairs them so.)  Gradients reach f0_candidates, freqs and amps."""

  def __init__(self, sinusoids_weight=1.0, harmonics_weight=1.0, sinusoids_scale=0.5,
               harmonics_scale=0.2, n_harmonic_points=10, n_harmonic_gaussians=30,
               softmin_temperature=1.0, sample_rate=16000, name=None):
    super().__init__(name)
    self.softmin_temperature = softmin_temperature
    self.sample_rate = sample_rate
    self.sinusoids_weight = sinusoids_weight
    self.harmonics_weight = harmonics_weight
    self.sinusoids_scale = sinusoids_scale
    self.n_harmonic_points = n_harmonic_points
    self.harmonics_scale = harmonics_scale
    self.n_harmonic_gaussians = n_harmonic_gaussians

  def call(self, f0_candidates, freqs, amps):
    """Scalar: the softmin over candidates of the weighted two terms."""
    sinusoids_loss, harmonics_loss = self.get_loss_tensors(f0_candidates, freqs, amps)
    combined_loss = (self.sinusoids_weight * sinusoids_loss +
                     self.harmonics_weight * harmonics_loss)
    softmin_loss = combined_loss * torch.softmax(
        -combined_loss / self.softmin_temperature, dim=-1)
    return torch.mean(softmin_loss)

  def predict_f0(self, f0_candidates, freqs, amps):
    """The candidate of least combined loss per frame, [batch, time, 1], on the
    inputs' device.  NaN losses are skipped and ties go to the first index, as with
    np.nanargmin; a frame whose losses are all NaN raises ValueError as it does."""
    with torch.no_grad():
      sinusoids_loss, harmonics_loss = self.get_loss_tensors(f0_candidates, freqs, amps)
      loss = (self.sinusoids_weight * sinusoids_loss +
              self.harmonics_weight * harmonics_loss)
      nan = torch.isnan(loss)
      if bool(torch.any(torch.all(nan, dim=-1))):
        raise ValueError('All-NaN slice encountered')
      idx = torch.argmin(torch.where(nan, torch.full_like(loss, math.inf), loss), dim=-1)
      # a frame whose least loss is +inf: the first +inf, not a skipped NaN before it
      first_inf = torch.argmax((loss == math.inf).to(torch.int32), dim=-1)
      least = torch.gather(loss, -1, idx[..., None])[..., 0]
      idx = torch.where(least == math.inf, first_inf, idx)
      return torch.gather(core.torch_float32(f0_candidates), -1, idx[..., None])

  def _check(self, f0_candidates, freqs, amps):
    _check_sinusoids('TWMLoss', [('amps, freqs', amps, freqs)])
    sc = core._shape(f0_candidates)
    if len(sc) != 3 or sc[:2] != core._shape(freqs)[:2]:
      raise ValueError(f'TWMLoss: f0_candidates must be [batch, time, candidates] with '
                       f'the [batch, time] of freqs {core._shape(freqs)[:2]}, got {sc}')
    if int(self.n_harmonic_points) < 1 or int(self.n_harmonic_gaussians) < 1:
      raise ValueError('TWMLoss: n_harmonic_points (%s) and n_harmonic_gaussians (%s) '
                       'must be at least 1' % (self.n_harmonic_points,
                                               self.n_harmonic_gaussians))
    _check_scale('TWMLoss', 'sinusoids_scale', self.sinusoids_scale)
    _check_scale('TWMLoss', 'harmonics_scale', self.harmonics_scale)

  def get_loss_tensors(self, f0_candidates, freqs, amps):
    """-log p(sinusoids | harmonics) and -log p(harmonics | sinusoids), each
    [batch, time, candidate]."""
    self._check(f0_candidates, freqs, amps)
    f0_candidates, freqs, amps = (
        core.torch_float32(x) for x in (f0_candidates, freqs, amps))
    sinusoids_loss = autograd.CombNLLFn.apply(
        f0_candidates, freqs, amps, int(self.n_harmonic_gaussians),
        float(self.harmonics_scale))

    harmonics = self.get_candidate_harmonics(f0_candidates, as_midi=True)
    b, t, c, n = harmonics.shape
    nll = autograd.MixtureNLLFn.apply(
        harmonics.reshape(b, t, c * n), hz_to_midi(freqs), _log_weights(amps),
        float(self.sinusoids_scale)).reshape(b, t, c, n)
    with torch.no_grad():
      # the prior on upper harmonics and the Nyquist mask, reweighted by the
      # number of harmonics below Nyquist: constants of the graph
      amps_prior = torch.linspace(1.0, 1.0 / n, n, device=harmonics.device)
      nyquist_mask = (harmonics < hz_to_midi(self.sample_rate / 2.0)).to(torch.float32)
      weights = amps_prior * safe_divide(
          nyquist_mask, torch.mean(nyquist_mask, dim=-1, keepdim=True))
    harmonics_loss = torch.mean(nll * weights, dim=-1)
    return sinusoids_loss, harmonics_loss

  def get_candidate_harmonics(self, f0_candidates, as_midi=True):
    """The harmonic series f0 * [1..n_harmonic_points] of each candidate,
    [batch, time, candidate, harmonic], in MIDI or in hertz.  In MIDI it is formed
    as hz_to_midi(f0) + 12 log2(n) (0 where f0 <= 0, as hz_to_midi(f0 n) gives),
    which keeps one [batch, time, candidate, harmonic] tensor in the graph instead
    of hz_to_midi's chain of them."""
    f0_candidates = core.torch_float32(f0_candidates)
    n = torch.arange(1, int(self.n_harmonic_points) + 1, dtype=torch.float32,
                     device=f0_candidates.device)
    if not as_midi:
      return f0_candidates[..., None] * n
    midi = hz_to_midi(f0_candidates)[..., None] + 12.0 * torch.log2(n)
    return torch.where(f0_candidates[..., None] <= 0.0, torch.zeros_like(midi), midi)


# ------------------------------------------------------------------------------
# Wasserstein consistency (losses.py:584-686)
# ------------------------------------------------------------------------------
def _check_wasserstein(u_values, v_values, u_weights, v_weights, p):
  """The checks of wasserstein_distance, before any device work; returns the batch shape
  and the two side lengths."""
  name = 'wasserstein_distance'
  if u_weights is None or v_weights is None:
    raise ValueError(f'{name}: u_weights and v_weights are required.  The reference '
                     'cannot evaluate None weights (it multiplies a float64 CDF by the '
                     'float32 values), and no normalised variant is offered.')
  su, sv = core._shape(u_values), core._shape(v_values)
  swu, swv = core._shape(u_weights), core._shape(v_weights)
  if len(su) < 1 or swu != su:
    raise ValueError(f'{name}: u_values {su} and u_weights {swu} must be one shape '
                     '[*batch, n_u]')
  if len(sv) < 1 or swv != sv:
    raise ValueError(f'{name}: v_values {sv} and v_weights {swv} must be one shape '
                     '[*batch, n_v]')
  if su[:-1] != sv[:-1]:
    raise ValueError(f'{name}: u has batch shape {su[:-1]}, v {sv[:-1]}')
  if su[-1] < 1 or sv[-1] < 1:
    raise ValueError(f'{name}: each side needs at least one value, got n_u={su[-1]} and '
                     f'n_v={sv[-1]} (the reference cannot evaluate an empty side)')
  p = float(p)
  if not (p > 0.0 and math.isfinite(p)):
    raise ValueError(f'{name}: p must be positive and finite, got {p}')
  limit = _lib.WASSERSTEIN_MAX_SIDE
  if su[-1] > limit or sv[-1] > limit:
    raise NotImplementedError(f'{name}: n_u={su[-1]} or n_v={sv[-1]} values exceed the '
                              f'{limit} per side the kernel sorts.')
  rows = math.prod(su[:-1])
  if rows > _lib.MAX_ROWS:
    raise NotImplementedError(f'{name}: {rows} rows exceed the {_lib.MAX_ROWS} '
                              'the kernel launches.')
  return su[:-1], su[-1], sv[-1]


@core.on_operands_device
def wasserstein_distance(u_values, v_values, u_weights, v_weights, p=1.0):
  """losses.wasserstein_distance (losses.py:641-686), [*batch], for values and weights
  [*batch, n_u] and [*batch, n_v]: (sum_i delta_i |U_i - V_i|^p)^(1/p) over the gaps
  delta_i of the sorted union, with U_i and V_i the cumulative weights at or below its
  i-th value.  As in the reference the cumulative weights are not normalised (its
  normalisation is computed and discarded), so weight totals that differ add their
  difference.  One launch of `autograd.WassersteinFn` forward and one backward, with
  gradients to all four inputs.  None weights, shapes that differ, empty sides and p
  not positive and finite raise ValueError, more than 4096 values per side
  NotImplementedError, before any device work."""
  batch, nu, nv = _check_wasserstein(u_values, v_values, u_weights, v_weights, p)
  u, v, wu, wv = (core.torch_float32(x) for x in (u_values, v_values, u_weights, v_weights))
  out = autograd.WassersteinFn.apply(u.reshape(-1, nu), v.reshape(-1, nv),
                                     wu.reshape(-1, nu), wv.reshape(-1, nv), float(p))
  return out.reshape(batch)


class WassersteinConsistencyLoss(Loss):
  """losses.WassersteinConsistencyLoss (losses.py:584-638): weight * the mean over
  [batch, time] of the p = 1 Wasserstein distance between the sinusoids a and b in MIDI
  (core.hz_to_midi: 0 Hz and below map to MIDI 0), amplitude-weighted.  As in the
  reference it is the plain number 0.0 unless weight > 0 and midi is true.  amps_a and
  freqs_a are [batch, time, n_a], amps_b and freqs_b [batch, time, n_b]; other shapes
  raise ValueError before any device work."""

  def __init__(self, weight=1.0, midi=True, name=None):
    super().__init__(name)
    self.weight = weight
    self.midi = midi

  def call(self, amps_a, freqs_a, amps_b, freqs_b):
    _check_sinusoids('WassersteinConsistencyLoss',
                     [('amps_a, freqs_a', amps_a, freqs_a),
                      ('amps_b, freqs_b', amps_b, freqs_b)])
    loss = 0.0
    if self.weight > 0.0 and self.midi:
      amps_a, freqs_a, amps_b, freqs_b = (
          core.torch_float32(x) for x in (amps_a, freqs_a, amps_b, freqs_b))
      dist = wasserstein_distance(hz_to_midi(freqs_a), hz_to_midi(freqs_b), amps_a, amps_b,
                                  p=1.0)
      loss = torch.mean(self.weight * dist)
    return loss


# ------------------------------------------------------------------------------
# HMM prior and MIDI transcription (losses.py:247-345)
# ------------------------------------------------------------------------------
class HmmTranscriber:
  """losses.HmmTranscriber (losses.py:247-345): an HMM over MIDI with one state per
  pitch 1..n_pitches - 1 and state 0 for "off", observing (f0 in MIDI, amplitude).

  The reference subclasses tfp's HiddenMarkovModel; here the two methods it uses run on
  the CUDA kernels of csrc/hmm.cuh: `log_prob` (the forward algorithm, differentiable in
  pitch and amplitude through `autograd.HmmLogProbFn`) and `posterior_mode` (Viterbi,
  ties to the lowest pitch).  The transitions are `hold` = 1 - 1 / avg_length on the
  diagonal and `other` = (1 - hold) / (n_pitches - 1) elsewhere; the HMM's parameters
  are constants.  Other tfp Distribution methods are not provided.

  pitch and amps other than [batch, n_timesteps, 1], n_pitches < 2, n_timesteps < 1
  and avg_length < 1 raise ValueError before any device work; n_pitches > 1024, and
  for `posterior_mode` more steps than `core.hmm_viterbi_takes` allows, raise
  NotImplementedError."""

  def __init__(self,
               avg_length=200,
               midi_std=0.5,
               amps_on_center=1.5,
               amps_on_scale=0.5,
               amps_off_center=0.0,
               amps_off_scale=0.1,
               n_timesteps=1000,
               n_pitches=128,
               weight=1.0,
               name='HiddenMarkovModel'):
    if not avg_length >= 1:
      raise ValueError(f'HmmTranscriber: avg_length must be at least 1 (hold = 1 - '
                       f'1 / avg_length), got {avg_length}')
    if int(n_pitches) != n_pitches or n_pitches < 2:
      raise ValueError(f'HmmTranscriber: n_pitches must be an integer >= 2, got {n_pitches}')
    if int(n_timesteps) != n_timesteps or n_timesteps < 1:
      raise ValueError(f'HmmTranscriber: n_timesteps must be an integer >= 1, got '
                       f'{n_timesteps}')
    self.avg_length = avg_length
    self.midi_std = midi_std
    self.n_timesteps = int(n_timesteps)
    self.n_pitches = int(n_pitches)
    self.weight = weight
    self.name = name
    self.hold = 1.0 - 1.0 / avg_length
    self.other = (1.0 - self.hold) / (self.n_pitches - 1)
    k = self.n_pitches
    self.loc = np.stack([np.r_[k / 2.0, np.arange(1, k)],
                         np.r_[amps_off_center, np.full(k - 1, amps_on_center)]],
                        axis=-1).astype(np.float32)
    self.scale = np.stack([np.r_[float(k), np.full(k - 1, midi_std)],
                           np.r_[amps_off_scale, np.full(k - 1, amps_on_scale)]],
                          axis=-1).astype(np.float32)
    self._params = {}   # device -> (loc, scale) on it

  def _on(self, device):
    if device not in self._params:
      self._params[device] = (core.torch_float32(self.loc, device=device),
                              core.torch_float32(self.scale, device=device))
    return self._params[device]

  def _check(self, name, x, last):
    s = core._shape(x)
    if len(s) != 3 or s[1] != self.n_timesteps or s[2] != last:
      raise ValueError(f'HmmTranscriber.{name}: expected [batch, {self.n_timesteps}, '
                       f'{last}], got {s}')

  def _supported(self, name, viterbi):
    k, t = self.n_pitches, self.n_timesteps
    if k > _lib.HMM_MAX_STATES:
      raise NotImplementedError(f'HmmTranscriber.{name}: {k} pitches exceed the '
                                f'{_lib.HMM_MAX_STATES} states the kernels run.')
    if viterbi and not core.hmm_viterbi_takes(t, k):
      raise NotImplementedError(f'HmmTranscriber.{name}: {t} steps of {k} states exceed '
                                'the back pointers the Viterbi kernel keeps.')

  def _observations(self, name, pitch, amps, viterbi=False):
    self._check(name, pitch, 1)
    self._check(name, amps, 1)
    if core._shape(pitch) != core._shape(amps):
      raise ValueError(f'HmmTranscriber.{name}: pitch {core._shape(pitch)} and amps '
                       f'{core._shape(amps)} differ')
    self._supported(name, viterbi)
    pitch = core.torch_float32(pitch)
    return torch.cat([pitch, core.torch_float32(amps, device=pitch.device)], dim=-1)

  def __call__(self, pitch, amps):
    return self.nll(pitch, amps)

  @staticmethod
  def straight_through(x, x_quant):
    """Straight through estimation: the value of x_quant, the gradient of x."""
    return x - (x - x_quant).detach()

  @core.on_operands_device
  def log_prob(self, pa):
    """log p(pa) [batch] for observations pa [batch, n_timesteps, 2] (pitch, amps)."""
    self._check('log_prob', pa, 2)
    self._supported('log_prob', False)
    x = core.torch_float32(pa)
    return core.hmm_log_prob(x, *self._on(x.device), self.hold, self.other)

  @core.on_operands_device
  def posterior_mode(self, pa):
    """The most likely state per step, [batch, n_timesteps] int64."""
    self._check('posterior_mode', pa, 2)
    self._supported('posterior_mode', True)
    x = core.torch_float32(pa)
    return core.hmm_posterior_mode(x, *self._on(x.device), self.hold, self.other)

  @core.on_operands_device
  def nll(self, pitch, amps, per_example_loss=False):
    """Negative log-likelihood per timestep: weight * mean_b(-log p_b / T), or the
    [batch] values with per_example_loss."""
    pa = self._observations('nll', pitch, amps)
    avg_nll = -self.log_prob(pa) / pa.shape[1]
    loss = avg_nll if per_example_loss else torch.mean(avg_nll)
    return self.weight * loss

  @core.on_operands_device
  def predict_midi(self, pitch, amps, channel_dim=True, dtype=torch.float32):
    """Viterbi decode of the most likely state as the quantized MIDI pitch,
    [batch, n_timesteps, 1] (or [batch, n_timesteps]) of `dtype`."""
    pa = self._observations('predict_midi', pitch, amps, viterbi=True)
    q_pitch = self.posterior_mode(pa).to(dtype)
    return q_pitch[:, :, None] if channel_dim else q_pitch
