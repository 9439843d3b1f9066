"""Effects processors that consume the decoder's audio: `Reverb`,
`ExpDecayReverb`, `FilteredNoiseReverb`, `FIRFilter` and `ModDelay` with the
reference's constructors and semantics (`ddsp/effects.py:28-394`; SURVEY 8f-3; the
next node after `Add` in `solo_instrument.gin:26-40`).

`Reverb` is a long linear time-invariant convolution (48000-tap impulse
response): `core.fft_convolve` routes one impulse response of 2048 taps and more
per item to the hand-written partitioned overlap-save convolution
(csrc/longconv.cuh); `FilteredNoiseReverb` draws that impulse response from a
`FilteredNoise` synthesizer; `FIRFilter` is the time-varying filter of
`FilteredNoise` applied to given audio and runs on the IR + FIR kernels."""
import itertools

import torch

from ddsp_b200 import core
from ddsp_b200 import processors
from ddsp_b200 import synths


class Reverb(processors.Processor):
  """Convolutional (FIR) reverb (effects.py:28-117)."""

  def __init__(self, trainable=False, reverb_length=48000, add_dry=True,
               name='reverb'):
    super().__init__(name=name, trainable=trainable)
    self._reverb_length = reverb_length
    self._add_dry = add_dry
    self._ir = None

  # build()'s variables: the reference's weight name -> the attribute that holds it
  _VARIABLES = {'ir': '_ir'}

  def named_variables(self):
    """[(name, torch.nn.Parameter)] of the variables build() created, with the
    reference's weight names: empty before the first call, or when not trainable.
    models.Autoencoder registers them as its parameters."""
    return [(name, getattr(self, attr)) for name, attr in self._VARIABLES.items()
            if getattr(self, attr) is not None]

  def _mask_dry_ir(self, ir):
    """effects.py:50-59: zero the first tap (the dry path)."""
    if ir.dim() == 1:
      ir = ir[None, :]
    if ir.dim() == 3:
      ir = ir[:, :, 0]
    dry_mask = torch.zeros((ir.shape[0], 1), dtype=torch.float32, device=ir.device)
    return torch.cat([dry_mask, ir[:, 1:]], dim=1)

  def _match_dimensions(self, audio, ir):
    """effects.py:61-68."""
    if ir.dim() == 1:
      ir = ir[None, :]
    return ir.repeat(int(audio.shape[0]), 1)

  def build(self, device=None):
    """effects.py:70-79: the single learned impulse response, N(0, 1e-6)."""
    if self.trainable and self._ir is None:
      self._ir = torch.nn.Parameter(1e-6 * torch.randn(
          self._reverb_length, dtype=torch.float32, device=device))

  def get_controls(self, audio, ir=None):
    """effects.py:81-101."""
    if not self.trainable and ir is None:          # before any device work
      raise ValueError('Must provide "ir" tensor if Reverb trainable=False.')
    audio = core.torch_float32(audio)
    if self.trainable:
      self.build(audio.device)
      ir = self._match_dimensions(audio, self._ir)
    return {'audio': audio, 'ir': ir}

  def get_signal(self, audio, ir):
    """effects.py:103-117."""
    audio, ir = core.torch_float32(audio), core.torch_float32(ir)
    ir = self._mask_dry_ir(ir)
    wet = core.fft_convolve(audio, ir, padding='same', delay_compensation=0)
    return (wet + audio) if self._add_dry else wet


class ExpDecayReverb(Reverb):
  """Impulse response = an exponential decay of white noise (effects.py:121-199):
  `(scale_fn(gain) * exp(-(2 + exp(decay)) * linspace(0, 1, L))) * noise`, one
  [1, L] noise row shared by the batch.  The noise is the library's Philox stream
  keyed by `seed` with a fresh offset per call (the reference draws fresh
  `tf.random.uniform` noise per call); set `injected_noise` to a [1, L] tensor to
  use that row instead.  The impulse response is one kernel with a CUDA backward to
  gain and decay; `get_signal` is Reverb's."""

  def __init__(self, trainable=False, reverb_length=48000, scale_fn=core.exp_sigmoid,
               add_dry=True, name='exp_decay_reverb', seed=0):
    super().__init__(name=name, add_dry=add_dry, trainable=trainable)
    self._reverb_length = reverb_length
    self._scale_fn = scale_fn
    self.seed = seed
    self._calls = itertools.count()
    self._gain = None
    self._decay = None
    # Test hook: a [1, reverb_length] tensor used instead of the Philox stream.
    self.injected_noise = None

  _VARIABLES = {'gain': '_gain', 'decay': '_decay'}

  def next_offset(self):
    """Per-call Philox counter offset, so successive calls draw fresh noise."""
    return next(self._calls)

  def build(self, device=None):
    """effects.py:153-166: the learned gain 2.0 and decay 4.0, shape [1]."""
    if self.trainable and self._gain is None:
      self._gain = torch.nn.Parameter(torch.full((1,), 2.0, dtype=torch.float32,
                                                 device=device))
      self._decay = torch.nn.Parameter(torch.full((1,), 4.0, dtype=torch.float32,
                                                  device=device))

  def _get_ir(self, gain, decay):
    """effects.py:144-151."""
    gain = core.torch_float32(gain)
    if self._scale_fn is not None:
      gain = self._scale_fn(gain)
    return core.exp_decay_ir(gain, core.torch_float32(decay), self._reverb_length,
                             noise=self.injected_noise, seed=self.seed,
                             offset=self.next_offset())

  def get_controls(self, audio, gain=None, decay=None):
    """effects.py:168-198."""
    if not self.trainable and (gain is None or decay is None):  # before device work
      raise ValueError('Must provide "gain" and "decay" tensors if '
                       'ExpDecayReverb trainable=False.')
    audio = core.torch_float32(audio)
    if self.trainable:
      self.build(audio.device)
      gain, decay = self._gain[None, :], self._decay[None, :]
    ir = self._get_ir(gain, decay)
    if self.trainable:
      ir = self._match_dimensions(audio, ir)
    return {'audio': audio, 'ir': ir}


class FilteredNoiseReverb(Reverb):
  """Impulse response = the output of a filtered-noise synthesizer
  (effects.py:202-278): `get_controls` runs `FilteredNoise(n_samples =
  reverb_length)` on the magnitudes (given per item, or ONE learned
  [n_frames, n_filter_banks] set tiled over the batch when trainable), `get_signal`
  is `Reverb`'s."""

  def __init__(self, trainable=False, reverb_length=48000, window_size=257,
               n_frames=1000, n_filter_banks=16, scale_fn=core.exp_sigmoid,
               initial_bias=-3.0, add_dry=True, name='filtered_noise_reverb'):
    super().__init__(name=name, add_dry=add_dry, trainable=trainable)
    self._n_frames = n_frames
    self._n_filter_banks = n_filter_banks
    self._synth = synths.FilteredNoise(n_samples=reverb_length,
                                       window_size=window_size,
                                       scale_fn=scale_fn,
                                       initial_bias=initial_bias)
    self._magnitudes = None

  _VARIABLES = {'magnitudes': '_magnitudes'}

  def build(self, device=None):
    """effects.py:240-249: the learned magnitudes, N(0, 1e-2)."""
    if self.trainable and self._magnitudes is None:
      self._magnitudes = torch.nn.Parameter(1e-2 * torch.randn(
          self._n_frames, self._n_filter_banks, dtype=torch.float32, device=device))

  def _synth_ir(self, magnitudes):
    """`self._synth(magnitudes)` (effects.py:272); with gradients to the magnitudes
    when they ask for them (the synthesizer's autograd node, exp_sigmoid as
    differentiable torch ops on the [n_frames, n_filter_banks] controls)."""
    if (isinstance(magnitudes, torch.Tensor) and magnitudes.requires_grad and
        torch.is_grad_enabled()):
      from ddsp_b200 import autograd as _ag
      syn = self._synth
      # the controls in float32, as on the inference path, whatever the caller's dtype
      magnitudes = core.torch_float32(magnitudes)
      if syn.scale_fn is core.exp_sigmoid:
        mags = _ag.exp_sigmoid(magnitudes + syn.initial_bias)
      elif syn.scale_fn is not None:
        mags = syn.scale_fn(magnitudes + syn.initial_bias)
      else:
        mags = magnitudes
      return _ag.FilteredNoiseFn.apply(mags, syn.n_samples, syn.window_size,
                                       syn.injected_noise, syn.seed,
                                       syn.next_offset())
    return self._synth(magnitudes)

  def get_controls(self, audio, magnitudes=None):
    """effects.py:251-277."""
    if not self.trainable and magnitudes is None:  # before any device work
      raise ValueError('Must provide "magnitudes" tensor if '
                       'FilteredNoiseReverb trainable=False.')
    audio = core.torch_float32(audio)
    if self.trainable:
      self.build(audio.device)
      magnitudes = self._magnitudes[None, :]
    ir = self._synth_ir(magnitudes)
    if self.trainable:
      ir = self._match_dimensions(audio, ir)
    return {'audio': audio, 'ir': ir}


class FIRFilter(processors.Processor):
  """Linear time-varying FIR filter (effects.py:283-325)."""

  def __init__(self, window_size=257, scale_fn=core.exp_sigmoid, name='fir_filter'):
    super().__init__(name=name)
    self.window_size = window_size
    self.scale_fn = scale_fn

  def get_controls(self, audio, magnitudes):
    if self.scale_fn is not None:
      magnitudes = self.scale_fn(core.torch_float32(magnitudes))
    return {'audio': audio, 'magnitudes': magnitudes}

  def get_signal(self, audio, magnitudes):
    return core.frequency_filter(audio, magnitudes, window_size=self.window_size)


class ModDelay(processors.Processor):
  """Modulated delay behind chorus, flanger and vibrato (effects.py:328-394).

  `get_signal` is one kernel: the phase mapping `phase * depth / max + center / max`,
  the delay line, the gain and the dry mix (core.mod_delay).  As in the reference,
  the mapped phase of the default `sigmoid` lies in (center / max, 1), which
  reaches the wrap region of core.variable_length_delay near 1 (no delay there)."""

  def __init__(self, center_ms=15.0, depth_ms=10.0, sample_rate=16000,
               gain_scale_fn=core.exp_sigmoid, phase_scale_fn=torch.sigmoid,
               add_dry=True, name='mod_delay'):
    super().__init__(name=name)
    self.center_ms = center_ms
    self.depth_ms = depth_ms
    self.sample_rate = sample_rate
    self.gain_scale_fn = gain_scale_fn
    self.phase_scale_fn = phase_scale_fn
    self.add_dry = add_dry

  def get_controls(self, audio, gain, phase):
    """effects.py:349-366."""
    if self.gain_scale_fn is not None:
      gain = self.gain_scale_fn(core.torch_float32(gain))
    if self.phase_scale_fn is not None:
      phase = self.phase_scale_fn(core.torch_float32(phase))
    return {'audio': audio, 'gain': gain, 'phase': phase}

  def get_signal(self, audio, gain, phase):
    """effects.py:368-394."""
    max_delay_ms = self.center_ms + self.depth_ms
    max_length_samples = int(self.sample_rate / 1000.0 * max_delay_ms)
    depth_phase = self.depth_ms / max_delay_ms
    center_phase = self.center_ms / max_delay_ms
    return core.mod_delay(audio, gain, phase, max_length_samples, scale=depth_phase,
                          offset=center_phase, add_dry=self.add_dry)
