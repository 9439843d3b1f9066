"""TensorToAudio, Harmonic, FilteredNoise, Wavetable and Sinusoidal synthesizers
with the reference's constructor arguments, method names and dict keys
(`ddsp/synths.py:23-323`)."""
import itertools

from ddsp_b200 import core
from ddsp_b200 import processors


class TensorToAudio(processors.Processor):
  """Identity "synth": the input samples without their channel axis
  (synths.py:23-52); a view."""

  def __init__(self, name='tensor_to_audio'):
    super().__init__(name=name)

  def get_controls(self, samples):
    return {'samples': samples}

  def get_signal(self, samples):
    """`tf.squeeze(samples, 2)`, which fails unless samples is [batch, time, 1]."""
    shape = core._shape(samples)   # pylint: disable=protected-access
    if len(shape) != 3 or shape[2] != 1:
      raise ValueError(f'TensorToAudio takes samples of shape [batch, time, 1]; got '
                       f'{shape}.')
    return samples[:, :, 0]


class Harmonic(processors.Processor):
  """Synthesize audio with a bank of harmonic sinusoidal oscillators
  (synths.py:55-146)."""

  def __init__(self,
               n_samples=64000,
               sample_rate=16000,
               scale_fn=core.exp_sigmoid,
               normalize_below_nyquist=True,
               amp_resample_method='window',
               use_angular_cumsum=False,
               name='harmonic'):
    super().__init__(name=name)
    self.n_samples = n_samples
    self.sample_rate = sample_rate
    self.scale_fn = scale_fn
    self.normalize_below_nyquist = normalize_below_nyquist
    self.amp_resample_method = amp_resample_method
    self.use_angular_cumsum = use_angular_cumsum

  def get_controls(self, amplitudes, harmonic_distribution, f0_hz):
    """synths.py:94-121.  exp_sigmoid scaling, Nyquist masking and row
    normalisation run as one kernel; any other scale_fn is applied by calling
    it (as the reference does) before the mask/normalise kernel."""
    f0_hz = core.torch_float32(f0_hz)
    fused_scale = self.scale_fn is core.exp_sigmoid
    if self.scale_fn is not None and not fused_scale:
      amplitudes = self.scale_fn(core.torch_float32(amplitudes))
      harmonic_distribution = self.scale_fn(
          core.torch_float32(harmonic_distribution))
    amplitudes, harmonic_distribution = core.harmonic_controls(
        amplitudes, harmonic_distribution, f0_hz, self.sample_rate,
        scale=fused_scale, normalize_below_nyquist=self.normalize_below_nyquist)
    return {'amplitudes': amplitudes,
            'harmonic_distribution': harmonic_distribution,
            'f0_hz': f0_hz}

  def get_signal(self, amplitudes, harmonic_distribution, f0_hz, out=None,
                 accumulate=False):
    """synths.py:123-146."""
    return core.harmonic_synthesis(
        frequencies=f0_hz,
        amplitudes=amplitudes,
        harmonic_distribution=harmonic_distribution,
        n_samples=self.n_samples,
        sample_rate=self.sample_rate,
        amp_resample_method=self.amp_resample_method,
        use_angular_cumsum=self.use_angular_cumsum,
        out=out, accumulate=accumulate)


class FilteredNoise(processors.Processor):
  """Synthesize audio by filtering white noise (synths.py:149-196).

  The reference draws fresh `tf.random.uniform` noise per call
  (synths.py:192-193).  Here the noise is Philox4x32-10 generated inside the
  filter kernel, keyed by `seed` with a per-call counter so successive calls
  differ; pass `noise=` to get_signal to inject a specific noise tensor
  (parity tests do).
  """

  def __init__(self,
               n_samples=64000,
               window_size=257,
               scale_fn=core.exp_sigmoid,
               initial_bias=-5.0,
               name='filtered_noise',
               seed=0):
    super().__init__(name=name)
    self.n_samples = n_samples
    self.window_size = window_size
    self.scale_fn = scale_fn
    self.initial_bias = initial_bias
    self.seed = seed
    self._calls = itertools.count()
    # Test hook: a [B, n_samples] tensor used instead of the Philox stream.
    self.injected_noise = None

  def next_offset(self):
    """Per-call Philox counter offset, so successive calls draw fresh noise."""
    return next(self._calls)

  def get_controls(self, magnitudes):
    """synths.py:165-179."""
    if self.scale_fn is core.exp_sigmoid:
      magnitudes = core.noise_controls(magnitudes, self.initial_bias, scale=True)
    elif self.scale_fn is not None:
      magnitudes = self.scale_fn(
          core.torch_float32(magnitudes) + self.initial_bias)
    else:
      magnitudes = core.torch_float32(magnitudes)
    return {'magnitudes': magnitudes}

  def get_signal(self, magnitudes, noise=None, out=None, accumulate=False,
                 offset=None):
    """synths.py:181-196."""
    if noise is None:
      noise = self.injected_noise
    return core.filtered_noise(
        magnitudes, self.n_samples, window_size=self.window_size, noise=noise,
        seed=self.seed, offset=self.next_offset() if offset is None else offset,
        out=out, accumulate=accumulate)


class Sinusoidal(processors.Processor):
  """Bank of arbitrary sinusoidal oscillators (synths.py:260-323).

  get_controls is frame-rate torch arithmetic; get_signal is one fused frame-rate
  oscillator bank with per-sinusoid exact phases
  (`ddsp_b200_sinusoidal_forward`) - the [batch, n_samples, n_sinusoids]
  envelopes of the reference are never materialised."""

  def __init__(self,
               n_samples=64000,
               sample_rate=16000,
               amp_scale_fn=core.exp_sigmoid,
               amp_resample_method='window',
               freq_scale_fn=core.frequencies_sigmoid,
               name='sinusoidal'):
    super().__init__(name=name)
    self.n_samples = n_samples
    self.sample_rate = sample_rate
    self.amp_scale_fn = amp_scale_fn
    self.amp_resample_method = amp_resample_method
    self.freq_scale_fn = freq_scale_fn

  def get_controls(self, amplitudes, frequencies):
    """synths.py:277-303."""
    amplitudes = core.torch_float32(amplitudes)
    frequencies = core.torch_float32(frequencies)
    if self.amp_scale_fn is not None:
      amplitudes = self.amp_scale_fn(amplitudes)
    if self.freq_scale_fn is not None:
      frequencies = self.freq_scale_fn(frequencies)
      amplitudes = core.remove_above_nyquist(frequencies, amplitudes,
                                             self.sample_rate)
    return {'amplitudes': amplitudes, 'frequencies': frequencies}

  def get_signal(self, amplitudes, frequencies):
    """synths.py:305-323.  One fused frame-rate kernel when the hop is an integer
    and the amplitudes are resampled by 'window' / 'linear' (differentiable in
    both inputs); otherwise the reference's own decomposition on the stand-alone
    kernels, which has no backward."""
    sa = core._shape(amplitudes)  # pylint: disable=protected-access
    if (self.amp_resample_method in core.AMP_METHODS and len(sa) == 3 and
        sa[1] > 0 and self.n_samples % sa[1] == 0 and
        (self.amp_resample_method != 'window' or sa[1] < self.n_samples)):
      return core.sinusoidal_synthesis(
          frequencies, amplitudes, n_samples=self.n_samples,
          sample_rate=self.sample_rate,
          amp_resample_method=self.amp_resample_method)
    # the resampled envelopes would be detached: refuse rather than drop the gradient
    core._no_grad_path('oscillator_bank', amplitudes, frequencies)  # pylint: disable=protected-access
    amplitude_envelopes = core.resample(amplitudes, self.n_samples,
                                        method=self.amp_resample_method)
    frequency_envelopes = core.resample(frequencies, self.n_samples)
    return core.oscillator_bank(frequency_envelopes=frequency_envelopes,
                                amplitude_envelopes=amplitude_envelopes,
                                sample_rate=self.sample_rate)


class Wavetable(processors.Processor):
  """Synthesize audio from a series of wavetables (synths.py:199-257).

  get_signal is one fused kernel (`core.wavetable_synthesis`) that reads the
  tables at frame rate; the reference's [batch, n_samples, n_wavetable] tables
  are never built."""

  def __init__(self,
               n_samples=64000,
               sample_rate=16000,
               scale_fn=core.exp_sigmoid,
               name='wavetable'):
    super().__init__(name=name)
    self.n_samples = n_samples
    self.sample_rate = sample_rate
    self.scale_fn = scale_fn

  def get_controls(self, amplitudes, wavetables, f0_hz):
    """synths.py:213-238: scale_fn on the amplitudes and the wavetables."""
    amplitudes = core.torch_float32(amplitudes)
    wavetables = core.torch_float32(wavetables)
    if self.scale_fn is not None:
      amplitudes = self.scale_fn(amplitudes)
      wavetables = self.scale_fn(wavetables)
    return {'amplitudes': amplitudes, 'wavetables': wavetables, 'f0_hz': f0_hz}

  def get_signal(self, amplitudes, wavetables, f0_hz):
    """synths.py:240-257.  The reference resamples 3-D tables to n_samples
    ('linear') and wavetable_synthesis then reads them one frame per sample; the
    kernel applies the same taps at frame rate.  2-D [batch, n_wavetable] tables
    are resampled along n_wavetable as time, as the reference does, and read as
    one static table of n_samples entries."""
    if len(core._shape(wavetables)) == 2:  # pylint: disable=protected-access
      wavetables = core.resample(wavetables, self.n_samples)
    return core.wavetable_synthesis(amplitudes=amplitudes, wavetables=wavetables,
                                    frequencies=f0_hz, n_samples=self.n_samples,
                                    sample_rate=self.sample_rate)
