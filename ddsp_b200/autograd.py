"""Differentiable wrappers of the synthesis kernels (C4: decoder forward +
backward through SpectralLoss).

The reference differentiates through every TF op of `core.harmonic_synthesis` /
`core.frequency_filter`; here forward and backward are the hand-written CUDA
kernels, exposed as `torch.autograd.Function`s:

  * `HarmonicSynthesisFn`  - d amplitudes, d harmonic_distribution, d f0 (the
    phase path, `models/inverse_synthesis.py:84-117`; computed only when f0
    requires grad);
  * `FilteredNoiseFn`      - d magnitudes (the filter is linear in them);
    `core.harmonic_synthesis` / `core.filtered_noise` route to these two under grad
    (DESIGN.md section 3.15 has the table of which shape goes where);
  * `HarmonicControlsFn` / `NoiseControlsFn` - `Harmonic.get_controls` and
    `FilteredNoise.get_controls` for any upstream gradient (a loss on the controls
    themselves as well as the synthesizer's), one backward launch each; routed to by
    `core.harmonic_controls` / `core.noise_controls` under grad.  With them the
    Processor API trains: `ProcessorGroup.get_controls` + `get_signal` and
    `group(features, return_outputs_dict=True)`;
  * `SinusoidalSynthesisFn` - d amplitudes and d frequencies of the frame-rate
    oscillator bank (`Sinusoidal.get_signal`, the synthesizer of
    `models/inverse_synthesis.py:84-105`; d frequencies only when they require
    grad); `core.sinusoidal_synthesis` routes to it under grad;
  * `OscillatorBankFn` / `AngularCumsumFn` - the stand-alone oscillator bank on
    audio-rate envelopes (d frequency and d amplitude envelopes) and the phase
    accumulation, routed to by `core.oscillator_bank` / `core.angular_cumsum` under
    grad;
  * `HarmonicOscillatorBankFn` - core.harmonic_oscillator_bank with a carried phase,
    differentiable in f0, amplitude envelopes and initial phase through the audio and the
    final phase; routed to by `core.harmonic_oscillator_bank` (and so by
    `core.streaming_harmonic_synthesis`) under grad;
  * `LinearLookupFn` - core.linear_lookup, d phase and d wavetables;
  * `WavetableSynthesisFn` - d f0, d amplitudes and d wavetables of the wavetable
    synthesizer (`Wavetable.get_signal`); `core.wavetable_synthesis` routes to it
    under grad;
  * `FftConvolveLtiFn` / `ModDelayFn` - the reverb convolution and the modulated
    delay, routed to by `core.fft_convolve` / `core.mod_delay` under grad;
  * `ResampleFn` / `AddFn` - core.resample (the transpose kernel) and core.add,
    routed to under grad;
  * `MixFn` / `ExpDecayIrFn` - processors.Mix's crossfade and the exponential
    decay impulse response of effects.ExpDecayReverb;
  * `FirTimeVaryingFn` / `FrequencyImpulseResponseFn` / `FrequencyFilterFn` - the
    direct-form time-varying FIR (impulse responses under 2048 taps: FIRFilter,
    short reverbs), the impulse-response synthesis and their composition, routed to
    by `core.fft_convolve` / `core.frequency_impulse_response` /
    `core.frequency_filter` under grad;
  * `SincImpulseResponseFn` / `SincFilterFn` - core.sinc_impulse_response and the
    fused core.sinc_filter, differentiable in the cutoff (and the audio); the taps
    are rebuilt on chip in the backward, never stored;
  * `MixtureNLLFn` / `CombNLLFn` - the Gaussian-mixture NLLs of the consistency
    losses (`losses.KDEConsistencyLoss`, `losses.TWMLoss`), evaluated per frame
    on-chip with gradients to every input;
  * `NoteMomentsFn` - nn.get_note_moments and nn.pool_over_notes, d x through the
    per-note mean and std;
  * `HmmLogProbFn` - the HMM log-likelihood of `losses.HmmTranscriber`, with
    gradients to the observations (pitch and amplitude); routed to by
    `core.hmm_log_prob` under grad;
  * `GruFn` - the Keras GRU of `nn.Rnn` / `decoders.RnnFcDecoder`: the recurrence and
    its backpropagation through time are one launch each (`csrc/gru.cuh`), the GEMMs
    around them cuBLAS;
  * `NormReluFn` - nn.Normalize followed by a ReLU at every site of `nn.ResNet`: one
    fused launch forward (`csrc/norm.cuh`), and one backward launch plus a fixed-order
    reduction of dscale and dshift; only the per-(item, group) mean and rstd are saved;
  * `NormResidualFn` - the residual site of `nn.DilatedConvStack`, x + normalize(y) s + h
    and its ReLU, with s and h per channel or read in place from a FiLM Dense output
    (`csrc/norm.cuh`): one launch forward, one or two backward;
  * `CrepeLossFramesFn` - the framing and per-frame normalisation of
    `losses.PretrainedCREPE`, d audio, which the embedding losses train through;
  * `DecoderFn` / `decoder_train` - the whole `ae.gin` decoder from RAW network
    outputs: forward is the fused two-kernel pipeline (`get_controls` in shared
    memory), backward is the two synthesizer backward kernels plus the
    `get_controls` backward kernels - no frame-rate torch op on either pass.

`harmonic_controls` / `exp_sigmoid` below are the same `get_controls` arithmetic as
differentiable torch ops, kept for callers that compose their own graphs.
"""
import ctypes
import math

import torch

from ddsp_b200 import _lib
from ddsp_b200 import core


class HarmonicSynthesisFn(torch.autograd.Function):
  """core.harmonic_synthesis (core.py:1048-1111), differentiable in
  amplitudes and harmonic_distribution."""

  @staticmethod
  def forward(ctx, f0_hz, amplitudes, harmonic_distribution, n_samples,
              sample_rate, amp_resample_method):
    f0_hz = core.torch_float32(f0_hz)
    amplitudes = core.torch_float32(amplitudes)
    harmonic_distribution = core.torch_float32(harmonic_distribution)
    ctx.save_for_backward(f0_hz, amplitudes, harmonic_distribution)
    ctx.cfg = (int(n_samples), float(sample_rate), amp_resample_method)
    return core.harmonic_synthesis(
        f0_hz, amplitudes, harmonic_distribution=harmonic_distribution,
        n_samples=n_samples, sample_rate=sample_rate,
        amp_resample_method=amp_resample_method)

  @staticmethod
  def backward(ctx, grad_audio):
    f0_hz, amplitudes, hd = ctx.saved_tensors
    n_samples, sample_rate, method = ctx.cfg
    b, f, k = hd.shape
    grad_audio = grad_audio.contiguous().to(torch.float32)
    g0 = torch.empty_like(hd)
    g1 = torch.empty_like(hd)
    core._launch('ddsp_b200_harmonic_backward', f0_hz, grad_audio, g0, g1, b, f, k,
                 n_samples, sample_rate, core.AMP_METHODS[method])
    # dL/d(amp * hd)[i] = g0[i] + g1[i-1], frame F being a copy of frame F-1
    dha = g0
    dha[:, 1:] += g1[:, :-1]
    dha[:, -1] += g1[:, -1]
    d_hd = dha * amplitudes
    d_amp = (dha * hd).sum(-1, keepdim=True)
    d_f0 = None
    if ctx.needs_input_grad[0]:
      d_f0 = _harmonic_d_f0(f0_hz, amplitudes, hd, grad_audio, n_samples, sample_rate,
                            method)
    return d_f0, d_amp, d_hd, None, None, None


def _harmonic_d_f0(f0_hz, amplitudes, hd, grad_audio, n_samples, sample_rate, method):
  """dL/d f0_hz [B, F, 1] through the phase (`ddsp_b200_harmonic_backward_f0`)."""
  b, f, k = hd.shape
  d_f0 = torch.empty((b, f, 1), dtype=torch.float32, device=hd.device)
  core._launch('ddsp_b200_harmonic_backward_f0', f0_hz, amplitudes, hd, grad_audio, d_f0,
               b, f, k, n_samples, sample_rate, core.AMP_METHODS[method],
               *core._workspace(12 * b * f, hd.device))
  return d_f0


class DecoderFn(torch.autograd.Function):
  """The `ae.gin` decoder (ae.gin:47-72) from raw network outputs, forward and
  backward entirely in the CUDA library.  Gradients: amps, harmonic_distribution,
  noise_magnitudes always; f0_hz when it requires grad."""

  @staticmethod
  def forward(ctx, amps, harmonic_distribution, f0_hz, noise_magnitudes, n_samples,
              sample_rate, amp_resample_method, normalize_below_nyquist, window_size,
              initial_bias, noise, seed, offset):
    amps = core.torch_float32(amps)
    hd = core.torch_float32(harmonic_distribution)
    f0_hz = core.torch_float32(f0_hz)
    mags = core.torch_float32(noise_magnitudes)
    noise = None if noise is None else core.torch_float32(noise)
    ctx.save_for_backward(amps, hd, f0_hz, mags)
    ctx.noise = noise
    ctx.cfg = (int(n_samples), float(sample_rate), amp_resample_method,
               bool(normalize_below_nyquist), int(window_size), float(initial_bias),
               int(seed), int(offset))
    return core.decoder_forward(
        amps, hd, f0_hz, mags, n_samples, sample_rate=sample_rate,
        amp_resample_method=amp_resample_method,
        normalize_below_nyquist=normalize_below_nyquist, window_size=window_size,
        initial_bias=initial_bias, noise=noise, seed=seed, offset=offset)

  @staticmethod
  def backward(ctx, grad_audio):
    amps, hd, f0_hz, mags = ctx.saved_tensors
    n_samples, sample_rate, method, nyq, window_size, bias, seed, offset = ctx.cfg
    b, f, k = hd.shape
    nb = mags.shape[-1]
    g = grad_audio.contiguous().to(torch.float32)
    flags = _lib.CTL_SCALE | (_lib.CTL_NYQUIST if nyq else 0)
    # harmonic: sample-rate reductions, then get_controls transposed at frame rate
    g0 = torch.empty_like(hd)
    g1 = torch.empty_like(hd)
    core._launch('ddsp_b200_harmonic_backward', f0_hz, g, g0, g1, b, f, k, n_samples,
                 sample_rate, core.AMP_METHODS[method])
    d_amps = torch.empty_like(amps)
    d_hd = torch.empty_like(hd)
    core._launch('ddsp_b200_harmonic_controls_backward', amps, hd, f0_hz, g0, g1, d_amps,
                 d_hd, b, f, k, sample_rate, flags)
    # noise: the filter is linear in the magnitudes
    dmags = torch.empty_like(mags)
    core._launch('ddsp_b200_filtered_noise_backward', g, ctx.noise, seed, offset, dmags, b,
                 f, nb, n_samples, window_size)
    d_mags = torch.empty_like(mags)
    core._launch('ddsp_b200_noise_controls_backward', mags, dmags, d_mags, mags.numel(),
                 bias)
    d_f0 = None
    if ctx.needs_input_grad[2]:
      # the phase path needs the synthesizer controls: one controls launch
      a_ctl, h_ctl = core.harmonic_controls(amps, hd, f0_hz, sample_rate, scale=True,
                                            normalize_below_nyquist=nyq)
      d_f0 = _harmonic_d_f0(f0_hz, a_ctl, h_ctl, g, n_samples, sample_rate, method)
    return (d_amps, d_hd, d_f0, d_mags) + (None,) * 9


class HarmonicControlsFn(torch.autograd.Function):
  """core.harmonic_controls (Harmonic.get_controls, synths.py:94-121), differentiable
  in the raw amplitudes and harmonic distribution for any upstream gradient on the two
  controls: one backward launch of `ddsp_b200_harmonic_controls_vjp`
  (csrc/controls_bwd.cuh).  f0_hz gets none: the Nyquist mask is piecewise constant
  (tf.where)."""

  @staticmethod
  def forward(ctx, amplitudes, harmonic_distribution, f0_hz, sample_rate, scale,
              normalize_below_nyquist):
    ctx.save_for_backward(amplitudes, harmonic_distribution, f0_hz)
    ctx.cfg = (float(sample_rate), bool(scale), bool(normalize_below_nyquist))
    ctx.set_materialize_grads(False)
    return core.harmonic_controls(amplitudes, harmonic_distribution, f0_hz, *ctx.cfg)

  @staticmethod
  def backward(ctx, d_amplitudes, d_hd):
    amps, hd, f0_hz = ctx.saved_tensors
    sample_rate, scale, nyq = ctx.cfg
    b, f, k = hd.shape
    if d_amplitudes is not None:
      d_amplitudes = d_amplitudes.contiguous().to(torch.float32)
    if d_hd is not None:
      d_hd = d_hd.contiguous().to(torch.float32)
    d_amps_raw = torch.empty_like(amps)
    d_hd_raw = torch.empty_like(hd)
    flags = (_lib.CTL_SCALE if scale else 0) | (_lib.CTL_NYQUIST if nyq else 0)
    core._launch('ddsp_b200_harmonic_controls_vjp', amps, hd, f0_hz, d_amplitudes, d_hd,
                 d_amps_raw, d_hd_raw, b, f, k, sample_rate, flags)
    want = ctx.needs_input_grad
    return (d_amps_raw if want[0] else None, d_hd_raw if want[1] else None, None, None,
            None, None)


class NoiseControlsFn(torch.autograd.Function):
  """core.noise_controls (FilteredNoise.get_controls, synths.py:165-179),
  differentiable in the raw magnitudes: `ddsp_b200_noise_controls_backward`.  Without
  `scale` the op is the identity and so is its gradient."""

  @staticmethod
  def forward(ctx, magnitudes, initial_bias, scale):
    ctx.save_for_backward(magnitudes)
    ctx.cfg = (float(initial_bias), bool(scale))
    return core.noise_controls(magnitudes, *ctx.cfg)

  @staticmethod
  def backward(ctx, d_mags):
    mags, = ctx.saved_tensors
    bias, scale = ctx.cfg
    if not scale:
      return d_mags, None, None
    d_mags = d_mags.contiguous().to(torch.float32)
    d_raw = torch.empty_like(mags)
    core._launch('ddsp_b200_noise_controls_backward', mags, d_mags, d_raw, mags.numel(),
                 bias)
    return d_raw, None, None


class FftConvolveLtiFn(torch.autograd.Function):
  """core.fft_convolve with one long impulse response per item (effects.Reverb,
  effects.py:103-117), differentiable in both operands:
    y[n]      = sum_s h[s] x[n + start - s]
    dL/dx[m]  = (g * reverse(h)) [m + S - 1 - start]
    dL/dh[s]  = (g * reverse(x)) [s + N - 1 - start]     (summed over the batch when
                                                          the IR is shared)
  - three calls of the same partitioned overlap-save kernels.  The crop ends at
  start + out_len, so audio samples and taps at or beyond it reach no output: their
  gradients are zero and only the taps / samples below it are convolved (an
  impulse response longer than the audio asks for a d IR crop past the end of
  g * reverse(x) otherwise)."""

  @staticmethod
  def forward(ctx, audio, ir, start, out_len):
    audio = core.torch_float32(audio)
    ir = core.torch_float32(ir)
    ctx.save_for_backward(audio, ir)
    ctx.cfg = (int(start), int(out_len))
    return core.fft_convolve_lti(audio, ir, start, out_len)

  @staticmethod
  def backward(ctx, g):
    audio, ir = ctx.saved_tensors
    start, out_len = ctx.cfg
    b, n = audio.shape
    ir_batch, s = ir.shape
    g = g.contiguous().to(torch.float32)
    end = start + out_len
    d_audio = d_ir = None
    if ctx.needs_input_grad[0]:
      live = min(n, end)
      off = s - 1 - start
      if off >= 0:
        d_audio = core.fft_convolve_lti(g, ir, off, live, reverse_ir=True)
      else:      # crop starts beyond the IR length: shift through a padded gradient
        gp = torch.nn.functional.pad(g, (-off, 0))
        d_audio = core.fft_convolve_lti(gp, ir, 0, live, reverse_ir=True)
      d_audio = torch.nn.functional.pad(d_audio, (0, n - live))
    if ctx.needs_input_grad[1]:
      live = min(s, end)
      off = n - 1 - start
      if off >= 0:
        d_ir = core.fft_convolve_lti(g, audio, off, live, reverse_ir=True)
      else:
        gp = torch.nn.functional.pad(g, (-off, 0))
        d_ir = core.fft_convolve_lti(gp, audio, 0, live, reverse_ir=True)
      d_ir = torch.nn.functional.pad(d_ir, (0, s - live))
      if ir_batch == 1 and b > 1:
        d_ir = d_ir.sum(0, keepdim=True)
    return d_audio, d_ir, None, None


class FirTimeVaryingFn(torch.autograd.Function):
  """core.fft_convolve on its direct-form route (impulse responses [1 or B, F, S]
  with S < FFT_CONVOLVE_MIN_IR), differentiable in audio and impulse response: one
  backward call of `ddsp_b200_fir_time_varying_backward` (csrc/fir_backward.cuh)
  computes the gradients asked for.  `delay` is the crop start (< 0: automatic)."""

  @staticmethod
  def forward(ctx, audio, ir, padding, delay):
    audio = core.torch_float32(audio)
    ir = core.torch_float32(ir)
    ctx.save_for_backward(audio, ir)
    ctx.cfg = (padding, int(delay))
    return core.fft_convolve(audio, ir, padding=padding, delay_compensation=delay)

  @staticmethod
  def backward(ctx, g):
    audio, ir = ctx.saved_tensors
    padding, delay = ctx.cfg
    b, n = audio.shape
    ir_batch, f, s = ir.shape
    g = g.contiguous().to(torch.float32)
    d_audio = torch.empty_like(audio) if ctx.needs_input_grad[0] else None
    d_ir = torch.empty_like(ir) if ctx.needs_input_grad[1] else None
    ws = (core._workspace('ddsp_b200_fir_time_varying_backward_workspace', audio.device, b,
                          n, f, s, ir_batch) if d_ir is not None else (None, 0))
    core._launch('ddsp_b200_fir_time_varying_backward', audio, ir, g, d_audio, d_ir, b, n,
                 f, s, ir_batch, _lib.PADDING[padding], delay, *ws)
    return d_audio, d_ir, None, None


class FrequencyImpulseResponseFn(torch.autograd.Function):
  """core.frequency_impulse_response, differentiable in the magnitudes:
  `ddsp_b200_frequency_impulse_response_backward` is the transpose of the windowed
  cosine sum."""

  @staticmethod
  def forward(ctx, magnitudes, window_size):
    magnitudes = core.torch_float32(magnitudes)
    ctx.cfg = (tuple(magnitudes.shape), int(window_size))
    return core.frequency_impulse_response(magnitudes, window_size=window_size)

  @staticmethod
  def backward(ctx, d_ir):
    shape, window_size = ctx.cfg
    nb = shape[-1]
    d_ir = d_ir.contiguous().to(torch.float32)
    d_mags = torch.empty(shape, dtype=torch.float32, device=d_ir.device)
    core._launch('ddsp_b200_frequency_impulse_response_backward', d_ir, d_mags,
                 d_mags.numel() // nb, nb, window_size)
    return d_mags, None


class FrequencyFilterFn(torch.autograd.Function):
  """core.frequency_filter on the direct-form route (impulse responses shorter than
  FFT_CONVOLVE_MIN_IR), differentiable in audio and magnitudes.  The forward's
  impulse responses are saved, not recomputed; one backward call of
  `ddsp_b200_frequency_filter_backward`, which picks the d magnitudes route."""

  @staticmethod
  def forward(ctx, audio, magnitudes, window_size, padding):
    audio = core.torch_float32(audio)
    magnitudes = core.torch_float32(magnitudes)
    ir = core.frequency_impulse_response(magnitudes, window_size=window_size)
    ctx.save_for_backward(audio, ir)
    ctx.cfg = (tuple(magnitudes.shape), int(window_size), padding)
    return core.fft_convolve(audio, ir, padding=padding)

  @staticmethod
  def backward(ctx, g):
    audio, ir = ctx.saved_tensors
    shape, window_size, padding = ctx.cfg
    b, n = audio.shape
    mb, nb = shape[0], shape[-1]
    f = shape[1] if len(shape) == 3 else 1
    pad = _lib.PADDING[padding]
    g = g.contiguous().to(torch.float32)
    d_audio = torch.empty_like(audio) if ctx.needs_input_grad[0] else None
    d_mags = (torch.empty(shape, dtype=torch.float32, device=audio.device)
              if ctx.needs_input_grad[1] else None)
    ws = (core._workspace('ddsp_b200_frequency_filter_backward_workspace', audio.device, b,
                          f, nb, n, mb, window_size, pad) if d_mags is not None else (None, 0))
    core._launch('ddsp_b200_frequency_filter_backward', audio, ir, g, d_audio, d_mags, b, f,
                 nb, n, mb, window_size, pad, *ws)
    return d_audio, d_mags, None, None


class SincImpulseResponseFn(torch.autograd.Function):
  """core.sinc_impulse_response, differentiable in the cutoff:
  `ddsp_b200_sinc_impulse_response_backward` recomputes each frame's taps and their
  derivative on chip (csrc/sinc.cuh)."""

  @staticmethod
  def forward(ctx, cutoff, s, shape, scale, high_pass):
    ctx.save_for_backward(cutoff)
    ctx.cfg = (s, scale, high_pass)
    return core.sinc_impulse_response_forward(cutoff, s, shape, scale, high_pass)

  @staticmethod
  def backward(ctx, d_ir):
    cutoff, = ctx.saved_tensors
    s, scale, high_pass = ctx.cfg
    d_ir = d_ir.contiguous().to(torch.float32)
    d_cutoff = torch.empty_like(cutoff)
    core._launch('ddsp_b200_sinc_impulse_response_backward', cutoff, d_ir, d_cutoff,
                 cutoff.numel(), s, scale, int(high_pass))
    return d_cutoff, None, None, None, None


class SincFilterFn(torch.autograd.Function):
  """core.sinc_filter on the fused route (fewer than FFT_CONVOLVE_MIN_IR taps),
  differentiable in audio and cutoff.  Nothing but the inputs is saved: one call of
  `ddsp_b200_sinc_filter_backward` rebuilds each frame's taps and computes the
  gradients asked for."""

  @staticmethod
  def forward(ctx, audio, cutoff, s, scale, high_pass, padding, cutoff_batch, n_frames):
    ctx.save_for_backward(audio, cutoff)
    ctx.cfg = (s, scale, high_pass, padding, cutoff_batch, n_frames)
    return core.sinc_filter_forward(audio, cutoff, s, scale, high_pass, padding,
                                    cutoff_batch, n_frames)

  @staticmethod
  def backward(ctx, g):
    audio, cutoff = ctx.saved_tensors
    s, scale, high_pass, padding, cutoff_batch, n_frames = ctx.cfg
    b, n = audio.shape
    g = g.contiguous().to(torch.float32)
    d_audio = torch.empty_like(audio) if ctx.needs_input_grad[0] else None
    d_cutoff = torch.empty_like(cutoff) if ctx.needs_input_grad[1] else None
    ws = (core._workspace('ddsp_b200_sinc_filter_backward_workspace', audio.device, b, n,
                          n_frames, s, cutoff_batch) if d_cutoff is not None else (None, 0))
    core._launch('ddsp_b200_sinc_filter_backward', audio, cutoff, g, d_audio, d_cutoff, b, n,
                 n_frames, s, cutoff_batch, scale, int(high_pass), _lib.PADDING[padding],
                 *ws)
    return d_audio, d_cutoff, None, None, None, None, None, None


class FilteredNoiseFn(torch.autograd.Function):
  """FilteredNoise.get_signal (synths.py:181-196), differentiable in magnitudes."""

  @staticmethod
  def forward(ctx, magnitudes, n_samples, window_size, noise, seed, offset):
    magnitudes = core.torch_float32(magnitudes)
    ctx.cfg = (int(n_samples), int(window_size), int(seed), int(offset),
               tuple(magnitudes.shape))
    ctx.noise = None if noise is None else core.torch_float32(noise)
    return core.filtered_noise(magnitudes, n_samples, window_size=window_size,
                               noise=ctx.noise, seed=seed, offset=offset)

  @staticmethod
  def backward(ctx, grad_audio):
    n_samples, window_size, seed, offset, (b, f, nb) = ctx.cfg
    grad_audio = grad_audio.contiguous().to(torch.float32)
    dmags = torch.empty((b, f, nb), dtype=torch.float32, device=grad_audio.device)
    core._launch('ddsp_b200_filtered_noise_backward', grad_audio, ctx.noise, seed, offset,
                 dmags, b, f, nb, n_samples, window_size)
    return dmags, None, None, None, None, None


class SinusoidalSynthesisFn(torch.autograd.Function):
  """core.sinusoidal_synthesis (Sinusoidal.get_signal, synths.py:305-323, on the
  fused route: 'window' / 'linear' amplitudes, an integer hop), differentiable in
  frequencies and amplitudes.  One backward call of `ddsp_b200_sinusoidal_backward`
  (csrc/sinusoidal.cuh); d frequencies, the phase path, only when asked for.  The
  Nyquist mask has subgradient 0 (tf.where)."""

  @staticmethod
  def forward(ctx, frequencies, amplitudes, n_samples, sample_rate, amp_resample_method):
    frequencies = core.torch_float32(frequencies)
    amplitudes = core.torch_float32(amplitudes)
    ctx.save_for_backward(frequencies, amplitudes)
    ctx.cfg = (int(n_samples), float(sample_rate), amp_resample_method)
    return core.sinusoidal_synthesis(frequencies, amplitudes, n_samples=n_samples,
                                     sample_rate=sample_rate,
                                     amp_resample_method=amp_resample_method)

  @staticmethod
  def backward(ctx, grad_audio):
    frequencies, amplitudes = ctx.saved_tensors
    n_samples, sample_rate, method = ctx.cfg
    b, f, k = amplitudes.shape
    g = grad_audio.contiguous().to(torch.float32)
    d_amp = torch.empty_like(amplitudes)
    d_freq = torch.empty_like(frequencies) if ctx.needs_input_grad[0] else None
    core._launch('ddsp_b200_sinusoidal_backward', frequencies, amplitudes, g, d_freq, d_amp,
                 b, f, k, n_samples, sample_rate, core.AMP_METHODS[method],
                 *core._workspace('ddsp_b200_sinusoidal_backward_workspace',
                                  amplitudes.device, b, f, k))
    return d_freq, d_amp if ctx.needs_input_grad[1] else None, None, None, None


class OscillatorBankFn(torch.autograd.Function):
  """core.oscillator_bank (core.py:911-962) on audio-rate envelopes [B, N, K],
  differentiable in frequency and amplitude envelopes.  One call of
  `ddsp_b200_oscillator_bank_backward` (csrc/oscbank.cuh) computes the gradients asked
  for from the saved inputs, on the forward's exact phase; the Nyquist mask has
  subgradient 0 (tf.where)."""

  @staticmethod
  def forward(ctx, f, a, sample_rate, sum_sinusoids):
    ctx.save_for_backward(f, a)
    ctx.cfg = (sample_rate, sum_sinusoids)
    return core.oscillator_bank_forward(f, a, sample_rate, sum_sinusoids)

  @staticmethod
  def backward(ctx, grad):
    f, a = ctx.saved_tensors
    sample_rate, sum_sinusoids = ctx.cfg
    b, n, k = f.shape
    g = grad.contiguous().to(torch.float32)
    want = ctx.needs_input_grad
    d_f = torch.empty_like(f) if want[0] else None
    d_a = torch.empty_like(a) if want[1] else None
    core._launch('ddsp_b200_oscillator_bank_backward', f, a, g, d_f, d_a, b, n, k,
                 sample_rate, int(sum_sinusoids))
    return d_f, d_a, None, None


class AngularCumsumFn(torch.autograd.Function):
  """core.angular_cumsum (core.py:799-866) on [batch, time, ...], differentiable in the
  angular frequency: the gradient is the reverse running sum of the upstream gradient
  along time (`ddsp_b200_angular_cumsum_backward`)."""

  @staticmethod
  def forward(ctx, x):
    ctx.shape = tuple(x.shape)
    return core.angular_cumsum_forward(x)

  @staticmethod
  def backward(ctx, grad):
    b, n, c = core._bnc(ctx.shape)
    g = grad.contiguous().to(torch.float32)
    d_x = torch.empty(ctx.shape, dtype=torch.float32, device=g.device)
    core._launch('ddsp_b200_angular_cumsum_backward', g, d_x, b, n, c)
    return d_x


class HarmonicOscillatorBankFn(torch.autograd.Function):
  """core.harmonic_oscillator_bank (core.py:966-1025) on f [B, N, 1], a [B, N, K] and
  init [B, 1, 1] or None, differentiable in all three through both outputs (audio and
  final phase).  One call of `ddsp_b200_harmonic_oscillator_bank_backward`
  (csrc/harmonic_bank.cuh) computes the gradients asked for on the forward's exact phase."""

  @staticmethod
  def forward(ctx, f, a, init, sample_rate, use_angular_cumsum):
    ctx.save_for_backward(f, a, init)
    ctx.sample_rate = sample_rate
    return core.harmonic_oscillator_bank_forward(f, a, init, sample_rate,
                                                 use_angular_cumsum)

  @staticmethod
  def backward(ctx, grad_audio, grad_final_phase):
    f, a, init = ctx.saved_tensors
    b, n, k = a.shape
    g = (torch.zeros((b, n), dtype=torch.float32, device=a.device) if grad_audio is None
         else grad_audio.contiguous().to(torch.float32))
    g_phi = (None if grad_final_phase is None
             else grad_final_phase.contiguous().to(torch.float32))
    want = ctx.needs_input_grad
    d_f = torch.empty_like(f) if want[0] else None
    d_a = torch.empty_like(a) if want[1] else None
    d_init = torch.empty_like(init) if init is not None and want[2] else None
    if b == 0:
      return d_f, d_a, d_init, None, None
    core._launch('ddsp_b200_harmonic_oscillator_bank_backward', f, a, init, g, g_phi, d_f,
                 d_a, d_init, b, n, k, ctx.sample_rate)
    return d_f, d_a, d_init, None, None


class LinearLookupFn(torch.autograd.Function):
  """core.linear_lookup (core.py:1168-1214) on phase [B, N] (or [B, N, 1]) and tables
  [B, W], [B, 1, W] or [B, N, W], differentiable in both: one call of
  `ddsp_b200_linear_lookup_backward` (csrc/lookup.cuh).  d phase follows TensorFlow's
  subgradients of abs and relu, so it is 0 on a grid point."""

  @staticmethod
  def forward(ctx, phase, wavetables, per_sample):
    ctx.save_for_backward(phase, wavetables)
    ctx.per_sample = per_sample
    return core.linear_lookup_forward(phase, wavetables, per_sample)

  @staticmethod
  def backward(ctx, grad):
    phase, wavetables = ctx.saved_tensors
    b, n = phase.shape[:2]
    w = wavetables.shape[-1]
    g = grad.contiguous().to(torch.float32)
    want = ctx.needs_input_grad
    d_phase = torch.empty_like(phase) if want[0] else None
    d_tab = torch.empty_like(wavetables) if want[1] else None
    if b == 0:
      return d_phase, d_tab, None
    core._launch('ddsp_b200_linear_lookup_backward', phase, wavetables, g, d_phase, d_tab,
                 b, n, w, int(ctx.per_sample))
    return d_phase, d_tab, None


class WavetableSynthesisFn(torch.autograd.Function):
  """core.wavetable_synthesis on the kernel's operands (f0 and amplitudes [B, F],
  tables [B, Fw, W]), differentiable in all three: one backward call of
  `ddsp_b200_wavetable_backward` (csrc/wavetable.cuh) computes the gradients that
  are asked for.  d f0 is 0 where the lookup position is an integer, TensorFlow's
  subgradient of linear_lookup."""

  @staticmethod
  def forward(ctx, f0, amplitudes, wavetables, n_samples, sample_rate, method):
    ctx.save_for_backward(f0, amplitudes, wavetables)
    ctx.cfg = (n_samples, sample_rate, method)
    return core.wavetable_forward(f0, amplitudes, wavetables, n_samples, sample_rate,
                                  method)

  @staticmethod
  def backward(ctx, grad_audio):
    f0, amplitudes, wavetables = ctx.saved_tensors
    n_samples, sample_rate, method = ctx.cfg
    b, f = amplitudes.shape
    _, fw, w = wavetables.shape
    g = grad_audio.contiguous().to(torch.float32)
    want = ctx.needs_input_grad
    d_f0 = torch.empty_like(f0) if want[0] else None
    d_amp = torch.empty_like(amplitudes) if want[1] else None
    d_tab = torch.empty_like(wavetables) if want[2] else None
    core._launch('ddsp_b200_wavetable_backward', f0, amplitudes, wavetables, g, d_f0, d_amp,
                 d_tab, b, f, n_samples, fw, w, sample_rate, core.AMP_METHODS[method],
                 *core._workspace('ddsp_b200_wavetable_backward_workspace',
                                  amplitudes.device, b, f, n_samples, fw, w))
    return d_f0, d_amp, d_tab, None, None, None


class ModDelayFn(torch.autograd.Function):
  """core.mod_delay (ModDelay.get_signal, effects.py:370-394, and
  core.variable_length_delay, core.py:1285-1314) on [B, N] operands,
  differentiable in audio, gain and phase; one backward kernel writes the three
  gradients (csrc/mod_delay.cuh).  gain may be None (variable_length_delay)."""

  @staticmethod
  def forward(ctx, audio, gain, phase, max_length, scale, offset, add_dry):
    ctx.save_for_backward(audio, gain, phase)
    ctx.cfg = (max_length, scale, offset, add_dry)
    return core.mod_delay_forward(audio, gain, phase, max_length, scale, offset,
                                  add_dry)

  @staticmethod
  def backward(ctx, grad_out):
    audio, gain, phase = ctx.saved_tensors
    max_length, scale, offset, add_dry = ctx.cfg
    g = grad_out.contiguous().to(torch.float32)
    want = ctx.needs_input_grad
    d_audio = torch.empty_like(audio) if want[0] else None
    d_gain = torch.empty_like(gain) if gain is not None and want[1] else None
    d_phase = torch.empty_like(phase) if want[2] else None
    b, n = audio.shape
    core._launch('ddsp_b200_mod_delay_backward', audio, phase, gain, g, d_audio, d_gain,
                 d_phase, b, n, max_length, scale, offset, int(add_dry))
    return d_audio, d_gain, d_phase, None, None, None, None


class ResampleFn(torch.autograd.Function):
  """core.resample / core.upsample_with_windows on [B, F, C] (core.py:573-714),
  differentiable in the input: the backward kernel is the forward's transpose
  (csrc/routing.cuh), every method and add_endpoint value."""

  @staticmethod
  def forward(ctx, inputs, n_timesteps, method, add_endpoint):
    ctx.cfg = (tuple(inputs.shape), int(n_timesteps), method, bool(add_endpoint))
    return core.resample_forward(inputs, n_timesteps, method, add_endpoint)

  @staticmethod
  def backward(ctx, g):
    (b, f, c), n, method, add_endpoint = ctx.cfg
    g = g.contiguous().to(torch.float32)
    d_in = torch.empty((b, f, c), dtype=torch.float32, device=g.device)
    core._launch('ddsp_b200_resample_backward', g, d_in, b, f, c, n,
                 core._RESAMPLE_METHODS[method], int(add_endpoint))
    return d_in, None, None, None


class AddFn(torch.autograd.Function):
  """core.add (processors.Add, processors.py:174-176): the gradient goes to each
  input, summed over the dimensions it was broadcast along."""

  @staticmethod
  def forward(ctx, a, b):
    ctx.shapes = (a.shape, b.shape)
    return core.add_forward(a, b)

  @staticmethod
  def backward(ctx, g):
    sa, sb = ctx.shapes
    want = ctx.needs_input_grad
    return (g.sum_to_size(sa) if want[0] else None,
            g.sum_to_size(sb) if want[1] else None)


class MixFn(torch.autograd.Function):
  """core.mix (processors.Mix.get_signal, processors.py:217-233), differentiable in
  both signals and the mix level: one backward kernel writes the gradients asked
  for (csrc/routing.cuh).  d mix_level is NaN where the level is exactly 0 or 1,
  as in the reference."""

  @staticmethod
  def forward(ctx, signal_one, signal_two, mix_level):
    ctx.save_for_backward(signal_one, signal_two, mix_level)
    return core.mix_forward(signal_one, signal_two, mix_level)

  @staticmethod
  def backward(ctx, g):
    s1, s2, m = ctx.saved_tensors
    b, n, c = s1.shape
    g = g.contiguous().to(torch.float32)
    want = ctx.needs_input_grad
    d1 = torch.empty_like(s1) if want[0] else None
    d2 = torch.empty_like(s2) if want[1] else None
    dm = torch.empty_like(m) if want[2] else None
    core._launch('ddsp_b200_mix_backward', s1, s2, m, g, d1, d2, dm, b, n, c)
    return d1, d2, dm


class ExpDecayIrFn(torch.autograd.Function):
  """core.exp_decay_ir (ExpDecayReverb._get_ir, effects.py:144-151) on [rows] scaled
  gain and raw decay, differentiable in both.  The backward regenerates the noise
  (or reads the injected row) instead of saving the impulse response."""

  @staticmethod
  def forward(ctx, gain, decay, reverb_length, noise, seed, offset):
    ctx.save_for_backward(gain, decay)
    ctx.noise = noise
    ctx.cfg = (int(reverb_length), int(seed), int(offset))
    return core.exp_decay_ir_forward(gain, decay, reverb_length, noise, seed, offset)

  @staticmethod
  def backward(ctx, g):
    gain, decay = ctx.saved_tensors
    length, seed, offset = ctx.cfg
    g = g.contiguous().to(torch.float32)
    want = ctx.needs_input_grad
    d_gain = torch.empty_like(gain) if want[0] else None
    d_decay = torch.empty_like(decay) if want[1] else None
    core._launch('ddsp_b200_exp_decay_ir_backward', gain, decay, ctx.noise, seed, offset, g,
                 d_gain, d_decay, gain.shape[0], length)
    return d_gain, d_decay, None, None, None, None


class MixtureNLLFn(torch.autograd.Function):
  """-log p(x | mixture) per query (csrc/consistency.cuh, mode A): for queries x
  [B, T, Q], components mu and log-weights lw [B, T, J] and a scalar scale, the
  Gaussian mixture NLL of each query under its own frame's mixture, [B, T, Q].  The
  mixture of `KDEConsistencyLoss.nll` and `TWMLoss`'s p(harmonics | sinusoids);
  differentiable in x, mu and lw by one backward launch.  With no components the
  logsumexp is over nothing: the NLL is +inf and every gradient 0.  With no queries
  the NLL is empty and nothing depends on mu or lw: their gradients are 0."""

  @staticmethod
  def forward(ctx, x, mu, lw, scale):
    x, mu, lw = (t.contiguous().to(torch.float32) for t in (x, mu, lw))
    b, t, q = x.shape
    j = mu.shape[-1]
    ctx.save_for_backward(x, mu, lw)
    ctx.scale = float(scale)
    if j == 0:
      return torch.full_like(x, math.inf)
    nll = torch.empty_like(x)
    core._launch('ddsp_b200_mixture_nll_forward', x, mu, lw, nll, b, t, q, j, ctx.scale)
    return nll

  @staticmethod
  def backward(ctx, grad):
    x, mu, lw = ctx.saved_tensors
    b, t, q = x.shape
    j = mu.shape[-1]
    g = grad.contiguous().to(torch.float32)
    if j == 0 or q == 0:
      # the kernel writes nothing when either is empty (include/ddsp_b200.h)
      dx, dmu, dlw = torch.zeros_like(x), torch.zeros_like(mu), torch.zeros_like(lw)
    else:
      dx, dmu, dlw = torch.empty_like(x), torch.empty_like(mu), torch.empty_like(lw)
      core._launch('ddsp_b200_mixture_nll_backward', x, mu, lw, g, dx, dmu, dlw, b, t, q,
                   j, ctx.scale)
    want = ctx.needs_input_grad
    return (dx if want[0] else None, dmu if want[1] else None,
            dlw if want[2] else None, None)


class CombNLLFn(torch.autograd.Function):
  """`TWMLoss`'s amplitude-weighted -log p(sinusoids | harmonics) (csrc/consistency.cuh,
  mode B): for candidates f0 [B, T, C], points f and amplitudes a [B, T, P], the
  `safe_divide`d mean over points of the comb NLL of f_p / f0_c, [B, T, C];
  differentiable in f0, f and a by one backward launch.  With no points the mean is
  0 / 1e-7 = 0."""

  @staticmethod
  def forward(ctx, f0, f, a, n_gaussians, scale):
    f0, f, a = (t.contiguous().to(torch.float32) for t in (f0, f, a))
    b, t, c = f0.shape
    p = f.shape[-1]
    ctx.save_for_backward(f0, f, a)
    ctx.cfg = (int(n_gaussians), float(scale))
    if p == 0:
      return torch.zeros_like(f0)
    out = torch.empty_like(f0)
    core._launch('ddsp_b200_comb_nll_forward', f0, f, a, out, b, t, c, p, *ctx.cfg)
    return out

  @staticmethod
  def backward(ctx, grad):
    f0, f, a = ctx.saved_tensors
    b, t, c = f0.shape
    p = f.shape[-1]
    g = grad.contiguous().to(torch.float32)
    if p == 0 or c == 0:
      d_f0, d_f, d_a = torch.zeros_like(f0), torch.zeros_like(f), torch.zeros_like(a)
    else:
      d_f0, d_f, d_a = torch.empty_like(f0), torch.empty_like(f), torch.empty_like(a)
      core._launch('ddsp_b200_comb_nll_backward', f0, f, a, g, d_f0, d_f, d_a, b, t, c, p,
                   *ctx.cfg)
    want = ctx.needs_input_grad
    return (d_f0 if want[0] else None, d_f if want[1] else None,
            d_a if want[2] else None, None, None)


class SinusoidalToHarmonicFn(torch.autograd.Function):
  """core.sinusoidal_to_harmonic, differentiable in sin_amps, sin_freqs and f0_hz.
  Nothing but the inputs is saved: one call of
  `ddsp_b200_sinusoidal_to_harmonic_backward` (csrc/consistency.cuh, mode C) recomputes
  each frame's weights and writes all three gradients, zeros where nothing contributes."""

  @staticmethod
  def forward(ctx, sin_amps, sin_freqs, f0_hz, n_harmonics, harmonic_width, sample_rate,
              normalize):
    ctx.save_for_backward(sin_amps, sin_freqs, f0_hz)
    ctx.cfg = (n_harmonics, harmonic_width, sample_rate, normalize)
    return core.sinusoidal_to_harmonic_forward(sin_amps, sin_freqs, f0_hz, *ctx.cfg)

  @staticmethod
  def backward(ctx, g_amp, g_dist):
    a, f, f0 = ctx.saved_tensors
    k, width, sample_rate, normalize = ctx.cfg
    b, t, s = a.shape
    g_amp = g_amp.contiguous().to(torch.float32)
    g_dist = g_dist.contiguous().to(torch.float32)
    d_a, d_f, d_f0 = torch.empty_like(a), torch.empty_like(f), torch.empty_like(f0)
    core._launch('ddsp_b200_sinusoidal_to_harmonic_backward', a, f, f0, g_amp, g_dist, d_a,
                 d_f, d_f0, b, t, s, k, width, sample_rate, int(normalize))
    want = ctx.needs_input_grad
    return (d_a if want[0] else None, d_f if want[1] else None, d_f0 if want[2] else None,
            None, None, None, None)


class HmmLogProbFn(torch.autograd.Function):
  """core.hmm_log_prob, differentiable in the observations [B, T, 2].  Nothing but the
  inputs is saved: `ddsp_b200_hmm_log_prob_backward` (csrc/hmm.cuh) re-runs the forward
  algorithm with a checkpoint every ~sqrt(T) steps ([B, ceil(T / seg), K] floats of
  scratch, 4 MB at B = 256, T = 1000, K = 128) and scans the posterior marginals back
  segment by segment."""

  @staticmethod
  def forward(ctx, x, loc, scale, hold, other):
    ctx.save_for_backward(x, loc, scale)
    ctx.cfg = (hold, other)
    return core.hmm_log_prob_forward(x, loc, scale, hold, other)

  @staticmethod
  def backward(ctx, g):
    x, loc, scale = ctx.saved_tensors
    b, t, _ = x.shape
    k = loc.shape[0]
    seg = core.hmm_segment(t, k)
    d_x = torch.empty_like(x)
    ckpt = torch.empty((b, -(-t // seg), k), dtype=torch.float32, device=x.device)
    core._launch('ddsp_b200_hmm_log_prob_backward', x, loc, scale,
                 g.contiguous().to(torch.float32), d_x, ckpt, seg, b, t, k, *ctx.cfg)
    return d_x, None, None, None, None



class WassersteinFn(torch.autograd.Function):
  """losses.wasserstein_distance on [R, Nu] values u and weights wu, [R, Nv] values v and
  weights wv (csrc/wasserstein.cuh): the [R] distances, differentiable in all four by one
  backward launch that re-sorts each row.  Nothing but the inputs is saved.  Empty sides
  are refused by the caller; R = 0 launches nothing."""

  @staticmethod
  def forward(ctx, u, v, wu, wv, p):
    u, v, wu, wv = (t.contiguous().to(torch.float32) for t in (u, v, wu, wv))
    ctx.save_for_backward(u, v, wu, wv)
    ctx.p = float(p)
    r, nu = u.shape
    out = torch.empty((r,), dtype=torch.float32, device=u.device)
    core._launch('ddsp_b200_wasserstein_forward', u, v, wu, wv, out, r, nu, v.shape[1],
                 ctx.p)
    return out

  @staticmethod
  def backward(ctx, grad):
    u, v, wu, wv = ctx.saved_tensors
    r, nu = u.shape
    du, dv, dwu, dwv = (torch.empty_like(t) for t in (u, v, wu, wv))
    core._launch('ddsp_b200_wasserstein_backward', u, v, wu, wv,
                 grad.contiguous().to(torch.float32), du, dv, dwu, dwv, r, nu, v.shape[1],
                 ctx.p)
    want = ctx.needs_input_grad
    return (du if want[0] else None, dv if want[1] else None, dwu if want[2] else None,
            dwv if want[3] else None, None)

class NoteMomentsFn(torch.autograd.Function):
  """nn.get_note_moments (pool=False) or nn.pool_over_notes (pool=True) on x [B,T,D] and
  a float mask [B,T,N] (csrc/notes.cuh): (mean, std) per note [B,N,D], or pooled back to
  the frames [B,T,D]; only the mean when `with_std` is false.  Differentiable in x only;
  the mask is a constant.  Grads are not materialised, so an output nobody uses adds no
  term: an unused std cannot turn the mean's gradient into 0 * inf = NaN.  Saves x, the
  mask and the per-note moments."""

  @staticmethod
  def forward(ctx, x, mask, pool, with_std):
    ctx.set_materialize_grads(False)
    b, t, d = x.shape
    n = mask.shape[2]
    mean = torch.empty((b, n, d), dtype=torch.float32, device=x.device)
    std = torch.empty_like(mean) if with_std else None
    pm = torch.empty_like(x) if pool else None
    ps = torch.empty_like(x) if pool and with_std else None
    core._launch('ddsp_b200_note_moments', x, mask, mean, std, pm, ps, b, t, n, d)
    ctx.save_for_backward(x, mask, mean, std)
    ctx.pool = pool
    outs = (pm, ps) if pool else (mean, std)
    return outs if with_std else outs[0]

  @staticmethod
  def backward(ctx, *grads):
    x, mask, mean, std = ctx.saved_tensors
    g = [None if a is None else a.contiguous().to(torch.float32) for a in grads]
    g += [None] * (2 - len(g))
    if g[0] is None and g[1] is None:
      return None, None, None, None
    b, t, d = x.shape
    n = mask.shape[2]
    gm, gs, gpm, gps = (None, None, g[0], g[1]) if ctx.pool else (g[0], g[1], None, None)
    dx = torch.empty_like(x)
    nbytes = 8 * b * n * d + 256 if b and n and d else 0   # A and C, [B,N,D] each
    core._launch('ddsp_b200_note_moments_backward', x, mask, mean, std, gm, gs, gpm, gps, dx,
                 *core._workspace(nbytes, x.device), b, t, n, d)
    return dx, None, None, None


class CrepeLossFramesFn(torch.autograd.Function):
  """losses.PretrainedCREPE.frame_audio on audio [B, N] (a contiguous float32 CUDA
  tensor): the frames [B, n_frames, 1024] of 1024 samples every `hop`, after 512 zeros
  on both sides when `center`, each normalised to (x - mean) / (sqrt(var) + 1e-5)
  (csrc/crepe.cuh).  Differentiable in the audio by one call of
  `ddsp_b200_crepe_frames_backward`, which recomputes each frame's statistics: only
  the audio is saved, not the frames.  A frame of variance 0 gives NaN gradients on the
  samples it covers, as TensorFlow does."""

  @staticmethod
  def forward(ctx, audio, hop, center):
    b, n = audio.shape
    padding = (_lib.PAD_CENTER if center else _lib.PAD_VALID) | _lib.CREPE_LOSS_FRAMES
    padded = n + (2 * (_lib.CREPE_FRAME // 2) if center else 0)
    n_frames = 1 + (padded - _lib.CREPE_FRAME) // hop if padded >= _lib.CREPE_FRAME else 0
    frames = torch.empty((b, n_frames, _lib.CREPE_FRAME), dtype=torch.float32,
                         device=audio.device)
    core._launch('ddsp_b200_crepe_frames', audio, frames, b, n, n_frames, hop, padding)
    ctx.save_for_backward(audio)
    ctx.cfg = (n_frames, hop, padding)
    return frames

  @staticmethod
  def backward(ctx, grad_frames):
    audio, = ctx.saved_tensors
    b, n = audio.shape
    d_audio = torch.empty_like(audio)
    core._launch('ddsp_b200_crepe_frames_backward', audio,
                 grad_frames.contiguous().to(torch.float32), d_audio, b, n, *ctx.cfg)
    return d_audio, None, None


class GruHandle:
  """A `ddsp_b200_gru` handle: the recurrent weights of one GRU layer packed for the
  recurrence kernels on one device.  Freed with the object.  Copying or pickling it
  raises TypeError: two objects would free one handle."""

  def __init__(self, units, device):
    self.units, self.device = int(units), torch.device(device)
    self.ptr = None
    self.loaded = None   # (data_ptr, version) of the weights the last load packed
    lib = _lib.load()
    out = ctypes.c_void_p()
    with torch.cuda.device(self.device):
      _lib.check(lib.ddsp_b200_gru_create(ctypes.byref(out), self.units))
    self.ptr = out.value

  def load(self, recurrent_kernel, recurrent_bias):
    core._launch('ddsp_b200_gru_load', self.ptr, recurrent_kernel, recurrent_bias)
    self.loaded = _weights_key(recurrent_kernel, recurrent_bias)

  def __del__(self):
    if self.ptr is not None:
      _lib.load().ddsp_b200_gru_destroy(self.ptr)
      self.ptr = None

  def _refuse_copy(self, *args):
    raise TypeError('GruHandle owns device memory and cannot be copied or pickled; '
                    'create a new handle (nn.Gru does so on its next call)')

  __copy__ = __deepcopy__ = __reduce_ex__ = _refuse_copy


def _weights_key(recurrent_kernel, recurrent_bias):
  return tuple((t.data_ptr(), t._version) for t in (recurrent_kernel, recurrent_bias))


class GruFn(torch.autograd.Function):
  """The Keras GRU (reset_after=True, gate columns z | r | h, h0 = 0) over x [B, T, in]
  with kernel [in, 3H], recurrent_kernel [H, 3H] and bias [2, 3H]: every state
  [B, T, H].  The input projection and the gradients' GEMMs run on cuBLAS; the
  recurrence is one `ddsp_b200_gru_forward` launch after one `ddsp_b200_gru_load`, and
  its backward one `ddsp_b200_gru_backward` launch.  The gate buffer [B, T, 4H] takes
  x W + b and then what the backward reads, so nothing else is stored.  `save` is
  whether to keep it for a backward (grad mode with an input that requires grad)."""

  @staticmethod
  def forward(ctx, x, kernel, recurrent_kernel, bias, handle, save):
    b, t, _ = x.shape
    h = handle.units
    gates = torch.empty((b, t, 4 * h), dtype=torch.float32, device=x.device)
    states = torch.empty((b, t + 1, h), dtype=torch.float32, device=x.device)
    states[:, 0].zero_()
    if b and t:
      torch.addmm(bias[0], x.reshape(b * t, -1), kernel,
                  out=gates.view(b * t, 4 * h)[:, :3 * h])
      handle.load(recurrent_kernel, bias[1])
      core._launch('ddsp_b200_gru_forward', handle.ptr, gates, states, b, t)
    if save:
      ctx.save_for_backward(x, kernel, recurrent_kernel, bias, gates, states)
      ctx.handle = handle
      ctx.key = _weights_key(recurrent_kernel, bias[1])
    return states[:, 1:]

  @staticmethod
  def backward(ctx, grad_out):
    x, kernel, recurrent_kernel, bias, gates, states = ctx.saved_tensors
    b, t, n_in = x.shape
    h = ctx.handle.units
    d_pre = torch.empty((b, t, 3 * h), dtype=torch.float32, device=x.device)
    # row t + 1 of each item is zero: d_rec and states then pair up row by row
    d_rec = torch.empty((b, t + 1, 3 * h), dtype=torch.float32, device=x.device)
    if b and t:
      if ctx.handle.loaded != ctx.key:   # another call of the layer packed other weights
        ctx.handle.load(recurrent_kernel, bias[1])
      core._launch('ddsp_b200_gru_backward', ctx.handle.ptr, gates, states,
                   grad_out.contiguous().to(torch.float32), d_pre, d_rec, b, t)
    else:
      d_pre.zero_()
      d_rec.zero_()
    d_pre2, d_rec2 = d_pre.view(b * t, 3 * h), d_rec.view(b * (t + 1), 3 * h)
    dx = (d_pre2 @ kernel.t()).view(b, t, n_in)
    d_kernel = x.reshape(b * t, n_in).t() @ d_pre2
    d_recurrent = states.view(b * (t + 1), h).t() @ d_rec2
    d_bias = torch.stack([d_pre2.sum(0), d_rec2.sum(0)])
    return dx, d_kernel, d_recurrent, d_bias, None, None


class NormReluFn(torch.autograd.Function):
  """relu(normalize(x) * scale + shift) on x [B, H, W, C] (a contiguous, 16-byte aligned
  float32 CUDA tensor) with scale and shift [C] and the channels in `groups` groups
  (csrc/norm.cuh): one `ddsp_b200_norm_relu_forward` launch, which also writes each
  (item, group)'s mean and rstd [B, groups]; those and x are all the backward keeps.
  The backward is one `ddsp_b200_norm_relu_backward` call (two launches) that gives dx,
  dscale and dshift."""

  @staticmethod
  def forward(ctx, x, scale, shift, groups):
    b, h, w, c = x.shape
    y = torch.empty_like(x)
    mean = torch.empty((b, groups), dtype=torch.float32, device=x.device)
    rstd = torch.empty_like(mean)
    if y.numel():
      core._launch('ddsp_b200_norm_relu_forward', x, scale, shift, y, mean, rstd, b, h * w,
                   c, groups, 1e-5)
    ctx.save_for_backward(x, scale, shift, mean, rstd)
    ctx.groups = groups
    return y

  @staticmethod
  def backward(ctx, grad_y):
    x, scale, shift, mean, rstd = ctx.saved_tensors
    b, h, w, c = x.shape
    if not x.numel():
      return torch.zeros_like(x), torch.zeros_like(scale), torch.zeros_like(shift), None
    dy = grad_y.to(torch.float32).contiguous()
    if dy.data_ptr() % 16:
      dy = dy.clone()
    dx = torch.empty_like(x)
    dscale, dshift = torch.empty_like(scale), torch.empty_like(shift)
    nbytes = 4 * 2 * _lib.NORM_CLUSTER * b * c   # partial [B, cluster, 2, C]
    core._launch('ddsp_b200_norm_relu_backward', x, scale, shift, mean, rstd, dy, dx, dscale,
                 dshift, *core._workspace(nbytes, x.device), b, h * w, c, ctx.groups)
    return dx, dscale, dshift, None


class NormResidualFn(torch.autograd.Function):
  """The residual site of nn.DilatedConvStack (csrc/norm.cuh): x_next = x +
  normalize(y) s + h and r = relu(x_next) over y, x [B, T, C] (contiguous, 16-byte
  aligned float32 CUDA tensors), with the channels in `groups` groups (0: no
  normalization).  s and h are scale and shift [C] (film None), or read in place from
  film [B, T, ld], the FiLM Dense output: scale in columns [0, C) and shift in [C, 2C),
  or the shift alone in [0, C) with shift_only.  Returns (x_next, r), or x_next alone
  without want_r.  One `ddsp_b200_norm_residual_forward` launch; x_next, y and the
  per-(item, group) mean and rstd are all the backward keeps.  The backward is one
  `ddsp_b200_norm_residual_backward` call: gradients to y, x and scale and shift (two
  launches) or film (one launch, written in film's layout)."""

  @staticmethod
  def forward(ctx, y, x, scale, shift, film, groups, shift_only, want_r):
    b, t, c = y.shape
    x_next = torch.empty_like(y)
    r = torch.empty_like(y) if want_r else None
    mean = torch.empty((b, groups), dtype=torch.float32, device=y.device) if groups else None
    rstd = torch.empty_like(mean) if groups else None
    ld, s, h = _norm_residual_affine(film, scale, shift, c, shift_only)
    if y.numel():
      core._launch('ddsp_b200_norm_residual_forward', y, x, s, h, ld, x_next, r, mean, rstd,
                   b, t, c, groups, 1e-5)
    ctx.save_for_backward(y, x_next, scale, film, mean, rstd)
    ctx.cfg = (groups, bool(shift_only))
    ctx.set_materialize_grads(False)
    return (x_next, r) if want_r else x_next

  @staticmethod
  def backward(ctx, gx, gr=None):
    y, x_next, scale, film, mean, rstd = ctx.saved_tensors
    groups, shift_only = ctx.cfg
    b, t, c = y.shape
    per_row = film is not None
    if gx is None and gr is None or not y.numel():
      zero = torch.zeros_like(y)
      return (zero, zero, None if per_row else torch.zeros_like(scale),
              None if per_row else torch.zeros_like(scale),
              torch.zeros_like(film) if per_row else None, None, None, None)

    def rows(g):
      g = g.to(torch.float32).contiguous()
      return g.clone() if g.data_ptr() % 16 else g

    gx = rows(gx) if gx is not None else torch.zeros_like(y)
    gr = rows(gr) if gr is not None else None
    dy, dx = torch.empty_like(y), torch.empty_like(y)
    if per_row:
      dfilm = torch.empty_like(film)   # film is [B, T, 2C], or [B, T, C] with shift_only
      ld, s, _ = _norm_residual_affine(film, None, None, c, shift_only)
      ds, dh = (None, dfilm) if shift_only else (dfilm.data_ptr(), dfilm.data_ptr() + 4 * c)
      core._launch('ddsp_b200_norm_residual_backward', y, s, ld, x_next, mean, rstd, gx, gr,
                   dy, dx, ds, dh, None, 0, b, t, c, groups)
      return dy, dx, None, None, dfilm, None, None, None
    dscale, dshift = torch.empty_like(scale), torch.empty_like(scale)
    nbytes = 4 * 2 * _lib.NORM_CLUSTER * b * c   # partial [B, cluster, 2, C]
    core._launch('ddsp_b200_norm_residual_backward', y, scale, 0, x_next, mean, rstd, gx, gr,
                 dy, dx, dscale, dshift, *core._workspace(nbytes, y.device), b, t, c, groups)
    return dy, dx, dscale, dshift, None, None, None, None


def _norm_residual_affine(film, scale, shift, c, shift_only):
  """(ld, scale, shift) arguments of the residual site's entry points: the per-channel
  tensors with ld 0, or film's row stride and the addresses of its scale and shift
  columns (scale None with shift_only)."""
  if film is None:
    return 0, scale, shift
  p, ld = film.data_ptr(), int(film.shape[-1])
  return (ld, None, film) if shift_only else (ld, p, p + 4 * c)


def exp_sigmoid(x, exponent=10.0, max_value=2.0, threshold=1e-7):
  """core.exp_sigmoid (core.py:386-404) as differentiable torch ops."""
  return max_value * torch.sigmoid(x)**math.log(exponent) + threshold


def harmonic_controls(amps, harmonic_distribution, f0_hz, sample_rate=16000,
                      normalize_below_nyquist=True):
  """Harmonic.get_controls (synths.py:94-121) as differentiable torch ops."""
  amps = exp_sigmoid(amps)
  hd = exp_sigmoid(harmonic_distribution)
  if normalize_below_nyquist:
    k = hd.shape[-1]
    ratios = torch.linspace(1.0, float(k), k, device=hd.device, dtype=hd.dtype)
    hd = torch.where(f0_hz * ratios >= sample_rate / 2.0, torch.zeros_like(hd), hd)
  denom = hd.sum(-1, keepdim=True)
  denom = torch.where(denom == 0.0, torch.full_like(denom, 1e-7), denom)
  return amps, hd / denom


def decoder_train(amps, harmonic_distribution, f0_hz, noise_magnitudes,
                  n_samples=64000, sample_rate=16000, window_size=0,
                  initial_bias=-5.0, noise=None, seed=0, offset=0,
                  amp_resample_method='window', normalize_below_nyquist=True):
  """The `ae.gin` decoder (ae.gin:47-72) with gradients to amps,
  harmonic_distribution, noise_magnitudes (and f0_hz if it requires grad) - one
  autograd node: fused forward pipeline, CUDA backward kernels for the two
  synthesizers and both `get_controls`."""
  return DecoderFn.apply(amps, harmonic_distribution, f0_hz, noise_magnitudes,
                         n_samples, sample_rate, amp_resample_method,
                         normalize_below_nyquist, window_size, initial_bias, noise,
                         seed, offset)


def decoder_train_unfused(amps, harmonic_distribution, f0_hz, noise_magnitudes,
                          n_samples=64000, sample_rate=16000, window_size=0,
                          initial_bias=-5.0, noise=None, seed=0, offset=0):
  """The same decoder with `get_controls` as differentiable torch ops around the two
  synthesizer Functions (the round-1 route; kept as a cross-check of DecoderFn)."""
  dev = core._device()
  amps = core.torch_float32(amps, dev) if not isinstance(amps, torch.Tensor) else amps
  a, h = harmonic_controls(amps, harmonic_distribution, f0_hz, sample_rate)
  harm = HarmonicSynthesisFn.apply(f0_hz, a, h, n_samples, sample_rate, 'window')
  mags = exp_sigmoid(noise_magnitudes + initial_bias)
  nz = FilteredNoiseFn.apply(mags, n_samples, window_size, noise, seed, offset)
  return harm + nz
