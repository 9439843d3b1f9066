"""Every public CUDA entry point on the tensors callers actually pass.

One table, one row per entry point: a builder of small float32 inputs, the call and
the inputs that take gradients.  The canonical call (contiguous float32 on the
current device, default stream) is checked once against the existing float64
references; every other form of the same values must give the canonical call's
bits:

  * float64, float16 and bfloat16 tensors and numpy float64 arrays (the canonical
    values being `x.float()`), strided views, `expand()`ed stride-0 batch views and
    contiguous views at storage offsets of 1, 2 and 3 floats (`data_ptr` 4, 8 or 12
    bytes off a 16-byte boundary, which selects other load paths in some kernels),
    also for `out=`;
  * the call inside `torch.cuda.stream(side)`;
  * the gradients of float16 / bfloat16 leaves (the float32 gradient cast to their
    dtype) and of offset or strided leaves (the canonical gradient);
  * a CUDA-graph capture of forward + backward, replayed.

No input is modified.  A recorder in place of the library checks, without launching
anything, that every launch goes to the operands' device and to that device's current
stream; with two devices the rows also run on cuda:1 while cuda:0 is current.
"""
import contextlib
import zlib

import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, core, effects, losses, processors, spectral_ops, synths
from oracle import ddsp_oracle as oracle
from tests import (consistency_ref, grad_ref, loudness_ref, mel_ref, mod_delay_ref,
                   routing_ref, sinc_ref, sinusoidal_ref, wavetable_ref)

B, F, N, K, NB = 2, 20, 1600, 8, 9
SR = 16000
OFFSETS = (1, 2, 3)


# ---- references ------------------------------------------------------------------
def _t(x):
  return torch.as_tensor(np.asarray(x, np.float64))


def _np(x):
  return x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)


def _phasor(x):
  """Wrapped phases compared as points on the circle (0 and 2 pi are one phase)."""
  x = np.asarray(x, np.float64)
  return np.stack([np.cos(x), np.sin(x)])


def _philox(rows, n, seed, offset=0):
  return np.asarray(oracle.philox_uniform_noise(rows, n, seed, offset), np.float64)


def _filtered_noise_ref(d, window_size):
  return oracle.noise_get_signal(d['mags'], d['noise'], window_size=window_size)


# ---- the case table --------------------------------------------------------------
class Row:
  """build(rng) -> {name: float32 array}; call(**tensors) -> output(s); grads: the
  inputs that take gradients; ref(**float64 arrays) -> the float64 output(s), with
  `cmp` (one function, or one per output, None for none) mapping both sides before
  the comparison at max-relative `tol`; out: shape of the `out=` the call takes as
  keyword `out`, or None; device_kw: the call takes `device=` (no tensor operands)."""

  def __init__(self, name, build, call, ref, tol=1e-5, grads=(), out=None, cmp=None,
               numpy=True, dtypes=True, device_kw=False):
    self.name, self.build, self.call, self.ref = name, build, call, ref
    self.tol, self.grads, self.out, self.cmp = tol, grads, out, cmp
    self.numpy, self.dtypes, self.device_kw = numpy, dtypes, device_kw

  def __call__(self, ins, device=None, **kw):
    """The call on the inputs `ins` (in the builder's order); `device` goes to the
    rows without tensor operands, which take their device as an argument."""
    if self.device_kw and device is not None:
      kw['device'] = device
    return self.call(*ins.values(), **kw)

  def inputs(self, device='cuda'):
    rng = np.random.default_rng(zlib.crc32(self.name.encode()))
    return {k: torch.as_tensor(np.asarray(v, np.float32), device=device)
            for k, v in self.build(rng).items()}


def u(rng, lo, hi, *shape):
  return rng.uniform(lo, hi, shape)


def _f0(rng):
  return u(rng, 100.0, 600.0, B, 1, 1) * (1.0 + 0.02 * u(rng, -1, 1, B, F, 1))


def _synth_inputs(rng):
  return {'amps': u(rng, 0.1, 1.0, B, F, 1), 'hd': u(rng, 0.0, 1.0, B, F, K),
          'f0': _f0(rng)}


def _raw_decoder(rng, f=F):
  f0 = u(rng, 100.0, 600.0, B, 1, 1) * (1.0 + 0.02 * u(rng, -1, 1, B, f, 1))
  return {'amps': rng.standard_normal((B, f, 1)), 'hd': rng.standard_normal((B, f, K)),
          'f0': f0, 'mags': rng.standard_normal((B, f, NB))}


def _fused_decoder(rng):
  """Hop 64: inside the fused decoder's regime."""
  return _raw_decoder(rng, N // 64)


def _audio(rng, n=N, b=B):
  return {'audio': u(rng, -1, 1, b, n)}


def _noise_row(name, f, nb, n, ws):
  def build(rng):
    return {'mags': u(rng, 0.0, 1.0, B, f, nb), 'noise': u(rng, -1, 1, B, n)}
  return Row(name, build,
             lambda mags, noise, out=None: core.filtered_noise(
                 mags, n, window_size=ws, noise=noise, out=out),
             lambda mags, noise: _filtered_noise_ref(
                 {'mags': mags, 'noise': noise}, ws),
             tol=1e-4, out=(B, n))


def _resample_row(method):
  n = N if method == 'window' else 3 * F
  return Row(f'resample_{method}', lambda rng: {'x': u(rng, -1, 1, B, F, 3)},
             lambda x: core.resample(x, n, method=method),
             lambda x: oracle.resample(x, n, method=method), grads=('x',))


def _kde(a_a, f_a, a_b, f_b):
  return losses.KDEConsistencyLoss()(a_a, f_a, a_b, f_b)


def _twm(f0c, freqs, amps):
  return losses.TWMLoss()(f0c, freqs, amps)


def _sinusoids(rng):
  return {'a_a': u(rng, 0.01, 1, B, 10, 6), 'f_a': u(rng, 100, 2000, B, 10, 6),
          'a_b': u(rng, 0.01, 1, B, 10, 5), 'f_b': u(rng, 100, 2000, B, 10, 5)}


def _new_group():
  """A fresh group per call: each call of a group advances its noise offset."""
  return processors.ProcessorGroup(dag=[
      (synths.Harmonic(n_samples=N), ['amps', 'harmonic_distribution', 'f0_hz']),
      (synths.FilteredNoise(n_samples=N, window_size=0, seed=3), ['noise_magnitudes']),
      (processors.Add(), ['filtered_noise/signal', 'harmonic/signal'])])


def _group(fused):
  return lambda amps, hd, f0, mags: (
      _new_group()({'amps': amps, 'harmonic_distribution': hd, 'f0_hz': f0,
             'noise_magnitudes': mags}) if fused else
      _new_group()({'amps': amps, 'harmonic_distribution': hd, 'f0_hz': f0,
             'noise_magnitudes': mags}, return_outputs_dict=True)['signal'])


def _decoder_ref(amps, hd, f0, mags, seed=3):
  return oracle.decoder(amps, hd, f0, mags, _philox(B, N, seed), n_samples=N,
                        window_size=0)['add']['signal']


ROWS = [
    Row('exp_sigmoid', lambda rng: {'x': rng.standard_normal((B, F, K))},
        core.exp_sigmoid, oracle.exp_sigmoid),
    *[_resample_row(m) for m in ('window', 'linear', 'nearest', 'cubic')],
    Row('harmonic_controls', _raw_decoder,
        lambda amps, hd, f0, mags: core.harmonic_controls(amps, hd, f0, SR),
        lambda amps, hd, f0, mags: [
            oracle.harmonic_get_controls(amps, hd, f0)[k]
            for k in ('amplitudes', 'harmonic_distribution')]),
    Row('noise_controls', lambda rng: {'x': rng.standard_normal((B, F, NB))},
        core.noise_controls, oracle.noise_get_controls),
    Row('angular_cumsum', lambda rng: {'x': u(rng, 0.0, 0.5, B, N, 2)},
        core.angular_cumsum, oracle.angular_cumsum, tol=2e-5, cmp=_phasor),
    Row('oscillator_bank', lambda rng: {'f': u(rng, 100, 3000, B, N, 3),
                                        'a': u(rng, 0, 1, B, N, 3)},
        lambda f, a: core.oscillator_bank(f, a, SR),
        lambda f, a: oracle.oscillator_bank(f, a, SR), tol=1e-4),
    Row('sinusoidal_synthesis', lambda rng: {'f': u(rng, 100, 3000, B, F, 4),
                                             'a': u(rng, 0, 1, B, F, 4)},
        lambda f, a, out=None: core.sinusoidal_synthesis(f, a, n_samples=N, out=out),
        lambda f, a: oracle.sinusoidal_get_signal(a, f, N), tol=1e-4, grads=('f', 'a'),
        out=(B, N)),
    Row('harmonic_synthesis', _synth_inputs,
        lambda amps, hd, f0, out=None: core.harmonic_synthesis(
            f0, amps, harmonic_distribution=hd, n_samples=N, out=out),
        lambda amps, hd, f0: oracle.harmonic_synthesis(
            f0, amps, harmonic_distribution=hd, n_samples=N), tol=1e-4, out=(B, N)),
    Row('harmonic_synthesis_shifts',
        lambda rng: dict(_synth_inputs(rng), shifts=u(rng, -0.02, 0.02, B, F, K)),
        lambda amps, hd, f0, shifts, out=None: core.harmonic_synthesis(
            f0, amps, harmonic_shifts=shifts, harmonic_distribution=hd, n_samples=N,
            out=out),
        lambda amps, hd, f0, shifts: oracle.harmonic_synthesis(
            f0, amps, harmonic_shifts=shifts, harmonic_distribution=hd, n_samples=N),
        tol=1e-4, out=(B, N)),
    Row('streaming_harmonic_synthesis',
        lambda rng: dict(_synth_inputs(rng), phase=u(rng, 0, 6, B, 1, 1)),
        lambda amps, hd, f0, phase: core.streaming_harmonic_synthesis(
            f0, amps, hd, initial_phase=phase, n_samples=N),
        lambda amps, hd, f0, phase: oracle.streaming_harmonic_synthesis(
            f0, amps, hd, initial_phase=phase, n_samples=N),
        tol=1e-4, cmp=(None, _phasor)),   # audio, final phase
    Row('frequency_impulse_response', lambda rng: {'m': u(rng, 0, 1, B, F, NB)},
        lambda m: core.frequency_impulse_response(m, window_size=11),
        lambda m: oracle.frequency_impulse_response(m, window_size=11), grads=('m',)),
    Row('fft_convolve_fir', lambda rng: dict(_audio(rng), ir=u(rng, -1, 1, B, F, 17)),
        lambda audio, ir, out=None: core.fft_convolve(audio, ir, out=out),
        lambda audio, ir: oracle.fft_convolve(audio, ir), grads=('audio', 'ir'),
        out=(B, N)),
    Row('fft_convolve_long_ir',
        lambda rng: dict(_audio(rng, 4000), ir=u(rng, -1, 1, B, 2048) * 0.05),
        lambda audio, ir: core.fft_convolve(audio, ir),
        lambda audio, ir: oracle.fft_convolve(audio, ir), tol=1e-5,
        grads=('audio', 'ir')),
    Row('fft_convolve_lti', lambda rng: dict(_audio(rng), ir=u(rng, -1, 1, 1, 300)),
        lambda audio, ir, out=None: core.fft_convolve_lti(audio, ir, 0, N, out=out),
        lambda audio, ir: _np(grad_ref.convolve_lti(_t(audio), _t(ir), 0, N)),
        out=(B, N)),
    Row('frequency_filter', lambda rng: dict(_audio(rng), m=u(rng, 0, 1, B, F, NB)),
        lambda audio, m: core.frequency_filter(audio, m, window_size=11),
        lambda audio, m: oracle.frequency_filter(audio, m, window_size=11),
        grads=('audio', 'm')),
    Row('sinc_impulse_response', lambda rng: {'c': u(rng, 0.05, 0.45, B, F, 1)},
        lambda c: core.sinc_impulse_response(c, window_size=64),
        lambda c: sinc_ref.sinc_impulse_response(c, window_size=64), grads=('c',)),
    Row('sinc_filter', lambda rng: dict(_audio(rng), c=u(rng, 0.05, 0.45, B, F, 1)),
        lambda audio, c: core.sinc_filter(audio, c, window_size=64),
        lambda audio, c: sinc_ref.sinc_filter(audio, c, window_size=64),
        grads=('audio', 'c')),
    Row('mod_delay', lambda rng: dict(_audio(rng), g=u(rng, 0, 1, B, N, 1),
                                      p=u(rng, 0.05, 0.95, B, N, 1)),
        lambda audio, g, p: core.mod_delay(audio, g, p, 100, add_dry=True),
        lambda audio, g, p: _np(mod_delay_ref.torch_mod_delay(
            _t(audio), _t(g)[..., 0], _t(p)[..., 0], 100, add_dry=True)),
        grads=('audio', 'g', 'p')),
    Row('variable_length_delay', lambda rng: dict(_audio(rng),
                                                  p=u(rng, 0.05, 0.95, B, N, 1)),
        lambda audio, p: core.variable_length_delay(p, audio, 100),
        lambda audio, p: mod_delay_ref.variable_length_delay(p, audio, 100),
        grads=('audio', 'p')),
    Row('wavetable_synthesis',
        lambda rng: {'f0': _f0(rng), 'a': u(rng, 0, 1, B, F, 1),
                     'w': u(rng, -1, 1, B, F, 64)},
        lambda f0, a, w: core.wavetable_synthesis(f0, a, w, n_samples=N),
        lambda f0, a, w: wavetable_ref.wavetable_synthesis(f0, a, w, N, SR), tol=1e-4,
        grads=('f0', 'a', 'w')),
    Row('mix', lambda rng: {'s1': u(rng, -1, 1, B, N, 1), 's2': u(rng, -1, 1, B, N, 1),
                            'm': u(rng, 0.05, 0.95, B, N, 1)},
        core.mix, lambda s1, s2, m: _np(routing_ref.mix(_t(s1), _t(s2), _t(m))),
        grads=('s1', 's2', 'm')),
    Row('exp_decay_ir',
        lambda rng: {'g': u(rng, 0.1, 1, B, 1), 'd': u(rng, 0, 2, B, 1),
                     'nz': u(rng, -1, 1, 1, 500)},
        lambda g, d, nz: core.exp_decay_ir(g, d, 500, noise=nz),
        lambda g, d, nz: _np(routing_ref.exp_decay_ir(_t(g), _t(d), 500, _t(nz))),
        grads=('g', 'd')),
    Row('uniform_noise', lambda rng: {},
        lambda device=None: core.uniform_noise(B, N, seed=5, device=device),
        lambda: _philox(B, N, 5), tol=0.0, device_kw=True),
    _noise_row('filtered_noise_ring', 25, 65, N, 0),
    _noise_row('filtered_noise_fused', F, NB, N, 0),
    _noise_row('filtered_noise_generic', F, 8, N, 0),
    Row('decoder_forward', lambda rng: dict(_fused_decoder(rng), noise=u(rng, -1, 1, B, N)),
        lambda amps, hd, f0, mags, noise: core.decoder_forward(
            amps, hd, f0, mags, N, noise=noise),
        lambda amps, hd, f0, mags, noise: oracle.decoder(
            amps, hd, f0, mags, noise, n_samples=N)['add']['signal'], tol=1e-4),
    Row('add', lambda rng: {'a': u(rng, -1, 1, B, N), 'b': u(rng, -1, 1, B, N)},
        lambda a, b, out=None: core.add(a, b, out=out), oracle.add_get_signal,
        tol=1e-7, grads=('a', 'b'), out=(B, N)),
    # spectral_ops
    Row('stft_cuda', _audio, lambda audio: spectral_ops.stft_cuda(audio, 256),
        lambda audio: _np(mel_ref.stft(_t(audio), 256)), tol=1e-5, grads=('audio',),
        cmp=lambda x: np.stack([np.real(_np(x)), np.imag(_np(x))])),
    Row('compute_loudness', _audio, spectral_ops.compute_loudness,
        lambda audio: _np(loudness_ref.compute_loudness(_t(audio))), tol=1e-4, grads=('audio',)),
    Row('compute_power', _audio, spectral_ops.compute_power,
        lambda audio: _np(loudness_ref.compute_power(_t(audio))),
        tol=1e-4),
    Row('compute_rms_energy', _audio, spectral_ops.compute_rms_energy,
        lambda audio: np.sqrt(np.mean(
            _np(loudness_ref.frames(_t(audio), 512, 64, 'center'))**2, -1)),
        tol=1e-5),
    Row('compute_mel', _audio, lambda audio: spectral_ops.compute_mel(audio, fft_size=256),
        lambda audio: _np(mel_ref.compute_mel(_t(audio), fft_size=256)), tol=1e-4,
        grads=('audio',)),
    Row('compute_logmel', _audio,
        lambda audio: spectral_ops.compute_logmel(audio, fft_size=256),
        lambda audio: _np(mel_ref.compute_logmel(_t(audio), fft_size=256)), tol=1e-4,
        grads=('audio',)),
    Row('compute_mfcc', _audio, lambda audio: spectral_ops.compute_mfcc(audio, fft_size=256),
        lambda audio: _np(mel_ref.compute_mfcc(_t(audio), fft_size=256)), tol=1e-4,
        grads=('audio',)),
    Row('compute_logmag', _audio,
        lambda audio: spectral_ops.compute_logmag(audio, size=256),
        lambda audio: _np(mel_ref.compute_logmag(_t(audio), size=256)), tol=1e-4,
        grads=('audio',), numpy=False),  # torch on the caller's tensor and device
    # losses
    Row('spectral_loss', lambda rng: {'t': u(rng, -1, 1, B, 4000),
                                      'audio': u(rng, -1, 1, B, 4000)},
        lambda t, audio: losses.SpectralLoss(fft_sizes=(512, 256, 128, 64),
                                             logmag_weight=1.0)(t, audio),
        lambda t, audio: _np(grad_ref.spectral_loss(_t(t), _t(audio), (512, 256, 128, 64),
                                                    logmag_weight=1.0)),
        tol=1e-4, grads=('audio',), numpy=False),
    Row('spectral_term', lambda rng: {'t': u(rng, -1, 1, B, N), 'audio': u(rng, -1, 1, B, N)},
        lambda t, audio: spectral_ops.SpectralTermFn.apply(
            spectral_ops.stft_cuda(t, 256).detach(), audio, 256, 64, 1.0, 1.0),
        lambda t, audio: _np(grad_ref.spectral_loss(_t(t), _t(audio), (256,),
                                                    logmag_weight=1.0)),
        tol=1e-4, grads=('audio',), numpy=False),
    Row('kde_consistency_loss', _sinusoids, _kde,
        lambda a_a, f_a, a_b, f_b: _np(consistency_ref.kde_loss(a_a, f_a, a_b, f_b)),
        tol=1e-4, grads=('a_a', 'f_a', 'a_b', 'f_b')),
    Row('twm_loss', lambda rng: {'f0c': u(rng, 80, 400, B, 10, 4),
                                 'freqs': u(rng, 100, 2000, B, 10, 6),
                                 'amps': u(rng, 0.01, 1, B, 10, 6)},
        _twm, lambda f0c, freqs, amps: _np(consistency_ref.twm_loss(f0c, freqs, amps)),
        tol=1e-4, grads=('f0c', 'freqs', 'amps')),
    # processors
    Row('Harmonic', _raw_decoder,
        lambda amps, hd, f0, mags: synths.Harmonic(n_samples=N)(amps, hd, f0),
        lambda amps, hd, f0, mags: oracle.harmonic_get_signal(
            **{'n_samples': N, **oracle.harmonic_get_controls(amps, hd, f0)}), tol=1e-4),
    Row('FilteredNoise', lambda rng: {'m': rng.standard_normal((B, F, NB))},
        lambda m: synths.FilteredNoise(n_samples=N, window_size=0, seed=3)(m),
        lambda m: oracle.noise_get_signal(oracle.noise_get_controls(m)['magnitudes'], _philox(B, N, 3),
                                          window_size=0), tol=1e-4),
    Row('Sinusoidal', lambda rng: {'a': rng.standard_normal((B, F, 4)),
                                   'f': rng.standard_normal((B, F, 4))},
        lambda a, f: synths.Sinusoidal(n_samples=N)(a, f),
        lambda a, f: oracle.sinusoidal_get_signal(
            n_samples=N, **oracle.sinusoidal_get_controls(a, f)), tol=1e-4,
        grads=('a', 'f')),
    Row('Wavetable', lambda rng: {'a': rng.standard_normal((B, F, 1)),
                                  'w': rng.standard_normal((B, F, 64)), 'f0': _f0(rng)},
        lambda a, w, f0: synths.Wavetable(n_samples=N)(a, w, f0),
        lambda a, w, f0: wavetable_ref.wavetable_synthesis(
            f0, oracle.exp_sigmoid(a), oracle.exp_sigmoid(w), N, SR), tol=1e-4,
        grads=('a', 'w', 'f0')),
    Row('Add', lambda rng: {'a': u(rng, -1, 1, B, N), 'b': u(rng, -1, 1, B, N)},
        lambda a, b: processors.Add()(a, b), oracle.add_get_signal, tol=1e-7,
        grads=('a', 'b')),
    Row('Mix', lambda rng: {'s1': u(rng, -1, 1, B, N, 1), 's2': u(rng, -1, 1, B, N, 1),
                            'm': rng.standard_normal((B, F, 1))},
        lambda s1, s2, m: processors.Mix()(s1, s2, m),
        lambda s1, s2, m: _np(routing_ref.mix_processor(_t(s1), _t(s2), _t(m))),
        grads=('s1', 's2', 'm')),
    Row('Crop', _audio, lambda audio: processors.Crop(64)(audio),
        lambda audio: audio[:, :-64], tol=0.0,
        dtypes=False, numpy=False),  # a view of the caller's tensor,
    Row('FIRFilter', lambda rng: dict(_audio(rng), m=rng.standard_normal((B, F, NB))),
        lambda audio, m: effects.FIRFilter(window_size=17)(audio, m),
        lambda audio, m: oracle.frequency_filter(audio, oracle.exp_sigmoid(m),
                                                 window_size=17), tol=1e-4,
        grads=('audio', 'm')),
    Row('ModDelay', lambda rng: dict(_audio(rng), g=rng.standard_normal((B, N, 1)),
                                     p=rng.standard_normal((B, N, 1))),
        lambda audio, g, p: effects.ModDelay()(audio, g, p),
        lambda audio, g, p: mod_delay_ref.mod_delay_get_signal(
            audio, oracle.exp_sigmoid(g), 1.0 / (1.0 + np.exp(-p))), tol=1e-4,
        grads=('audio', 'g', 'p')),
    Row('Reverb', lambda rng: dict(_audio(rng), ir=u(rng, -0.1, 0.1, B, 300)),
        lambda audio, ir: effects.Reverb(reverb_length=300)(audio, ir),
        lambda audio, ir: _np(routing_ref.reverb(_t(audio), _t(ir))), tol=1e-5,
        grads=('audio', 'ir')),
    Row('ExpDecayReverb', lambda rng: dict(_audio(rng), g=rng.standard_normal((B, 1)),
                                           d=u(rng, 0, 2, B, 1)),
        lambda audio, g, d: effects.ExpDecayReverb(reverb_length=300)(audio, g, d),
        lambda audio, g, d: _np(routing_ref.exp_decay_reverb(
            _t(audio), _t(g), _t(d), _t(_philox(1, 300, 0)), 300)), tol=1e-5,
        grads=('audio', 'g', 'd')),
    Row('FilteredNoiseReverb',
        lambda rng: dict(_audio(rng), m=rng.standard_normal((B, 10, 16))),
        lambda audio, m: effects.FilteredNoiseReverb(
            reverb_length=300, n_frames=10, window_size=0)(audio, m),
        lambda audio, m: _np(routing_ref.reverb(_t(audio), _t(oracle.noise_get_signal(
            oracle.noise_get_controls(m, initial_bias=-3.0)['magnitudes'], _philox(B, 300, 0),
            window_size=0)))), tol=1e-4,
        grads=('audio', 'm')),
    Row('ProcessorGroup_fused', _fused_decoder, _group(True), _decoder_ref, tol=1e-4),
    Row('ProcessorGroup_nodes', _raw_decoder, _group(False), _decoder_ref, tol=1e-4),
]
ROW_IDS = [r.name for r in ROWS]
GRAD_ROWS = [r for r in ROWS if r.grads]
OUT_ROWS = [r for r in ROWS if r.out]


# ---- helpers ----------------------------------------------------------------------
def _flat(res):
  if isinstance(res, dict):
    return [t for k in sorted(res) for t in _flat(res[k])]
  if isinstance(res, (list, tuple)):
    return [t for x in res for t in _flat(x)]
  return [res]


def _bits(t):
  t = t.detach()
  if t.is_complex():
    t = torch.view_as_real(t)
  return t.contiguous().reshape(-1).view(torch.uint8)


def assert_same_bits(got, want, what):
  got, want = _flat(got), _flat(want)
  assert len(got) == len(want), what
  for i, (g, w) in enumerate(zip(got, want)):
    assert g.shape == w.shape and g.dtype == w.dtype, (what, i, g.shape, w.shape)
    assert torch.equal(_bits(g), _bits(w)), (
        what, i, float((g.double() - w.double()).abs().max())
        if not g.is_complex() else 'complex')


def at_offset(x, off):
  """The values of x in a contiguous view whose storage begins `off` elements into a
  fresh buffer (data_ptr 4 * off bytes past a 256-byte allocation boundary)."""
  buf = torch.full((x.numel() + off + 5,), 7.0, dtype=x.dtype, device=x.device)
  v = buf[off:off + x.numel()].view(x.shape)
  v.copy_(x)
  return v


def strided(x):
  """The values of x in a view with a stride of 2 in the last dimension."""
  buf = torch.full(tuple(x.shape) + (2,), 7.0, dtype=x.dtype, device=x.device)
  v = buf[..., 0]
  v.copy_(x)
  return v


def expanded(x):
  """Item 0 of x broadcast over the batch (stride 0), and its canonical values."""
  if x.dim() == 0 or x.shape[0] != B:
    return x, x
  v = x[:1].expand(x.shape)
  return v, v.contiguous()


def variants(row, t):
  """(label, inputs passed, canonical float32 inputs holding the same values)."""
  for dt in (torch.float64, torch.float16, torch.bfloat16) if row.dtypes else ():
    yield str(dt).split('.')[-1], {k: v.to(dt) for k, v in t.items()}, {
        k: v.to(dt).float() for k, v in t.items()}
  if row.numpy:
    yield 'numpy', {k: v.double().cpu().numpy() for k, v in t.items()}, t
  yield 'strided', {k: strided(v) for k, v in t.items()}, t
  ex = {k: expanded(v) for k, v in t.items()}
  yield 'expand', {k: v[0] for k, v in ex.items()}, {k: v[1] for k, v in ex.items()}
  for off in OFFSETS:
    yield f'offset{off}', {k: at_offset(v, off) for k, v in t.items()}, t


def upstream(outs):
  gen = torch.Generator('cuda').manual_seed(3)
  res = []
  for o in _flat(outs):
    if o.is_complex():
      res.append(torch.randn(o.shape, generator=gen, device=o.device,
                             dtype=torch.float32).to(o.dtype))
    else:
      res.append(torch.randn(o.shape, generator=gen, device=o.device, dtype=o.dtype))
  return res


def run_grad(row, ins, gs=None):
  """Forward and backward with a fixed upstream gradient; (outputs, grads)."""
  for k in row.grads:
    ins[k].grad = None
  outs = row(ins)
  flat = _flat(outs)
  torch.autograd.backward(flat, upstream(flat) if gs is None else gs)
  return outs, {k: ins[k].grad for k in row.grads}


def with_leaves(row, t):
  """t with the inputs in row.grads made leaves that require grad (same storage)."""
  return {k: v.detach().requires_grad_(True) if k in row.grads else v
          for k, v in t.items()}


def snapshot(ins):
  return {k: (v.detach().clone() if torch.is_tensor(v) else np.array(v, copy=True))
          for k, v in ins.items()}


def assert_unchanged(before, ins, what):
  for k, v in ins.items():
    if torch.is_tensor(v):
      assert torch.equal(_bits(v), _bits(before[k])), (what, k, 'input modified')
    else:
      assert np.array_equal(v, before[k]), (what, k, 'input modified')


def needs_gpu():
  if not torch.cuda.is_available():
    pytest.skip('needs a CUDA device')


# ---- CPU-side checks of the table -------------------------------------------------
def test_table_covers_the_public_entry_points():
  names = set(ROW_IDS)
  assert len(names) == len(ROWS)
  for want in ('exp_sigmoid', 'harmonic_synthesis', 'harmonic_synthesis_shifts',
               'streaming_harmonic_synthesis', 'fft_convolve_fir',
               'fft_convolve_long_ir', 'fft_convolve_lti', 'filtered_noise_ring',
               'filtered_noise_fused', 'filtered_noise_generic', 'add', 'stft_cuda',
               'spectral_loss', 'ProcessorGroup_fused', 'ProcessorGroup_nodes'):
    assert want in names


def test_filtered_noise_rows_take_the_routes_they_name():
  for row in ROWS:
    if row.name.startswith('filtered_noise_'):
      shapes = {k: v.shape for k, v in row.build(np.random.default_rng(0)).items()}
      _, f, nb = shapes['mags']
      n = shapes['noise'][1]
      assert grad_ref.noise_route(f, nb, n, 0) == row.name.split('_')[-1]


@pytest.mark.parametrize('row', ROWS, ids=ROW_IDS)
def test_references_run_on_the_host(row):
  """The float64 side of every canonical check runs without a device."""
  d = {k: np.asarray(v, np.float64) for k, v in row.build(np.random.default_rng(0)).items()}
  want = row.ref(*d.values())
  for w in _flat(want):
    assert np.all(np.isfinite(np.asarray(_np(w), np.complex128)))


# ---- on the GPU -------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('row', ROWS, ids=ROW_IDS)
def test_canonical_call_matches_float64_reference(row):
  t = row.inputs()
  with torch.no_grad():
    got = _flat(row(t))
  want = _flat(row.ref(*[v.double().cpu().numpy() for v in t.values()]))
  assert len(got) == len(want), (row.name, len(got), len(want))
  cmps = row.cmp if isinstance(row.cmp, tuple) else (row.cmp,) * len(want)
  for g, w, cmp in zip(got, want, cmps):
    g = _np(g)
    w = _np(w)
    if cmp is not None:
      g, w = cmp(g), cmp(w)
    g = np.asarray(g, np.complex128)
    w = np.asarray(w, np.complex128)
    assert g.shape == w.shape, (row.name, g.shape, w.shape)
    peak = max(np.abs(w).max(), 1e-30)
    assert np.abs(g - w).max() <= row.tol * peak, (row.name, np.abs(g - w).max() / peak)


@pytest.mark.gpu
@pytest.mark.parametrize('row', ROWS, ids=ROW_IDS)
def test_input_forms_give_the_canonical_bits(row):
  t = row.inputs()
  with torch.no_grad():
    for label, ins, canon in variants(row, t):
      want = row(canon)
      before = snapshot(ins)
      got = row(ins)
      assert_same_bits(got, want, (row.name, label))
      assert_unchanged(before, ins, (row.name, label))


@pytest.mark.gpu
@pytest.mark.parametrize('row', OUT_ROWS, ids=[r.name for r in OUT_ROWS])
def test_out_at_every_offset(row):
  t = row.inputs()
  with torch.no_grad():
    want = row(t)
    numel = int(np.prod(row.out))
    for off in (0,) + OFFSETS:
      buf = torch.full((numel + off + 5,), 7.0, device='cuda')
      out = buf[off:off + numel].view(row.out)
      before = snapshot(t)
      got = row(t, out=out)
      assert got.data_ptr() == out.data_ptr(), (row.name, off)
      assert_same_bits(out, want, (row.name, 'out', off))
      rest = torch.cat([buf[:off], buf[off + numel:]])
      assert torch.all(rest == 7.0), (row.name, off, 'out= written outside its region')
      assert_unchanged(before, t, (row.name, 'out', off))


@pytest.mark.gpu
@pytest.mark.parametrize('row', ROWS, ids=ROW_IDS)
def test_side_stream_gives_the_canonical_bits(row):
  t = row.inputs()
  with torch.no_grad():
    want = row(t)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
      got = row(t)
    side.synchronize()
  assert_same_bits(got, want, row.name)


@pytest.mark.gpu
@pytest.mark.parametrize('row', GRAD_ROWS, ids=[r.name for r in GRAD_ROWS])
def test_gradient_forms(row):
  t = row.inputs()
  _, want = run_grad(row, with_leaves(row, t))
  for dt in (torch.float16, torch.bfloat16):
    lo = {k: v.to(dt) for k, v in t.items()}
    _, c_grad = run_grad(row, with_leaves(row, {k: v.float() for k, v in lo.items()}))
    before = snapshot(lo)
    _, grad = run_grad(row, with_leaves(row, lo))
    assert_unchanged(before, lo, (row.name, dt))
    for k in row.grads:
      assert grad[k].dtype == dt, (row.name, k, grad[k].dtype)
      assert_same_bits(grad[k], c_grad[k].to(dt), (row.name, k, dt))
  forms = [('strided', strided)] + [(f'offset{o}', lambda v, o=o: at_offset(v, o))
                                    for o in OFFSETS]
  for label, form in forms:
    ins = {k: form(v) for k, v in t.items()}
    before = snapshot(ins)
    _, grad = run_grad(row, with_leaves(row, ins))
    assert_unchanged(before, ins, (row.name, label))
    for k in row.grads:
      assert_same_bits(grad[k].contiguous(), want[k], (row.name, k, label))


@pytest.mark.gpu
@pytest.mark.parametrize('row', GRAD_ROWS, ids=[r.name for r in GRAD_ROWS])
def test_cuda_graph_replay_equals_eager(row):
  t = row.inputs()
  ins = with_leaves(row, t)
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  gs = upstream(row(ins))
  with torch.cuda.stream(side):
    for _ in range(2):
      outs, grads = run_grad(row, ins, gs)
      eager = [o.detach().clone() for o in _flat(outs)]
      eager_grads = {k: g.clone() for k, g in grads.items()}
  torch.cuda.current_stream().wait_stream(side)
  for k in row.grads:
    ins[k].grad = None
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    static = _flat(row(ins))
    torch.autograd.backward(static, gs)
  graph.replay()
  torch.cuda.synchronize()
  assert_same_bits(static, eager, row.name)
  for k in row.grads:
    assert_same_bits(ins[k].grad, eager_grads[k], (row.name, k))


@pytest.mark.gpu
def test_stft_frame_size_not_a_multiple_of_four_raises():
  audio = torch.zeros((2, 1600), device='cuda')
  with pytest.raises(ValueError):
    spectral_ops.stft_cuda(audio, 250)


@pytest.mark.gpu
def test_spectral_term_target_at_any_offset_or_stride():
  """SpectralTermFn hands the caller's target STFT to spectral_l1, which reads 16-byte
  vectors: a complex64 view at an odd element offset, or a strided one, must give the
  contiguous target's loss and gradient bits."""
  rng = np.random.default_rng(5)
  t = torch.as_tensor(u(rng, -1, 1, B, N), dtype=torch.float32, device='cuda')
  audio = torch.as_tensor(u(rng, -1, 1, B, N), dtype=torch.float32, device='cuda')
  xt = spectral_ops.stft_cuda(t, 256)

  def run(target):
    a = audio.clone().requires_grad_(True)
    loss = spectral_ops.SpectralTermFn.apply(target, a, 256, 64, 1.0, 1.0)
    loss.backward()
    return loss.detach(), a.grad

  want = run(xt)
  for label, target in [('strided', strided(xt))] + [
      (f'offset{o}', at_offset(xt, o)) for o in OFFSETS]:
    before = target.clone()
    got = run(target)
    assert_same_bits(got, want, label)
    assert torch.equal(_bits(target), _bits(before)), (label, 'target modified')


# ---- stream and device routing, with nothing launched -----------------------------
_PASS_THROUGH = ('ddsp_b200_ir_size', 'ddsp_b200_last_error', 'ddsp_b200_launch_count',
                 'ddsp_b200_version')


class Recorder:
  """Stands in for the loaded library: the functions that launch nothing go to the
  real one; every launching entry point records (name, current device, stream
  argument) and returns 0."""

  def __init__(self, real):
    self.real = real
    self.calls = []

  def __getattr__(self, name):
    if name.endswith(('_workspace', '_takes')) or name in _PASS_THROUGH:
      return getattr(self.real, name)
    assert name in _lib.SIGNATURES, name

    def launch(*args):
      self.calls.append((name, torch.cuda.current_device(), args[-1]))
      return 0
    return launch


@pytest.fixture
def recorder(monkeypatch):
  rec = Recorder(_lib.load())
  monkeypatch.setattr(_lib, 'load', lambda: rec)
  return rec


def _record(row, rec, device, stream=None):
  """The row's calls on `device` (inside `stream` when given); returns the launches."""
  rec.calls.clear()
  t = {k: v.to(device) for k, v in row.inputs().items()}
  ctx = torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext()
  with ctx:
    if row.grads:
      outs = _flat(row(with_leaves(row, t), device))
      torch.autograd.backward(outs, [torch.ones_like(o) for o in outs])
    else:
      with torch.no_grad():
        row(t, device)
  torch.cuda.synchronize(device)
  return list(rec.calls)


def _check_launches(row, calls, device, stream):
  assert calls or row.name in ('compute_logmag', 'Crop'), (row.name, 'no launch recorded')
  for name, dev, st in calls:
    assert dev == device.index, (row.name, name, 'launched on device', dev)
    assert st == stream.cuda_stream, (row.name, name, 'launched on stream', st)


@pytest.mark.gpu
@pytest.mark.parametrize('row', ROWS, ids=ROW_IDS)
def test_launches_name_the_operands_stream(row, recorder):
  dev = torch.device('cuda', torch.cuda.current_device())
  side = torch.cuda.Stream(dev)
  calls = _record(row, recorder, dev, side)
  _check_launches(row, calls, dev, side)


def needs_two_devices():
  if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
    pytest.skip('needs two CUDA devices')


@pytest.mark.gpu
@pytest.mark.parametrize('row', ROWS, ids=ROW_IDS)
def test_launches_name_the_operands_device(row, recorder):
  needs_two_devices()
  dev = torch.device('cuda', 1)
  with torch.cuda.device(0):
    calls = _record(row, recorder, dev)
  _check_launches(row, calls, dev, torch.cuda.current_stream(dev))


# ---- two devices ------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('row', ROWS, ids=ROW_IDS)
def test_operands_on_a_non_current_device(row):
  needs_two_devices()
  t = {k: v.to('cuda:1') for k, v in row.inputs('cuda:1').items()}
  with torch.no_grad():
    with torch.cuda.device(1):
      want = row(t, 'cuda:1')
    with torch.cuda.device(0):
      got = row(t, 'cuda:1')
  torch.cuda.synchronize(1)
  for g in _flat(got):
    assert g.device == torch.device('cuda', 1), row.name
  assert_same_bits(got, want, row.name)


@pytest.mark.gpu
@pytest.mark.parametrize('row', [r for r in ROWS if len(r.build(np.random.default_rng(0))) > 1],
                         ids=[r.name for r in ROWS if len(r.build(np.random.default_rng(0))) > 1])
def test_operands_on_two_devices_raise(row):
  needs_two_devices()
  t = row.inputs('cuda:1')
  first = next(iter(t))
  t[first] = t[first].to('cuda:0')
  with torch.no_grad(), pytest.raises(ValueError):
    row(t)
