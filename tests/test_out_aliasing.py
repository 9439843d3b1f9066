"""Outputs that alias their inputs.

The C ABI states, per forward entry point, which outputs may BE which inputs (the
same pointer and extent) and which must not overlap them; every other overlap is
refused with E_INVALID before any launch.  `ALIAS_RULES` restates that table and is
checked to cover exactly the header's candidates: every forward entry point with a
float output and a float input.

The Python `out=` paths promise that `out=` never changes the result: a call whose
`out` is, or partly overlaps, an input gives the bits of the same call with a fresh
output (plus the old output with accumulate), records the write in `out`'s autograd
version counter, and refuses an `out` that requires grad under grad mode.
"""
import json
import os
import re
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, core, processors, synths
from oracle import ddsp_oracle as oracle
from tests import grad_ref, mod_delay_ref, routing_ref
from tests.test_gpu_input_conventions import Recorder
from tests.util import rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# may alias: the output may BE the input (same pointer and extent), else disjoint;
# may overlap: any overlap is allowed; must not overlap: disjoint only
MAY, ANY, MUST_NOT = 'may alias', 'may overlap', 'must not overlap'


def _rules(default, **exceptions):
  return default, exceptions


# entry point -> (rule of every (output, input) pair, {'output:input': other rule})
ALIAS_RULES = {
    'ddsp_b200_harmonic_controls': _rules(MUST_NOT, **{'amps_out:amps_in': MAY,
                                                       'hd_out:hd_in': MAY}),
    'ddsp_b200_noise_controls': _rules(MAY),
    'ddsp_b200_add': _rules(MAY),
    'ddsp_b200_mix_forward': _rules(MAY),
    'ddsp_b200_resample': _rules(MUST_NOT),
    'ddsp_b200_fir_time_varying': _rules(MUST_NOT),
    'ddsp_b200_filtered_noise_forward': _rules(MUST_NOT),
    'ddsp_b200_decoder_forward': _rules(MUST_NOT),
    'ddsp_b200_fft_convolve_lti': _rules(ANY),
    'ddsp_b200_mod_delay_forward': _rules(MAY, **{'out:audio': MUST_NOT}),
    'ddsp_b200_sinc_filter': _rules(MUST_NOT),
    'ddsp_b200_sinusoidal_forward': _rules(MUST_NOT),
    'ddsp_b200_harmonic_forward': _rules(MUST_NOT),
    'ddsp_b200_streaming_harmonic_forward': _rules(MUST_NOT),
    'ddsp_b200_wavetable_forward': _rules(MUST_NOT),
    'ddsp_b200_linear_lookup_forward': _rules(MUST_NOT),
    'ddsp_b200_oscillator_bank': _rules(MUST_NOT),
    'ddsp_b200_oscillator_bank_tf_sequential': _rules(MUST_NOT),
    'ddsp_b200_harmonic_oscillator_bank': _rules(MUST_NOT),
    'ddsp_b200_mel_forward': _rules(MUST_NOT),
    'ddsp_b200_comb_nll_forward': _rules(MUST_NOT),
    'ddsp_b200_wasserstein_forward': _rules(MUST_NOT),
    'ddsp_b200_frequency_impulse_response': _rules(MUST_NOT),
    'ddsp_b200_sinc_impulse_response': _rules(MUST_NOT),
    'ddsp_b200_angular_cumsum': _rules(MUST_NOT),
    'ddsp_b200_frame_window': _rules(MUST_NOT),
    'ddsp_b200_frame_window_adjoint': _rules(MUST_NOT),
    # spectral_terms' grad_value may be an STFT except with delta_time (refused, tested
    # with the loss)
    'ddsp_b200_spectral_l1': _rules(MUST_NOT, **{'grad_value:stft_value': MAY}),
    'ddsp_b200_spectral_terms': _rules(MAY),
    'ddsp_b200_exp_decay_ir': _rules(MUST_NOT),
    'ddsp_b200_loudness_forward': _rules(MUST_NOT),
    'ddsp_b200_rms_power': _rules(MUST_NOT),
    'ddsp_b200_crepe_frames': _rules(MUST_NOT),
    'ddsp_b200_crepe_decode': _rules(MUST_NOT),
    'ddsp_b200_mixture_nll_forward': _rules(MUST_NOT),
    'ddsp_b200_sinusoidal_to_harmonic': _rules(MUST_NOT),
    'ddsp_b200_hmm_log_prob': _rules(MUST_NOT),
    'ddsp_b200_note_mask': _rules(MUST_NOT),
    'ddsp_b200_note_moments': _rules(MUST_NOT),
}
# forward entry points with float outputs and inputs that have no row, and why
EXCLUDED = {
    'ddsp_b200_decoder_forward_host':
        'its pointers are host buffers, copied through the pipeline\'s own device staging',
}


def _prototypes():
  """{entry point: [(is_const, type, name)]} of every prototype in the header."""
  text = re.sub(r'/\*.*?\*/|//[^\n]*', ' ', _lib._read_header(), flags=re.S)
  protos = {}
  for m in re.finditer(r'\b(ddsp_b200_\w+)\s*\(([^()]*)\)\s*;', text):
    params = []
    for p in m[2].split(','):
      p = p.strip()
      if p == 'void':
        continue
      name = re.search(r'(\w+)$', p)[1]
      params.append(('const' in p.split(), re.sub(r'\bconst\b|\s|\w+$', '', p), name))
    protos[m[1]] = params
  assert set(protos) == set(_lib.SIGNATURES)
  return protos


def _float_pairs(params):
  outs = [n for c, t, n in params if t == 'float*' and not c]
  ins = [n for c, t, n in params if t == 'float*' and c]
  return [(o, i) for o in outs for i in ins]


def _candidates():
  """Every forward entry point (backward and vector-Jacobian products are called by
  ddsp_b200.autograd alone, which allocates their outputs) with a non-const float*
  output and a const float* input: {entry point: [(output, input)]}."""
  return {name: _float_pairs(params) for name, params in _prototypes().items()
          if not re.search(r'_(backward|vjp)(_\w+)?$', name) and _float_pairs(params)}


def _rule(entry, out, inp):
  default, exceptions = ALIAS_RULES[entry]
  return exceptions.get(f'{out}:{inp}', default)


def test_alias_rules_cover_the_header():
  cands = _candidates()
  assert not set(ALIAS_RULES) & set(EXCLUDED)
  named = set(ALIAS_RULES) | set(EXCLUDED)
  assert named == set(cands), (
      'ALIAS_RULES and EXCLUDED must name exactly the header\'s candidates; missing '
      f'{sorted(set(cands) - named)}, extra {sorted(named - set(cands))}')
  for entry, (default, exceptions) in ALIAS_RULES.items():
    assert default in (MAY, ANY, MUST_NOT), entry
    pairs = {f'{o}:{i}' for o, i in cands[entry]}
    assert set(exceptions) <= pairs, (entry, set(exceptions) - pairs)
    assert all(r in (MAY, ANY, MUST_NOT) for r in exceptions.values()), entry
  for entry in ('ddsp_b200_harmonic_controls', 'ddsp_b200_noise_controls', 'ddsp_b200_add',
                'ddsp_b200_mix_forward', 'ddsp_b200_resample', 'ddsp_b200_fir_time_varying',
                'ddsp_b200_filtered_noise_forward', 'ddsp_b200_decoder_forward',
                'ddsp_b200_fft_convolve_lti', 'ddsp_b200_mod_delay_forward',
                'ddsp_b200_sinc_filter', 'ddsp_b200_sinusoidal_forward',
                'ddsp_b200_harmonic_forward', 'ddsp_b200_wavetable_forward',
                'ddsp_b200_linear_lookup_forward'):
    assert entry in cands, entry


# ---- must not overlap: refused on the host, before any launch --------------------
SR = 16000.0
_B, _F, _K, _N, _NB = 2, 4, 3, 64, 5


class Call:
  """A valid call of `entry` on fake device pointers: `extents` {operand: floats},
  `args(p)` the argument tuple for pointers p {operand: int} (the stream last), and
  `row` the floats of one output row; overlaps move by multiples of `align` floats
  (the alignment the entry point requires)."""

  def __init__(self, entry, extents, args, row, align=1):
    self.entry, self.extents, self.args, self.row = entry, extents, args, row
    self.align = align


def _ws(n=1 << 30):
  return (0x7000000000, n)   # a workspace pointer and a size no check refuses


CALLS = [
    Call('ddsp_b200_harmonic_controls',
         dict(amps_in=_B * _F, hd_in=_B * _F * _K, f0_hz=_B * _F, amps_out=_B * _F,
              hd_out=_B * _F * _K),
         lambda p: (p['amps_in'], p['hd_in'], p['f0_hz'], p['amps_out'], p['hd_out'], _B, _F,
                    _K, SR, 3, None), _F * _K),
    Call('ddsp_b200_resample', {'in': _B * _F * 2, 'out': _B * _N * 2},
         lambda p: (p['in'], p['out'], _B, _F, 2, _N, 1, 1, None), _N * 2),
    Call('ddsp_b200_fir_time_varying', dict(audio=_B * _N, ir=_B * _F * 9, out=_B * _N),
         lambda p: (p['audio'], p['ir'], p['out'], _B, _N, _F, 9, _B, 0, -1, 0, None), _N),
    # the fused route, then the impulse responses + FIR (1025 bands)
    Call('ddsp_b200_filtered_noise_forward',
         dict(mags=_B * _F * _NB, noise=_B * _N, audio=_B * _N),
         lambda p: (p['mags'], p['noise'], 1, 0, p['audio'], _B, _F, _NB, _N, 0, 0, *_ws(),
                    None), _N),
    Call('ddsp_b200_filtered_noise_forward',
         dict(mags=_B * _F * 1025, noise=_B * _N, audio=_B * _N),
         lambda p: (p['mags'], p['noise'], 1, 0, p['audio'], _B, _F, 1025, _N, 0, 0, *_ws(),
                    None), _N),
    # hop 64: the fused decoder's regime
    Call('ddsp_b200_decoder_forward',
         dict(amps_raw=_B * _F, hd_raw=_B * _F * _K, f0_hz=_B * _F, mags_raw=_B * _F * _NB,
              noise=_B * 256, audio=_B * 256),
         lambda p: (p['amps_raw'], p['hd_raw'], p['f0_hz'], p['mags_raw'], p['noise'], 1, 0,
                    p['audio'], _B, _F, _K, _NB, 256, SR, 0, 3, 0, -5.0, None), 256),
    Call('ddsp_b200_mod_delay_forward',
         dict(audio=_B * _N, phase=_B * _N, gain=_B * _N, out=_B * _N),
         lambda p: (p['audio'], p['phase'], p['gain'], p['out'], _B, _N, 10, 1.0, 0.0, 1,
                    None), _N),
    Call('ddsp_b200_sinc_filter', dict(audio=_B * _N, cutoff=_B * _F, out=_B * _N),
         lambda p: (p['audio'], p['cutoff'], p['out'], _B, _N, _F, 9, _B, 1.0, 0, 0, 0,
                    None), _N),
    Call('ddsp_b200_sinusoidal_forward',
         dict(frequencies=_B * _F * _K, amplitudes=_B * _F * _K, audio=_B * _N),
         lambda p: (p['frequencies'], p['amplitudes'], p['audio'], _B, _F, _K, _N, SR, 0, 0,
                    *_ws(), None), _N),
    Call('ddsp_b200_harmonic_forward',
         dict(f0_hz=_B * _F, amps=_B * _F, hd=_B * _F * _K, audio=_B * _N),
         lambda p: (p['f0_hz'], p['amps'], p['hd'], p['audio'], _B, _F, _K, _N, SR, 0, 0, 0,
                    None), _N),
    Call('ddsp_b200_streaming_harmonic_forward',
         dict(f0_hz=_B * _F, amps=_B * _F, hd=_B * _F * _K, initial_phase=_B, audio=_B * _N,
              final_phase=_B),
         lambda p: (p['f0_hz'], p['amps'], p['hd'], p['initial_phase'], p['audio'],
                    p['final_phase'], _B, _F, _K, _N, SR, 0, None), _N),
    Call('ddsp_b200_wavetable_forward',
         dict(f0_hz=_B * _F, amplitudes=_B * _F, wavetables=_B * _F * 16, audio=_B * _N),
         lambda p: (p['f0_hz'], p['amplitudes'], p['wavetables'], p['audio'], _B, _F, _N, _F,
                    16, SR, 0, *_ws(), None), _N),
    Call('ddsp_b200_linear_lookup_forward', dict(phase=_B * _N, wavetables=_B * 16, out=_B * _N),
         lambda p: (p['phase'], p['wavetables'], p['out'], _B, _N, 16, 0, None), _N),
    Call('ddsp_b200_oscillator_bank',
         dict(frequency_envelopes=_B * _N * _K, amplitude_envelopes=_B * _N * _K, out=_B * _N),
         lambda p: (p['frequency_envelopes'], p['amplitude_envelopes'], p['out'], _B, _N, _K,
                    SR, 1, *_ws(), None), _N),
    Call('ddsp_b200_oscillator_bank_tf_sequential',
         dict(frequency_envelopes=_B * _N * _K, amplitude_envelopes=_B * _N * _K,
              out=_B * _N * _K),
         lambda p: (p['frequency_envelopes'], p['amplitude_envelopes'], p['out'], _B, _N, _K,
                    SR, 0, 1000, None), _N * _K),
    Call('ddsp_b200_harmonic_oscillator_bank',
         dict(frequency=_B * _N, amplitude_envelopes=_B * _N * _K, initial_phase=_B,
              audio=_B * _N, final_phase=_B),
         lambda p: (p['frequency'], p['amplitude_envelopes'], p['initial_phase'], p['audio'],
                    p['final_phase'], _B, _N, _K, SR, 1, None), _N),
    # fft_size 16, hop 8, pad_end: 8 frames of 4 mel bins
    Call('ddsp_b200_mel_forward', dict(audio=_B * _N, window=16, out=_B * 8 * 4),
         lambda p: (p['audio'], p['window'], 0x6000000000, p['out'], _B, _N, 8, 16, 16, 8, 1,
                    4, 4, _lib.MEL, None), 8 * 4),
    Call('ddsp_b200_comb_nll_forward', dict(f0=_B * 3 * 4, f=_B * 3 * 5, a=_B * 3 * 5,
                                            out=_B * 3 * 4),
         lambda p: (p['f0'], p['f'], p['a'], p['out'], _B, 3, 4, 5, 3, 0.1, None), 3 * 4),
    Call('ddsp_b200_wasserstein_forward', dict(u=4 * 3, v=4 * 5, wu=4 * 3, wv=4 * 5, out=4),
         lambda p: (p['u'], p['v'], p['wu'], p['wv'], p['out'], 4, 3, 5, 1.0, None), 2),
    Call('ddsp_b200_noise_controls', dict(mag_in=_B * _F * _NB, mag_out=_B * _F * _NB),
         lambda p: (p['mag_in'], p['mag_out'], _B * _F * _NB, -5.0, 1, None), _F * _NB),
    Call('ddsp_b200_add', dict(a=_B * _N, b=_B * _N, out=_B * _N),
         lambda p: (p['a'], p['b'], p['out'], _B * _N, None), _N),
    # C = 2: out may not be mix_level, whose extent is half of out's
    Call('ddsp_b200_mix_forward',
         dict(signal_one=_B * _N * 2, signal_two=_B * _N * 2, mix_level=_B * _N,
              out=_B * _N * 2),
         lambda p: (p['signal_one'], p['signal_two'], p['mix_level'], p['out'], _B, _N, 2,
                    None), _N * 2),
    Call('ddsp_b200_frequency_impulse_response',
         dict(mags=8 * _NB, ir=8 * _lib.load().ddsp_b200_ir_size(_NB, 0)),
         lambda p: (p['mags'], p['ir'], 8, _NB, 0, None), _lib.load().ddsp_b200_ir_size(_NB, 0)),
    Call('ddsp_b200_sinc_impulse_response', dict(cutoff=8, ir=8 * 9),
         lambda p: (p['cutoff'], p['ir'], 8, 9, 1.0, 0, None), 9),
    # mode 0 (exact, three passes) and mode 1 (tf.cumsum order) check on their own
    Call('ddsp_b200_angular_cumsum', dict(angular_frequency=_B * _N * 2, phase=_B * _N * 2),
         lambda p: (p['angular_frequency'], p['phase'], _B, _N, 2, 1000, 0, *_ws(), None),
         _N * 2),
    Call('ddsp_b200_angular_cumsum', dict(angular_frequency=_B * _N * 2, phase=_B * _N * 2),
         lambda p: (p['angular_frequency'], p['phase'], _B, _N, 2, 1000, 1, *_ws(), None),
         _N * 2),
    # 8 frames of 16 every 8 samples; window and frames 16-byte aligned
    Call('ddsp_b200_frame_window', dict(audio=_B * _N, window=16, frames=_B * 8 * 16),
         lambda p: (p['audio'], p['window'], p['frames'], _B, _N, 8, 16, 8, None), 8 * 16,
         align=4),
    Call('ddsp_b200_frame_window_adjoint',
         dict(grad_frames=_B * 8 * 16, window=16, scale_device=1, grad_audio=_B * _N),
         lambda p: (p['grad_frames'], p['window'], p['grad_audio'], _B, _N, 8, 16, 8,
                    p['scale_device'], 0, None), _N),
    # 6 frames of 9 bins; 16-byte aligned complex values
    Call('ddsp_b200_spectral_l1',
         dict(stft_target=2 * 54, stft_value=2 * 54, grad_value=2 * 54),
         lambda p: (p['stft_target'], p['stft_value'], p['grad_value'], 0x6000000000, 54, 1.0,
                    1.0, 9, 16, None), 2 * 9, align=4),
    Call('ddsp_b200_spectral_terms',
         dict(stft_target=2 * _B * 3 * 9, stft_value=2 * _B * 3 * 9,
              grad_value=2 * _B * 3 * 9),
         lambda p: (p['stft_target'], p['stft_value'], p['grad_value'], 0x6000000000, _B, 3,
                    9, _lib.TERM_MAG, _lib.LOSS_L1, 1.0, 0.0, 0.0, 0.0, 0.0, None), 2 * 9,
         align=2),
    Call('ddsp_b200_exp_decay_ir', dict(gain=4, decay=4, noise=16, ir=4 * 16),
         lambda p: (p['gain'], p['decay'], p['noise'], 1, 0, p['ir'], 4, 16, None), 16),
    # n_fft 16 every 8 samples, centred: 9 frames
    Call('ddsp_b200_loudness_forward', dict(audio=_B * _N, weights=9, loudness=_B * 9),
         lambda p: (p['audio'], p['weights'], p['loudness'], _B, _N, 9, 16, 8,
                    _lib.PAD_CENTER, 70.0, 20.7, None), 9),
    Call('ddsp_b200_rms_power', dict(audio=_B * _N, power_db=_B * 9),
         lambda p: (p['audio'], p['power_db'], _B, _N, 9, 16, 8, _lib.PAD_CENTER, 1, 70.0,
                    20.7, None), 9),
    # 2048 samples, hop 512, 'valid': 3 frames
    Call('ddsp_b200_crepe_frames', dict(audio=_B * 2048, frames=_B * 3 * 1024),
         lambda p: (p['audio'], p['frames'], _B, 2048, 3, 512, _lib.PAD_VALID, None), 3 * 1024),
    Call('ddsp_b200_crepe_decode', dict(activations=4 * 360, f0=4, confidence=4),
         lambda p: (p['activations'], None, p['f0'], p['confidence'], 4, None), 4),
    Call('ddsp_b200_mixture_nll_forward',
         dict(x=_B * 3 * 4, mu=_B * 3 * 5, lw=_B * 3 * 5, nll=_B * 3 * 4),
         lambda p: (p['x'], p['mu'], p['lw'], p['nll'], _B, 3, 4, 5, 0.5, None), 3 * 4),
    Call('ddsp_b200_sinusoidal_to_harmonic',
         dict(sin_amps=_B * 3 * 4, sin_freqs=_B * 3 * 4, f0_hz=_B * 3, harm_amp=_B * 3,
              harm_dist=_B * 3 * 5),
         lambda p: (p['sin_amps'], p['sin_freqs'], p['f0_hz'], p['harm_amp'], p['harm_dist'],
                    _B, 3, 4, 5, 0.1, SR, 1, None), 3 * 5),
    Call('ddsp_b200_hmm_log_prob', dict(obs=_B * 5 * 2, loc=3 * 2, scale=3 * 2, log_prob=_B),
         lambda p: (p['obs'], p['loc'], p['scale'], p['log_prob'], _B, 5, 3, 0.9, 0.05, None),
         1),
    Call('ddsp_b200_note_mask', dict(q=_B * 6, onset=_B * 6, mask=_B * 6 * 3),
         lambda p: (p['q'], p['onset'], p['mask'], None, 0, _B, 6, 3, 0, None), 6 * 3),
    Call('ddsp_b200_note_moments',
         dict(x=_B * 6 * 4, mask=_B * 6 * 3, mean=_B * 3 * 4, std=_B * 3 * 4,
              pooled_mean=_B * 6 * 4, pooled_std=_B * 6 * 4),
         lambda p: (p['x'], p['mask'], p['mean'], p['std'], p['pooled_mean'], p['pooled_std'],
                    _B, 6, 3, 4, None), 3 * 4),
]
CALLS_BY_ENTRY = {}
for _c in CALLS:
  CALLS_BY_ENTRY.setdefault(_c.entry, []).append(_c)


def _checked_pairs():
  """(entry point, output, input, rule) of every pair the library refuses some overlap
  of: all but `may overlap`."""
  return [(e, o, i, _rule(e, o, i)) for e, pairs in sorted(_candidates().items())
          if e in ALIAS_RULES for o, i in pairs if _rule(e, o, i) != ANY]


def test_every_checked_row_has_a_call():
  assert {e for e, _, _, _ in _checked_pairs()} == set(CALLS_BY_ENTRY)
  for c in CALLS:
    assert set(c.extents) >= {n for pair in _candidates()[c.entry] for n in pair}, c.entry


def test_filtered_noise_calls_take_both_routes():
  lib = _lib.load()
  routes = [lib.ddsp_b200_filtered_noise_workspace(_B, _F, nb, _N, 0) == 0
            for nb in (_NB, 1025)]
  assert routes == [True, False]


def _shifts(call, out, inp, rule):
  """Where `out` is put, in floats after `inp`: the exact alias (refused unless the
  rule allows it and the extents agree) and the overlaps among +-`align` and +-half a
  row (of the shorter operand when that is less than a row)."""
  a = call.align
  half = max(a, min(call.row, call.extents[out], call.extents[inp]) // 2 // a * a)
  exact_ok = rule == MAY and call.extents[out] == call.extents[inp]
  # a shift past the end of either operand overlaps nothing (a one-float input)
  moved = [d for d in dict.fromkeys([a, -a, half, -half])
           if -call.extents[out] < d < call.extents[inp]]
  return ([] if exact_ok else [0]) + moved


def _refusals():
  """Every checked pair on fake device pointers, each operand at its own address and
  then `out` moved onto `inp` by each of _shifts.  Returns [entry, out, inp, call
  index, shift, status, last error, launches made]."""
  lib = _lib.load()
  rows = []
  for entry, out, inp, rule in _checked_pairs():
    for index, call in enumerate(CALLS_BY_ENTRY[entry]):
      base = {n: (k + 1) << 32 for k, n in enumerate(sorted(call.extents))}
      for shift in _shifts(call, out, inp, rule):
        p = dict(base)
        p[out] = base[inp] + 4 * shift
        assert shift == 0 or p[out] < p[inp] + 4 * call.extents[inp] and (
            p[inp] < p[out] + 4 * call.extents[out])
        launches = lib.ddsp_b200_launch_count()
        rc = getattr(lib, entry)(*call.args(p))
        rows.append([entry, out, inp, index, shift, rc, lib.ddsp_b200_last_error().decode(),
                     lib.ddsp_b200_launch_count() - launches])
  return rows


@pytest.fixture(scope='module')
def refusals():
  """_refusals() in a child process that sees no CUDA device, so that an entry point
  that lacked its check fails the launch instead of touching a fake address."""
  proc = subprocess.run(
      [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [
          '-c', 'import json; from tests.test_out_aliasing import _refusals; '
                'print(json.dumps(_refusals()))'],
      cwd=ROOT, env=dict(os.environ, CUDA_VISIBLE_DEVICES=''), capture_output=True,
      text=True)
  assert proc.returncode == 0, proc.stderr
  rows = json.loads(proc.stdout.strip().splitlines()[-1])
  by_pair = {}
  for entry, out, inp, *result in rows:
    by_pair.setdefault((entry, out, inp), []).append(result)
  return by_pair


@pytest.mark.parametrize('entry,out,inp,rule', _checked_pairs(),
                         ids=[f'{e[len("ddsp_b200_"):]}-{o}-{i}' for e, o, i, _ in _checked_pairs()])
def test_overlap_is_refused_before_any_launch(entry, out, inp, rule, refusals):
  """E_INVALID naming both operands, and no launch, for each overlap of _refusals."""
  results = refusals[(entry, out, inp)]
  calls = CALLS_BY_ENTRY[entry]
  assert len(results) == sum(len(_shifts(c, out, inp, rule)) for c in calls)
  assert {r[0] for r in results} == set(range(len(calls)))
  fn = entry[len('ddsp_b200_'):]
  want = (f'{fn}: {out} must not overlap {inp}' if rule == MUST_NOT else
          f'{fn}: {out} must be {inp} or not overlap it')
  for index, shift, rc, msg, launches in results:
    assert rc == _lib.E_INVALID, (entry, out, inp, index, shift, rc, msg)
    assert msg == want, (index, shift, msg)
    assert launches == 0, (entry, out, inp, index, shift)


# ---- may alias: the C ABI in place ----------------------------------------------
def _rng(name):
  return np.random.default_rng(zlib.crc32(name.encode()))


def _cuda(x):
  return torch.as_tensor(np.asarray(x, np.float32), device='cuda')


def _assert_close(got, want, tol, what):
  e_max, e_l2 = rel_err(got.detach().cpu().numpy() if torch.is_tensor(got) else got, want)
  assert e_max < tol and e_l2 < tol, (what, e_max, e_l2)


def _in_place(symbol, ins, out_name, alias, args):
  """The kernel `symbol` on inputs `ins` (a dict in the entry's argument order) with
  a fresh output, and with `alias`'s own buffer as the output: (fresh, in place)."""
  fresh = torch.empty_like(ins[alias]).fill_(7.0)
  _launch_with(symbol, ins, {out_name: fresh}, args)
  aliased = {k: v.clone() for k, v in ins.items()}
  _launch_with(symbol, aliased, {out_name: aliased[alias]}, args)
  torch.cuda.synchronize()
  return fresh, aliased[alias]


def _launch_with(symbol, ins, outs, args):
  core._launch(symbol, *args(dict(ins, **outs)))


@pytest.mark.gpu
@pytest.mark.parametrize('K', [1, 31, 32, 33, 100, 260])
def test_harmonic_controls_in_place(K):
  B, F = 3, 250
  rng = _rng(f'controls{K}')
  amps, hd = rng.standard_normal((B, F, 1)), rng.standard_normal((B, F, K))
  f0 = rng.uniform(20.0, 4000.0, (B, F, 1))
  want = oracle.harmonic_get_controls(amps, hd, f0)
  t = {'a': _cuda(amps), 'h': _cuda(hd), 'f': _cuda(f0)}

  def run(a_out, h_out, ins):
    core._launch('ddsp_b200_harmonic_controls', ins['a'], ins['h'], ins['f'], a_out, h_out,
                 B, F, K, 16000.0, _lib.CTL_SCALE | _lib.CTL_NYQUIST)

  fa, fh = torch.empty_like(t['a']), torch.empty_like(t['h'])
  run(fa, fh, t)
  ins = {k: v.clone() for k, v in t.items()}
  run(ins['a'], ins['h'], ins)
  torch.cuda.synchronize()
  assert torch.equal(ins['a'], fa) and torch.equal(ins['h'], fh), K
  _assert_close(ins['a'], want['amplitudes'], 1e-5, ('amps', K))
  _assert_close(ins['h'], want['harmonic_distribution'], 1e-5, ('hd', K))


@pytest.mark.gpu
def test_noise_controls_in_place():
  x = _rng('noise_controls').standard_normal((3, 250, 65))
  n = x.size
  fresh, aliased = _in_place(
      'ddsp_b200_noise_controls', {'x': _cuda(x)}, 'y', 'x',
      lambda p: (p['x'], p['y'], n, -5.0, 1))
  assert torch.equal(aliased, fresh)
  _assert_close(aliased, oracle.noise_get_controls(x)['magnitudes'], 1e-5, 'noise_controls')


@pytest.mark.gpu
@pytest.mark.parametrize('alias', ['a', 'b'])
def test_add_in_place(alias):
  rng = _rng('add')
  a, b = rng.uniform(-1, 1, (3, 64000)), rng.uniform(-1, 1, (3, 64000))
  fresh, aliased = _in_place('ddsp_b200_add', {'a': _cuda(a), 'b': _cuda(b)}, 'out', alias,
                             lambda p: (p['a'], p['b'], p['out'], a.size))
  assert torch.equal(aliased, fresh)
  _assert_close(aliased, np.float32(a) + np.float32(b).astype(np.float64), 1e-7, alias)


@pytest.mark.gpu
@pytest.mark.parametrize('alias', ['s1', 's2', 'm'])
def test_mix_in_place(alias):
  rng = _rng('mix')
  B, N = 3, 16000
  v = {'s1': rng.uniform(-1, 1, (B, N, 1)), 's2': rng.uniform(-1, 1, (B, N, 1)),
       'm': rng.uniform(0.05, 0.95, (B, N, 1))}
  fresh, aliased = _in_place(
      'ddsp_b200_mix_forward', {k: _cuda(x) for k, x in v.items()}, 'out', alias,
      lambda p: (p['s1'], p['s2'], p['m'], p['out'], B, N, 1))
  assert torch.equal(aliased, fresh)
  want = routing_ref.mix(*(torch.as_tensor(np.float32(v[k]), dtype=torch.float64)
                           for k in ('s1', 's2', 'm')))
  _assert_close(aliased, want.numpy(), 1e-5, alias)


@pytest.mark.gpu
@pytest.mark.parametrize('alias', ['phase', 'gain'])
def test_mod_delay_in_place(alias):
  rng = _rng('mod_delay')
  B, N, L = 3, 16000, 100
  v = {'audio': rng.uniform(-1, 1, (B, N)), 'phase': rng.uniform(0.05, 0.95, (B, N)),
       'gain': rng.uniform(0, 1, (B, N))}
  fresh, aliased = _in_place(
      'ddsp_b200_mod_delay_forward', {k: _cuda(x) for k, x in v.items()}, 'out', alias,
      lambda p: (p['audio'], p['phase'], p['gain'], p['out'], B, N, L, 1.0, 0.0, 1))
  assert torch.equal(aliased, fresh)
  t = {k: torch.as_tensor(np.float32(x), dtype=torch.float64) for k, x in v.items()}
  want = mod_delay_ref.torch_mod_delay(t['audio'], t['gain'], t['phase'], L, add_dry=True)
  _assert_close(aliased, want.numpy(), 1e-5, alias)


@pytest.mark.gpu
@pytest.mark.parametrize('alias', ['audio', 'ir'])
def test_fft_convolve_lti_in_place(alias):
  """out = audio or the impulse response, several 1024-sample blocks per item."""
  rng = _rng('lti')
  B, N = 2, 5000
  v = {'audio': rng.uniform(-1, 1, (B, N)), 'ir': rng.uniform(-1, 1, (B, N)) * 0.02}
  ins = {k: _cuda(x) for k, x in v.items()}
  for accumulate in (0, 1):
    fresh, aliased = _in_place(
        'ddsp_b200_fft_convolve_lti', ins, 'out', alias,
        lambda p: (p['audio'], p['ir'], p['out'], B, N, N, B, 0, N, accumulate, 0,
                   *core._workspace('ddsp_b200_fft_convolve_lti_workspace',
                                    p['audio'].device, B, N, N, B)))
    # with accumulate the fresh output started at 7, the aliased one at the input
    base = ins[alias].double() if accumulate else 0.0
    want = grad_ref.convolve_lti(*(torch.as_tensor(np.float32(v[k]), dtype=torch.float64)
                                   for k in ('audio', 'ir')), 0, N)
    _assert_close(aliased, (want + (base.cpu() if accumulate else 0)).numpy(), 1e-4,
                  (alias, accumulate))
    if not accumulate:
      assert torch.equal(aliased, fresh)


# ---- every Python out= path -------------------------------------------------------
B, F, N = 2, 20, 1600
HOP = N // F


class Case:
  """A Python out= path: build(rng) -> {name: array}; call(ins, out, accumulate);
  `audio_rate`: the inputs of out's [B, N] extent; `frame`: its frame size in floats;
  `launches`: the library calls the route makes (checked with the recorder);
  ref(arrays) -> the float64 result; grad: the inputs that require grad (the
  route under grad)."""

  def __init__(self, name, build, call, audio_rate, frame, launches, ref, tol,
               grad=(), n=N, check=None):
    self.name, self.build, self.call = name, build, call
    self.audio_rate, self.frame, self.launches = audio_rate, frame, launches
    self.ref, self.tol, self.grad, self.n, self.check = ref, tol, grad, n, check

  def arrays(self):
    return {k: np.asarray(v, np.float32) for k, v in self.build(_rng(self.name)).items()}


def _u(rng, lo, hi, *shape):
  return rng.uniform(lo, hi, shape)


def _conv(ir_shape, n):
  return lambda rng: {'audio': _u(rng, -1, 1, B, n), 'ir': _u(rng, -1, 1, *ir_shape) * 0.05}


def _noise_case(name, nb, fused):
  def check():
    ws = _lib.load().ddsp_b200_filtered_noise_workspace(B, F, nb, N, 0)
    assert (ws == 0) == fused, (name, ws)
  return Case(name, lambda rng: {'mags': _u(rng, 0, 1, B, F, nb), 'noise': _u(rng, -1, 1, B, N)},
              lambda t, out, acc: core.filtered_noise(t['mags'], N, window_size=0,
                                                      noise=t['noise'], out=out,
                                                      accumulate=acc),
              ('noise',), HOP, ['ddsp_b200_filtered_noise_forward'],
              lambda a: oracle.noise_get_signal(a['mags'], a['noise'], window_size=0), 1e-4,
              check=check)


CASES = [
    Case('fft_convolve_partitioned', _conv((B, 2048), 4096),
         lambda t, out, acc: core.fft_convolve(t['audio'], t['ir'], out=out, accumulate=acc),
         ('audio',), 1024, ['ddsp_b200_fft_convolve_lti'],
         lambda a: oracle.fft_convolve(a['audio'], a['ir']), 1e-4, n=4096),
    Case('fft_convolve_long_ir', _conv((B, 2, 2048), 4096),
         lambda t, out, acc: core.fft_convolve(t['audio'], t['ir'], out=out, accumulate=acc),
         ('audio',), 2048, [], lambda a: oracle.fft_convolve(a['audio'], a['ir']), 1e-4,
         n=4096),
    Case('fft_convolve_fir', _conv((B, F, 17), N),
         lambda t, out, acc: core.fft_convolve(t['audio'], t['ir'], out=out, accumulate=acc),
         ('audio',), HOP, ['ddsp_b200_fir_time_varying'],
         lambda a: oracle.fft_convolve(a['audio'], a['ir']), 1e-5),
    Case('fft_convolve_grad', _conv((B, F, 17), N),
         lambda t, out, acc: core.fft_convolve(t['audio'], t['ir'], out=out, accumulate=acc),
         ('audio',), HOP, ['ddsp_b200_fir_time_varying'],
         lambda a: oracle.fft_convolve(a['audio'], a['ir']), 1e-5, grad=('ir',)),
    Case('fft_convolve_lti', lambda rng: {'audio': _u(rng, -1, 1, B, N),
                                          'ir': _u(rng, -1, 1, 1, 300)},
         lambda t, out, acc: core.fft_convolve_lti(t['audio'], t['ir'], 0, N, out=out,
                                                   accumulate=acc),
         ('audio',), 1024, ['ddsp_b200_fft_convolve_lti'],
         lambda a: grad_ref.convolve_lti(torch.as_tensor(a['audio'], dtype=torch.float64),
                                         torch.as_tensor(a['ir'], dtype=torch.float64),
                                         0, N).numpy(), 1e-4),
    _noise_case('filtered_noise_fused', 9, True),
    _noise_case('filtered_noise_ir_fir', 8, False),
    Case('FilteredNoise_get_signal',
         lambda rng: {'mags': _u(rng, 0, 1, B, F, 9), 'noise': _u(rng, -1, 1, B, N)},
         lambda t, out, acc: synths.FilteredNoise(n_samples=N, window_size=0).get_signal(
             t['mags'], noise=t['noise'], out=out, accumulate=acc),
         ('noise',), HOP, ['ddsp_b200_filtered_noise_forward'],
         lambda a: oracle.noise_get_signal(a['mags'], a['noise'], window_size=0), 1e-4),
    Case('add', lambda rng: {'a': _u(rng, -1, 1, B, N), 'b': _u(rng, -1, 1, B, N)},
         lambda t, out, acc: core.add(t['a'], t['b'], out=out),
         ('a', 'b'), HOP, ['ddsp_b200_add'], lambda a: oracle.add_get_signal(
             a['a'].astype(np.float64), a['b']), 1e-7),
    Case('harmonic_synthesis',
         lambda rng: {'f0': _u(rng, 100, 600, B, F, 1), 'amps': _u(rng, 0.1, 1, B, F, 1),
                      'hd': _u(rng, 0, 1, B, F, 8)},
         lambda t, out, acc: core.harmonic_synthesis(
             t['f0'], t['amps'], harmonic_distribution=t['hd'], n_samples=N, out=out,
             accumulate=acc),
         (), HOP, ['ddsp_b200_harmonic_forward'],
         lambda a: oracle.harmonic_synthesis(a['f0'], a['amps'],
                                             harmonic_distribution=a['hd'], n_samples=N),
         1e-4),
    Case('sinusoidal_synthesis',
         lambda rng: {'f': _u(rng, 100, 3000, B, F, 4), 'a': _u(rng, 0, 1, B, F, 4)},
         lambda t, out, acc: core.sinusoidal_synthesis(t['f'], t['a'], n_samples=N, out=out,
                                                       accumulate=acc),
         (), HOP, ['ddsp_b200_sinusoidal_forward'],
         lambda a: oracle.sinusoidal_get_signal(a['a'], a['f'], N), 1e-4),
]
CONTROL_INPUT = {'harmonic_synthesis': 'f0', 'sinusoidal_synthesis': 'f'}


def _tensors(case, arrays):
  t = {k: _cuda(v) for k, v in arrays.items()}
  for k in case.grad:
    t[k].requires_grad_(True)
  return t


def _grad_ctx(case):
  return torch.enable_grad() if case.grad else torch.no_grad()


def _forms(case):
  """(input, shift) pairs: shift None is an exact alias, an int s puts the input at
  float s of one storage and out at float 0 (negative: out at -s, input at 0)."""
  forms = []
  for x in case.audio_rate:
    forms += [(x, None)] + [(x, s) for s in (1, -1, case.frame, -case.frame)]
  if case.name in CONTROL_INPUT:
    forms += [(CONTROL_INPUT[case.name], s) for s in (1, case.frame, -1)]
  return forms


def _shares_memory(a, b):
  a0, b0 = a.data_ptr(), b.data_ptr()
  return a0 < b0 + 4 * b.numel() and b0 < a0 + 4 * a.numel()


def _layout(arrays, name, shift, out_numel, seed):
  """One storage holding input `name` (its values) and out (random values where the
  input does not cover it); returns (input view, out view)."""
  x = arrays[name]
  n = x.size
  a, o = (shift, 0) if shift >= 0 else (0, -shift)
  size = max(a + n, o + out_numel)
  g = torch.Generator(device='cuda').manual_seed(seed)
  store = torch.rand(size, device='cuda', generator=g) * 2 - 1
  xv = store[a:a + n].view(x.shape)
  xv.copy_(torch.as_tensor(x))
  return xv, store[o:o + out_numel]


PY_FORMS = [(c, x, s, acc) for c in CASES for x, s in _forms(c) for acc in (False, True)
            if not (acc and c.name == 'add')]


@pytest.mark.gpu
@pytest.mark.parametrize('case,inp,shift,accumulate', PY_FORMS,
                         ids=[f'{c.name}-{x}-{"alias" if s is None else s}-'
                              f'{"acc" if a else "set"}' for c, x, s, a in PY_FORMS])
def test_python_out_aliasing_an_input(case, inp, shift, accumulate, monkeypatch):
  arrays = case.arrays()
  shape = (B, case.n)
  if case.check:
    case.check()
  t = _tensors(case, arrays)
  if shift is None:
    out = t[inp].detach().view(shape) if case.grad else t[inp].view(shape)
  else:
    t[inp], flat = _layout(arrays, inp, shift, B * case.n, zlib.crc32(case.name.encode()))
    out = flat.view(shape)
    assert _shares_memory(t[inp], out)
  old_out, old_in = out.detach().clone(), {k: v.detach().clone() for k, v in t.items()}
  # the same call with a fresh output holding out's old values
  want = old_out.clone()
  with _grad_ctx(case):
    case.call(_tensors(case, {k: v.cpu().numpy() for k, v in old_in.items()}), want,
              accumulate)
  torch.cuda.synchronize()
  # the route, recorded without launching
  rec = Recorder(_lib.load())
  monkeypatch.setattr(_lib, 'load', lambda: rec)
  with _grad_ctx(case):
    case.call({k: v.clone().requires_grad_(k in case.grad) for k, v in old_in.items()},
              old_out.clone(), accumulate)
  monkeypatch.undo()
  assert [c[0] for c in rec.calls] == case.launches, (case.name, rec.calls)
  version = out._version
  with _grad_ctx(case):
    got = case.call(t, out, accumulate)
  torch.cuda.synchronize()
  assert torch.equal(out.detach(), want.detach()), (
      case.name, inp, shift, accumulate, rel_err(out.detach().cpu().numpy(),
                                                 want.detach().cpu().numpy()))
  assert got.data_ptr() == out.data_ptr()
  assert out._version > version, case.name
  assert case.grad == () or got.requires_grad


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[c.name for c in CASES])
def test_python_out_matches_float64(case):
  """The fresh-output call those comparisons stand on, against float64, at the op's
  tolerance; with accumulate the old output is added."""
  arrays = case.arrays()
  old = np.linspace(-1, 1, B * case.n, dtype=np.float32).reshape(B, case.n)
  want = case.ref({k: v.astype(np.float64) for k, v in arrays.items()})
  for accumulate in ((False, True) if case.name != 'add' else (False,)):
    out = _cuda(old)
    with _grad_ctx(case):
      case.call(_tensors(case, arrays), out, accumulate)
    _assert_close(out, want + (old if accumulate else 0), case.tol, (case.name, accumulate))


# ---- autograd ---------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[c.name for c in CASES])
def test_out_overwriting_a_saved_tensor_fails_backward(case):
  t = _tensors(case, case.arrays())
  buf = torch.zeros(B, case.n, device='cuda')
  w = torch.ones_like(buf, requires_grad=True)
  loss = (w * buf).sum()
  with _grad_ctx(case):
    case.call(t, buf, False)
  with pytest.raises(RuntimeError, match='modified by an inplace operation'):
    loss.backward()


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[c.name for c in CASES])
def test_out_that_requires_grad_is_refused(case, monkeypatch):
  t = _tensors(case, case.arrays())
  out = torch.zeros(B, case.n, device='cuda', requires_grad=True)
  rec = Recorder(_lib.load())
  monkeypatch.setattr(_lib, 'load', lambda: rec)
  with torch.enable_grad(), pytest.raises(RuntimeError, match='requires grad'):
    case.call(t, out, False)
  assert rec.calls == [], rec.calls
  assert out._version == 0 and not out.detach().any()


@pytest.mark.gpu
def test_processor_group_refuses_a_harmonic_signal_that_requires_grad():
  """Outside the fused decoder the signal-only ProcessorGroup call adds the noise into
  the harmonic buffer with out=.  When only the harmonic inputs require grad, it
  refuses with the way to train before any noise launch, not with the out= error."""
  b, f, n = 2, 50, 1600   # hop 32: outside the fused decoder
  rng = _rng('group')
  t = {'amps': _cuda(rng.standard_normal((b, f, 1))).requires_grad_(),
       'harmonic_distribution': _cuda(rng.standard_normal((b, f, 8))).requires_grad_(),
       'f0_hz': _cuda(rng.uniform(100, 400, (b, f, 1))),
       'noise_magnitudes': _cuda(rng.standard_normal((b, f, 9)))}
  group = processors.ProcessorGroup(dag=[
      (synths.Harmonic(n_samples=n), ['amps', 'harmonic_distribution', 'f0_hz']),
      (synths.FilteredNoise(n_samples=n, window_size=0), ['noise_magnitudes']),
      (processors.Add(), ['filtered_noise/signal', 'harmonic/signal'])])
  with pytest.raises(RuntimeError, match='return_outputs_dict=True'):
    group(t)
  out = group(t, return_outputs_dict=True)['signal']
  out.square().sum().backward()
  assert t['amps'].grad.abs().sum() > 0
