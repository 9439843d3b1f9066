"""Host-side contract tests that need no GPU: the C ABI surface, argument
validation (which happens before any launch), and the Processor /
ProcessorGroup / DAG semantics of the reference (processors_test.py, dags.py).
"""
import ctypes
import os
import re

import numpy as np
import pytest

import ddsp_b200
from ddsp_b200 import _lib, core, dags, processors, synths

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- C ABI ------------------------------------------------------------------
def _header_symbols():
  text = open(os.path.join(ROOT, 'include', 'ddsp_b200.h')).read()
  return sorted(set(re.findall(r'\b(ddsp_b200_[a-z0-9_]+)\s*\(', text)))


def test_library_exports_every_declared_symbol():
  lib = ctypes.CDLL(_lib.LIB_PATH)
  names = _header_symbols()
  assert len(names) >= 13
  for name in names:
    assert hasattr(lib, name), name
    assert name in _lib.SIGNATURES, f'{name} is not bound in _lib.SIGNATURES'
  assert set(_lib.SIGNATURES) == set(names)
  assert _lib.load().ddsp_b200_version() == 200


def test_abi_validates_before_launching():
  """Shape errors come back as E_INVALID with a message - no CUDA call made."""
  lib = _lib.load()
  fake = ctypes.c_void_p(0x1000)   # never dereferenced on the host
  # N not divisible by F
  rc = lib.ddsp_b200_harmonic_forward(fake, fake, fake, fake, 1, 7, 4, 100,
                                      16000.0, 0, 0, 0, None)
  assert rc == _lib.E_INVALID
  assert b'divisible' in lib.ddsp_b200_last_error()
  with pytest.raises(ValueError):
    _lib.check(rc)
  # NULL harmonic_distribution with K > 1
  rc = lib.ddsp_b200_harmonic_forward(fake, fake, None, fake, 1, 10, 4, 100,
                                      16000.0, 0, 0, 0, None)
  assert rc == _lib.E_INVALID
  # bad enum values
  assert lib.ddsp_b200_harmonic_forward(fake, fake, fake, fake, 1, 10, 4, 100,
                                        16000.0, 7, 0, 0, None) == _lib.E_INVALID
  assert lib.ddsp_b200_harmonic_forward(fake, fake, fake, fake, 1, 10, 4, 100,
                                        16000.0, 0, 9, 0, None) == _lib.E_INVALID
  # fir: batch mismatch / frame mismatch / bad padding (core.py:1441-1457,1367)
  assert lib.ddsp_b200_fir_time_varying(fake, fake, fake, 2, 1000, 10, 16, 3, 0,
                                        -1, 0, None) == _lib.E_INVALID
  assert b'Batch size' in lib.ddsp_b200_last_error()
  assert lib.ddsp_b200_fir_time_varying(fake, fake, fake, 1, 1000, 999, 16, 1, 0,
                                        -1, 0, None) == _lib.E_INVALID
  assert b'Number of Audio frames' in lib.ddsp_b200_last_error()
  assert lib.ddsp_b200_fir_time_varying(fake, fake, fake, 1, 1000, 10, 16, 1, 5,
                                        -1, 0, None) == _lib.E_INVALID
  # null pointers
  assert lib.ddsp_b200_add(None, fake, fake, 4, None) == _lib.E_INVALID
  assert lib.ddsp_b200_harmonic_controls(fake, fake, fake, fake, None, 1, 1, 1,
                                         16000.0, 3, None) == _lib.E_INVALID
  # too few frequencies for an irfft
  assert lib.ddsp_b200_ir_size(1, 0) == _lib.E_INVALID
  # empty batches are no-ops, not errors
  assert lib.ddsp_b200_harmonic_forward(fake, fake, fake, fake, 0, 10, 4, 640,
                                        16000.0, 0, 0, 0, None) == 0


P = 0x1000        # a device pointer the library never dereferences on the host
SR = 16000.0
E_INVALID, E_UNSUPPORTED, E_WORKSPACE = _lib.E_INVALID, _lib.E_UNSUPPORTED, _lib.E_WORKSPACE

# (case, entry point, arguments, status or size, the full last_error or None).  An
# error row fails one check alone and passes every check before it; a 0 row is an
# empty-batch no-op; a *_workspace / ir_size row is a size query.  None of them
# reaches a CUDA call.
_ABI_CASES = [
    ('harmonic_forward-null', 'harmonic_forward', (P, P, P, None, 1, 10, 4, 100, SR, 0, 0, 0, None), E_INVALID, b'harmonic_forward: null pointer'),
    ('harmonic_forward-B', 'harmonic_forward', (P, P, P, P, -1, 10, 4, 100, SR, 0, 0, 0, None), E_INVALID, b'harmonic_forward: bad shape B=-1 F=10 K=4 N=100'),
    ('harmonic_forward-F', 'harmonic_forward', (P, P, P, P, 1, 0, 4, 100, SR, 0, 0, 0, None), E_INVALID, b'harmonic_forward: bad shape B=1 F=0 K=4 N=100'),
    ('harmonic_forward-K', 'harmonic_forward', (P, P, P, P, 1, 10, 0, 100, SR, 0, 0, 0, None), E_INVALID, b'harmonic_forward: bad shape B=1 F=10 K=0 N=100'),
    ('harmonic_forward-N', 'harmonic_forward', (P, P, P, P, 1, 10, 4, 0, SR, 0, 0, 0, None), E_INVALID, b'harmonic_forward: bad shape B=1 F=10 K=4 N=0'),
    ('harmonic_forward-hd', 'harmonic_forward', (P, P, None, P, 1, 10, 4, 100, SR, 0, 0, 0, None), E_INVALID, b'harmonic_forward: harmonic_distribution is NULL but K=4'),
    ('harmonic_forward-amp_method', 'harmonic_forward', (P, P, P, P, 1, 10, 4, 100, SR, 7, 0, 0, None), E_INVALID, b'harmonic_forward: bad amp_method 7'),
    ('harmonic_forward-phase_mode', 'harmonic_forward', (P, P, P, P, 1, 10, 4, 100, SR, 0, 9, 0, None), E_INVALID, b'harmonic_forward: bad phase_mode 9'),
    ('harmonic_forward-divisible', 'harmonic_forward', (P, P, P, P, 1, 7, 4, 100, SR, 0, 0, 0, None), E_INVALID, b'harmonic_forward: n_samples (100) must be divisible by the number of frames (7)'),
    ('harmonic_forward-window', 'harmonic_forward', (P, P, P, P, 1, 10, 4, 10, SR, 0, 0, 0, None), E_INVALID, b'harmonic_forward: window upsampling cannot downsample (frames 10 >= timesteps 10)'),
    ('harmonic_forward-sample_rate', 'harmonic_forward', (P, P, P, P, 1, 10, 4, 100, 0.0, 0, 0, 0, None), E_INVALID, b'harmonic_forward: sample_rate must be positive'),
    ('harmonic_forward-B0', 'harmonic_forward', (P, P, P, P, 0, 10, 4, 640, SR, 0, 0, 0, None), 0, None),
    ('harmonic_forward-B0-linear-F_eq_N', 'harmonic_forward', (P, P, P, P, 0, 10, 4, 10, SR, 1, 0, 0, None), 0, None),
    ('harmonic_forward-grid', 'harmonic_forward', (P, P, P, P, 65536, 10, 4, 100, SR, 0, 0, 0, None), E_INVALID, b'harmonic_forward: B=65536 exceeds the 65535 grid limit'),
    ('add-null', 'add', (None, P, P, 4, None), E_INVALID, b'add: null pointer'),
    ('harmonic_controls-null', 'harmonic_controls', (P, P, P, P, None, 1, 1, 1, SR, 3, None), E_INVALID, b'harmonic_controls: null pointer'),
    ('streaming_harmonic_forward-null', 'streaming_harmonic_forward', (None, P, P, None, P, None, 1, 10, 4, 640, SR, 0, None), E_INVALID, b'streaming_harmonic_forward: null pointer'),
    ('streaming_harmonic_forward-B', 'streaming_harmonic_forward', (P, P, P, None, P, None, -1, 10, 4, 640, SR, 0, None), E_INVALID, b'streaming_harmonic_forward: bad shape B=-1 F=10 K=4 N=640'),
    ('streaming_harmonic_forward-K', 'streaming_harmonic_forward', (P, P, P, None, P, None, 1, 10, 0, 640, SR, 0, None), E_INVALID, b'streaming_harmonic_forward: bad shape B=1 F=10 K=0 N=640'),
    ('streaming_harmonic_forward-hd', 'streaming_harmonic_forward', (P, P, None, None, P, None, 1, 10, 4, 640, SR, 0, None), E_INVALID, b'streaming_harmonic_forward: harmonic_distribution is NULL but K=4'),
    ('streaming_harmonic_forward-amp_method', 'streaming_harmonic_forward', (P, P, P, None, P, None, 1, 10, 4, 640, SR, 2, None), E_INVALID, b'streaming_harmonic_forward: bad amp_method 2'),
    ('streaming_harmonic_forward-divisible', 'streaming_harmonic_forward', (P, P, P, None, P, None, 1, 10, 4, 645, SR, 0, None), E_INVALID, b'streaming_harmonic_forward: n_samples (645) must be divisible by the number of frames (10)'),
    ('streaming_harmonic_forward-sample_rate', 'streaming_harmonic_forward', (P, P, P, None, P, None, 1, 10, 4, 640, -1.0, 0, None), E_INVALID, b'streaming_harmonic_forward: sample_rate must be positive'),
    ('streaming_harmonic_forward-B0', 'streaming_harmonic_forward', (P, P, P, None, P, None, 0, 10, 4, 640, SR, 0, None), 0, None),
    ('streaming_harmonic_forward-B0-window-F_eq_N', 'streaming_harmonic_forward', (P, P, P, None, P, None, 0, 10, 4, 10, SR, 0, None), 0, None),
    ('streaming_harmonic_forward-grid', 'streaming_harmonic_forward', (P, P, P, None, P, None, 65536, 10, 4, 640, SR, 0, None), E_INVALID, b'streaming_harmonic_forward: B=65536 exceeds the 65535 grid limit'),
    ('streaming_harmonic_forward-smem', 'streaming_harmonic_forward', (P, P, P, None, P, None, 1, 10, 30000, 640, SR, 0, None), E_UNSUPPORTED, b'streaming_harmonic_forward: K=30000 needs more shared memory than one CTA has'),
    ('decoder_forward-null', 'decoder_forward', (P, None, P, P, None, 0, 0, P, 1, 1000, 60, 65, 64000, SR, 0, 3, 257, -5.0, None), E_INVALID, b'decoder_forward: null pointer'),
    ('decoder_forward-B', 'decoder_forward', (P, P, P, P, None, 0, 0, P, -1, 1000, 60, 65, 64000, SR, 0, 3, 257, -5.0, None), E_INVALID, b'decoder_forward: bad shape B=-1 F=1000 K=60 N=64000'),
    ('decoder_forward-F', 'decoder_forward', (P, P, P, P, None, 0, 0, P, 1, 0, 60, 65, 64000, SR, 0, 3, 257, -5.0, None), E_INVALID, b'decoder_forward: bad shape B=1 F=0 K=60 N=64000'),
    ('decoder_forward-K', 'decoder_forward', (P, P, P, P, None, 0, 0, P, 1, 1000, 0, 65, 64000, SR, 0, 3, 257, -5.0, None), E_INVALID, b'decoder_forward: bad shape B=1 F=1000 K=0 N=64000'),
    ('decoder_forward-nb', 'decoder_forward', (P, P, P, P, None, 0, 0, P, 1, 1000, 60, 1, 64000, SR, 0, 3, 257, -5.0, None), E_INVALID, b'decoder_forward: need n_frequencies >= 2 (got 1)'),
    ('decoder_forward-N', 'decoder_forward', (P, P, P, P, None, 0, 0, P, 1, 1000, 60, 65, 0, SR, 0, 3, 257, -5.0, None), E_INVALID, b'decoder_forward: bad shape B=1 F=1000 K=60 N=0'),
    ('decoder_forward-amp_method', 'decoder_forward', (P, P, P, P, None, 0, 0, P, 1, 1000, 60, 65, 64000, SR, 3, 3, 257, -5.0, None), E_INVALID, b'decoder_forward: bad amp_method 3'),
    ('decoder_forward-flags0', 'decoder_forward', (P, P, P, P, None, 0, 0, P, 1, 1000, 60, 65, 64000, SR, 0, 0, 257, -5.0, None), E_INVALID, b'decoder_forward: bad harmonic_flags 0'),
    ('decoder_forward-flags4', 'decoder_forward', (P, P, P, P, None, 0, 0, P, 1, 1000, 60, 65, 64000, SR, 0, 4, 257, -5.0, None), E_INVALID, b'decoder_forward: bad harmonic_flags 4'),
    ('decoder_forward-sample_rate', 'decoder_forward', (P, P, P, P, None, 0, 0, P, 1, 1000, 60, 65, 64000, 0.0, 0, 3, 257, -5.0, None), E_INVALID, b'decoder_forward: sample_rate must be positive'),
    ('decoder_forward-B0', 'decoder_forward', (P, P, P, P, None, 0, 0, P, 0, 1000, 60, 65, 64000, SR, 0, 3, 257, -5.0, None), 0, None),
    ('decoder_forward-divisible', 'decoder_forward', (P, P, P, P, None, 0, 0, P, 1, 1000, 60, 65, 64001, SR, 0, 3, 257, -5.0, None), E_UNSUPPORTED, b'decoder_forward: shape outside the fused decoder path (needs hop % 64 == 0, n_frequencies <= 129)'),
    ('decoder_forward-grid', 'decoder_forward', (P, P, P, P, None, 0, 0, P, 65536, 1000, 60, 65, 64000, SR, 0, 3, 257, -5.0, None), E_UNSUPPORTED, b'decoder_forward: shape outside the fused decoder path (needs hop % 64 == 0, n_frequencies <= 129)'),
    ('decoder_forward-hop32', 'decoder_forward', (P, P, P, P, None, 0, 0, P, 1, 1000, 60, 65, 32000, SR, 0, 3, 257, -5.0, None), E_UNSUPPORTED, b'decoder_forward: shape outside the fused decoder path (needs hop % 64 == 0, n_frequencies <= 129)'),
    ('decoder_forward-hop8256', 'decoder_forward', (P, P, P, P, None, 0, 0, P, 1, 1, 60, 65, 8256, SR, 0, 3, 257, -5.0, None), E_UNSUPPORTED, b'decoder_forward: shape outside the fused decoder path (needs hop % 64 == 0, n_frequencies <= 129)'),
    ('decoder_forward-K1025', 'decoder_forward', (P, P, P, P, None, 0, 0, P, 1, 1000, 1025, 65, 64000, SR, 0, 3, 257, -5.0, None), E_UNSUPPORTED, b'decoder_forward: shape outside the fused decoder path (needs hop % 64 == 0, n_frequencies <= 129)'),
    ('decoder_forward-nb1025', 'decoder_forward', (P, P, P, P, None, 0, 0, P, 1, 1000, 60, 1025, 64000, SR, 0, 3, 0, -5.0, None), E_UNSUPPORTED, b'decoder_forward: shape outside the fused decoder path (needs hop % 64 == 0, n_frequencies <= 129)'),
    ('harmonic_backward-null', 'harmonic_backward', (P, P, P, None, 1, 10, 4, 640, SR, 0, None), E_INVALID, b'harmonic_backward: null pointer'),
    ('harmonic_backward-B', 'harmonic_backward', (P, P, P, P, -1, 10, 4, 640, SR, 0, None), E_INVALID, b'harmonic_backward: bad shape B=-1 F=10 K=4 N=640'),
    ('harmonic_backward-K', 'harmonic_backward', (P, P, P, P, 1, 10, 0, 640, SR, 0, None), E_INVALID, b'harmonic_backward: bad shape B=1 F=10 K=0 N=640'),
    ('harmonic_backward-divisible', 'harmonic_backward', (P, P, P, P, 1, 10, 4, 645, SR, 0, None), E_INVALID, b'harmonic_backward: bad shape B=1 F=10 K=4 N=645'),
    ('harmonic_backward-amp_method', 'harmonic_backward', (P, P, P, P, 1, 10, 4, 640, SR, 5, None), E_INVALID, b'harmonic_backward: bad amp_method 5'),
    ('harmonic_backward-sample_rate', 'harmonic_backward', (P, P, P, P, 1, 10, 4, 640, 0.0, 0, None), E_INVALID, b'harmonic_backward: sample_rate must be positive'),
    ('harmonic_backward-B0', 'harmonic_backward', (P, P, P, P, 0, 10, 4, 640, SR, 0, None), 0, None),
    ('harmonic_backward-hop65', 'harmonic_backward', (P, P, P, P, 1, 10, 4, 650, SR, 0, None), E_UNSUPPORTED, b'harmonic_backward: needs hop % 64 == 0 (hop = 65)'),
    ('harmonic_backward-hop8256', 'harmonic_backward', (P, P, P, P, 1, 1, 4, 8256, SR, 0, None), E_UNSUPPORTED, b'harmonic_backward: needs hop % 64 == 0 (hop = 8256)'),
    ('harmonic_backward-grid-limit', 'harmonic_backward', (P, P, P, P, 65536, 10, 4, 640, SR, 0, None), E_UNSUPPORTED, b'harmonic_backward: B=65536 exceeds the 65535 grid limit'),
    ('harmonic_backward_f0-null', 'harmonic_backward_f0', (P, P, P, P, None, 1, 10, 4, 640, SR, 0, P, 120, None), E_INVALID, b'harmonic_backward_f0: null pointer'),
    ('harmonic_backward_f0-B', 'harmonic_backward_f0', (P, P, P, P, P, -1, 10, 4, 640, SR, 0, P, 120, None), E_INVALID, b'harmonic_backward_f0: bad shape B=-1 F=10 K=4 N=640'),
    ('harmonic_backward_f0-N', 'harmonic_backward_f0', (P, P, P, P, P, 1, 10, 4, 0, SR, 0, P, 120, None), E_INVALID, b'harmonic_backward_f0: bad shape B=1 F=10 K=4 N=0'),
    ('harmonic_backward_f0-divisible', 'harmonic_backward_f0', (P, P, P, P, P, 1, 10, 4, 645, SR, 0, P, 120, None), E_INVALID, b'harmonic_backward_f0: bad shape B=1 F=10 K=4 N=645'),
    ('harmonic_backward_f0-hd', 'harmonic_backward_f0', (P, P, None, P, P, 1, 10, 4, 640, SR, 0, P, 120, None), E_INVALID, b'harmonic_backward_f0: harmonic_distribution is NULL but K=4'),
    ('harmonic_backward_f0-amp_method', 'harmonic_backward_f0', (P, P, P, P, P, 1, 10, 4, 640, SR, 2, P, 120, None), E_INVALID, b'harmonic_backward_f0: bad amp_method 2'),
    ('harmonic_backward_f0-sample_rate', 'harmonic_backward_f0', (P, P, P, P, P, 1, 10, 4, 640, 0.0, 0, P, 120, None), E_INVALID, b'harmonic_backward_f0: sample_rate must be positive'),
    ('harmonic_backward_f0-B0', 'harmonic_backward_f0', (P, P, P, P, P, 0, 10, 4, 640, SR, 0, P, 120, None), 0, None),
    ('harmonic_backward_f0-grid', 'harmonic_backward_f0', (P, P, P, P, P, 65536, 10, 4, 640, SR, 0, P, 120, None), E_INVALID, b'harmonic_backward_f0: B=65536 exceeds the 65535 grid limit'),
    ('harmonic_backward_f0-workspace-null', 'harmonic_backward_f0', (P, P, P, P, P, 1, 10, 4, 640, SR, 0, None, 120, None), E_WORKSPACE, b'harmonic_backward_f0: workspace of 120 B needed, 120 given'),
    ('harmonic_backward_f0-workspace-short', 'harmonic_backward_f0', (P, P, P, P, P, 1, 10, 4, 640, SR, 0, P, 119, None), E_WORKSPACE, b'harmonic_backward_f0: workspace of 120 B needed, 119 given'),
    ('harmonic_backward_f0-smem', 'harmonic_backward_f0', (P, P, P, P, P, 1, 10, 30000, 640, SR, 0, P, 120, None), E_UNSUPPORTED, b'harmonic_backward_f0: K=30000 needs more shared memory than one CTA has'),
    ('fir_time_varying-null', 'fir_time_varying', (P, None, P, 1, 1000, 10, 16, 1, 0, -1, 0, None), E_INVALID, b'fir_time_varying: null pointer'),
    ('fir_time_varying-B', 'fir_time_varying', (P, P, P, -1, 1000, 10, 16, 1, 0, -1, 0, None), E_INVALID, b'fir_time_varying: bad shape B=-1 N=1000 F=10 S=16'),
    ('fir_time_varying-S', 'fir_time_varying', (P, P, P, 1, 1000, 10, 0, 1, 0, -1, 0, None), E_INVALID, b'fir_time_varying: bad shape B=1 N=1000 F=10 S=0'),
    ('fir_time_varying-batch', 'fir_time_varying', (P, P, P, 2, 1000, 10, 16, 3, 0, -1, 0, None), E_INVALID, b'Batch size of audio (2) and impulse response (3) must be the same.'),
    ('fir_time_varying-padding', 'fir_time_varying', (P, P, P, 1, 1000, 10, 16, 1, 5, -1, 0, None), E_INVALID, b"Padding must be 'valid' or 'same' (got code 5)"),
    ('fir_time_varying-frames', 'fir_time_varying', (P, P, P, 1, 1000, 999, 16, 1, 0, -1, 0, None), E_INVALID, b'Number of Audio frames (500) and impulse response frames (999) do not match. For small hop size = ceil(audio_size / n_ir_frames), number of impulse response frames must be a multiple of the audio size.'),
    ('fir_time_varying-B0', 'fir_time_varying', (P, P, P, 0, 1000, 10, 16, 0, 0, -1, 0, None), 0, None),
    ('fir_time_varying-grid', 'fir_time_varying', (P, P, P, 65536, 1000, 10, 16, 1, 0, -1, 0, None), E_INVALID, b'fir_time_varying: B=65536 exceeds the 65535 grid limit'),
    ('fir_time_varying-delay', 'fir_time_varying', (P, P, P, 1, 1000, 10, 2, 1, 0, -1, 0, None), E_UNSUPPORTED, b'fir_time_varying: impulse response of 2 taps gives a negative automatic delay; pass delay_compensation >= 0'),
    ('fir_time_varying-smem', 'fir_time_varying', (P, P, P, 1, 1000, 10, 60000, 1, 0, -1, 0, None), E_UNSUPPORTED, b'fir_time_varying: impulse response of 60000 taps is beyond the shared-memory FIR (long-IR convolution is not built yet)'),
    ('filtered_noise_forward-null', 'filtered_noise_forward', (None, None, 0, 0, P, 1, 10, 1025, 640, 0, 0, None, 0, None), E_INVALID, b'filtered_noise_forward: null pointer'),
    ('filtered_noise_forward-F', 'filtered_noise_forward', (P, None, 0, 0, P, 1, 0, 1025, 640, 0, 0, None, 0, None), E_INVALID, b'filtered_noise_forward: bad shape B=1 F=0 N=640'),
    ('filtered_noise_forward-nb', 'filtered_noise_forward', (P, None, 0, 0, P, 1, 10, 1, 640, 0, 0, None, 0, None), E_INVALID, b'filtered_noise_forward: need n_frequencies >= 2 (got 1)'),
    ('filtered_noise_forward-frames', 'filtered_noise_forward', (P, None, 0, 0, P, 1, 999, 1025, 1000, 0, 0, None, 0, None), E_INVALID, b'Number of Audio frames (500) and impulse response frames (999) do not match. For small hop size = ceil(audio_size / n_ir_frames), number of impulse response frames must be a multiple of the audio size.'),
    ('filtered_noise_forward-B0', 'filtered_noise_forward', (P, None, 0, 0, P, 0, 10, 1025, 640, 0, 0, None, 0, None), 0, None),
    ('filtered_noise_forward-workspace', 'filtered_noise_forward', (P, None, 0, 0, P, 1, 10, 1025, 640, 0, 0, None, 0, None), E_WORKSPACE, b'filtered_noise_forward: workspace of 84736 B needed, 0 given'),
    ('filtered_noise_backward-null', 'filtered_noise_backward', (P, None, 0, 0, None, 1, 10, 65, 640, 257, None), E_INVALID, b'filtered_noise_backward: null pointer'),
    ('filtered_noise_backward-nb', 'filtered_noise_backward', (P, None, 0, 0, P, 1, 10, 1, 640, 257, None), E_INVALID, b'filtered_noise_backward: bad shape B=1 F=10 nb=1 N=640'),
    ('filtered_noise_backward-N', 'filtered_noise_backward', (P, None, 0, 0, P, 1, 10, 65, 0, 257, None), E_INVALID, b'filtered_noise_backward: bad shape B=1 F=10 nb=65 N=0'),
    ('filtered_noise_backward-frames', 'filtered_noise_backward', (P, None, 0, 0, P, 1, 999, 65, 1000, 257, None), E_INVALID, b'Number of Audio frames (500) and impulse response frames (999) do not match. For small hop size = ceil(audio_size / n_ir_frames), number of impulse response frames must be a multiple of the audio size.'),
    ('filtered_noise_backward-B0', 'filtered_noise_backward', (P, None, 0, 0, P, 0, 10, 65, 640, 257, None), 0, None),
    ('filtered_noise_backward-short-ir', 'filtered_noise_backward', (P, None, 0, 0, P, 1, 10, 2, 640, 0, None), E_UNSUPPORTED, b'filtered_noise_backward: impulse response too short'),
    ('filtered_noise_backward-tiles', 'filtered_noise_backward', (P, None, 0, 0, P, 1048576, 65536, 65, 65536, 257, None), E_INVALID, b'filtered_noise_backward: too many tiles'),
    ('filtered_noise_backward-smem', 'filtered_noise_backward', (P, None, 0, 0, P, 1, 10, 1025, 640, 0, None), E_UNSUPPORTED, b'filtered_noise_backward: shape needs 690560 B of shared memory'),
    ('oscillator_bank-null', 'oscillator_bank', (None, P, P, 1, 640, 4, SR, 1, None, 0, None), E_INVALID, b'oscillator_bank: null pointer'),
    ('oscillator_bank-K', 'oscillator_bank', (P, P, P, 1, 640, 0, SR, 1, None, 0, None), E_INVALID, b'oscillator_bank: bad shape B=1 N=640 K=0'),
    ('oscillator_bank-sample_rate', 'oscillator_bank', (P, P, P, 1, 640, 4, 0.0, 1, None, 0, None), E_INVALID, b'oscillator_bank: sample_rate must be positive'),
    ('oscillator_bank-B0', 'oscillator_bank', (P, P, P, 0, 640, 4, SR, 1, None, 0, None), 0, None),
    ('oscillator_bank-grid', 'oscillator_bank', (P, P, P, 65536, 640, 4, SR, 1, None, 0, None), E_INVALID, b'oscillator_bank: B=65536 exceeds the 65535 grid limit'),
    ('oscillator_bank-workspace', 'oscillator_bank', (P, P, P, 1, 640, 4, SR, 1, None, 0, None), E_WORKSPACE, b'oscillator_bank: workspace of 416 B needed, 0 given'),
    ('angular_cumsum-mode', 'angular_cumsum', (P, P, 1, 640, 4, 1000, 3, None, 0, None), E_INVALID, b'angular_cumsum: bad mode 3'),
    ('angular_cumsum-chunk', 'angular_cumsum', (P, P, 1, 640, 4, 0, 2, None, 0, None), E_INVALID, b'angular_cumsum: chunk_size must be positive'),
    ('angular_cumsum-B0', 'angular_cumsum', (P, P, 0, 640, 4, 1000, 0, None, 0, None), 0, None),
    ('angular_cumsum-grid', 'angular_cumsum', (P, P, 65536, 640, 4, 1000, 0, None, 0, None), E_INVALID, b'angular_cumsum: B=65536 exceeds the 65535 grid limit'),
    ('angular_cumsum-workspace', 'angular_cumsum', (P, P, 1, 640, 4, 1000, 0, None, 0, None), E_WORKSPACE, b'angular_cumsum: workspace of 416 B needed, 0 given'),
    ('fft_convolve_lti-null', 'fft_convolve_lti', (P, P, None, 1, 1000, 100, 1, 0, 1000, 0, 0, None, 0, None), E_INVALID, b'fft_convolve_lti: null pointer'),
    ('fft_convolve_lti-S', 'fft_convolve_lti', (P, P, P, 1, 1000, 0, 1, 0, 1000, 0, 0, None, 0, None), E_INVALID, b'fft_convolve_lti: bad shape B=1 N=1000 S=0'),
    ('fft_convolve_lti-batch', 'fft_convolve_lti', (P, P, P, 2, 1000, 100, 3, 0, 1000, 0, 0, None, 0, None), E_INVALID, b'Batch size of audio (2) and impulse response (3) must be the same.'),
    ('fft_convolve_lti-crop', 'fft_convolve_lti', (P, P, P, 1, 1000, 100, 1, 100, 1000, 0, 0, None, 0, None), E_INVALID, b'fft_convolve_lti: crop [100, 1100) leaves the convolution of length 1099'),
    ('fft_convolve_lti-B0', 'fft_convolve_lti', (P, P, P, 0, 1000, 100, 1, 0, 1000, 0, 0, None, 0, None), 0, None),
    ('fft_convolve_lti-out_len0', 'fft_convolve_lti', (P, P, P, 1, 1000, 100, 1, 0, 0, 0, 0, None, 0, None), 0, None),
    ('fft_convolve_lti-grid', 'fft_convolve_lti', (P, P, P, 65536, 1000, 100, 1, 0, 1000, 0, 0, None, 0, None), E_INVALID, b'fft_convolve_lti: B=65536 exceeds the 65535 grid limit'),
    ('fft_convolve_lti-workspace', 'fft_convolve_lti', (P, P, P, 1, 1000, 100, 1, 0, 1000, 0, 0, None, 0, None), E_WORKSPACE, b'fft_convolve_lti: workspace of 57600 B needed, 0 given'),
    ('fft_convolve_lti-flags', 'fft_convolve_lti', (P, P, P, 1, 1000, 100, 1, 0, 1000, 0, 4, P, 1073741824, None), E_INVALID, b'fft_convolve_lti: bad flags 4'),
    ('sinusoidal_forward-null', 'sinusoidal_forward', (P, None, P, 1, 10, 4, 640, SR, 0, 0, None, 0, None), E_INVALID, b'sinusoidal_forward: null pointer'),
    ('sinusoidal_forward-window', 'sinusoidal_forward', (P, P, P, 1, 10, 4, 10, SR, 0, 0, None, 0, None), E_INVALID, b'sinusoidal_forward: window upsampling cannot downsample (frames 10 >= timesteps 10)'),
    ('sinusoidal_forward-B0', 'sinusoidal_forward', (P, P, P, 0, 10, 4, 640, SR, 0, 0, None, 0, None), 0, None),
    ('sinusoidal_forward-smem', 'sinusoidal_forward', (P, P, P, 1, 10, 30000, 640, SR, 0, 0, None, 0, None), E_UNSUPPORTED, b'sinusoidal_forward: K=30000 needs more shared memory than one CTA has'),
    ('sinusoidal_forward-workspace', 'sinusoidal_forward', (P, P, P, 1, 10, 4, 640, SR, 0, 0, None, 0, None), E_WORKSPACE, b'sinusoidal_forward: workspace of 288 B needed, 0 given'),
    ('sinusoidal_backward-null', 'sinusoidal_backward', (P, P, P, None, None, 1, 10, 4, 640, SR, 0, None, 0, None), E_INVALID, b'sinusoidal_backward: null pointer'),
    ('sinusoidal_backward-divisible', 'sinusoidal_backward', (P, P, P, None, P, 1, 10, 4, 645, SR, 0, None, 0, None), E_INVALID, b'sinusoidal_backward: n_samples (645) must be divisible by the number of frames (10)'),
    ('sinusoidal_backward-B0', 'sinusoidal_backward', (P, P, P, None, P, 0, 10, 4, 640, SR, 0, None, 0, None), 0, None),
    ('sinusoidal_backward-workspace', 'sinusoidal_backward', (P, P, P, None, P, 1, 10, 4, 640, SR, 0, None, 0, None), E_WORKSPACE, b'sinusoidal_backward: workspace of 1344 B needed, 0 given'),
    ('filtered_noise_workspace-0-1000-65-64000-257', 'filtered_noise_workspace', (0, 1000, 65, 64000, 257), 0, None),
    ('filtered_noise_workspace-0-250-65-64000-0', 'filtered_noise_workspace', (0, 250, 65, 64000, 0), 0, None),
    ('filtered_noise_workspace-0-10-1025-640-0', 'filtered_noise_workspace', (0, 10, 1025, 640, 0), 0, None),
    ('filtered_noise_workspace-0-10-129-641-64', 'filtered_noise_workspace', (0, 10, 129, 641, 64), 0, None),
    ('filtered_noise_workspace-0-10-1-640-0', 'filtered_noise_workspace', (0, 10, 1, 640, 0), 0, None),
    ('oscillator_bank_workspace-0-1-1', 'oscillator_bank_workspace', (0, 1, 1), 0, None),
    ('oscillator_bank_workspace-0-640-4', 'oscillator_bank_workspace', (0, 640, 4), 0, None),
    ('oscillator_bank_workspace-0-64000-100', 'oscillator_bank_workspace', (0, 64000, 100), 0, None),
    ('oscillator_bank_workspace-0-0-4', 'oscillator_bank_workspace', (0, 0, 4), 0, None),
    ('fft_convolve_lti_workspace-0-1000-100-1', 'fft_convolve_lti_workspace', (0, 1000, 100, 1), 0, None),
    ('fft_convolve_lti_workspace-0-64000-64000-1', 'fft_convolve_lti_workspace', (0, 64000, 64000, 1), 0, None),
    ('fft_convolve_lti_workspace-0-64000-16000-0', 'fft_convolve_lti_workspace', (0, 64000, 16000, 0), 0, None),
    ('fft_convolve_lti_workspace-0-10-1-2', 'fft_convolve_lti_workspace', (0, 10, 1, 2), 0, None),
    ('sinusoidal_workspace-0-1-1', 'sinusoidal_workspace', (0, 1, 1), 0, None),
    ('sinusoidal_backward_workspace-0-1-1', 'sinusoidal_backward_workspace', (0, 1, 1), 0, None),
    ('sinusoidal_workspace-0-250-100', 'sinusoidal_workspace', (0, 250, 100), 0, None),
    ('sinusoidal_backward_workspace-0-250-100', 'sinusoidal_backward_workspace', (0, 250, 100), 0, None),
    ('sinusoidal_workspace-0-1000-420', 'sinusoidal_workspace', (0, 1000, 420), 0, None),
    ('sinusoidal_backward_workspace-0-1000-420', 'sinusoidal_backward_workspace', (0, 1000, 420), 0, None),
    ('sinusoidal_workspace-0-10-30000', 'sinusoidal_workspace', (0, 10, 30000), 0, None),
    ('sinusoidal_backward_workspace-0-10-30000', 'sinusoidal_backward_workspace', (0, 10, 30000), 0, None),
    ('sinusoidal_workspace-0-0-4', 'sinusoidal_workspace', (0, 0, 4), 0, None),
    ('sinusoidal_backward_workspace-0-0-4', 'sinusoidal_backward_workspace', (0, 0, 4), 0, None),
    ('filtered_noise_workspace-1-1000-65-64000-257', 'filtered_noise_workspace', (1, 1000, 65, 64000, 257), 0, None),
    ('filtered_noise_workspace-1-250-65-64000-0', 'filtered_noise_workspace', (1, 250, 65, 64000, 0), 0, None),
    ('filtered_noise_workspace-1-10-1025-640-0', 'filtered_noise_workspace', (1, 10, 1025, 640, 0), 84736, None),
    ('filtered_noise_workspace-1-10-129-641-64', 'filtered_noise_workspace', (1, 10, 129, 641, 64), 5340, None),
    ('filtered_noise_workspace-1-10-1-640-0', 'filtered_noise_workspace', (1, 10, 1, 640, 0), 0, None),
    ('oscillator_bank_workspace-1-1-1', 'oscillator_bank_workspace', (1, 1, 1), 264, None),
    ('oscillator_bank_workspace-1-640-4', 'oscillator_bank_workspace', (1, 640, 4), 416, None),
    ('oscillator_bank_workspace-1-64000-100', 'oscillator_bank_workspace', (1, 64000, 100), 400256, None),
    ('oscillator_bank_workspace-1-0-4', 'oscillator_bank_workspace', (1, 0, 4), 0, None),
    ('fft_convolve_lti_workspace-1-1000-100-1', 'fft_convolve_lti_workspace', (1, 1000, 100, 1), 57600, None),
    ('fft_convolve_lti_workspace-1-64000-64000-1', 'fft_convolve_lti_workspace', (1, 64000, 64000, 1), 2343168, None),
    ('fft_convolve_lti_workspace-1-64000-16000-1', 'fft_convolve_lti_workspace', (1, 64000, 16000, 1), 1188096, None),
    ('fft_convolve_lti_workspace-1-10-1-2', 'fft_convolve_lti_workspace', (1, 10, 1, 2), 0, None),
    ('sinusoidal_workspace-1-1-1', 'sinusoidal_workspace', (1, 1, 1), 264, None),
    ('sinusoidal_backward_workspace-1-1-1', 'sinusoidal_backward_workspace', (1, 1, 1), 540, None),
    ('sinusoidal_workspace-1-250-100', 'sinusoidal_workspace', (1, 250, 100), 13056, None),
    ('sinusoidal_backward_workspace-1-250-100', 'sinusoidal_backward_workspace', (1, 250, 100), 513312, None),
    ('sinusoidal_workspace-1-1000-420', 'sinusoidal_workspace', (1, 1000, 420), 420256, None),
    ('sinusoidal_backward_workspace-1-1000-420', 'sinusoidal_backward_workspace', (1, 1000, 420), 8820512, None),
    ('sinusoidal_workspace-1-10-30000', 'sinusoidal_workspace', (1, 10, 30000), 2400256, None),
    ('sinusoidal_backward_workspace-1-10-30000', 'sinusoidal_backward_workspace', (1, 10, 30000), 8400512, None),
    ('sinusoidal_workspace-1-0-4', 'sinusoidal_workspace', (1, 0, 4), 0, None),
    ('sinusoidal_backward_workspace-1-0-4', 'sinusoidal_backward_workspace', (1, 0, 4), 0, None),
    ('filtered_noise_workspace-3-1000-65-64000-257', 'filtered_noise_workspace', (3, 1000, 65, 64000, 257), 0, None),
    ('filtered_noise_workspace-3-250-65-64000-0', 'filtered_noise_workspace', (3, 250, 65, 64000, 0), 0, None),
    ('filtered_noise_workspace-3-10-1025-640-0', 'filtered_noise_workspace', (3, 10, 1025, 640, 0), 253696, None),
    ('filtered_noise_workspace-3-10-129-641-64', 'filtered_noise_workspace', (3, 10, 129, 641, 64), 15508, None),
    ('filtered_noise_workspace-3-10-1-640-0', 'filtered_noise_workspace', (3, 10, 1, 640, 0), 0, None),
    ('oscillator_bank_workspace-3-1-1', 'oscillator_bank_workspace', (3, 1, 1), 280, None),
    ('oscillator_bank_workspace-3-640-4', 'oscillator_bank_workspace', (3, 640, 4), 736, None),
    ('oscillator_bank_workspace-3-64000-100', 'oscillator_bank_workspace', (3, 64000, 100), 1200256, None),
    ('oscillator_bank_workspace-3-0-4', 'oscillator_bank_workspace', (3, 0, 4), 0, None),
    ('fft_convolve_lti_workspace-3-1000-100-1', 'fft_convolve_lti_workspace', (3, 1000, 100, 1), 139520, None),
    ('fft_convolve_lti_workspace-3-64000-64000-1', 'fft_convolve_lti_workspace', (3, 64000, 64000, 1), 4964608, None),
    ('fft_convolve_lti_workspace-3-64000-16000-3', 'fft_convolve_lti_workspace', (3, 64000, 16000, 3), 3563776, None),
    ('fft_convolve_lti_workspace-3-10-1-2', 'fft_convolve_lti_workspace', (3, 10, 1, 2), 0, None),
    ('sinusoidal_workspace-3-1-1', 'sinusoidal_workspace', (3, 1, 1), 280, None),
    ('sinusoidal_backward_workspace-3-1-1', 'sinusoidal_backward_workspace', (3, 1, 1), 596, None),
    ('sinusoidal_workspace-3-250-100', 'sinusoidal_workspace', (3, 250, 100), 38656, None),
    ('sinusoidal_backward_workspace-3-250-100', 'sinusoidal_backward_workspace', (3, 250, 100), 1538912, None),
    ('sinusoidal_workspace-3-1000-420', 'sinusoidal_workspace', (3, 1000, 420), 1260256, None),
    ('sinusoidal_backward_workspace-3-1000-420', 'sinusoidal_backward_workspace', (3, 1000, 420), 26460512, None),
    ('sinusoidal_workspace-3-10-30000', 'sinusoidal_workspace', (3, 10, 30000), 7200256, None),
    ('sinusoidal_backward_workspace-3-10-30000', 'sinusoidal_backward_workspace', (3, 10, 30000), 25200512, None),
    ('sinusoidal_workspace-3-0-4', 'sinusoidal_workspace', (3, 0, 4), 0, None),
    ('sinusoidal_backward_workspace-3-0-4', 'sinusoidal_backward_workspace', (3, 0, 4), 0, None),
    ('ir_size-1-0', 'ir_size', (1, 0), E_INVALID, None),
    ('ir_size-2-0', 'ir_size', (2, 0), 2, None),
    ('ir_size-65-257', 'ir_size', (65, 257), 128, None),
    ('ir_size-1025-0', 'ir_size', (1025, 0), 2048, None),
    ('ir_size-513-22', 'ir_size', (513, 22), 21, None),
]


@pytest.mark.parametrize('fn,args,want,msg', [c[1:] for c in _ABI_CASES],
                         ids=[c[0] for c in _ABI_CASES])
def test_abi_check_table(fn, args, want, msg):
  """Every check of the touched entry points, one row each: the status and the full
  message come back before any CUDA call, and nothing is launched, so this runs
  without a GPU."""
  lib = _lib.load()
  launches = lib.ddsp_b200_launch_count()
  assert getattr(lib, 'ddsp_b200_' + fn)(*args) == want
  assert lib.ddsp_b200_launch_count() == launches
  if msg is not None:
    assert lib.ddsp_b200_last_error() == msg
    error = {E_INVALID: ValueError, E_UNSUPPORTED: NotImplementedError,
             E_WORKSPACE: RuntimeError}[want]
    with pytest.raises(error):
      _lib.check(want)


@pytest.mark.parametrize('nb,ws,want', [(1025, 0, 2048), (1025, 257, 257),
                                        (513, 22, 21), (513, 2048, 1024),
                                        (65, 0, 128), (65, 257, 128), (100, 50, 49)])
def test_ir_size_table(nb, ws, want):
  """core_test.py:825-855: window_size if odd, -1 if even, fft size if none."""
  assert _lib.load().ddsp_b200_ir_size(nb, ws) == want


def test_missing_library_is_loud(monkeypatch):
  monkeypatch.setattr(_lib, '_lib', None)
  monkeypatch.setattr(_lib, 'LIB_PATH', '/nonexistent/libddsp_b200.so')
  with pytest.raises(RuntimeError, match='no CPU fallback'):
    _lib.load()


# ---- Python error conventions (raised before any device work) ----------------
def test_harmonic_synthesis_value_errors():
  f0 = np.zeros((1, 10, 1), np.float32)
  amp = np.zeros((1, 10, 1), np.float32)
  with pytest.raises(ValueError, match='is invalid'):        # core.py:632-634
    core.harmonic_synthesis(f0, amp, n_samples=640, amp_resample_method='bogus')
  with pytest.raises(ValueError, match='only supports 3 dimensions'):
    core.harmonic_synthesis(f0[0], amp[0], n_samples=640)    # core.py:670-672
  with pytest.raises(ValueError, match='downsampling'):      # core.py:682-685
    core.harmonic_synthesis(f0, amp, n_samples=5)
  with pytest.raises(ValueError, match='divisible'):         # core.py:687-693
    core.harmonic_synthesis(f0, amp, n_samples=645)
  with pytest.raises(ValueError, match='harmonic_shifts'):
    core.harmonic_synthesis(f0, amp, harmonic_shifts=np.zeros((1, 9, 4), np.float32),
                            n_samples=640)


def test_fft_convolve_value_errors():
  """core_test.py:787-823."""
  audio = np.zeros((1, 1000), np.float32)
  with pytest.raises(ValueError, match='Batch size'):
    core.fft_convolve(audio, np.zeros((2, 1000), np.float32))
  for padding in ('', 'saaammmeee'):
    with pytest.raises(ValueError, match='Padding'):
      core.fft_convolve(audio, audio, padding=padding)
  for n_frames in (1010, 999):
    with pytest.raises(ValueError, match='Number of Audio frames'):
      core.fft_convolve(audio, np.zeros((1, n_frames, 1000), np.float32))


def test_filtered_noise_value_errors():
  with pytest.raises(ValueError, match='Number of Audio frames'):
    core.filtered_noise(np.zeros((1, 999, 65), np.float32), 1000)
  with pytest.raises(ValueError, match='noise must be'):
    core.filtered_noise(np.zeros((1, 10, 65), np.float32), 640,
                        noise=np.zeros((1, 64), np.float32))


def test_get_fft_size():
  """core.py:1317-1335."""
  assert core.get_fft_size(64, 128) == 256
  assert core.get_fft_size(64, 257) == 512
  assert core.get_fft_size(1000, 10) == 1024


# ---- dict helpers (core.py:39-129) --------------------------------------------
def test_nested_lookup_and_to_dict():
  d = {'a': {'b': {'c': 3}}, 'x': 1}
  assert core.nested_lookup('a/b/c', d) == 3
  assert core.nested_keys(d) == ['a/b/c', 'x']
  with pytest.raises(KeyError, match='available keys'):
    core.nested_lookup('a/z', d)
  assert core.to_dict([1, 2], ['p', 'q']) == {'p': 1, 'q': 2}
  assert core.to_dict({'k': 1}, ['ignored']) == {'k': 1}
  with pytest.raises(ValueError):
    core.to_dict([1, 2, 3], ['p', 'q'])
  assert core.make_iterable(None) == []
  arr = np.zeros(3)
  assert core.make_iterable(arr)[0] is arr


# ---- Processor / ProcessorGroup / DAG (processors.py:37-176, dags.py:57-195) --
class _Scale(processors.Processor):
  """A host-only processor: lets the DAG logic run without a GPU."""

  def __init__(self, gain, name):
    super().__init__(name=name)
    self.gain = gain

  def get_controls(self, x):
    return {'x': np.asarray(x) * 1.0}

  def get_signal(self, x):
    return x * self.gain


class _HostAdd(processors.Processor):

  def __init__(self, name='add'):
    super().__init__(name=name)

  def get_controls(self, signal_one, signal_two):
    return {'signal_one': signal_one, 'signal_two': signal_two}

  def get_signal(self, signal_one, signal_two):
    return signal_one + signal_two


def test_processor_call_protocol():
  """processors.py:53-68: drops training/mask, optional outputs dict."""
  p = _Scale(3.0, 'scale')
  x = np.ones((2, 4))
  assert np.all(p(x) == 3.0)
  out = p(x, return_outputs_dict=True, training=True, mask=None)
  assert set(out) == {'signal', 'controls'} and set(out['controls']) == {'x'}
  with pytest.raises(NotImplementedError):
    processors.Processor('base').get_controls()


def test_processor_group_dag_semantics():
  """processors_test.py:57-87 key set; dags.py:149-193 outputs / 'out' alias."""
  a, b, add = _Scale(2.0, 'a'), _Scale(5.0, 'b'), _HostAdd('add')
  dag = [(a, ['inputs/u']), (b, ['v']), (add, ['a/signal', 'b/signal'])]
  group = processors.ProcessorGroup(dag=dag, name='processor_group')
  assert group.dag == [['a', ['inputs/u']], ['b', ['v']],
                       ['add', ['a/signal', 'b/signal']]]
  assert group.processors == [a, b, add] and group.a is a
  feats = {'u': np.ones((1, 3)), 'v': np.ones((1, 3))}
  outs = group.get_controls(feats)
  for key in ['u', 'v', 'inputs/u', 'a/signal', 'a/controls/x', 'b/signal',
              'b/controls/x', 'add/signal', 'add/controls/signal_one',
              'add/controls/signal_two', 'out/signal']:
    assert isinstance(core.nested_lookup(key, outs), np.ndarray), key
  assert np.all(outs['out']['signal'] == 7.0)
  assert np.all(group.get_signal(outs) == 7.0)
  assert np.all(group(feats) == 7.0)
  full = group(feats, return_outputs_dict=True)
  assert set(full) == {'signal', 'controls'}
  # string nodes resolve through kwarg processors (dags.py:104-106)
  g2 = processors.ProcessorGroup(dag=[('a', ['u']), ('add', ['a/signal', 'u'])],
                                 a=a, add=add)
  assert np.all(g2({'u': np.ones((1, 3))}) == 3.0)
  with pytest.raises(KeyError):
    group.get_controls({'u': np.ones((1, 3))})          # 'v' missing


def test_dag_layer_non_processor_modules_and_output_keys():
  """dags.py:171-186: plain modules are called, tuples zipped with output keys."""

  class Split:
    name = 'split'

    def __call__(self, x):
      return x + 1, x - 1

  layer = dags.DAGLayer([(Split(), ['x'], ['hi', 'lo'])])
  out = layer({'x': np.zeros(2)})
  assert np.all(out['split']['hi'] == 1) and np.all(out['out']['lo'] == -1)
  bad = dags.DAGLayer([(Split(), ['x'], ['only_one'])])
  with pytest.raises(ValueError):
    bad({'x': np.zeros(2)})


def test_synth_constructors_match_reference_defaults():
  """synths.py:59-66, 153-158; processors.py:166."""
  h = synths.Harmonic()
  assert (h.n_samples, h.sample_rate, h.normalize_below_nyquist,
          h.amp_resample_method, h.use_angular_cumsum, h.name) == (
              64000, 16000, True, 'window', False, 'harmonic')
  assert h.scale_fn is core.exp_sigmoid
  n = synths.FilteredNoise()
  assert (n.n_samples, n.window_size, n.initial_bias, n.name) == (
      64000, 257, -5.0, 'filtered_noise')
  assert processors.Add().name == 'add'
  assert dags.is_processor(h) and dags.is_processor(n)


def test_decoder_pattern_detection():
  h, n, add = synths.Harmonic(), synths.FilteredNoise(), processors.Add()
  g = processors.ProcessorGroup(dag=[
      (h, ['amps', 'hd', 'f0_hz']), (n, ['mags']),
      (add, ['filtered_noise/signal', 'harmonic/signal'])])
  assert g._decoder_pattern() is not None
  g2 = processors.ProcessorGroup(dag=[(h, ['amps', 'hd', 'f0_hz'])])
  assert g2._decoder_pattern() is None
  g3 = processors.ProcessorGroup(dag=[
      (h, ['amps', 'hd', 'f0_hz']), (n, ['mags']),
      (add, ['harmonic/signal', 'harmonic/signal'])])
  assert g3._decoder_pattern() is None


def test_resample_value_errors():
  """core_test.py:178-198, 295-381 - raised before any device work."""
  for dims in (1, 2, 4):
    with pytest.raises(ValueError, match='only supports 3 dimensions'):
      core.upsample_with_windows(np.ones([5] * dims, np.float32), 16000)
  for add_endpoint in (True, False):
    with pytest.raises(ValueError, match='downsampling'):
      core.upsample_with_windows(np.ones([1, 16000, 1], np.float32), 5, add_endpoint)
  with pytest.raises(ValueError, match='divisible'):
    core.upsample_with_windows(np.ones([1, 5, 1], np.float32), 16)
  with pytest.raises(ValueError, match='divisible'):
    core.upsample_with_windows(np.ones([1, 5, 1], np.float32), 15, add_endpoint=False)
  with pytest.raises(ValueError, match='is invalid'):
    core.resample(np.ones([1, 5, 1], np.float32), 10, method='bogus')


def test_host_pipeline_validates_without_a_gpu():
  """ddsp_b200_host_pipeline_*: argument errors come back as status codes before
  any CUDA call; a null handle is rejected by the forward entry point."""
  import ctypes
  lib = _lib.load()
  h = ctypes.c_void_p()
  assert lib.ddsp_b200_host_pipeline_create(ctypes.byref(h), 0, 10, 4, 5, 640, 2) == _lib.E_INVALID
  assert not h.value
  assert lib.ddsp_b200_decoder_forward_host(None, 1, 1, 1, 1, 0, 0, 1, 1, 1, 16000.0,
                                            0, 3, 0, -5.0, None) == _lib.E_INVALID
  assert b'null handle' in lib.ddsp_b200_last_error()
  assert lib.ddsp_b200_host_pipeline_destroy(None) == 0


def test_host_decoder_rejects_non_decoder_dags():
  import ddsp_b200
  harm = ddsp_b200.Harmonic(n_samples=640)
  group = ddsp_b200.ProcessorGroup(dag=[(harm, ['a', 'h', 'f'])])
  with pytest.raises(ValueError):
    ddsp_b200.HostDecoder(group, 2, 10, 4, 5)


def test_window_and_crop_helpers_match_oracle_and_reference():
  """core.apply_window_to_impulse_response (core.py:1477-1531) and
  core.crop_and_compensate_delay (1338-1379): host-side torch ops, so they run on
  the CPU - against the oracle and the unmodified reference's results
  (tests/golden/host_helpers.npz, make_golden.py)."""
  import os
  import torch
  from oracle import ddsp_oracle as o
  from tests.golden import make_golden as mg
  ref = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden',
                             'host_helpers.npz'))
  irs, audio = mg.host_helper_inputs()
  for i, ((_, ws, causal), ir) in enumerate(zip(mg.WINDOW_CASES, irs)):
    got = core.apply_window_to_impulse_response(ir, ws, causal)
    assert isinstance(got, torch.Tensor) and not got.is_cuda
    want = o.apply_window_to_impulse_response(ir, ws, causal, dtype=np.float32)
    assert tuple(got.shape) == want.shape == ref['window_%d' % i].shape
    assert np.abs(got.numpy() - want).max() < 1e-6
    assert np.abs(got.numpy() - ref['window_%d' % i]).max() < 1e-6
  for i, ((_, n, s, pad, dc), a) in enumerate(zip(mg.CROP_CASES, audio)):
    got = core.crop_and_compensate_delay(a, n, s, pad, dc).numpy()
    want = o.crop_and_compensate_delay(a, n, s, pad, dc)
    assert np.array_equal(got, want)
    start, length = (int(v) for v in ref['crop_%d' % i])
    assert np.array_equal(got, a[:, start:start + length])
  with pytest.raises(ValueError, match="Padding must be 'valid' or 'same'"):
    core.crop_and_compensate_delay(np.zeros((1, 10), np.float32), 5, 3, 'full', 0)

