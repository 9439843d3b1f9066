"""The kernels that take a shape when a fused kernel declines it, and the kernels
behind the stand-alone core ops, against float64 at the shapes where their code
branches.

  A. harmonic_generic_kernel (harmonic.cuh): hops 1 .. 8256 (every hop that is
     not a multiple of 64, and 'direct' at 64), K 1 .. 20000, both phase modes,
     every f0 regime plus 'alllive' (the recurrence's whole chain live at every
     sample), every tile regime (FT = 2048, set by ft_fill, = F, halved by
     fit_tile to 2 and to 1) and the shared-memory limit;
  B. oscbank_* (oscbank.cuh): core.oscillator_bank and core.angular_cumsum over
     1 .. 8 blocks of 128 oscillators and 1 .. 500 chunks of 128 samples, and
     core.harmonic_synthesis where it runs resample + oscillator_bank;
  C. resample_kernel (controls.cuh): four methods, both add_endpoint values,
     up- and downsampling by non-integer ratios, 1-D .. 4-D inputs, a grid-stride
     loop that runs more than once;
  D. ir_kernel + fir_kernel (noise.cuh) behind frequency_impulse_response,
     fft_convolve (shared and per-item impulse responses, several frames,
     'valid', explicit delays, N < S, accumulate) and frequency_filter, and the
     multi-frame long-IR route of fft_convolve on cuFFT.

Shapes whose [B, N, K] is large for the NumPy oracle are checked against
tests/grad_ref.py's float64 restatements on the GPU (pinned to the oracle at
<= 1e-12 by tests/test_grad_ref.py); harmonic tile widths are restated in
grad_ref.harmonic_generic_tile and pinned by tests/test_forward_routing.py.
"""
import numpy as np
import pytest
import torch

from ddsp_b200 import _lib
from ddsp_b200 import core
from ddsp_b200 import effects
from oracle import ddsp_oracle as o
from tests import grad_ref
from tests.util import rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')
TOL = 1e-4
ORACLE_ELEMS = 4_000_000        # largest [B, N, K] handed to the NumPy oracle
CHUNK_ELEMS = 20_000_000        # per batch chunk of the float64 GPU reference
TWO_PI32 = float(np.float32(2 * np.pi))


def _np(x):
  return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _gate(got, want, tol=TOL):
  got, want = _np(got), _np(want)
  assert got.shape == want.shape, (got.shape, want.shape)
  assert np.isfinite(got).all()
  emax, el2 = rel_err(got, want)
  assert emax < tol and el2 < tol, (emax, el2)
  return emax, el2


def _n_sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


def _launches():
  return _lib.load().ddsp_b200_launch_count()


# ---------------------------------------------------------------------------
# A. harmonic_generic_kernel
# ---------------------------------------------------------------------------
def _harmonic_inputs(B, F, K, sr, regime, seed):
  f0 = grad_ref.low_f0_regime(regime, B, F, sr, seed=seed, n_harmonics=K).to(DEV)
  gen = torch.Generator(device='cpu').manual_seed(seed)
  amp = (torch.rand(B, F, 1, generator=gen) + 0.2).to(DEV)
  hd = torch.rand(B, F, K, generator=gen)
  hd = (hd / hd.sum(-1, keepdim=True)).to(DEV)
  return f0, amp, hd


def _harmonic_ref(f0, amp, hd, N, sr, method):
  """[B, N] float64 harmonic synthesis with the Nyquist decision in float32: the
  NumPy oracle for small shapes, grad_ref.harmonic on the GPU in batch chunks
  otherwise."""
  B, _, K = hd.shape
  if B * N * K <= ORACLE_ELEMS:
    return torch.from_numpy(o.harmonic_synthesis(
        _np(f0), _np(amp), harmonic_distribution=_np(hd), n_samples=N, sample_rate=sr,
        amp_resample_method=method)).to(DEV)
  step = max(1, CHUNK_ELEMS // (N * K))
  return torch.cat([grad_ref.harmonic(f0[i:i + step], amp[i:i + step], hd[i:i + step], N,
                                      sr, method) for i in range(0, B, step)])


@pytest.mark.parametrize('B,F,K,hop,sr,method,regime,mode,acc,ft',
                         grad_ref.GENERIC_HARMONIC_CASES)
def test_harmonic_generic_every_hop_k_mode_and_tile(B, F, K, hop, sr, method, regime, mode,
                                                    acc, ft):
  """core.harmonic_synthesis on harmonic_generic_kernel against float64: hops 1 ..
  8256, K 1 .. 20000, both phase modes, both amplitude methods, 16 / 44.1 / 48
  kHz, every f0 regime, accumulate onto a base, and the tiles FT = 2048, set by
  ft_fill (a strided f0 prefix over thousands of frames), = F, and halved by
  fit_tile.  The last tile of every item reads its frame F as frame F - 1."""
  assert grad_ref.harmonic_route(B, F, K, hop, mode, _n_sms()) == 'generic'
  assert grad_ref.harmonic_generic_tile(B, F, K, hop, _n_sms()) == ft
  N = F * hop
  f0, amp, hd = _harmonic_inputs(B, F, K, sr, regime, seed=K + hop + F)
  base = None
  if acc:
    base = 0.5 * torch.randn(B, N, device=DEV,
                             generator=torch.Generator(device=DEV).manual_seed(hop))
  out = base.clone() if acc else None
  got = core.harmonic_synthesis(f0, amp, harmonic_distribution=hd, n_samples=N,
                                sample_rate=sr, amp_resample_method=method, out=out,
                                accumulate=acc, phase_mode=mode)
  want = _harmonic_ref(f0, amp, hd, N, sr, method)
  _gate(got.double() - base.double() if acc else got, want)


def test_harmonic_generic_refuses_k_past_shared_memory_before_launching():
  """K = 25584 is the largest K one frame's rows fit in 200 KB; one more raises
  E_UNSUPPORTED (NotImplementedError) without a launch, in both phase modes."""
  assert grad_ref.harmonic_generic_tile(1, 3, 25584, 8256, _n_sms()) == 1
  assert grad_ref.harmonic_generic_tile(1, 3, 25585, 8256, _n_sms()) is None
  K, F, hop = 25585, 3, 8256
  f0, amp, hd = _harmonic_inputs(1, F, K, 16000, 'glide', seed=1)
  torch.cuda.synchronize()
  for mode in ('recurrence', 'direct'):
    before = _launches()
    with pytest.raises(NotImplementedError, match='shared memory'):
      core.harmonic_synthesis(f0, amp, harmonic_distribution=hd, n_samples=F * hop,
                              phase_mode=mode)
    assert _launches() == before


# ---------------------------------------------------------------------------
# B. oscillator_bank, angular_cumsum and the unfused harmonic routes
# ---------------------------------------------------------------------------
def _oscbank_inputs(B, N, K, sr, seed):
  """Frequencies in [-0.3, 0.55] sr (negative ones and masked ones above Nyquist);
  every 7th sample of oscillator 0 exactly at sr / 2 (silenced: the mask is >=)
  and of oscillator 1 one float32 ulp below it (live)."""
  gen = torch.Generator(device=DEV).manual_seed(seed)
  f = (torch.rand(B, N, K, device=DEV, generator=gen) * 0.85 - 0.3) * sr
  a = torch.rand(B, N, K, device=DEV, generator=gen) + 0.1
  nyq = np.float32(sr / 2.0)
  f[:, ::7, 0] = float(nyq)
  if K > 1:
    f[:, ::7, 1] = float(np.nextafter(nyq, np.float32(0)))
  return f, a


@pytest.mark.parametrize('sum_sinusoids', [True, False])
@pytest.mark.parametrize('B,N,K,sr', [
    (1, 1, 1, 16000),
    (64, 127, 127, 16000),
    (5, 128, 128, 44100),
    (3, 129, 129, 16000),
    (2, 12345, 300, 48000),       # 97 chunks, three blocks of 128 oscillators
    (1, 64000, 1000, 16000),      # 500 chunks, eight blocks
    (7, 12345, 1, 44100),
])
def test_oscillator_bank_over_oscillator_blocks_and_chunks(B, N, K, sr, sum_sinusoids):
  """core.oscillator_bank against float64: K over 1 .. 8 blocks of 128 threads (the
  per-warp partial sums accumulate across blocks), N over 1 .. 500 chunks,
  negative frequencies, and the Nyquist mask at and one ulp below sr / 2."""
  f, a = _oscbank_inputs(B, N, K, sr, seed=N + K)
  got = core.oscillator_bank(f, a, sample_rate=sr, sum_sinusoids=sum_sinusoids)
  want = grad_ref.oscillator_bank(f, a, sr, sum_sinusoids)
  _gate(got, want)
  if not sum_sinusoids:
    assert not got[:, ::7, 0].any()
    if K > 1 and N > 1:
      live = got[:, 7::7, 1].double()
      assert float((live - want[:, 7::7, 1]).abs().max()) < 1e-5
      assert float(live.abs().max()) > 0.1


def _landing_input(B, N, C, seed):
  """[B, N, C] float32 angular frequencies in (-pi, pi) whose float64 running sum
  lands, every 10 samples, on a multiple of 2 pi plus one of 0, +-1e-8, +-3e-8,
  +-1e-7 rad (to within ~4e-9: a coarse step to 0.04 short of the multiple, then a
  fine step of ~0.04, whose float32 spacing is 3.7e-9)."""
  rng = np.random.default_rng(seed)
  x = rng.uniform(-np.pi, np.pi, (B, N, C)).astype(np.float32)
  deltas = [0.0, 1e-8, -1e-8, 3e-8, -3e-8, 1e-7, -1e-7]
  two_pi = 2 * np.pi
  s = np.zeros((B, C))
  for t in range(N):
    if t % 10 == 8:
      m = np.floor(s / two_pi) + 1.0
      x[:, t] = (m * two_pi - 0.04 - s).astype(np.float32)
    elif t % 10 == 9:
      m = np.round((s + 0.04) / two_pi)
      x[:, t] = (m * two_pi + deltas[(t // 10) % len(deltas)] - s).astype(np.float32)
    s = s + x[:, t].astype(np.float64)
  return x


def _wrapped(got, want):
  d = np.mod(_np(got).astype(np.float64) - _np(want), 2 * np.pi)
  return np.minimum(d, 2 * np.pi - d)


@pytest.mark.parametrize('shape,landing', [
    ((3, 1), False), ((2, 127), True), ((4, 129, 1), True), ((1, 128, 127), False),
    ((2, 12345, 3, 43), True),          # 4-D, 129 channels
    ((1, 12345, 300), False), ((1, 64000, 1000), False), ((64, 1000, 2, 2), True),
])
def test_angular_cumsum_exact_and_wrapped(shape, landing):
  """core.angular_cumsum (exact mode) on 2-D .. 4-D inputs against the float64
  running sum, as a distance on the circle, with running sums that land on and
  within 1e-7 rad of multiples of 2 pi.  Values lie in [0, float32(2 pi)]: a
  phase within half a float32 ulp below 2 pi rounds up to float32(2 pi)."""
  B, N = shape[:2]
  C = int(np.prod(shape[2:])) if len(shape) > 2 else 1
  if landing:
    x = torch.from_numpy(_landing_input(B, N, C, seed=N).reshape(shape)).to(DEV)
  else:
    gen = torch.Generator(device=DEV).manual_seed(N)
    x = (torch.rand(shape, device=DEV, generator=gen) * 2 - 1) * np.pi
  got = core.angular_cumsum(x)
  assert tuple(got.shape) == shape
  want = grad_ref.angular_cumsum(x)
  g = _np(got)
  assert np.isfinite(g).all() and g.min() >= 0.0 and g.max() <= TWO_PI32
  assert _wrapped(got, want).max() < 1e-6


@pytest.mark.parametrize('B,F,K,N,method', [
    (2, 50, 60, 16000, 'nearest'),
    (1, 40, 300, 12800, 'cubic'),
    (2, 250, 60, 16001, 'linear'),      # hop 64.004: not an integer
    (1, 101, 300, 44100, 'linear'),     # hop 436.6
    (1, 250, 60, 64000, 'cubic'),       # 500 chunks
    (3, 33, 60, 10000, 'nearest'),
])
def test_harmonic_synthesis_through_resample_and_oscillator_bank(B, F, K, N, method):
  """core.harmonic_synthesis where the fused kernels do not apply ('nearest' /
  'cubic' amplitudes, non-integer hops): resample + resample + oscillator_bank.

  This route materialises the frame-rate harmonic frequencies f0 * k and
  amplitudes amp * hd in float32, as the reference does, and accumulates every
  harmonic's phase from its float32 frequency.  The float32 rounding of f0 * k is
  constant over a frame, so that harmonic's phase drifts from k times the exact
  fundamental phase, and the audio sits 1.1e-4 .. 2e-4 (max-abs / peak) from the
  all-float64 oracle at 16000 .. 64000 samples.  The reference here is the float64
  decomposition fed those float32 frame-rate values: resample with TensorFlow's
  float32 index arithmetic (which the resample kernel follows), the Nyquist
  decision on the float32 envelopes, and the oscillator bank in float64."""
  sr = 16000 if N != 44100 else 44100
  f0, amp, hd = _harmonic_inputs(B, F, K, sr, 'glide', seed=F + K)
  got = core.harmonic_synthesis(f0, amp, harmonic_distribution=hd, n_samples=N,
                                sample_rate=sr, amp_resample_method=method)
  hf = o.get_harmonic_frequencies(_np(f0), K, np.float32)
  ha = (_np(amp) * _np(hd)).astype(np.float32)
  fe = o.resample(hf, N, tf_index_math=True)
  ae = o.resample(ha, N, method=method, tf_index_math=True)
  mask = o.resample(hf, N, dtype=np.float32, tf_index_math=True) >= np.float32(sr / 2.0)
  want = o.oscillator_bank(fe, ae, sample_rate=sr, nyquist_mask=mask)
  _gate(got, want)
  # and against the all-float64 oracle within the drift stated above
  wide = o.harmonic_synthesis(_np(f0), _np(amp), harmonic_distribution=_np(hd),
                              n_samples=N, sample_rate=sr, amp_resample_method=method,
                              tf_index_math=True)
  _gate(got, wide, tol=5e-4)


# ---------------------------------------------------------------------------
# C. resample_kernel
# ---------------------------------------------------------------------------
def _resample_input(shape, seed):
  return np.random.default_rng(seed).uniform(-1, 1, shape).astype(np.float32)


def _resample_check(x, n, method, ep):
  got = _np(core.resample(torch.from_numpy(x).to(DEV), n, method=method, add_endpoint=ep))
  want = o.resample(x, n, method=method, add_endpoint=ep, tf_index_math=True)
  assert got.shape == want.shape
  assert np.isfinite(got).all()
  assert np.abs(got - want).max() <= 1e-6, np.abs(got - want).max()


@pytest.mark.parametrize('ep', [True, False])
@pytest.mark.parametrize('method', ['linear', 'nearest', 'cubic'])
@pytest.mark.parametrize('F,N', [(7, 1000), (13, 641), (1000, 7), (641, 13), (1, 5),
                                 (5, 1), (9, 9), (4, 3), (3, 5), (9, 17), (11, 5)])
def test_resample_ratios_against_tf_index_math(F, N, method, ep):
  """Non-integer up- and downsampling ratios, F = 1, N = 1 and F = N, on [2, F, 3];
  (4, 3), (3, 5), (9, 17) and (11, 5) put exact ties t * scale = m + 1/2 on
  'nearest' with add_endpoint=False (roundf rounds them away from zero)."""
  _resample_check(_resample_input((2, F, 3), F * 100 + N), N, method, ep)


@pytest.mark.parametrize('method', ['linear', 'nearest', 'cubic', 'window'])
@pytest.mark.parametrize('shape,n', [((13,), 641), ((3, 7), 1000), ((2, 7, 1025), 1001),
                                     ((2, 5, 3, 4), 120), ((4, 7, 300), 1000)])
def test_resample_input_ranks_channels_and_grid_stride(shape, n, method):
  """1-D .. 4-D inputs, C = 1, 3, 1025, and [4, 1000, 300] (1.2e6 outputs: more
  than 16 CTAs x 132 SMs x 256 threads, so every thread's grid-stride loop runs
  again); 'window' refuses 4-D inputs and non-dividing sizes before launching."""
  x = _resample_input(shape, sum(shape) + n)
  if method == 'window':
    f = shape[1] if len(shape) > 1 else shape[0]
    if len(shape) == 4 or n % f:
      before = _launches()
      with pytest.raises(ValueError):
        core.resample(torch.from_numpy(x).to(DEV), n, method='window')
      assert _launches() == before
      return
  _resample_check(x, n, method, True)


@pytest.mark.parametrize('ep', [True, False])
@pytest.mark.parametrize('hop', [1, 2, 3, 441, 1000])
def test_resample_window_every_hop(hop, ep):
  """upsample_with_windows at hops 1 .. 1000, both add_endpoint values; hop 1 (as
  many frames as timesteps) raises before launching, as the reference does."""
  F = 5
  n = hop * (F if ep else F - 1)
  x = _resample_input((2, F, 3), hop)
  if hop == 1:
    before = _launches()
    with pytest.raises(ValueError):
      core.resample(torch.from_numpy(x).to(DEV), n, method='window', add_endpoint=ep)
    with pytest.raises(ValueError):
      o.resample(x, n, method='window', add_endpoint=ep)
    assert _launches() == before
    return
  _resample_check(x, n, 'window', ep)


# ---------------------------------------------------------------------------
# D. ir_kernel, fir_kernel and the multi-frame long-IR route
# ---------------------------------------------------------------------------
def _windows(nb):
  """window sizes for nb bins: the whole IR, odd and even padded, clamped.  A
  window of 1 or 2 taps on a longer IR is the known corner of DESIGN.md section
  3.1 (iii) (the reference's slicing keeps two taps, the kernel one) and is left
  out."""
  s0 = 2 * (nb - 1)
  odd = (s0 // 2) | 1
  even = (s0 // 2) & ~1
  return sorted({0, s0 + 7} | {w for w in (odd, even) if 2 < w < s0})


@pytest.mark.parametrize('nb', [2, 3, 4, 64, 65, 2049, 5000, 5120])
def test_frequency_impulse_response_every_band_count(nb):
  """ir_kernel at 2 .. 5120 bins (5120: 10 nb - 2 floats, the last that fit in
  200 KB), odd / even padded and clamped windows, 21 frames (not a multiple of
  the kernel's 8 frames per CTA), against float64 to 1e-6 abs."""
  m = np.random.default_rng(nb).uniform(0, 1, (3, 7, nb)).astype(np.float32)
  for ws in _windows(nb):
    want = o.frequency_impulse_response(m, ws)
    got = _np(core.frequency_impulse_response(torch.from_numpy(m).to(DEV), ws))
    assert got.shape == want.shape, ws
    assert np.isfinite(got).all()
    assert np.abs(got - want).max() < 1e-6, (ws, np.abs(got - want).max())


def test_frequency_impulse_response_refuses_too_many_bins_before_launching():
  m = torch.rand(2, 5121, device=DEV)
  torch.cuda.synchronize()
  before = _launches()
  with pytest.raises(NotImplementedError, match='too large'):
    core.frequency_impulse_response(m, 0)
  assert _launches() == before


def _conv_inputs(B, N, F, S, ir_batch, seed):
  rng = np.random.default_rng(seed)
  audio = rng.standard_normal((B, N)).astype(np.float32)
  ir = (rng.standard_normal((ir_batch, F, S)) / np.sqrt(S)).astype(np.float32)
  return audio, ir


def _conv_ref(audio, ir, padding, delay):
  B = audio.shape[0]
  return o.fft_convolve(audio, np.broadcast_to(ir, (B,) + ir.shape[1:]), padding=padding,
                        delay_compensation=delay)


# (B, N, F, S, ir_batch, padding, delay, accumulate)
FIR_CASES = [
    (2, 1000, 1, 3, 2, 'same', -1, False),
    (3, 1000, 7, 128, 1, 'same', -1, False),     # shared IR, ragged last frame
    (3, 1000, 7, 129, 1, 'valid', 0, True),
    (2, 1000, 1000, 129, 2, 'same', 64, False),  # one frame per sample
    (2, 300, 300, 3, 2, 'valid', -1, False),
    (1, 100, 1, 2047, 1, 'same', -1, False),     # N < S
    (2, 100, 7, 2047, 2, 'valid', 0, False),     # N < S, several frames
    (1, 1, 1, 3, 1, 'same', -1, False),          # N = 1
    (2, 1000, 1, 129, 2, 'same', 300, True),     # delay past S
    (3, 2000, 7, 2047, 1, 'same', 1023, False),  # delay S / 2
    (2, 777, 7, 1, 2, 'valid', 0, False),        # one tap, explicit delay
    (2, 64, 64, 2047, 2, 'same', 1023, True),
    (2, 1000, 1, 129, 1, 'valid', 300, False),   # delay past S, 'valid', shared IR
]


@pytest.mark.parametrize('B,N,F,S,ir_batch,padding,delay,acc', FIR_CASES)
def test_fft_convolve_short_impulse_responses(B, N, F, S, ir_batch, padding, delay, acc):
  """core.fft_convolve on fir_kernel (S < 2048): S = 1 .. 2047, one IR shared by
  every item (Reverb's layout) or one per item, 1, 7, 16 and N frames, ragged
  last frames, 'valid' and 'same', delay_compensation -1, 0, S / 2 and past S,
  N < S, N = 1, and out= with accumulate."""
  frame = -(-N // F)
  total = (F - 1) * frame + core.get_fft_size(frame, S)
  _, out_len, crop = core._crop_range(total, N, S, padding, delay)
  assert out_len == crop > 0                 # a non-degenerate crop
  audio, ir = _conv_inputs(B, N, F, S, ir_batch, seed=N + S + F)
  want = _conv_ref(audio, ir, padding, delay)
  a, h = torch.from_numpy(audio).to(DEV), torch.from_numpy(ir).to(DEV)
  base = None
  out = None
  if acc:
    base = torch.randn(B, crop, device=DEV, generator=torch.Generator(device=DEV)
                       .manual_seed(S))
    out = base.clone()
  got = core.fft_convolve(a, h, padding=padding, delay_compensation=delay, out=out,
                          accumulate=acc)
  _gate(got.double() - base.double() if acc else got, want)


@pytest.mark.parametrize('S', [1, 2])
def test_fir_refuses_negative_automatic_delay(S):
  """An impulse response of one or two taps gives the automatic delay -1: the
  reference's slice is then empty, and so is core.fft_convolve's result; the C
  ABI refuses the crop with E_UNSUPPORTED before launching."""
  audio, ir = _conv_inputs(2, 100, 1, S, 2, seed=S)
  want = _conv_ref(audio, ir, 'same', -1)
  got = core.fft_convolve(torch.from_numpy(audio).to(DEV), torch.from_numpy(ir).to(DEV))
  assert tuple(got.shape) == want.shape == (2, 0)
  lib = _lib.load()
  a, h = torch.from_numpy(audio).to(DEV), torch.from_numpy(ir).to(DEV)
  out = torch.empty(2, 100, device=DEV)
  torch.cuda.synchronize()
  before = _launches()
  rc = lib.ddsp_b200_fir_time_varying(a.data_ptr(), h.data_ptr(), out.data_ptr(), 2, 100,
                                      1, S, 2, _lib.PAD_SAME, -1, 0,
                                      torch.cuda.current_stream().cuda_stream)
  assert rc == _lib.E_UNSUPPORTED
  assert _launches() == before


@pytest.mark.parametrize('B,F,nb,N,ws', [(3, None, 65, 1000, 0), (2, None, 129, 777, 101),
                                         (3, 7, 65, 1000, 64), (2, 20, 33, 1280, 0)])
def test_frequency_filter_and_fir_filter(B, F, nb, N, ws):
  """core.frequency_filter and effects.FIRFilter with 2-D magnitudes (one IR per
  item) and with several frames, against float64."""
  shape = (B, nb) if F is None else (B, F, nb)
  rng = np.random.default_rng(nb + N)
  mags = rng.uniform(0.0, 1.0, shape).astype(np.float32)
  audio = rng.uniform(-1, 1, (B, N)).astype(np.float32)
  want = o.frequency_filter(audio, mags, window_size=ws)
  a, m = torch.from_numpy(audio).to(DEV), torch.from_numpy(mags).to(DEV)
  _gate(core.frequency_filter(a, m, window_size=ws), want)
  fir = effects.FIRFilter(window_size=ws, scale_fn=None)
  _gate(fir(a, m), want)


@pytest.mark.parametrize('B,N,F,S,ir_batch,padding', [
    (2, 6000, 2, 2048, 2, 'same'),
    (3, 6000, 5, 3000, 1, 'valid'),
    (2, 16000, 16, 2049, 1, 'same'),
    (3, 4001, 5, 4096, 3, 'valid'),
    (2, 16000, 16, 2500, 2, 'same'),
])
def test_fft_convolve_long_impulse_responses_several_frames(B, N, F, S, ir_batch, padding):
  """The multi-frame long-IR route of core.fft_convolve (S >= 2048, several frames:
  the reference's framed algorithm on cuFFT) against grad_ref.fft_convolve in
  float64 on the GPU, shared and per-item impulse responses."""
  frame = -(-N // F)
  total = (F - 1) * frame + core.get_fft_size(frame, S)
  _, out_len, crop = core._crop_range(total, N, S, padding, -1)
  assert out_len == crop > 0 and S >= core.FFT_CONVOLVE_MIN_IR
  audio, ir = _conv_inputs(B, N, F, S, ir_batch, seed=N + S)
  a, h = torch.from_numpy(audio).to(DEV), torch.from_numpy(ir).to(DEV)
  got = core.fft_convolve(a, h, padding=padding)
  want = grad_ref.fft_convolve(a.double(), h.double(), padding=padding)
  _gate(got, want)
