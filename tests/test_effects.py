"""Reverb / FIRFilter (SURVEY 8f-3) and the long-impulse-response path of
core.fft_convolve (framed FFT convolution on torch.fft / cuFFT).

CPU: the FFT formulation against the oracle's literal restatement of
core.py:1382-1473, for single-frame (reverb) and multi-frame IRs.  GPU: the
processors against the float64 oracle through both routes of fft_convolve."""
import numpy as np
import pytest
import torch

from oracle import ddsp_oracle as o
from ddsp_b200 import core
from tests.util import rel_err


def _fft_path(audio, ir, padding, delay):
  b, n = audio.shape
  ir3 = ir if ir.ndim == 3 else ir[:, None, :]
  f, s = ir3.shape[1], ir3.shape[2]
  frame = int(np.ceil(n / f))
  fft_size = core.get_fft_size(frame, s, power_of_2=True)
  total = (f - 1) * frame + fft_size
  start, out_len, crop = core._crop_range(total, n, s, padding, delay)
  assert out_len == crop
  return core._fft_convolve_cufft(torch.from_numpy(audio), torch.from_numpy(ir3), f,
                                  frame, fft_size, int(start), int(crop)).numpy()


@pytest.mark.parametrize('n,frames,taps,padding,delay', [
    (4000, 1, 3000, 'same', 0), (4000, 1, 3000, 'same', -1), (1000, 1, 100, 'valid', -1),
    (1280, 20, 129, 'same', -1), (1280, 5, 300, 'valid', -1), (999, 1, 4096, 'same', 0)])
def test_fft_formulation_matches_oracle(n, frames, taps, padding, delay):
  rng = np.random.default_rng(n + taps)
  audio = rng.standard_normal((2, n)).astype(np.float32)
  ir = (rng.standard_normal((2, frames, taps)) / np.sqrt(taps)).astype(np.float32)
  want = o.fft_convolve(audio, ir, padding=padding, delay_compensation=delay)
  got = _fft_path(audio, ir, padding, delay)
  assert got.shape == want.shape
  assert np.abs(got - want).max() < 1e-4 * max(1.0, np.abs(want).max())


def test_reverb_value_errors_and_masking():
  """effects.py:81-101 (ValueError without an IR) and 50-59 (dry tap masked)."""
  from ddsp_b200 import effects
  rev = effects.Reverb(trainable=False)
  ir = torch.arange(1.0, 6.0)[None, :].repeat(2, 1)
  masked = rev._mask_dry_ir(ir)
  assert masked.tolist() == [[0.0, 2.0, 3.0, 4.0, 5.0]] * 2
  assert rev._mask_dry_ir(ir[..., None]).shape == (2, 5)
  assert rev._match_dimensions(torch.zeros(3, 10), torch.ones(4)).shape == (3, 4)


def test_filtered_noise_reverb_constructor_and_errors():
  """effects.py:205-238, 266-270."""
  from ddsp_b200 import effects
  rev = effects.FilteredNoiseReverb()
  assert (rev.name, rev.trainable, rev._add_dry, rev._n_frames, rev._n_filter_banks) == (
      'filtered_noise_reverb', False, True, 1000, 16)
  syn = rev._synth
  assert (syn.n_samples, syn.window_size, syn.initial_bias) == (48000, 257, -3.0)
  assert syn.scale_fn is core.exp_sigmoid
  with pytest.raises(ValueError, match='Must provide "magnitudes" tensor'):
    rev.get_controls(np.zeros((2, 100), np.float32))
  with pytest.raises(ValueError, match='Must provide "ir" tensor'):
    effects.Reverb().get_controls(np.zeros((2, 100), np.float32))


@pytest.mark.parametrize('trainable', [False, True])
def test_filtered_noise_reverb_composition_matches_reference(monkeypatch, trainable):
  """The host logic of FilteredNoiseReverb (effects.py:202-278 on top of Reverb's
  28-117) against the UNMODIFIED reference class run on the NumPy shim, with the
  same noise and, when trainable, the same learned magnitudes.  The CUDA kernels
  are replaced by the oracle here (they have their own parity tests): what is under
  test is the composition - scale + bias, synthesis of the impulse response, tiling
  of the single learned response, dry-tap masking, 'same' convolution with zero
  delay compensation, dry mix.  The reference's results, with its random draw pinned
  to the same noise, are tests/golden/reverb_composition.npz (make_golden.py)."""
  import os
  from ddsp_b200 import effects
  from tests.golden import make_golden as mg
  B, N, L, F, NB, WS = (mg.REVERB[k] for k in ('B', 'N', 'L', 'F', 'NB', 'WS'))
  audio, mags, noise = mg.reverb_inputs(trainable)
  want = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden',
                              'reverb_composition.npz'))['out_trainable_%d' % trainable]

  # ---- ours, kernels swapped for the oracle ----
  def t32(x, device=None):
    return torch.as_tensor(np.asarray(x.detach() if isinstance(x, torch.Tensor) else x,
                                      dtype=np.float32))
  monkeypatch.setattr(core, 'torch_float32', t32)
  monkeypatch.setattr(core, 'noise_controls', lambda m, bias, scale=True: torch.from_numpy(
      o.noise_get_controls(t32(m).numpy(), initial_bias=bias, scale=scale,
                           dtype=np.float32)['magnitudes']))
  monkeypatch.setattr(core, 'filtered_noise', lambda m, n, window_size=257, noise=None, **kw:
                      torch.from_numpy(o.noise_get_signal(t32(m).numpy(), t32(noise).numpy(),
                                                          window_size=window_size,
                                                          dtype=np.float32)))
  monkeypatch.setattr(core, 'fft_convolve', lambda a, ir, padding='same',
                      delay_compensation=-1, **kw: torch.from_numpy(
                          o.fft_convolve(t32(a).numpy(), t32(ir).numpy(), padding=padding,
                                         delay_compensation=delay_compensation,
                                         dtype=np.float32)))
  rev = effects.FilteredNoiseReverb(trainable=trainable, reverb_length=L, window_size=WS,
                                    n_frames=F, n_filter_banks=NB)
  rev._synth.injected_noise = torch.from_numpy(noise)
  with torch.no_grad():
    if trainable:
      rev._magnitudes = torch.from_numpy(mags[0]).requires_grad_(True)
      got = rev(audio).numpy()
    else:
      got = rev(audio, mags).numpy()
  assert got.shape == want.shape == (B, N)
  assert np.abs(got - want).max() < 2e-5 * max(1.0, np.abs(want).max())


@pytest.mark.gpu
@pytest.mark.parametrize('taps,add_dry', [(3000, True), (48000, False), (200, True)])
def test_reverb_matches_oracle(taps, add_dry):
  import ddsp_b200
  rng = np.random.default_rng(taps)
  B, N = 2, 16000
  audio = rng.standard_normal((B, N)).astype(np.float32)
  ir = (rng.standard_normal((B, taps)) * np.exp(-np.arange(taps) / (taps / 6.0)) /
        np.sqrt(taps)).astype(np.float32)
  rev = ddsp_b200.Reverb(add_dry=add_dry)
  with pytest.raises(ValueError):
    rev.get_controls(audio)
  got = rev(audio, ir).cpu().numpy()
  masked = ir.copy()
  masked[:, 0] = 0.0
  want = o.fft_convolve(audio, masked, padding='same', delay_compensation=0)
  if add_dry:
    want = want + audio
  assert got.shape == (B, N)
  emax, el2 = rel_err(got, want)
  assert emax < 1e-4 and el2 < 1e-4, (emax, el2)


@pytest.mark.gpu
def test_trainable_reverb_and_fir_filter():
  import ddsp_b200
  rng = np.random.default_rng(3)
  B, N, F, nb = 2, 6400, 100, 65
  audio = rng.standard_normal((B, N)).astype(np.float32)
  rev = ddsp_b200.Reverb(trainable=True, reverb_length=4000)
  out = rev(audio)
  assert tuple(out.shape) == (B, N) and rev._ir.requires_grad
  out.square().mean().backward()
  assert rev._ir.grad is not None and float(rev._ir.grad.abs().sum()) > 0
  mags = rng.standard_normal((B, F, nb)).astype(np.float32)
  filt = ddsp_b200.FIRFilter(window_size=257)
  got = filt(audio, mags).cpu().numpy()
  scaled = o.exp_sigmoid(mags.astype(np.float64))
  want = o.frequency_filter(audio, scaled, window_size=257)
  emax, el2 = rel_err(got, want)
  assert emax < 1e-4 and el2 < 1e-4, (emax, el2)


@pytest.mark.gpu
@pytest.mark.parametrize('B,n,taps,ir_batch,padding,delay', [
    (2, 64000, 48000, 2, 'same', 0),        # effects.Reverb at the ae.gin length
    (3, 64000, 48000, 1, 'same', 0),        # one trainable IR shared by the batch
    (2, 16000, 2048, 2, 'same', -1),        # smallest IR on this route, auto delay
    (2, 5000, 9000, 2, 'valid', 0),         # IR longer than the audio, full tail
    (1, 1023, 2049, 1, 'same', 0),          # ragged against the 1024-sample blocks
    (2, 4097, 4096, 2, 'same', 5),
    (2, 1, 2048, 2, 'same', 0),             # one-sample audio
    (1, 2, 2049, 1, 'valid', 0),
    (2, 1025, 3072, 2, 'same', 0),          # one sample past a block, S = 3 blocks
    (2, 2047, 3073, 1, 'valid', 0),         # 'valid' with S > n, shared IR
    (2, 16000, 48000, 2, 'same', -1),       # auto delay: start 23998, j_first = 15
    (2, 4000, 3000, 2, 'same', 1500),       # positive delay past one block
    (5, 3001, 2048, 1, 'same', 0)])         # IR batch 1 at B = 5
def test_long_impulse_response_convolution_kernel(B, n, taps, ir_batch, padding, delay):
  """`ddsp_b200_fft_convolve_lti` (partitioned overlap-save, hand-written FFTs)
  behind core.fft_convolve for 2-D / single-frame impulse responses >= 2048 taps,
  against the oracle's restatement of core.py:1382-1473.  The kernel packs the two
  time-halves of the audio (n2 = ceil(n / 2) samples apart) into one complex
  signal and produces only the 1024-sample output blocks the crop reads, from
  max(0, start - n2) on: the automatic delay of a 48000-tap IR over 16000 samples
  starts that range at block 15."""
  rng = np.random.default_rng(n + taps)
  audio = rng.standard_normal((B, n)).astype(np.float32)
  ir = (rng.standard_normal((ir_batch, taps)) * np.exp(-np.arange(taps) / (taps / 5.0))
        ).astype(np.float32)
  want = o.fft_convolve(audio, np.broadcast_to(ir, (B, taps)) if ir_batch == 1 else ir,
                        padding=padding, delay_compensation=delay)
  got = core.fft_convolve(audio, ir, padding=padding, delay_compensation=delay)
  assert tuple(got.shape) == want.shape
  emax, el2 = rel_err(got.cpu().numpy(), want)
  assert emax < 1e-4 and el2 < 1e-4, (emax, el2)
  # accumulate into an existing buffer (the wet + dry sum of Reverb)
  base = torch.full(tuple(got.shape), 0.25, device='cuda')
  acc = core.fft_convolve(audio, ir, padding=padding, delay_compensation=delay,
                          out=base.clone(), accumulate=True)
  assert float((acc - (got + 0.25)).abs().max()) < 1e-5


# (B, n, S, ir_batch, padding, a, b): padding 'same' / 'valid' runs core.fft_convolve
# with delay_compensation a (b unused); padding None runs FftConvolveLtiFn on the
# crop [a, a + b), which the public API cannot always ask for.
LONG_CONV_BACKWARD_CASES = [
    (3, 6000, 5000, 1, 'same', 0, None),      # shared trainable IR, B > 1
    (3, 6000, 5000, 3, 'same', 0, None),
    (2, 16000, 48000, 2, 'same', 0, None),    # Reverb's crop with S > n: d IR past end
    (2, 1000, 3000, 1, 'same', 0, None),      # n < 1024, S > n, shared
    (2, 2047, 3073, 2, 'valid', 0, None),     # odd n, full tail
    (2, 1600, 4800, 1, 'same', -1, None),     # auto delay: start > n - 1 (d IR off < 0)
    (2, 5001, 2048, 2, None, 2500, 1500),     # start > S - 1: d audio off < 0
    (1, 1000, 2048, 1, None, 2500, 500),      # both offsets < 0, S > end
    (2, 3001, 9000, 2, None, 100, 3000),      # end = 3100: d IR zero past it
]


@pytest.mark.gpu
@pytest.mark.parametrize('B,n,S,ir_batch,padding,a,b', LONG_CONV_BACKWARD_CASES)
def test_long_convolution_backward_matches_autograd(B, n, S, ir_batch, padding, a, b):
  """FftConvolveLtiFn (the trainable Reverb): d audio and d impulse response from
  the same kernels on reversed operands, each with its own crop offset
  (S - 1 - start, n - 1 - start) and a padded-gradient branch where that offset is
  negative.  Checked (a) elementwise against float64 autograd of
  grad_ref.convolve_lti, (b) exactly 0 for samples and taps at or past start +
  out_len, which reach no output, and (c) by the linearity identity against the
  oracle's full convolution for three random directions of each operand."""
  from ddsp_b200 import autograd as ag
  from tests import grad_ref
  from tests.util import linearity
  if padding is None:
    start, out_len = a, b
  else:
    start, out_len, crop = core._crop_range(core.get_fft_size(n, S), n, S, padding, a)
    assert out_len == crop
  gen = torch.Generator().manual_seed(n + S)
  audio = torch.randn(B, n, generator=gen).cuda()
  ir = (torch.randn(ir_batch, S, generator=gen) *
        torch.exp(-torch.arange(S) / (S / 5.0))).cuda()
  g = torch.randn(B, out_len, generator=gen).cuda()
  a1, h1 = audio.clone().requires_grad_(True), ir.clone().requires_grad_(True)
  if padding is None:
    y = ag.FftConvolveLtiFn.apply(a1, h1, start, out_len)
  else:
    y = core.fft_convolve(a1, h1, padding=padding, delay_compensation=a)
  (y * g).sum().backward()
  a2, h2 = audio.double().requires_grad_(True), ir.double().requires_grad_(True)
  yr = grad_ref.convolve_lti(a2, h2, start, out_len)
  (yr * g.double()).sum().backward()
  assert tuple(y.shape) == tuple(yr.shape) == (B, out_len)
  for name, got, want, tol_max, tol_l2 in (('y', y, yr, 1e-4, 1e-4),
                                           ('d audio', a1.grad, a2.grad, 2e-4, 1e-4),
                                           ('d ir', h1.grad, h2.grad, 2e-4, 1e-4)):
    assert torch.isfinite(got).all(), name
    emax, el2 = rel_err(got.detach().cpu().numpy(), want.detach().cpu().numpy())
    assert emax < tol_max and el2 < tol_l2, (name, emax, el2)
  end = start + out_len
  assert not a1.grad[:, end:].any() and not h1.grad[:, end:].any()
  a64, h64 = audio.double().cpu().numpy(), ir.double().cpu().numpy()

  def full(x, h):
    h = np.broadcast_to(h, (B, h.shape[-1]))
    return o.fft_convolve(x, h, padding='valid', delay_compensation=0)

  linearity(a1.grad, g, lambda d: full(d, h64)[:, start:end], (B, n), seed=n)
  linearity(h1.grad, g, lambda d: full(a64, d)[:, start:end], (ir_batch, S), seed=S)


@pytest.mark.gpu
def test_trainable_reverb_with_impulse_response_longer_than_audio():
  """Reverb(trainable=True) at the default 48000 taps on one second of audio, with
  the dry tap masked and the IR tiled over the batch, through .backward():
  d audio and d IR against float64 autograd."""
  import ddsp_b200
  from tests import grad_ref
  B, n, S = 2, 16000, 48000
  gen = torch.Generator().manual_seed(11)
  audio = torch.randn(B, n, generator=gen).cuda()
  ir = (torch.randn(S, generator=gen) * torch.exp(-torch.arange(S) / 8000.0)).cuda()
  g = torch.randn(B, n, generator=gen).cuda()
  rev = ddsp_b200.Reverb(trainable=True, reverb_length=S)
  rev._ir = ir.clone().requires_grad_(True)
  a1 = audio.clone().requires_grad_(True)
  out = rev(a1)
  (out * g).sum().backward()
  a2, h2 = audio.double().requires_grad_(True), ir.double().requires_grad_(True)
  masked = torch.cat([h2.new_zeros(1), h2[1:]])[None, :]
  ref = grad_ref.convolve_lti(a2, masked, 0, n) + a2
  (ref * g.double()).sum().backward()
  for name, got, want, tol_max in (('out', out, ref, 1e-4), ('d audio', a1.grad, a2.grad, 2e-4),
                                   ('d ir', rev._ir.grad, h2.grad, 2e-4)):
    emax, el2 = rel_err(got.detach().cpu().numpy(), want.detach().cpu().numpy())
    assert emax < tol_max and el2 < 1e-4, (name, emax, el2)
  assert float(rev._ir.grad[0]) == 0.0 and not rev._ir.grad[n:].any()


@pytest.mark.gpu
@pytest.mark.parametrize('B,n,S,ir_batch,start,out_len', [
    (2, 3001, 2048, 2, 0, 3001), (1, 1000, 5000, 1, 700, 4000), (3, 4096, 3000, 1, 2500, 3000)])
def test_long_convolution_reverse_flags(B, n, S, ir_batch, start, out_len):
  """LTI_REVERSE_AUDIO / LTI_REVERSE_IR of `ddsp_b200_fft_convolve_lti` (the
  backward's time-reversed operands) against the same call on flipped tensors."""
  from tests import grad_ref
  gen = torch.Generator().manual_seed(n)
  audio = torch.randn(B, n, generator=gen).cuda()
  ir = torch.randn(ir_batch, S, generator=gen).cuda()
  for ra, ri in ((True, False), (False, True), (True, True)):
    got = core.fft_convolve_lti(audio, ir, start, out_len, reverse_audio=ra, reverse_ir=ri)
    x = audio.flip(-1).contiguous() if ra else audio
    h = ir.flip(-1).contiguous() if ri else ir
    want = core.fft_convolve_lti(x, h, start, out_len)
    peak = float(want.abs().max())
    assert float((got - want).abs().max()) <= 1e-6 * peak, (ra, ri)
    ref = grad_ref.convolve_lti(x.double(), h.double(), start, out_len)
    emax, el2 = rel_err(got.cpu().numpy(), ref.cpu().numpy())
    assert emax < 1e-4 and el2 < 1e-4, (ra, ri, emax, el2)
