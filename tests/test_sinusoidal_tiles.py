"""The Sinusoidal kernels (csrc/sinusoidal.cuh) at every tile height they choose.

`ddsp_b200_sinusoidal_forward` and `_backward` give a CTA FT frames: FT starts at
min(16, F) and halves, rounding up, while the tile's tables, (32 FT + 8) K bytes of
shared memory, exceed 200 KB.  For F >= 16 that is

  FT = 16 for K <= 393, 8 for 394 .. 775, 4 for 776 .. 1505, 2 for 1506 .. 2844,
  1 for 2845 .. 5120, and K >= 5121 is refused (E_UNSUPPORTED).

FT sets the number of tiles (and so the length of the tile-offset scan), the per-tile
phase tables of the forward and the prologue through which the backward rebuilds a
frame's phase from its tile's offset.  The GPU cases sit on both edges of every K
range, with one tile, several tiles and a last tile of 1 or FT - 1 frames.

CPU: the tile height and the workspace it implies, the refusal at K = 5121 before any
launch, and that every GPU case below lands on the tile height its id names.  GPU:
audio, d amplitudes and d frequencies against float64 autograd of
tests/sinusoidal_ref.py at every FT; the amplitude-only backward; accumulate=True on
ragged last tiles; and core.harmonic_synthesis on its routes into these kernels."""
import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, core
from tests import sinusoidal_ref as ref
from tests.util import rel_err

P = 0x1000        # a device pointer the library never dereferences on the host
SMEM = 200 * 1024
WINDOW, LINEAR = _lib.AMP_WINDOW, _lib.AMP_LINEAR


def tile_frames(F, K):
  """Frames per CTA of the Sinusoidal kernels (sinus_tile_frames)."""
  ft = min(16, F)
  while ft > 1 and (32 * ft + 8) * K > SMEM:
    ft = (ft + 1) // 2
  return ft


def _workspace(B, F, K, ft):
  """Bytes of the forward's workspace: one 64-bit phase offset per (b, tile, k)."""
  return 8 * B * -(-F // ft) * K + 256


# (K, FT) on both sides of every boundary, for F >= 16
EDGES = [(1, 16), (393, 16), (394, 8), (775, 8), (776, 4), (1505, 4), (1506, 2),
         (2844, 2), (2845, 1), (5120, 1)]

# (FT, B, F, K, hop, sample rate, amplitude method, frequency regime)
CASES = [
    (16, 2, 17, 393, 63, 44100, 'window', 'random'),    # last tile 1 frame
    (16, 1, 31, 1, 441, 48000, 'linear', 'glide'),      # last tile 15 frames
    (16, 2, 16, 393, 2, 16000, 'linear', 'above'),      # one tile
    (16, 1, 17, 200, 4096, 16000, 'window', 'zero'),
    (8, 2, 17, 394, 64, 16000, 'window', 'glide'),      # 8 + 8 + 1
    (8, 1, 15, 775, 441, 44100, 'linear', 'random'),    # FT 15 -> 8: 8 + 7
    (8, 1, 48, 775, 1, 48000, 'linear', 'above'),       # six full tiles
    (8, 2, 23, 600, 2, 44100, 'window', 'zero'),        # 8 + 8 + 7
    (4, 1, 17, 776, 63, 48000, 'linear', 'zero'),       # 4 x 4 + 1
    (4, 1, 7, 1505, 441, 16000, 'window', 'glide'),     # FT 7 -> 4: 4 + 3
    (4, 1, 4, 1000, 4096, 44100, 'window', 'random'),   # one tile
    (4, 1, 40, 1505, 2, 48000, 'window', 'above'),      # ten full tiles
    (2, 1, 7, 1506, 64, 16000, 'linear', 'random'),     # FT 7 -> 4 -> 2: 2 x 3 + 1
    (2, 2, 9, 2844, 63, 44100, 'window', 'above'),      # 2 x 4 + 1
    (2, 1, 2, 2844, 441, 48000, 'window', 'glide'),     # one tile
    (2, 1, 101, 2000, 1, 16000, 'linear', 'zero'),      # 51 tiles
    (1, 1, 3, 2845, 441, 44100, 'window', 'random'),
    (1, 1, 64, 5120, 2, 48000, 'linear', 'glide'),
    (1, 1, 2000, 2845, 1, 16000, 'linear', 'above'),    # a scan over 2000 tiles
    (1, 2, 1, 5120, 64, 16000, 'window', 'zero'),       # one frame
]

# (FT, B, F, K, hop, sample rate): ragged last tiles (FT = 1 has none)
RAGGED = [
    (16, 2, 17, 393, 63, 44100),      # last tile 1 frame
    (16, 1, 31, 100, 64, 16000),      # 15
    (8, 2, 17, 394, 64, 16000),       # 1
    (8, 1, 15, 775, 441, 44100),      # 7
    (4, 1, 17, 776, 63, 48000),       # 1
    (4, 1, 7, 1505, 441, 16000),      # 3
    (2, 2, 9, 2844, 63, 44100),       # 1
    (1, 1, 3, 2845, 441, 48000),
    (1, 1, 64, 5120, 2, 16000),
]

# (FT, B, F, K, hop, sample rate, amplitude method) of core.harmonic_synthesis with
# harmonic_shifts, on both sides of K = 775 and K = 1505
HARMONIC_SHIFTS = [
    (8, 1, 20, 775, 64, 16000, 'window'),
    (4, 1, 20, 776, 63, 44100, 'linear'),
    (4, 1, 20, 1505, 441, 48000, 'window'),
    (2, 1, 20, 1506, 2, 16000, 'linear'),
]
# without shifts, under grad, at a hop the fused harmonic backward refuses
HARMONIC_NO_SHIFTS = [
    (4, 1, 20, 1000, 441, 16000, 'window'),
    (2, 1, 20, 2000, 441, 44100, 'linear'),
]


def _id(c):
  """FT{ft}-K{K}-B{B}-F{F}-hop{hop}-... of a case (FT, B, F, K, hop, ...)."""
  ft, B, F, K, hop, *rest = c
  return '-'.join([f'FT{ft}', f'K{K}', f'B{B}', f'F{F}', f'hop{hop}'] + [str(x) for x in rest])


# ---- CPU ---------------------------------------------------------------------
@pytest.mark.parametrize('F', [16, 17, 1000])
def test_tile_height_table(F):
  """The rule restated here gives the documented table at every boundary."""
  for K, ft in EDGES:
    assert tile_frames(F, K) == ft, (F, K)


def test_tile_height_starts_below_16_for_short_items():
  """Fewer than 16 frames: FT starts at F and halves rounding up (7 -> 4 -> 2 -> 1)."""
  assert [tile_frames(7, K) for K in (100, 1000, 2000, 5000)] == [7, 4, 2, 1]
  assert [tile_frames(15, K) for K in (100, 700, 1000, 2000, 5000)] == [15, 8, 4, 2, 1]
  assert [tile_frames(3, K) for K in (100, 2000, 5000)] == [3, 2, 1]
  assert tile_frames(1, 5120) == 1


@pytest.mark.parametrize('F', [1, 3, 7, 15, 16, 17, 1000])
@pytest.mark.parametrize('B', [1, 3])
def test_workspace_follows_tile_height(B, F):
  """The workspaces hold one phase offset per (b, tile, k), so they pin the number
  of tiles the library chose at every K boundary; the backward adds its five
  float partials per (b, frame, k)."""
  lib = _lib.load()
  for K in sorted({k for k, _ in EDGES} | {100, 1000, 2000, 5000}):
    ft = tile_frames(F, K)
    want = _workspace(B, F, K, ft)
    assert lib.ddsp_b200_sinusoidal_workspace(B, F, K) == want, (F, K, ft)
    assert lib.ddsp_b200_sinusoidal_backward_workspace(B, F, K) == (
        want + 4 * 5 * B * F * K + 256), (F, K, ft)


@pytest.mark.parametrize('F', [1, 16, 1000])
@pytest.mark.parametrize('method', [WINDOW, LINEAR], ids=['window', 'linear'])
def test_k_past_shared_memory_is_refused_before_launching(F, method):
  """K = 5121 does not fit one frame's tables: both entry points return
  E_UNSUPPORTED with their message and launch nothing.  K = 5120 passes that check
  and stops at the missing workspace."""
  lib = _lib.load()
  N = F * 64
  launches = lib.ddsp_b200_launch_count()
  assert lib.ddsp_b200_sinusoidal_forward(
      P, P, P, 2, F, 5121, N, 16000.0, method, 0, P, 1 << 40, None) == _lib.E_UNSUPPORTED
  assert lib.ddsp_b200_last_error() == (
      b'sinusoidal_forward: K=5121 needs more shared memory than one CTA has')
  assert lib.ddsp_b200_sinusoidal_backward(
      P, P, P, P, P, 2, F, 5121, N, 16000.0, method, P, 1 << 40, None) == _lib.E_UNSUPPORTED
  assert lib.ddsp_b200_last_error() == (
      b'sinusoidal_backward: K=5121 needs more shared memory than one CTA has')
  with pytest.raises(NotImplementedError):
    _lib.check(_lib.E_UNSUPPORTED)
  assert lib.ddsp_b200_sinusoidal_forward(
      P, P, P, 2, F, 5120, N, 16000.0, method, 0, None, 0, None) == _lib.E_WORKSPACE
  assert lib.ddsp_b200_sinusoidal_backward(
      P, P, P, P, P, 2, F, 5120, N, 16000.0, method, None, 0, None) == _lib.E_WORKSPACE
  assert lib.ddsp_b200_launch_count() == launches


def test_every_gpu_case_lands_on_its_tile_height():
  """The FT in each GPU case's id is the library's: by the rule and by the workspace.
  Each FT has both amplitude methods, both edges of its K range and, but for FT = 1,
  a ragged last tile of 1 and of FT - 1 frames."""
  lib = _lib.load()
  for ft, B, F, K, hop, *_ in CASES + RAGGED + HARMONIC_SHIFTS + HARMONIC_NO_SHIFTS:
    assert tile_frames(F, K) == ft, (F, K)
    assert lib.ddsp_b200_sinusoidal_workspace(B, F, K) == _workspace(B, F, K, ft)
    assert B * F * hop * K <= 2.1e7, (B, F, K, hop)
  for ft in (16, 8, 4, 2, 1):
    cases = [c for c in CASES if c[0] == ft]
    assert {c[6] for c in cases} == {'window', 'linear'}, ft
    assert {c[3] for c in cases} >= {k for k, f in EDGES if f == ft}, ft
    if ft > 1:
      last = {c[2] % ft for c in RAGGED if c[0] == ft}
      assert last == {1, ft - 1}, ft
  assert {c[4] for c in CASES} >= {1, 2, 63, 64, 441, 4096}
  assert {c[5] for c in CASES} == {16000, 44100, 48000}
  assert {c[7] for c in CASES} == {'random', 'glide', 'zero', 'above'}
  assert all(c[6] == 'linear' for c in CASES if c[4] == 1)


# ---- GPU ---------------------------------------------------------------------
DEV = 'cuda'


def _check(name, got, want, tol_max, tol_l2):
  got = got.detach().double().cpu().numpy()
  want = want.detach().double().cpu().numpy()
  assert np.isfinite(got).all(), name
  emax, el2 = rel_err(got, want)
  assert emax < tol_max and el2 < tol_l2, (name, emax, el2)


def _inputs(B, F, K, hop, sr, regime):
  """Frequencies of the regime, amplitudes in [0.1, 1.1) and an upstream gradient."""
  f = torch.from_numpy(ref.regime(regime, B, F, K, sr, seed=F * K + hop)).to(DEV)
  gen = torch.Generator(device='cpu').manual_seed(K + hop)
  a = (torch.rand((B, F, K), generator=gen) + 0.1).to(DEV)
  g = torch.randn((B, F * hop), generator=gen).to(DEV)
  return f, a, g


@pytest.mark.gpu
@pytest.mark.parametrize('ft,B,F,K,hop,sr,method,regime', CASES, ids=[_id(c) for c in CASES])
def test_forward_and_backward_against_float64(ft, B, F, K, hop, sr, method, regime):
  """Audio, d amplitudes and d frequencies against float64 autograd through the
  restatement, given the forward's float32 Nyquist mask.  A sinusoid above Nyquist
  in every frame gets exactly zero gradients."""
  assert tile_frames(F, K) == ft
  N = F * hop
  f, a, g = _inputs(B, F, K, hop, sr, regime)
  f1 = f.clone().requires_grad_(True)
  a1 = a.clone().requires_grad_(True)
  out = core.sinusoidal_synthesis(f1, a1, n_samples=N, sample_rate=sr,
                                  amp_resample_method=method)
  out.backward(g)
  want, d_f, d_a = ref.float64_grads(f, a, g, N, sr, method)
  _check('audio', out, want, 1e-4, 1e-4)
  _check('d amplitudes', a1.grad, d_a, 2e-4, 1e-4)
  _check('d frequencies', f1.grad, d_f, 5e-4, 2e-4)
  if regime == 'above':
    assert bool((a1.grad[..., 0] == 0).all()) and bool((f1.grad[..., 0] == 0).all())


@pytest.mark.gpu
@pytest.mark.parametrize('method', ['window', 'linear'])
@pytest.mark.parametrize('ft,B,F,K,hop,sr', RAGGED, ids=[_id(c) for c in RAGGED])
def test_amplitudes_only_backward_is_bit_identical(ft, B, F, K, hop, sr, method):
  """With only the amplitudes requiring grad the backward skips the phase path; its
  d amplitudes are bit for bit those of the call that also asks for d frequencies."""
  assert tile_frames(F, K) == ft
  N = F * hop
  f, a, g = _inputs(B, F, K, hop, sr, 'glide')
  a1, f1 = a.clone().requires_grad_(True), f.clone().requires_grad_(True)
  core.sinusoidal_synthesis(f1, a1, n_samples=N, sample_rate=sr,
                            amp_resample_method=method).backward(g)
  a2 = a.clone().requires_grad_(True)
  core.sinusoidal_synthesis(f, a2, n_samples=N, sample_rate=sr,
                            amp_resample_method=method).backward(g)
  assert f.grad is None and f1.grad is not None
  assert bool(torch.isfinite(a1.grad).all()) and float(a1.grad.abs().max()) > 0
  assert torch.equal(a1.grad, a2.grad)


@pytest.mark.gpu
@pytest.mark.parametrize('method', ['window', 'linear'])
@pytest.mark.parametrize('ft,B,F,K,hop,sr', RAGGED, ids=[_id(c) for c in RAGGED])
def test_accumulate_adds_to_out_and_writes_nothing_past_it(ft, B, F, K, hop, sr, method):
  """accumulate=True onto a known signal gives that signal plus the float64 audio;
  `out` sits between two guard bands of a larger buffer, and neither changes."""
  assert tile_frames(F, K) == ft
  N = F * hop
  f, a, _ = _inputs(B, F, K, hop, sr, 'glide')
  gen = torch.Generator(device='cpu').manual_seed(N)
  base = (0.5 * torch.randn((B, N), generator=gen)).to(DEV)
  guard = max(N, 1024)
  buf = torch.full((guard + B * N + guard,), 1234.5, device=DEV)
  out = buf[guard:guard + B * N].view(B, N)
  out.copy_(base)
  got = core.sinusoidal_synthesis(f, a, n_samples=N, sample_rate=sr,
                                  amp_resample_method=method, out=out, accumulate=True)
  assert got.data_ptr() == out.data_ptr()
  mask = torch.from_numpy(ref.nyquist_mask(f.cpu().numpy(), N, sr)).to(DEV)
  want = ref.torch_sinusoidal(f.double(), a.double(), N, sr, method, mask=mask)
  _check('accumulated audio', out.double() - base.double(), want, 1e-4, 1e-4)
  assert bool((buf[:guard] == 1234.5).all()) and bool((buf[guard + B * N:] == 1234.5).all())


# ---- core.harmonic_synthesis on the Sinusoidal kernels -------------------------
def _harmonic_inputs(B, F, K, hop, sr, seed):
  """f0 so that harmonic K sits between 0.6 and 1.4 times Nyquist: the top
  harmonics cross it from frame to frame.  Returns f0, amplitudes, distribution,
  shifts and an upstream gradient."""
  g = torch.Generator().manual_seed(seed)
  f0 = (0.5 * sr / K) * (0.6 + 0.8 * torch.rand(B, F, 1, generator=g))
  amps = 0.2 + torch.rand(B, F, 1, generator=g)
  hd = torch.rand(B, F, K, generator=g)
  shifts = 0.02 * torch.randn(B, F, K, generator=g)
  up = torch.randn(B, F * hop, generator=g)
  return [t.to(DEV) for t in (f0, amps, hd, shifts, up)]


@pytest.fixture
def sinusoidal_calls(monkeypatch):
  """The shapes core.sinusoidal_synthesis is called with."""
  calls = []
  real = core.sinusoidal_synthesis

  def spy(frequencies, amplitudes, *args, **kwargs):
    calls.append(tuple(frequencies.shape))
    return real(frequencies, amplitudes, *args, **kwargs)
  monkeypatch.setattr(core, 'sinusoidal_synthesis', spy)
  return calls


@pytest.mark.gpu
@pytest.mark.parametrize('ft,B,F,K,hop,sr,method', HARMONIC_SHIFTS,
                         ids=[_id(c) for c in HARMONIC_SHIFTS])
def test_harmonic_shifts_forward_against_float64(sinusoidal_calls, ft, B, F, K, hop, sr,
                                                 method):
  """harmonic_shifts without grad: (f0 k)(1 + shifts) on the Sinusoidal kernels."""
  assert tile_frames(F, K) == ft
  N = F * hop
  f0, amps, hd, shifts, _ = _harmonic_inputs(B, F, K, hop, sr, seed=K)
  out = core.harmonic_synthesis(f0, amps, harmonic_shifts=shifts, harmonic_distribution=hd,
                                n_samples=N, sample_rate=sr, amp_resample_method=method)
  assert sinusoidal_calls == [(B, F, K)]
  want = ref.harmonic_sinusoidal64(f0.double(), amps.double(), hd.double(), shifts.double(),
                                   N, sr, method)
  _check('audio', out, want, 1e-4, 1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize('ft,B,F,K,hop,sr,method,with_shifts',
                         [c + (True,) for c in HARMONIC_SHIFTS] +
                         [c + (False,) for c in HARMONIC_NO_SHIFTS],
                         ids=[_id(c + ('shifts',)) for c in HARMONIC_SHIFTS] +
                         [_id(c + ('no_shifts',)) for c in HARMONIC_NO_SHIFTS])
def test_harmonic_sinusoidal_route_backward_against_float64(
    sinusoidal_calls, ft, B, F, K, hop, sr, method, with_shifts):
  """Gradients to f0, amplitudes, distribution and shifts through the Sinusoidal
  backward against float64 autograd, with the tolerances of the K = 20 test of this
  route (test_processor_api_training.test_harmonic_shifts_and_other_hops_against_float64).
  Without shifts the hop is one the fused harmonic backward refuses."""
  assert tile_frames(F, K) == ft
  N = F * hop
  f0, amps, hd, shifts, up = _harmonic_inputs(B, F, K, hop, sr, seed=K + 1)
  if not with_shifts:
    shifts = None
    assert not core._harmonic_backward_takes(B, F, N)
  leaves = [t.clone().requires_grad_(True) for t in (f0, amps, hd)]
  s1 = shifts.clone().requires_grad_(True) if with_shifts else None
  out = core.harmonic_synthesis(leaves[0], leaves[1], harmonic_shifts=s1,
                                harmonic_distribution=leaves[2], n_samples=N,
                                sample_rate=sr, amp_resample_method=method)
  out.backward(up)
  assert sinusoidal_calls and set(sinusoidal_calls) == {(B, F, K)}
  l64 = [t.double().requires_grad_(True) for t in (f0, amps, hd)]
  s64 = shifts.double().requires_grad_(True) if with_shifts else None
  want = ref.harmonic_sinusoidal64(l64[0], l64[1], l64[2], s64, N, sr, method)
  want.backward(up.double())
  _check('audio', out, want, 1e-4, 1e-4)
  for name, got, r in zip(('f0', 'amps', 'hd'), leaves, l64):
    _check(name, got.grad, r.grad, 2e-3, 1e-3)
  if with_shifts:
    _check('shifts', s1.grad, s64.grad, 2e-3, 1e-3)


@pytest.mark.gpu
def test_harmonic_shifts_past_shared_memory_raise_but_plain_harmonics_do_not(
    sinusoidal_calls):
  """K = 5121 with harmonic_shifts takes the Sinusoidal kernel, which refuses it
  with its message before launching, with or without grad.  Without shifts the same
  K runs on the harmonic kernel, whose tables are per frame, not per sinusoid."""
  B, F, K, hop, sr = 1, 4, 5121, 64, 16000
  N = F * hop
  f0, amps, hd, shifts, _ = _harmonic_inputs(B, F, K, hop, sr, seed=5)
  lib = _lib.load()
  msg = 'sinusoidal_forward: K=5121 needs more shared memory than one CTA has'
  torch.cuda.synchronize()
  before = lib.ddsp_b200_launch_count()
  with pytest.raises(NotImplementedError, match=msg):
    core.harmonic_synthesis(f0, amps, harmonic_shifts=shifts, harmonic_distribution=hd,
                            n_samples=N, sample_rate=sr)
  with pytest.raises(NotImplementedError, match=msg):
    core.harmonic_synthesis(f0, amps, harmonic_shifts=shifts.clone().requires_grad_(True),
                            harmonic_distribution=hd, n_samples=N, sample_rate=sr)
  assert lib.ddsp_b200_launch_count() == before
  assert sinusoidal_calls and set(sinusoidal_calls) == {(B, F, K)}
  del sinusoidal_calls[:]
  # every harmonic below Nyquist, so no float32 Nyquist decision is in question
  f0 = 1.0 + 0.5 * torch.rand(B, F, 1, device=DEV,
                              generator=torch.Generator(device=DEV).manual_seed(5))
  out = core.harmonic_synthesis(f0, amps, harmonic_distribution=hd, n_samples=N,
                                sample_rate=sr)
  assert sinusoidal_calls == []
  # the harmonic kernel multiplies the phase of f0, not a float32 product f0 k
  hf = f0.double() * torch.arange(1, K + 1, device=DEV, dtype=torch.float64)
  assert float(hf.max()) < sr / 2
  want = ref.torch_sinusoidal(hf, amps.double() * hd.double(), N, sr, 'window')
  _check('audio', out, want, 1e-4, 1e-4)
