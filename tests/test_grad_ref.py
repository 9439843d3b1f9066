"""The float64 references of the backward tests (tests/grad_ref.py) against the
oracle, which is pinned to the reference itself: both must reproduce
`oracle.harmonic_synthesis` / `oracle.frequency_filter` to 1e-12 of the peak on
every shape the GPU tests use."""
import numpy as np
import pytest
import torch

from oracle import ddsp_oracle as o
from tests import grad_ref


def _rel(got, want):
  got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
  return np.abs(got - want).max() / max(np.abs(want).max(), 1e-300)


@pytest.mark.parametrize('B,F,K,hop,sr,method,regime', grad_ref.HARMONIC_CASES)
def test_harmonic_reference_matches_oracle(B, F, K, hop, sr, method, regime):
  N = F * hop
  f0 = grad_ref.low_f0_regime(regime, B, F, sr, seed=K + hop)
  g = torch.Generator().manual_seed(F * K)
  amp = torch.rand(B, F, 1, generator=g) + 0.2
  hd = torch.rand(B, F, K, generator=g)
  got = grad_ref.harmonic(f0, amp, hd, N, sr, method)
  want = o.harmonic_synthesis(f0.numpy(), amp.numpy(), harmonic_distribution=hd.numpy(),
                              n_samples=N, sample_rate=sr, amp_resample_method=method)
  assert got.shape == want.shape == (B, N)
  assert np.abs(want).max() > 0
  assert _rel(got.numpy(), want) <= 1e-12


@pytest.mark.parametrize('B,F,nb,ws,frame,ragged',
                         grad_ref.NOISE_CASES + [(2, 33, 65, 31, 50, True),
                                                 (1, 7, 65, 1, 64, False),
                                                 (2, 5, 65, 2, 48, True),
                                                 (1, 4, 17, 2, 30, False)])
def test_noise_reference_matches_oracle(B, F, nb, ws, frame, ragged):
  """Includes window_size 1 and 2, where the reference's slicing yields two taps
  and its crop then starts at -1, so 'same' returns an empty signal (DESIGN.md
  section 3.1 (iii)); the oracle follows the reference there, and so must this."""
  N = F * frame - (7 if ragged else 0)
  rng = np.random.default_rng(nb * 1000 + ws)
  mags = rng.uniform(0.05, 1.0, (B, F, nb))
  noise = rng.uniform(-1.0, 1.0, (B, N))
  ir = grad_ref.impulse_response(torch.from_numpy(mags), ws).numpy()
  ir_want = o.frequency_impulse_response(mags, ws)
  assert ir.shape == ir_want.shape
  assert _rel(ir, ir_want) <= 1e-12
  got = grad_ref.frequency_filter(torch.from_numpy(noise), torch.from_numpy(mags), ws)
  want = o.frequency_filter(noise, mags, window_size=ws)
  assert got.shape == want.shape
  if ws in (1, 2):
    assert want.shape == (B, 0)
    return
  assert want.shape == (B, N)
  assert _rel(got.numpy(), want) <= 1e-12


def test_references_are_differentiable_in_float64():
  f0 = grad_ref.low_f0_regime('jump', 1, 4, 16000, seed=1)
  amp = torch.rand(1, 4, 1, dtype=torch.float64, requires_grad=True)
  hd = torch.rand(1, 4, 5, dtype=torch.float64, requires_grad=True)
  f64 = f0.double().requires_grad_(True)
  grad_ref.harmonic(f64, amp, hd, 256).sum().backward()
  assert all(t.grad is not None and t.grad.dtype == torch.float64 for t in (amp, hd, f64))
  mags = torch.rand(1, 4, 9, dtype=torch.float64, requires_grad=True)
  grad_ref.frequency_filter(torch.rand(1, 200, dtype=torch.float64), mags, 7).sum().backward()
  assert mags.grad is not None and torch.isfinite(mags.grad).all()
