"""Time of core.sinusoidal_to_harmonic (csrc/consistency.cuh, mode C) against a float32
torch composition of the reference formulation (core.py:733-781).

Shape: the self-supervised pitch model's, B = 32, T = 1000 frames, S = 100 sinusoids
(ResnetSinusoidalEncoder) and K = 100 harmonics (SinusoidalToHarmonicEncoder), 16 kHz,
harmonic_width 0.1, with normalize off and on; forward, and forward + backward to all
three inputs.  The composition forms the reference's [B, T, K, S] tensors
(1.28 GB each) and differentiates them with autograd.

  python tools/sinusoidal_to_harmonic_time.py [--iters 20] [--rounds 3] [--out FILE]

Times are CUDA events after warm-up, the median of `rounds` alternated rounds; peak
memory is torch.cuda.max_memory_allocated above the inputs.  Harmonic-sinusoid pairs
are counted from shapes, B T K S per forward.  Prints the card name and power limit read
in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import core  # noqa: E402
from tools import measure  # noqa: E402

DEV = 'cuda'
B, T, S, K = 32, 1000, 100, 100


def _safe_divide(n, d, eps=1e-7):
  return n / torch.where(d == 0.0, torch.full_like(d, eps), d)


def ref_s2h(sin_amps, sin_freqs, f0_hz, harmonic_width=0.1, n_harmonics=K, sample_rate=16000,
            normalize=False):
  """The reference formulation in float32 torch, pairwise tensors and all."""
  ratios = torch.linspace(1.0, float(n_harmonics), n_harmonics, device=f0_hz.device)
  harm_freqs = f0_hz * ratios
  freqs_diff = sin_freqs[:, :, None, :] - harm_freqs[..., None]
  freqs_ratio = torch.abs(_safe_divide(freqs_diff, f0_hz[..., None]))
  weights = torch.exp(-(freqs_ratio / harmonic_width)**2.0)
  if normalize:
    weights_sum = torch.sum(weights, -1, keepdim=True)
    weights = torch.where(weights_sum > 1.0, _safe_divide(weights, weights_sum), weights)
  harm_amps = torch.sum(weights * sin_amps[:, :, None, :], -1)
  harm_amps = torch.where(harm_freqs >= sample_rate / 2.0, torch.zeros_like(harm_amps),
                          harm_amps)
  harm_amp = torch.sum(harm_amps, -1, keepdim=True)
  return harm_amp, _safe_divide(harm_amps, harm_amp)


def _inputs(seed=1):
  """Noisy harmonics of f0 in 80 .. 400 Hz with a fifth of the sinusoids elsewhere."""
  rng = np.random.default_rng(seed)
  f0 = np.exp(rng.uniform(np.log(80.0), np.log(400.0), (B, T, 1)))
  freqs = f0 * rng.integers(1, 20, (B, T, S)) * np.exp(rng.normal(0.0, 0.02, (B, T, S)))
  freqs = np.where(rng.uniform(size=(B, T, S)) < 0.2, rng.uniform(20, 8000, (B, T, S)), freqs)
  amps = rng.uniform(0.05, 1.0, (B, T, S))
  return [torch.as_tensor(v, dtype=torch.float32, device=DEV) for v in (amps, freqs, f0)]


def _fwd_bwd(fn, inputs, normalize):
  g = torch.randn((B, T, K), device=DEV, generator=torch.Generator(DEV).manual_seed(0))

  def run():
    for x in inputs:
      x.grad = None
    amp, dist = fn(*inputs, normalize=normalize)
    (amp.sum() + (dist * g).sum()).backward()
  return run


def configs():
  plain = _inputs()
  leaves = [x.clone().requires_grad_(True) for x in plain]
  rows = []
  for norm in (False, True):
    tag = 'normalize' if norm else 'plain'
    rows.append(('forward_' + tag,
                 lambda n=norm: core.sinusoidal_to_harmonic(*plain, n_harmonics=K, normalize=n),
                 lambda n=norm: ref_s2h(*plain, normalize=n), B * T * K * S))
    rows.append(('forward_backward_' + tag,
                 _fwd_bwd(lambda *x, normalize: core.sinusoidal_to_harmonic(
                     *x, n_harmonics=K, normalize=normalize), leaves, norm),
                 _fwd_bwd(ref_s2h, leaves, norm), 2 * B * T * K * S))
  return rows


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('sinusoidal_to_harmonic_time.py')
  card = measure.card()
  rows = []
  for name, ours, theirs, pairs in configs():
    t = measure.alternate({'ms': ours, 'torch_ms': theirs}, args.rounds,
                          {'ms': args.iters, 'torch_ms': max(2, args.iters // 4)}, 3)
    torch.cuda.empty_cache()
    row = {'config': name, 'B': B, 'T': T, 'S': S, 'K': K, **t,
           'peak_mb': measure.peak_bytes(ours) / 2**20,
           'torch_peak_mb': measure.peak_bytes(theirs) / 2**20, 'pairs': pairs}
    row['pairs_per_s'] = pairs / (row['ms'] * 1e-3)
    row.update(card)
    rows.append(row)
    print(json.dumps(row), flush=True)
    torch.cuda.empty_cache()
  if args.out:
    measure.append_rows(args.out, rows)


if __name__ == '__main__':
  main()
