"""Times losses.SpectralLoss at the C4 shape (B = 128, N = 64000, FFT sizes 2048 .. 64)
on the fused path (SpectralLossFn with spectral_terms) against the torch path
(`SpectralLoss._call_spectrograms`: unfold framing, rfft, abs, core.diff / cumsum,
mean_difference, autograd), for each of delta_time, delta_freq and cumsum_freq alone
(with mag), all five terms together, and plain 'L2' on mag (which SpectralLoss keeps
on the torch path), forward and forward + backward.

CUDA events; the two paths alternate within each round, and each time is the median
over rounds.  Also records each path's peak memory for forward + backward and the
largest relative difference between the two losses, and prints the card name and
power limit read in the same run.

  python tools/spectral_loss_time.py [--iters 5] [--rounds 3] [--out FILE]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import losses, spectral_ops  # noqa: E402
from tools import measure  # noqa: E402

B, N = 128, 64000
SIZES = (2048, 1024, 512, 256, 128, 64)
CONFIGS = {
    'delta_time': dict(mag_weight=1.0, delta_time_weight=1.0),
    'delta_freq': dict(mag_weight=1.0, delta_freq_weight=1.0),
    'cumsum_freq': dict(mag_weight=1.0, cumsum_freq_weight=1.0),
    'all_terms': dict(mag_weight=1.0, delta_time_weight=1.0, delta_freq_weight=1.0,
                      cumsum_freq_weight=1.0, logmag_weight=1.0),
    'l2_mag': dict(loss_type='L2', mag_weight=1.0),
}


def _fused(loss, target, audio):
  return spectral_ops.SpectralLossFn.apply(
      target, audio, SIZES, loss.mag_weight, loss.logmag_weight, loss.delta_time_weight,
      loss.delta_freq_weight, loss.cumsum_freq_weight, loss.loss_type)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=5)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('spectral_loss_time.py')
  gen = torch.Generator(device='cuda').manual_seed(0)
  target = 0.1 * torch.randn(B, N, device='cuda', generator=gen)
  audio = (0.7 * target + 0.05 * torch.randn(B, N, device='cuda', generator=gen))
  a = audio.clone().requires_grad_(True)
  res = {'card': measure.card(), 'shape': [B, N], 'fft_sizes': list(SIZES), 'configs': {}}
  for name, kw in CONFIGS.items():
    loss = losses.SpectralLoss(fft_sizes=SIZES, **kw)
    paths = {
        'fused': lambda: _fused(loss, target, a),
        'torch': lambda: loss._call_spectrograms(target, a, None),
    }
    values = {}
    for p, f in paths.items():          # warm-up: cuFFT plans, caches
      values[p] = float(f().detach())
      f().backward()
    timed = {}
    for p, f in paths.items():
      timed[p + '_forward_ms'] = torch.no_grad()(f)
      timed[p + '_forward_backward_ms'] = lambda f=f: f().backward()
    r = measure.alternate(timed, args.rounds, args.iters, 0)
    for p, f in paths.items():
      r[p + '_peak_mib'] = measure.peak_bytes(lambda: f().backward()) / 2**20
    r['loss_rel_diff'] = abs(values['fused'] - values['torch']) / abs(values['torch'])
    r['fused_routed'] = loss._fusable(target, a, None)
    res['configs'][name] = r
    a.grad = None
  print(json.dumps(res))
  if args.out:
    measure.append_rows(args.out, [res])


if __name__ == '__main__':
  main()
