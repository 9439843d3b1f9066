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
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import losses, spectral_ops  # noqa: E402
from tools.oscillator_bank_time import _card  # noqa: E402

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


def _time(fn, iters):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(iters):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / iters


def _peak(fn):
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  base = torch.cuda.memory_allocated()
  fn()
  torch.cuda.synchronize()
  return (torch.cuda.max_memory_allocated() - base) / 2**20


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=5)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  gen = torch.Generator(device='cuda').manual_seed(0)
  target = 0.1 * torch.randn(B, N, device='cuda', generator=gen)
  audio = (0.7 * target + 0.05 * torch.randn(B, N, device='cuda', generator=gen))
  a = audio.clone().requires_grad_(True)
  res = {'card': _card(), 'shape': [B, N], 'fft_sizes': list(SIZES), 'configs': {}}
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
    times = {p + k: [] for p in paths for k in ('_forward_ms', '_forward_backward_ms')}
    for _ in range(args.rounds):
      for p, f in paths.items():
        with torch.no_grad():
          times[p + '_forward_ms'].append(_time(f, args.iters))
        times[p + '_forward_backward_ms'].append(_time(lambda: f().backward(), args.iters))
    r = {k: statistics.median(v) for k, v in times.items()}
    for p, f in paths.items():
      r[p + '_peak_mib'] = _peak(lambda: f().backward())
    r['loss_rel_diff'] = abs(values['fused'] - values['torch']) / abs(values['torch'])
    r['fused_routed'] = loss._fusable(target, a, None)
    res['configs'][name] = r
    a.grad = None
  line = json.dumps(res)
  print(line)
  if args.out:
    with open(args.out, 'a') as fh:
      fh.write(line + '\n')


if __name__ == '__main__':
  main()
