"""Kernel time of the ModDelay forward and backward (csrc/mod_delay.cuh) at
B = 256, N = 64000, L = 400 (ModDelay's default max_length at 16 kHz), with CUDA
events over a ring of input sets larger than twice the L2, and the achieved
fraction of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s).

  python tools/mod_delay_time.py [--iters 50] [--warmup 10]

Algorithmic bytes per sample: forward 16 (read phase, gain, audio; write out),
backward 28 (read phase, gain, audio, upstream gradient; write three gradients).
The backward's CTAs also re-read phase, gain and gradient over an (L - 1) halo per
1024-sample tile: 12 (L - 1) / 1024 B per sample more, reported separately.
Prints the card name and power limit read in the same run."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import _lib  # noqa: E402
from ddsp_b200 import core  # noqa: E402
from tools import measure  # noqa: E402

BWD_TILE = 1024      # md_::kTile


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, default=256)
  ap.add_argument('--n', type=int, default=64000)
  ap.add_argument('--max-length', type=int, default=400)
  ap.add_argument('--iters', type=int, default=50)
  ap.add_argument('--warmup', type=int, default=10)
  args = ap.parse_args()
  measure.require_cuda('mod_delay_time.py')
  B, N, L = args.batch, args.n, args.max_length
  lib = _lib.load()
  st = torch.cuda.current_stream().cuda_stream
  set_bytes = 4 * 4 * B * N                      # audio, phase, gain, gradient
  n_sets = measure.ring_len(set_bytes)
  gen = torch.Generator(device='cuda').manual_seed(0)
  t = torch.arange(N, device='cuda') / 16000.0
  sets = []
  for _ in range(n_sets):
    audio = torch.randn((B, N), device='cuda', generator=gen)
    phase = 0.8 + 0.2 * torch.sin(2 * torch.pi * (2.0 + 4.0 * torch.rand(
        (B, 1), device='cuda', generator=gen)) * t)
    gain = torch.rand((B, N), device='cuda', generator=gen)
    grad = torch.randn((B, N), device='cuda', generator=gen)
    sets.append((audio, phase, gain, grad))
  out = torch.empty((B, N), device='cuda')
  d = [torch.empty((B, N), device='cuda') for _ in range(3)]

  def fwd(s):
    audio, phase, gain, _ = s
    _lib.check(lib.ddsp_b200_mod_delay_forward(
        audio.data_ptr(), phase.data_ptr(), gain.data_ptr(), out.data_ptr(), B, N, L,
        0.4, 0.6, 1, st))

  def bwd(s):
    audio, phase, gain, grad = s
    _lib.check(lib.ddsp_b200_mod_delay_backward(
        audio.data_ptr(), phase.data_ptr(), gain.data_ptr(), grad.data_ptr(),
        d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), B, N, L, 0.4, 0.6, 1, st))

  # the timed calls are the ones ModDelay makes (same kernels as core.mod_delay)
  with torch.no_grad():
    core.mod_delay(sets[0][0], sets[0][2], sets[0][1], L, 0.4, 0.6, True)
  samples = B * N
  res = {'card': measure.card(), 'B': B, 'N': N, 'L': L, 'input_sets': n_sets,
         'ring_bytes': n_sets * set_bytes, 'l2_bytes': measure.l2_bytes()}
  for name, fn, per_sample, halo in (('forward', fwd, 16, 0.0),
                                     ('backward', bwd, 28, 12.0 * (L - 1) / BWD_TILE)):
    sec = measure.event_ms(fn, args.iters, args.warmup, sets) * 1e-3
    res[name] = {
        'us': sec * 1e6,
        'algorithmic_bytes': per_sample * samples,
        'halo_bytes': halo * samples,
        'achieved_TBps': per_sample * samples / sec / 1e12,
        'fraction_of_hbm_peak': per_sample * samples / sec / measure.HBM_BYTES_PER_S,
        'fraction_with_halo': (per_sample + halo) * samples / sec / measure.HBM_BYTES_PER_S,
    }
  print(json.dumps(res))


if __name__ == '__main__':
  main()
