"""Times synths.Sinusoidal.get_signal: the fused frame-rate oscillator bank against the
reference's decomposition (resample + resample + oscillator_bank over [B, N, K]), and
its training step: forward + backward of `core.sinusoidal_synthesis` (d amplitudes
and d frequencies, `ddsp_b200_sinusoidal_backward`) at the InverseSynthesis shape
(B = 32, F = 125, K = 100, N = 64000: hop 512) and at F = 1000 (hop 64), against
float32 torch autograd through the materialised [B, N, K] envelopes.  CUDA events;
prints the card name and power limit read in the same run.

  python tools/sinusoidal_time.py [--iters 20] [--profile]"""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import core  # noqa: E402
from tools import measure  # noqa: E402


def _torch_decomposition(f, a, n, sr=16000.0):
  """Sinusoidal.get_signal as float32 torch ops over [B, N, K] ('window' amplitudes,
  linear frequencies, Nyquist mask, cumsum phase) - what autograd would run."""
  b, n_frames, k = f.shape
  hop = n // n_frames
  r = torch.arange(hop, device=f.device, dtype=torch.float32)
  frac = (r / hop)[None, None, :, None]
  w1 = 0.5 - 0.5 * torch.cos(math.pi * frac)
  f_next = torch.cat([f[:, 1:], f[:, -1:]], 1)
  a_next = torch.cat([a[:, 1:], a[:, -1:]], 1)
  fe = (f[:, :, None] + (f_next - f)[:, :, None] * frac).reshape(b, n, k)
  amp = (a[:, :, None] * (1 - w1) + a_next[:, :, None] * w1).reshape(b, n, k)
  amp = torch.where(fe >= sr / 2, torch.zeros_like(amp), amp)
  return (amp * torch.sin(torch.cumsum(fe * (2 * math.pi / sr), 1))).sum(-1)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--profile', action='store_true',
                  help='also list the per-kernel device times (torch.profiler)')
  args = ap.parse_args()
  measure.require_cuda('sinusoidal_time.py')
  print(json.dumps(measure.card()), flush=True)
  rng = np.random.default_rng(0)

  # inference: fused against the reference's decomposition on our kernels
  for B, K in ((8, 100), (32, 100)):
    F, N = 1000, 64000
    freqs = torch.from_numpy(rng.uniform(50, 7000, (B, F, K)).astype(np.float32)).cuda()
    amps = torch.from_numpy(rng.uniform(0, 1, (B, F, K)).astype(np.float32)).cuda()

    def fused():
      return core.sinusoidal_synthesis(freqs, amps, n_samples=N)

    def materialised():
      return core.oscillator_bank(core.resample(freqs, N),
                                  core.resample(amps, N, method='window'))
    for name, fn in (('fused frame-rate bank', fused),
                     ('resample + resample + oscillator_bank', materialised)):
      print('B=%d K=%d %-40s %.3f ms' % (B, K, name, measure.event_ms(fn, 5, 2)),
            flush=True)
    print('  max |fused - materialised| = %.2e' % (fused() - materialised()).abs().max().item())
    del freqs, amps

  # training: forward and forward + backward
  for B, F, K, N in ((32, 125, 100, 64000), (32, 1000, 100, 64000)):
    freqs = torch.from_numpy(rng.uniform(20, 7900, (B, F, K)).astype(np.float32)).cuda()
    amps = torch.from_numpy(rng.uniform(0, 0.05, (B, F, K)).astype(np.float32)).cuda()
    g = torch.randn((B, N), device='cuda')
    f1, a1 = freqs.clone().requires_grad_(True), amps.clone().requires_grad_(True)

    def fwd():
      with torch.no_grad():
        return core.sinusoidal_synthesis(freqs, amps, n_samples=N)

    def fwd_bwd(both=True):
      f1.grad = a1.grad = None
      fr = f1 if both else freqs
      core.sinusoidal_synthesis(fr, a1, n_samples=N).backward(g)

    def torch_fwd_bwd():
      f1.grad = a1.grad = None
      _torch_decomposition(f1, a1, N).backward(g)
    t_f = measure.event_ms(fwd, args.iters, 3)
    t_fb = measure.event_ms(fwd_bwd, args.iters, 3)
    t_fa = measure.event_ms(lambda: fwd_bwd(False), args.iters, 3)
    t_torch = measure.event_ms(torch_fwd_bwd, 3, 1)
    print('B=%d F=%d K=%d N=%d hop=%d' % (B, F, K, N, N // F))
    print('  forward                              %8.3f ms' % t_f)
    print('  forward + backward (d amp, d freq)   %8.3f ms   backward %.3f ms = %.2fx forward'
          % (t_fb, t_fb - t_f, (t_fb - t_f) / t_f))
    print('  forward + backward (d amp only)      %8.3f ms   backward %.3f ms = %.2fx forward'
          % (t_fa, t_fa - t_f, (t_fa - t_f) / t_f))
    print('  float32 torch autograd over [B,N,K]  %8.3f ms' % t_torch, flush=True)
    if args.profile:      # per-kernel device time of one forward + backward
      from torch.profiler import ProfilerActivity, profile
      with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fwd_bwd()
        torch.cuda.synchronize()
      for ev in prof.key_averages():
        if ev.device_type.name == 'CUDA' and 'sinus' in ev.key:
          print('    %-60s %8.1f us' % (ev.key[:60], ev.device_time_total))
    del freqs, amps, g, f1, a1
    torch.cuda.empty_cache()


if __name__ == '__main__':
  main()
