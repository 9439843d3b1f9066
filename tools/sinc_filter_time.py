"""Kernel time of core.sinc_filter (csrc/sinc.cuh) at four shapes, with CUDA events
after warm-up:

  (a) B = 32,  N = 64000, cutoff [B, 1000, 1], window 512 (513 taps)
  (b) B = 256, N = 64000, cutoff [B, 1000, 1], window 512
  (c) B = 32,  N = 64000, static cutoff [1, 1, 1], window 1024 (1025 taps)
  (d) B = 8,   N = 64000, audio-rate cutoff [B, N, 1], window 512

For each: the fused forward, the fused backward (both gradients), the composition
sinc_impulse_response + fft_convolve (forward), and float32 torch autograd of the
reference's framed-FFT formulation (forward + backward; skipped where its framed
tensors would not fit).  FMA rates count B N S multiply-adds for the forward and twice
that for the backward (d audio and d cutoff), from shapes.  Prints the card name and
power limit read in the same run.

  python tools/sinc_filter_time.py [--iters 20] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import core  # noqa: E402
from tools import measure  # noqa: E402

FMA_PEAK = measure.FP32_FLOPS_PER_S / 2     # an FMA is two FLOPs

SHAPES = {
    'a': (32, 64000, (32, 1000, 1), 512),
    'b': (256, 64000, (256, 1000, 1), 512),
    'c': (32, 64000, (1, 1, 1), 1024),
    'd': (8, 64000, (8, 64000, 1), 512),
}


def _torch_reference(audio, cutoff, s):
  """float32 torch: sinc taps [.., S], then the reference's framed FFT convolution."""
  half = s // 2
  idx = torch.arange(-half, half + 1, dtype=torch.float32, device=audio.device)
  x = cutoff * idx
  x = torch.where(x.abs() < 1e-20, torch.full_like(x, 1e-20), x) * np.pi
  w = torch.hamming_window(s, periodic=False, device=audio.device)
  u = w * torch.sin(x) / x
  h = u / u.sum(-1, keepdim=True).abs()
  b, n = audio.shape
  f = h.shape[1]
  frame = -(-n // f)
  fft = int(2**np.ceil(np.log2(frame + s - 1)))
  return core._fft_convolve_cufft(audio, h, f, frame, fft, half - 1, n)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('sinc_filter_time.py')
  res = {'card': measure.card(), 'shapes': {}}
  rng = np.random.default_rng(0)

  def seconds(fn):
    return measure.event_ms(fn, args.iters, args.warmup) * 1e-3

  for key, (b, n, cshape, ws) in SHAPES.items():
    s = 2 * (ws // 2) + 1
    audio = torch.from_numpy(rng.standard_normal((b, n)).astype(np.float32)).cuda()
    cutoff = torch.from_numpy(rng.uniform(0.05, 0.95, cshape).astype(np.float32)).cuda()
    g = torch.randn(b, n, device='cuda')
    row = {'B': b, 'N': n, 'cutoff': list(cshape), 'taps': s, 'fma': b * n * s}
    with torch.no_grad():
      row['fused_fwd_s'] = seconds(lambda: core.sinc_filter(audio, cutoff, window_size=ws))
      row['composition_fwd_s'] = seconds(
          lambda: core.fft_convolve(audio, core.sinc_impulse_response(cutoff, window_size=ws)))
    xa = audio.clone().requires_grad_(True)
    ct = cutoff.clone().requires_grad_(True)
    y = core.sinc_filter(xa, ct, window_size=ws)
    row['fused_bwd_s'] = seconds(
        lambda: torch.autograd.grad(y, (xa, ct), g, retain_graph=True))
    row['fused_fwd_fma_per_s'] = row['fma'] / row['fused_fwd_s']
    row['fused_fwd_share_of_fp32_peak'] = row['fused_fwd_fma_per_s'] / FMA_PEAK
    row['fused_bwd_share_of_fp32_peak'] = 2 * row['fma'] / row['fused_bwd_s'] / FMA_PEAK
    frames = cshape[1] if len(cshape) == 3 else 1
    frame = -(-n // frames)
    fft = int(2**np.ceil(np.log2(frame + s - 1)))
    if b * frames * fft * 4 * 8 < 20e9:
      def ref_step():
        xr = audio.clone().requires_grad_(True)
        cr = cutoff.clone().requires_grad_(True)
        yr = _torch_reference(xr, cr, s)
        torch.autograd.grad(yr, (xr, cr), g)
      row['torch_fwd_bwd_s'] = measure.event_ms(ref_step, max(3, args.iters // 4), 2) * 1e-3
    else:
      row['torch_fwd_bwd_s'] = None
    del y, xa, ct
    torch.cuda.empty_cache()
    res['shapes'][key] = row
    print(key, json.dumps(row), flush=True)
  print(json.dumps(res['card']))
  if args.out:
    measure.append_rows(args.out, [res])


if __name__ == '__main__':
  main()
