"""Time of the loudness and RMS power kernels (csrc/loudness.cuh).

  * compute_loudness forward and backward at B = 128, N = 64000, 16 kHz, 250
    frames/s ('center'), with n_fft = 2048 (SpectralLoss's loudness term) and 512
    (the preprocessors' default), alternated in the same run with float32 torch
    autograd of the framing + rfft + A-weighting composition;
  * SpectralLoss forward + backward (ae.gin: mag + logmag, L1) with and without
    loudness_weight = 1 at B = 128;
  * compute_power at B = 256, N = 64000, frame_size 64 and 1024.

  python tools/loudness_time.py [--iters 20] [--rounds 3] [--out FILE]

Times are CUDA events after warm-up, the median of `rounds` alternated rounds.
FLOP counts come from shapes: per frame a complex FFT of M = n_fft / 2 points
(5 M log2 M), the split step and weighted power (~12 (M + 1)) and the window
(2 n_fft); the backward is counted as two transforms plus 30 M + 4 n_fft, and does
(n_fft - hop + own) / own times that work because each CTA recomputes its halo
frames (own = max(4096, n_fft) samples per CTA).  Algorithmic bytes: the audio once,
the output once (and the upstream gradient / d audio in the backward).  Share of peak
is against the H100 SXM data sheet (67 TFLOP/s FP32, 3.35 TB/s); the kernels are
bound by neither: their radix-2 stages run out of shared memory.  Prints the card
name and power limit read in the same run."""
import argparse
import json
import math
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import losses, spectral_ops  # noqa: E402
from tools import measure  # noqa: E402

DEV = 'cuda'


def torch_loudness(audio, n_fft, hop=64, sample_rate=16000):
  """The reference's composition in float32 torch ops (autograd-able)."""
  x = torch.nn.functional.pad(audio, (n_fft // 2, n_fft // 2))
  frames = x.unfold(-1, n_fft, hop)
  window = spectral_ops._hann(n_fft, audio.device)
  spec = torch.fft.rfft(frames * window, dim=-1)
  power = spec.real ** 2 + spec.imag ** 2
  weighted = (power * spectral_ops.a_weighting(sample_rate, n_fft, audio.device)).mean(-1)
  db = 10.0 * torch.log10(torch.maximum(weighted, torch.full_like(weighted, 1e-8)))
  return torch.maximum(db, torch.full_like(db, -80.0))


def _flops(n_frames, n_fft, backward, n=64000, hop=64):
  m = n_fft // 2
  fft = 5.0 * m * math.log2(max(m, 2))
  if not backward:
    return n_frames * (fft + 12.0 * (m + 1) + 2.0 * n_fft)
  own = max(4096, n_fft)
  recompute = (n_fft - hop + own) / own
  return n_frames * recompute * (2 * fft + 30.0 * m + 4.0 * n_fft)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('loudness_time.py')
  torch.backends.cuda.matmul.allow_tf32 = False
  res = {'card': measure.card(), 'rows': []}
  gen = torch.Generator(DEV).manual_seed(0)
  B, N = 128, 64000
  audio = torch.rand((B, N), device=DEV, generator=gen) * 2 - 1
  for n_fft in (2048, 512):
    T = spectral_ops.get_framed_lengths(N, n_fft, 64, 'center')[0]
    g = torch.randn((B, T), device=DEV, generator=gen)
    a = audio.clone().requires_grad_(True)

    def ours_fwd():
      with torch.no_grad():
        spectral_ops.compute_loudness(audio, n_fft=n_fft)

    def ours_fb():
      a.grad = None
      spectral_ops.compute_loudness(a, n_fft=n_fft).backward(g)

    def torch_fwd():
      with torch.no_grad():
        torch_loudness(audio, n_fft)

    def torch_fb():
      a.grad = None
      torch_loudness(a, n_fft).backward(g)

    few = max(2, args.iters // 4)
    runs = (('ours_fwd', ours_fwd, args.iters), ('torch_fwd', torch_fwd, few),
            ('ours_fwd_bwd', ours_fb, args.iters), ('torch_fwd_bwd', torch_fb, few))
    times = {k: [] for k, _, _ in runs}
    for _ in range(args.rounds):     # alternated rounds, each kept for the spread
      for k, fn, n in runs:
        times[k].append(measure.event_ms(fn, n, 3))
    t = {k: statistics.median(v) * 1e-3 for k, v in times.items()}
    t_bwd = t['ours_fwd_bwd'] - t['ours_fwd']
    f_fwd, f_bwd = _flops(B * T, n_fft, False), _flops(B * T, n_fft, True)
    bytes_fwd, bytes_bwd = 4.0 * (B * N + B * T), 4.0 * (2 * B * N + B * T)
    fp32, hbm = measure.FP32_FLOPS_PER_S, measure.HBM_BYTES_PER_S
    row = {'what': 'loudness', 'B': B, 'N': N, 'n_fft': n_fft, 'frames': B * T,
           'fwd_ms': t['ours_fwd'] * 1e3, 'bwd_ms': t_bwd * 1e3,
           'fwd_bwd_ms': t['ours_fwd_bwd'] * 1e3,
           'torch_fwd_ms': t['torch_fwd'] * 1e3, 'torch_fwd_bwd_ms': t['torch_fwd_bwd'] * 1e3,
           'fwd_tflops': f_fwd / t['ours_fwd'] / 1e12, 'bwd_tflops': f_bwd / t_bwd / 1e12,
           'fwd_share_of_peak': max(f_fwd / fp32, bytes_fwd / hbm) / t['ours_fwd'],
           'bwd_share_of_peak': max(f_bwd / fp32, bytes_bwd / hbm) / t_bwd,
           'bound': 'FP32' if f_fwd / fp32 > bytes_fwd / hbm else 'HBM',
           'spread_fwd_ms': [round(x, 4) for x in times['ours_fwd']]}
    res['rows'].append(row)
    print(json.dumps(row), flush=True)
    del a, g
    torch.cuda.empty_cache()

  target = torch.rand((B, N), device=DEV, generator=gen) * 2 - 1
  a = audio.clone().requires_grad_(True)
  for lw in (0.0, 1.0):
    loss_obj = losses.SpectralLoss(mag_weight=1.0, logmag_weight=1.0, loudness_weight=lw)

    def step():
      a.grad = None
      loss_obj(target, a).backward()
    ts = [measure.event_ms(step, max(2, args.iters // 2), 3) for _ in range(args.rounds)]
    row = {'what': 'spectral_loss_fwd_bwd', 'B': B, 'N': N, 'loudness_weight': lw,
           'ms': statistics.median(ts), 'spread_ms': [round(x, 4) for x in ts]}
    res['rows'].append(row)
    print(json.dumps(row), flush=True)
  del a, target
  torch.cuda.empty_cache()

  B2 = 256
  audio2 = torch.rand((B2, N), device=DEV, generator=gen) * 2 - 1
  for frame in (64, 1024):
    ts = [measure.event_ms(lambda: spectral_ops.compute_power(audio2, frame_size=frame),
                           args.iters, 3) for _ in range(args.rounds)]
    T = spectral_ops.get_framed_lengths(N, frame, 64, 'center')[0]
    t = statistics.median(ts) * 1e-3
    nbytes = 4.0 * (B2 * N + B2 * T)
    row = {'what': 'rms_power', 'B': B2, 'N': N, 'frame_size': frame, 'ms': t * 1e3,
           'hbm_share': nbytes / measure.HBM_BYTES_PER_S / t, 'flops': 2.0 * B2 * T * frame,
           'fp32_share': 2.0 * B2 * T * frame / measure.FP32_FLOPS_PER_S / t}
    res['rows'].append(row)
    print(json.dumps(row), flush=True)
  print(json.dumps(res['card']))
  if args.out:
    measure.append_rows(args.out, [res])


if __name__ == '__main__':
  main()
