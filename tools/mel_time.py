"""Time of the mel / log-mel / MFCC kernels (csrc/mel.cuh).

At B = 128, N = 64000, 16 kHz, three configurations:
  * mfcc:   the ae.gin encoder's compute_mfcc (fft_size 1024, overlap 0.5, 128 mel
            bins -> 30 coefficients, 20-8000 Hz);
  * logmel: the ICML-2020 pretraining encoder's compute_logmel (2048, 0.75, 229 bins,
            0-8000 Hz);
  * mel:    compute_mel's defaults (2048, 0.75, 64 bins, 0-8000 Hz);
forward and forward + backward, alternated in the same run with a float32 torch
composition (unfold + Hann + torch.fft.rfft (cuFFT) + abs + dense matmul + safe_log
+ DCT matmul, TF32 off).

  python tools/mel_time.py [--iters 20] [--rounds 3] [--out FILE]

Times are CUDA events after warm-up, the median of `rounds` alternated rounds.  FLOP
counts come from shapes: per frame a complex FFT of M = L / 2 points (5 M log2 M), the
window (L), magnitudes (~12 (M + 1)), the sparse projection (2 x 2 (M + 1)) and the DCT
(2 bins C).  The backward is counted as the forward plus an inverse transform, the
projection's transpose and the DCT's, 4 L more, times (fft_size - hop + own) / own for
the halo frames each CTA recomputes (own = max(4096, fft_size)).  Prints the card name
and power limit read in the same run."""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import spectral_ops  # noqa: E402
from tools import measure  # noqa: E402

DEV = 'cuda'
CONFIGS = [
    ('mfcc', 'compute_mfcc', dict(lo_hz=20.0, hi_hz=8000.0, fft_size=1024, mel_bins=128,
                                  mfcc_bins=30, overlap=0.5)),
    ('logmel', 'compute_logmel', dict(lo_hz=0.0, hi_hz=8000.0, bins=229, fft_size=2048,
                                      overlap=0.75)),
    ('mel', 'compute_mel', dict()),
]


def _params(fn, kw):
  a = dict(fft_size=2048, overlap=0.75, bins=64, lo_hz=0.0, hi_hz=8000.0)
  if fn == 'compute_mfcc':
    a.update(bins=kw['mel_bins'], n_out=kw['mfcc_bins'])
  a.update({k: v for k, v in kw.items() if k not in ('mel_bins', 'mfcc_bins')})
  a.setdefault('n_out', a['bins'])
  return a


def torch_features(audio, fn, p, sample_rate=16000):
  """The reference's composition in float32 torch ops (autograd-able)."""
  fft_size, hop = p['fft_size'], int(p['fft_size'] * (1.0 - p['overlap']))
  fft_length = 1 << (fft_size - 1).bit_length()
  n = audio.shape[-1]
  n_frames = -(-n // hop)
  x = torch.nn.functional.pad(audio, (0, (n_frames - 1) * hop + fft_size - n))
  frames = x.unfold(-1, fft_size, hop)
  mag = torch.fft.rfft(frames * spectral_ops._hann(fft_size, audio.device), n=fft_length,
                       dim=-1).abs()
  key = ('w', p['bins'], fft_length, p['lo_hz'], p['hi_hz'])
  if key not in _CACHE:
    _CACHE[key] = torch.as_tensor(spectral_ops.linear_to_mel_weight_matrix(
        p['bins'], fft_length // 2 + 1, sample_rate, p['lo_hz'], p['hi_hz']),
        dtype=torch.float32, device=audio.device)
  mel = mag @ _CACHE[key]
  if fn == 'compute_mel':
    return mel
  logmel = spectral_ops.safe_log(mel)
  if fn == 'compute_logmel':
    return logmel
  key = ('dct', p['bins'], p['n_out'])
  if key not in _CACHE:
    b = p['bins']
    nn = torch.arange(b, dtype=torch.float64)[:, None]
    k = torch.arange(p['n_out'], dtype=torch.float64)[None, :]
    _CACHE[key] = (2.0 * torch.cos(math.pi * k * (2 * nn + 1) / (2 * b)) /
                   math.sqrt(2.0 * b)).float().to(audio.device)
  return logmel @ _CACHE[key]


_CACHE = {}


def _flops(p, n_frames, backward, n=64000):
  fft_size, hop = p['fft_size'], int(p['fft_size'] * (1.0 - p['overlap']))
  L = 1 << (fft_size - 1).bit_length()
  m = L // 2
  fwd = 5.0 * m * math.log2(max(m, 2)) + L + 12.0 * (m + 1) + 4.0 * (m + 1) + \
      2.0 * p['bins'] * p['n_out']
  if not backward:
    return n_frames * fwd
  own = max(4096, fft_size)
  recompute = (fft_size - hop + own) / own
  per = 2 * fwd + 12.0 * (m + 1) + 4.0 * L
  return n_frames * (fwd + recompute * per)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('mel_time.py')
  torch.backends.cuda.matmul.allow_tf32 = False
  res = {'card': measure.card(), 'B': 128, 'N': 64000, 'rows': []}
  gen = torch.Generator(DEV).manual_seed(0)
  B, N = 128, 64000
  audio = torch.rand((B, N), device=DEV, generator=gen) * 2 - 1
  for name, fn, kw in CONFIGS:
    p = _params(fn, kw)
    feat = getattr(spectral_ops, fn)
    out = feat(audio, **kw)
    ref = torch_features(audio, fn, p)
    assert out.shape == ref.shape, (out.shape, ref.shape)
    g = torch.randn(out.shape, device=DEV, generator=gen)
    a = audio.clone().requires_grad_(True)

    def ours_fwd():
      with torch.no_grad():
        feat(audio, **kw)

    def ours_fb():
      a.grad = None
      feat(a, **kw).backward(g)

    def torch_fwd():
      with torch.no_grad():
        torch_features(audio, fn, p)

    def torch_fb():
      a.grad = None
      torch_features(a, fn, p).backward(g)

    t = measure.alternate({'ours_fwd': ours_fwd, 'torch_fwd': torch_fwd, 'ours_fb': ours_fb,
                           'torch_fb': torch_fb}, args.rounds, args.iters, 3)
    T = out.shape[1]
    ffw, ffb = _flops(p, B * T, False), _flops(p, B * T, True)
    row = {'config': name, 'fn': fn, 'kwargs': kw, 'frames': T,
           'ours_fwd_ms': t['ours_fwd'], 'ours_fwd_bwd_ms': t['ours_fb'],
           'torch_fwd_ms': t['torch_fwd'], 'torch_fwd_bwd_ms': t['torch_fb'],
           'fwd_gflop': ffw / 1e9, 'fwd_bwd_gflop': ffb / 1e9,
           'fwd_fp32_share': ffw / (t['ours_fwd'] * 1e-3) / measure.FP32_FLOPS_PER_S,
           'fwd_bwd_fp32_share': ffb / (t['ours_fb'] * 1e-3) / measure.FP32_FLOPS_PER_S,
           'max_abs_vs_torch': float((out - ref).abs().max())}
    res['rows'].append(row)
    print(json.dumps(row), flush=True)
  print(json.dumps({'card': res['card']}))
  if args.out:
    measure.append_rows(args.out, [res])


if __name__ == '__main__':
  main()
