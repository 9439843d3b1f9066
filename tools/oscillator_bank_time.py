"""Times `core.oscillator_bank` on audio-rate envelopes [B, N, K]: the forward, the
backward with both gradients (`ddsp_b200_oscillator_bank_backward`, d f and d a), the
backward with d a only, and float32 torch autograd of the reference formulation
(`where`, `cumsum`, `sin`, `sum`) on the same inputs; and `core.angular_cumsum` with its
backward.  Shapes: B = 32, N = 64000, K = 100 with both `sum_sinusoids` values,
B = 4, N = 64000, K = 16, and angular_cumsum at [32, 64000, 100].

Each timed call takes the next input set of a ring larger than twice the L2 cache, so
no call finds its operands in L2.  CUDA events; the backward is timed as a direct call
of the entry point on saved inputs (no forward inside).  Prints the card name and power
limit read in the same run, and the time against the byte floor of the backward (f and
a read once, d f and d a written once) at 3.35 TB/s.

  python tools/oscillator_bank_time.py [--iters 20] [--out FILE]"""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import core  # noqa: E402
from tools import measure  # noqa: E402


def _torch_reference(f, a, sr, sum_sinusoids):
  amp = torch.where(f >= sr / 2.0, torch.zeros_like(a), a)
  out = amp * torch.sin(torch.cumsum(f * (2.0 * math.pi / sr), dim=1))
  return out.sum(-1) if sum_sinusoids else out


def _bank(B, N, K, sum_sinusoids, iters, sr=16000.0):
  gen = torch.Generator(device='cuda').manual_seed(B * K + sum_sinusoids)
  g_shape = (B, N) if sum_sinusoids else (B, N, K)
  set_bytes = 4 * (2 * B * N * K + math.prod(g_shape))
  n = measure.ring_len(set_bytes)
  fs = [torch.rand(B, N, K, device='cuda', generator=gen) * 7900 + 20 for _ in range(n)]
  as_ = [torch.rand(B, N, K, device='cuda', generator=gen) * 0.05 for _ in range(n)]
  gs = [torch.randn(g_shape, device='cuda', generator=gen) for _ in range(n)]
  df, da = torch.empty_like(fs[0]), torch.empty_like(fs[0])

  def fwd(i):
    return core.oscillator_bank(fs[i], as_[i], sample_rate=sr, sum_sinusoids=sum_sinusoids)

  def bwd(i, want_df=True):
    core._launch('ddsp_b200_oscillator_bank_backward', fs[i], as_[i], gs[i],
                 df if want_df else None, da, B, N, K, sr, int(sum_sinusoids))

  leaves = [(f.clone().requires_grad_(True), a.clone().requires_grad_(True))
            for f, a in zip(fs[:1], as_[:1])]

  def torch_fwd_bwd():
    f, a = leaves[0]
    f.grad = a.grad = None
    _torch_reference(f, a, sr, sum_sinusoids).backward(gs[0])

  ring = range(n)
  t_f = measure.event_ms(fwd, iters, 2 * n, ring)
  t_b = measure.event_ms(bwd, iters, 2 * n, ring)
  t_ba = measure.event_ms(lambda i: bwd(i, False), iters, 2 * n, ring)
  t_torch_f = measure.event_ms(lambda i: _torch_reference(fs[i], as_[i], sr, sum_sinusoids),
                               3, n, ring)
  t_torch = measure.event_ms(torch_fwd_bwd, 3, 1)
  floor = 4 * 4 * B * N * K / measure.HBM_BYTES_PER_S * 1e3
  row = dict(B=B, N=N, K=K, sum_sinusoids=sum_sinusoids, ring=n, forward_ms=t_f,
             backward_ms=t_b, backward_da_only_ms=t_ba, torch_forward_ms=t_torch_f,
             torch_fwd_bwd_ms=t_torch, byte_floor_ms=floor)
  print('B=%d N=%d K=%d sum_sinusoids=%d (ring of %d input sets)' % (B, N, K, sum_sinusoids, n))
  print('  forward                                 %8.3f ms' % t_f)
  print('  backward, d f and d a                   %8.3f ms = %.2fx forward, %.2fx the %.3f ms '
        'byte floor' % (t_b, t_b / t_f, t_b / floor, floor))
  print('  backward, d a only                      %8.3f ms = %.2fx forward' % (t_ba, t_ba / t_f))
  print('  float32 torch forward                   %8.3f ms' % t_torch_f)
  print('  float32 torch autograd forward+backward %8.3f ms (ours: %.3f ms, %.1fx faster)'
        % (t_torch, t_f + t_b, t_torch / (t_f + t_b)), flush=True)
  del fs, as_, gs, df, da, leaves
  torch.cuda.empty_cache()
  return row


def _cumsum(B, N, C, iters):
  gen = torch.Generator(device='cuda').manual_seed(5)
  n = measure.ring_len(4 * 2 * B * N * C)
  xs = [torch.rand(B, N, C, device='cuda', generator=gen) * 0.5 for _ in range(n)]
  gs = [torch.randn(B, N, C, device='cuda', generator=gen) for _ in range(n)]
  d = torch.empty_like(xs[0])
  x_leaf = xs[0].clone().requires_grad_(True)

  def torch_fwd_bwd():
    x_leaf.grad = None
    torch.remainder(torch.cumsum(x_leaf, 1), 2 * math.pi).backward(gs[0])

  t_f = measure.event_ms(lambda i: core.angular_cumsum(xs[i]), iters, 2 * n, range(n))
  t_b = measure.event_ms(
      lambda i: core._launch('ddsp_b200_angular_cumsum_backward', gs[i], d, B, N, C),
      iters, 2 * n, range(n))
  t_torch = measure.event_ms(torch_fwd_bwd, 3, 1)
  floor = 2 * 4 * B * N * C / measure.HBM_BYTES_PER_S * 1e3
  print('angular_cumsum [%d, %d, %d] (ring of %d)' % (B, N, C, n))
  print('  forward %8.3f ms   backward %8.3f ms = %.2fx the %.3f ms byte floor   float32 '
        'torch autograd forward+backward %8.3f ms' % (t_f, t_b, t_b / floor, floor, t_torch),
        flush=True)
  del xs, gs, d, x_leaf
  torch.cuda.empty_cache()
  return dict(op='angular_cumsum', B=B, N=N, C=C, ring=n, forward_ms=t_f, backward_ms=t_b,
              torch_fwd_bwd_ms=t_torch, byte_floor_ms=floor)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--out', default=None, help='also append the rows as one JSON line')
  args = ap.parse_args()
  measure.require_cuda('oscillator_bank_time.py')
  card = measure.card()
  print(json.dumps(card), flush=True)
  rows = [_bank(32, 64000, 100, True, args.iters), _bank(32, 64000, 100, False, args.iters),
          _bank(4, 64000, 16, True, args.iters), _bank(4, 64000, 16, False, args.iters),
          _cumsum(32, 64000, 100, args.iters)]
  if args.out:
    measure.append_rows(args.out, [dict(card=card, rows=rows)])


if __name__ == '__main__':
  main()
