"""Times `core.harmonic_oscillator_bank` at B = 32, N = 64000, K = 64, and at two shapes
that expose its scaling (B = 1, N = 10^6, K = 1: one backward cluster per item and the
forward's re-read of f dominate; B = 1, N = 64000, K = 64): the forward, the backward with
every gradient (`ddsp_b200_harmonic_oscillator_bank_backward`: d f, d a,
d initial_phase, with an upstream gradient on the final phase), the backward with d a
only, and float32 torch autograd of the reference formulation (`cumsum`, `remainder`,
`sin` of the [B, N, K] phases, `sum`) on the same inputs.

Each timed call takes the next input set of a ring larger than twice the L2 cache, so
no call finds its operands in L2.  CUDA events; the backward is timed as a direct call
of the entry point on saved inputs.  Prints the card name and power limit read in the
same run, and each time beside the floor of its bytes at 3.35 TB/s (forward: f and a
read once, audio written; backward: a read, d a written, f, g and d f once).  Both
directions are timed as direct calls of the entry points on preallocated outputs.  The
torch side runs at the first shape only.

  python tools/harmonic_oscillator_bank_time.py [--iters 20] [--out FILE]"""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import core  # noqa: E402
from tools import measure  # noqa: E402


def _torch_reference(f, a, init, sr):
  phases = torch.remainder(torch.cumsum(f * (2.0 * math.pi / sr), dim=1), 2.0 * math.pi) + init
  k = torch.arange(1, a.shape[-1] + 1, dtype=a.dtype, device=a.device)
  return (a * torch.sin(phases * k)).sum(-1), phases[:, -1:, 0:1]


def _shape(B, N, K, iters, with_torch, sr=16000.0):
  gen = torch.Generator(device='cuda').manual_seed(B * K)
  n = measure.ring_len(4 * (2 * B * N * K + 3 * B * N))
  fs = [torch.rand(B, N, 1, device='cuda', generator=gen) * 600 + 60 for _ in range(n)]
  as_ = [torch.rand(B, N, K, device='cuda', generator=gen) * 0.05 for _ in range(n)]
  ps = [torch.rand(B, 1, 1, device='cuda', generator=gen) * 6 for _ in range(n)]
  gs = [torch.randn(B, N, device='cuda', generator=gen) for _ in range(n)]
  gp = torch.ones(B, 1, 1, device='cuda')
  audio, final = torch.empty(B, N, device='cuda'), torch.empty(B, 1, 1, device='cuda')
  df, da, dp = torch.empty(B, N, 1, device='cuda'), torch.empty(B, N, K, device='cuda'), \
      torch.empty(B, 1, 1, device='cuda')

  def fwd(i):
    core._launch('ddsp_b200_harmonic_oscillator_bank', fs[i], as_[i], ps[i], audio, final,
                 B, N, K, sr, 1)

  def bwd(i, all_grads=True):
    core._launch('ddsp_b200_harmonic_oscillator_bank_backward', fs[i], as_[i], ps[i], gs[i],
                 gp, df if all_grads else None, da, dp if all_grads else None, B, N, K, sr)

  def torch_train(i):
    f, a, p = (x.clone().requires_grad_() for x in (fs[i], as_[i], ps[i]))
    out, fin = _torch_reference(f, a, p, sr)
    ((out * gs[i]).sum() + fin.sum()).backward()

  ring, few = range(n), max(3, iters // 4)
  res = {'shape': [B, N, K]}
  res['forward_ms'] = measure.event_ms(fwd, iters, 2 * n, ring)
  res['backward_ms'] = measure.event_ms(bwd, iters, 2 * n, ring)
  res['backward_da_only_ms'] = measure.event_ms(lambda i: bwd(i, False), iters, 2 * n, ring)
  if with_torch:
    res['torch_forward_ms'] = measure.event_ms(
        lambda i: _torch_reference(fs[i], as_[i], ps[i], sr), few, 2 * n, ring)
    res['torch_forward_backward_ms'] = measure.event_ms(torch_train, few, 2 * n, ring)
  res['forward_floor_ms'] = 4 * (B * N * K + 2 * B * N) / measure.HBM_BYTES_PER_S * 1e3
  res['backward_floor_ms'] = 4 * (2 * B * N * K + 3 * B * N) / measure.HBM_BYTES_PER_S * 1e3
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('harmonic_oscillator_bank_time.py')
  res = {'card': measure.card(),
         'shapes': [_shape(32, 64000, 64, args.iters, True),
                    _shape(1, 1000000, 1, args.iters, False),
                    _shape(1, 64000, 64, args.iters, False)]}
  print(json.dumps(res))
  if args.out:
    measure.append_rows(args.out, [res])


if __name__ == '__main__':
  main()
