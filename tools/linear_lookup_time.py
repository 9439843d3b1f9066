"""Times `core.linear_lookup` forward and backward (d phase and d wavetables) with
per-item tables [B, W] (B = 32, N = 64000, W = 2048) and per-sample tables [B, N, W]
(B = 4, N = 16000, W = 512), and float32 torch autograd of the reference formulation
([B, N, W + 1] distances, relu weights, sum).  The torch side of the per-item case runs
on the first N / 16 samples (its [B, N, W + 1] intermediates would otherwise take tens of
GB) and its time is reported scaled by 16, marked as such.

Each timed call takes the next input set of a ring larger than twice the L2 cache.  CUDA
events; both directions are timed as direct calls of the entry points on preallocated
outputs, without the Python wrapper.  Prints the card name and power limit read in the
same run, and each time beside the floor of the bytes it must move at 3.35 TB/s:
forward, phase read and out written, plus one 32-byte sector of each per-sample table
row (the at most two columns read); backward, phase and g read and d phase written, plus
the table gradient written once (per item: B W floats; per sample: the whole [B, N, W]).

  python tools/linear_lookup_time.py [--iters 20] [--out FILE]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import core  # noqa: E402
from tools import measure  # noqa: E402


def _torch_reference(phase, tab):
  if tab.dim() == 2:
    tab = tab[:, None, :]
  w = tab.shape[-1]
  tab = torch.cat([tab, tab[..., :1]], -1)
  lin = torch.linspace(0.0, 1.0, w + 1, device=phase.device)
  weights = torch.relu(1.0 - torch.abs(phase[..., None] - lin) * w)
  return (weights * tab).sum(-1)


def _case(B, N, W, per_sample, iters):
  gen = torch.Generator(device='cuda').manual_seed(W)
  tshape = (B, N, W) if per_sample else (B, W)
  n = measure.ring_len(4 * (3 * B * N + 2 * B * (N if per_sample else 1) * W))
  ph = [torch.rand(B, N, device='cuda', generator=gen) for _ in range(n)]
  tabs = [torch.randn(tshape, device='cuda', generator=gen) for _ in range(n)]
  gs = [torch.randn(B, N, device='cuda', generator=gen) for _ in range(n)]
  dp, dt = torch.empty(B, N, device='cuda'), torch.empty(tshape, device='cuda')
  out = torch.empty(B, N, device='cuda')
  nt = N if per_sample else N // 16         # samples of the torch side
  scale = N / nt

  def fwd(i):
    core._launch('ddsp_b200_linear_lookup_forward', ph[i], tabs[i], out, B, N, W,
                 int(per_sample))

  def bwd(i):
    core._launch('ddsp_b200_linear_lookup_backward', ph[i], tabs[i], gs[i], dp, dt, B, N, W,
                 int(per_sample))

  def torch_tab(i):
    return tabs[i][:, :nt] if per_sample else tabs[i]

  def torch_train(i):
    p, t = ph[i][:, :nt].clone().requires_grad_(), torch_tab(i).clone().requires_grad_()
    (_torch_reference(p, t) * gs[i][:, :nt]).sum().backward()

  tab_bytes = 4 * B * (N if per_sample else 1) * W
  ring, few = range(n), max(3, iters // 4)
  res = {'tables': list(tshape)}
  res['forward_ms'] = measure.event_ms(fwd, iters, 2 * n, ring)
  res['backward_ms'] = measure.event_ms(bwd, iters, 2 * n, ring)
  res['torch_forward_ms'] = scale * measure.event_ms(
      lambda i: _torch_reference(ph[i][:, :nt], torch_tab(i)), few, 2 * n, ring)
  res['torch_forward_backward_ms'] = scale * measure.event_ms(torch_train, few, 2 * n, ring)
  if scale != 1:
    res['torch_note'] = 'torch run on %d samples per item, times scaled by %g' % (nt, scale)
  res['forward_floor_ms'] = ((8 * B * N + (32 * B * N if per_sample else 0)) /
                             measure.HBM_BYTES_PER_S * 1e3)
  res['backward_floor_ms'] = (12 * B * N + tab_bytes) / measure.HBM_BYTES_PER_S * 1e3
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('linear_lookup_time.py')
  res = {'card': measure.card(), 'per_item': _case(32, 64000, 2048, False, args.iters),
         'per_sample': _case(4, 16000, 512, True, args.iters)}
  print(json.dumps(res))
  if args.out:
    measure.append_rows(args.out, [res])


if __name__ == '__main__':
  main()
