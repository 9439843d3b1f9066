"""Time of nn.get_note_mask followed by nn.pool_over_notes on their CUDA kernels
(csrc/notes.cuh) against the reference's formulas as float32 torch ops on the same GPU,
at the MIDI autoencoder's size (z_midiae.gin): B = 32, T = 1000 frames,
max_regions = 100, z_dims = 128.

Rows, each alternated in the same run with the torch restatement:
  * forward:          get_note_mask(q) then pool_over_notes(z, mask) (mean and std);
  * forward+backward: the same with a loss on the pooled mean, backward to z.
The torch formulas build the reference's [B, T, R, D] products; their peak memory
(torch.cuda.max_memory_allocated above the inputs) is reported beside the kernels'.  The
largest |difference| of the two pooled means is printed with each row.

  python tools/notes_time.py [--iters 20] [--rounds 3] [--out FILE]

Times are CUDA events after warm-up, the median of `rounds` alternated rounds.  Prints
the card name and power limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import nn  # noqa: E402
from tools import measure  # noqa: E402

DEV = 'cuda'
B, T, R, D = 32, 1000, 100, 128


# ---- the reference's formulas (training/nn.py:375-547) in float32 torch ----------------
def _safe_divide(a, b):
  return a / torch.where(b == 0.0, torch.full_like(b, 1e-7), b)


def _moments(x, m):
  md = m[..., None]
  lengths = md.sum(1)
  mean = _safe_divide((x[:, :, None, :] * md).sum(1), lengths)
  num = (((x[:, :, None, :] - mean[:, None]) * md)**2.0).sum(1)
  return mean, _safe_divide(num, lengths)**0.5


def torch_mask(q, r=R):
  edges = torch.abs(q[:, 1:] - q[:, :-1]) > 0
  edges = torch.cat([torch.ones_like(edges[:, :1]), edges[:, :-1],
                     torch.zeros_like(edges[:, :1])], dim=1)
  idx = torch.cumsum(edges.to(torch.int32), dim=1) - 1
  mask = (idx[..., None] == torch.arange(r, device=q.device)).to(torch.float32)
  pitches = _moments(q[:, :, None], mask)[0][..., 0]
  return mask * (pitches > 0.0).to(torch.float32)[:, None, :]


def torch_pool(z, m):
  mean, std = _moments(z, m)
  return (mean[:, None] * m[..., None]).sum(2), (std[:, None] * m[..., None]).sum(2)


def _inputs(seed=0):
  rng = np.random.default_rng(seed)
  q = np.zeros((B, T), np.float32)
  for i in range(B):
    k = 0
    while k < T:
      n = 1 + int(rng.exponential(15.0))
      q[i, k:k + n] = rng.integers(-10, 80) if rng.uniform() < 0.7 else 0.0
      k += n
  z = rng.normal(size=(B, T, D)).astype(np.float32)
  return torch.as_tensor(q, device=DEV), torch.as_tensor(z, device=DEV)


def _run(mask_fn, pool_fn, q, z, w, backward):
  zz = z.detach().requires_grad_(backward)
  mean, _ = pool_fn(zz, mask_fn(q))
  if backward:
    (mean * w).sum().backward()
  return mean


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--out', default=None)
  a = ap.parse_args()
  measure.require_cuda('notes_time.py')
  card = measure.card()
  q, z = _inputs()
  w = torch.randn((B, T, D), device=DEV)
  ours = (lambda x: nn.get_note_mask(x, R), nn.pool_over_notes)
  ref = (torch_mask, torch_pool)
  rows = []
  for backward in (False, True):
    fns = {name: (lambda f=f: _run(*f, q, z, w, backward)) for name, f in
           (('cuda', ours), ('torch', ref))}
    diff = float((fns['cuda']().detach() - fns['torch']().detach()).abs().max())
    t = measure.alternate(fns, a.rounds, a.iters, 1)
    row = dict(card, config=f'B={B} T={T} R={R} D={D}',
               what='forward+backward' if backward else 'forward',
               cuda_ms=t['cuda'], torch_ms=t['torch'],
               cuda_peak_bytes=measure.peak_bytes(fns['cuda']),
               torch_peak_bytes=measure.peak_bytes(fns['torch']),
               max_abs_diff_pooled_mean=diff, iters=a.iters, rounds=a.rounds)
    rows.append(row)
    print(json.dumps(row), flush=True)
  if a.out:
    measure.append_rows(a.out, rows)


if __name__ == '__main__':
  main()
