"""Time of losses.wasserstein_distance on its CUDA kernels (csrc/wasserstein.cuh) against
a float32 torch composition of the reference formula.

Configurations (values in MIDI, amplitude weights, p = 1):
  * icml:   B = 32, T = 125 frames, 100 against 100 sinusoids (the ICML 2020
            self-supervised pitch model's size, as in tools/consistency_time.py);
  * long:   B = 256, T = 1000, 100 against 100;
  * wide:   B = 32, T = 125, 1024 against 1024.
Each is timed forward, and forward + backward, alternated in the same run with the
reference formula in float32 torch (torch.sort, searchsorted, gather, cumsum, with
autograd), whose peak memory (torch.cuda.max_memory_allocated above the inputs) is
reported too.  The largest |difference| of the two forwards is printed with each row.

  python tools/wasserstein_time.py [--iters 20] [--rounds 3] [--out FILE]

Times are CUDA events after warm-up, the median of `rounds` alternated rounds.  Prints
the card name and power limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import losses  # noqa: E402
from tools import measure  # noqa: E402

DEV = 'cuda'


# ---- the reference formula, float32 torch ----------------------------------------
def _cdf(values, weights, points):
  sorted_values, sorter = torch.sort(values, dim=-1)
  idx = torch.searchsorted(sorted_values, points.detach().contiguous(), right=True)
  cum = torch.cumsum(torch.gather(weights, -1, sorter), dim=-1)
  return torch.gather(torch.cat([torch.zeros_like(cum[..., :1]), cum], -1), -1, idx)


def ref_distance(u, v, wu, wv, p=1.0):
  s, _ = torch.sort(torch.cat([u, v], -1), dim=-1)
  deltas = s[..., 1:] - s[..., :-1]
  d = _cdf(u, wu, s[..., :-1]) - _cdf(v, wv, s[..., :-1])
  return torch.sum(deltas * torch.abs(d)**p, -1)**(1.0 / p)


# ---- inputs ----------------------------------------------------------------------
def _inputs(b, t, n, seed):
  rng = np.random.default_rng(seed)
  cast = lambda x: torch.as_tensor(x, dtype=torch.float32, device=DEV)
  u = cast(rng.uniform(30.0, 110.0, (b, t, n)))
  v = cast(rng.uniform(30.0, 110.0, (b, t, n)))
  wu = cast(rng.uniform(0.0, 1.0, (b, t, n)))
  wv = cast(rng.uniform(0.0, 1.0, (b, t, n)))
  return [u, v, wu, wv]


def _fwd_bwd(fn, inputs):
  def run():
    for x in inputs:
      x.grad = None
    fn(*inputs).sum().backward()
  return run


def configs():
  for name, (b, t, n) in (('icml', (32, 125, 100)), ('long', (256, 1000, 100)),
                          ('wide', (32, 125, 1024))):
    plain = _inputs(b, t, n, 7)
    grad = [x.clone().requires_grad_(True) for x in plain]
    yield (name + '_forward', lambda x=plain: losses.wasserstein_distance(*x),
           lambda x=plain: ref_distance(*x), plain)
    yield (name + '_forward_backward', _fwd_bwd(losses.wasserstein_distance, grad),
           _fwd_bwd(ref_distance, grad), plain)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('wasserstein_time.py')
  card = measure.card()
  rows = []
  for name, ours, theirs, plain in configs():
    with torch.no_grad():
      a, b = losses.wasserstein_distance(*plain), ref_distance(*plain)
      diff = float(torch.max(torch.abs(a - b)))
      scale = float(torch.max(torch.abs(b)))
    t = measure.alternate({'ms': ours, 'torch_ms': theirs}, args.rounds, args.iters, 3)
    torch.cuda.empty_cache()
    row = {'config': name, **t, 'peak_mb': measure.peak_bytes(ours) / 2**20,
           'torch_peak_mb': measure.peak_bytes(theirs) / 2**20,
           'max_abs_diff': diff, 'max_abs_value': scale, 'rows': int(plain[0][..., 0].numel())}
    row['speedup'] = row['torch_ms'] / row['ms']
    row.update(card)
    rows.append(row)
    print(json.dumps(row), flush=True)
    torch.cuda.empty_cache()
  if args.out:
    measure.append_rows(args.out, rows)


if __name__ == '__main__':
  main()
