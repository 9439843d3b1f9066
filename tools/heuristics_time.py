"""Time of heuristics.midi_heuristic followed by heuristics.note_table (mean pick) on their
CUDA kernels (csrc/heuristics.cuh) against a float32 torch composition of the same steps
on the same GPU: unfold statistics for the pooled outliers and the strided test, and
run-length encoding by torch ops for remove_short and the note table.  Sizes:
B = 32, T = 1001 (4 s at 250 Hz) and B = 8, T = 15001 (60 s).

  python tools/heuristics_time.py [--iters 20] [--rounds 3] [--out FILE]
  python tools/heuristics_time.py --reference [--out FILE]   # CPU: the reference on the
                                                             # NumPy shim, per item

Times are CUDA events after warm-up, the median of `rounds` alternated rounds; each row
prints how many frames of the two masks and how many notes differ.  Prints the card name
and power limit read in the same run.  --reference times the unmodified reference's
segment_notes_batch(midi_heuristic, mean_f0, median_amps) on the CPU (it needs the
reference sources) and labels the line as CPU."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests.golden import make_heuristics_golden as mk  # noqa: E402
from tools import measure  # noqa: E402

SIZES = ((32, 1001), (8, 15001))


def _inputs(b, t):
  f0, amps = zip(*(mk.track(t, 100 + i) for i in range(b)))
  return np.stack(f0), np.stack(amps)


# ---- the composition in float32 torch ------------------------------------------------------
def _pad(torch, v, before, after):
  e0 = torch.trunc(v[:, :1]).expand(-1, before)
  e1 = torch.trunc(v[:, -1:]).expand(-1, after)
  return torch.cat([e0, v, e1], dim=1)


def torch_midi_heuristic(torch, f0, amps):
  la = torch.log(amps)
  w = _pad(torch, la, 40, 39).unfold(1, 80, 1)
  pooled = (w.mean(-1) - 2.0 * w.std(-1, unbiased=False)) < la
  ln2 = torch.log(torch.tensor(2.0, device=f0.device))
  midi = 12.0 * (torch.log(torch.where(f0 <= 0, torch.ones_like(f0), f0)) / ln2 -
                 torch.log(torch.tensor(440.0, device=f0.device)) / ln2) + 69.0
  midi = torch.where(f0 <= 0, torch.zeros_like(midi), midi)
  tr = torch.ones_like(f0, dtype=torch.bool)
  for width in (2, 4, 8, 16, 32):
    fr = _pad(torch, midi, width - 1, 0).unfold(1, width, 1)
    change = torch.abs(fr[..., 0] - fr[..., -1]) > 0.75
    allon = torch.cat([tr[:, :1].expand(-1, width - 1), tr], 1).unfold(1, width, 1).all(-1)
    tr = tr & ~(allon & change)
  on = tr & (f0 > 0) & pooled
  # remove_short(min_samples=10) by run-length encoding
  b, t = on.shape
  change = torch.ones_like(on)
  change[:, 1:] = on[:, 1:] != on[:, :-1]
  run = torch.cumsum(change.reshape(-1).to(torch.int64), 0) - 1
  length = torch.bincount(run)
  last = torch.zeros_like(length)
  last.scatter_reduce_(0, run, torch.arange(b * t, device=f0.device) % t, 'amax')
  short = (length[run] < 10) & (last[run] < t - 1)
  return on & ~short.reshape(b, t)


def torch_note_table(torch, mask, f0):
  b, t = mask.shape
  m = mask.to(torch.int8)
  d = torch.diff(torch.nn.functional.pad(m, (1, 1)), dim=1)
  sb, ss = torch.nonzero(d == 1, as_tuple=True)
  _, se = torch.nonzero(d == -1, as_tuple=True)
  csum = torch.nn.functional.pad(torch.cumsum(f0.to(torch.float64), 1), (1, 0))
  mean = ((csum[sb, se] - csum[sb, ss]) / (se - ss)).to(torch.float32)
  ln2 = torch.log(torch.tensor(2.0, device=f0.device))
  midi = 12.0 * (torch.log(mean) / ln2 - torch.log(torch.tensor(440.0, device=f0.device)) /
                 ln2) + 69.0
  pitch = torch.round(torch.where(mean <= 0, torch.zeros_like(midi), midi)).to(torch.int32)
  return sb, ss, se, pitch


def gpu(args):
  import torch
  measure.require_cuda('heuristics_time.py')
  from ddsp_b200 import heuristics as h
  rows = []
  for b, t in SIZES:
    f0, amps = _inputs(b, t)
    f0 = torch.as_tensor(f0, device='cuda')
    amps = torch.as_tensor(amps, device='cuda')
    c = {'f0_hz': f0, 'harmonic': {'controls': {'amplitudes': amps}}}
    f2, a2 = f0[..., 0].contiguous(), amps[..., 0].contiguous()

    def ours():
      return h.note_table(h.midi_heuristic(c), f0)

    def theirs():
      m = torch_midi_heuristic(torch, f2, a2)
      return m, torch_note_table(torch, m, f2)

    times = measure.alternate({'cuda_ms': ours, 'torch_ms': theirs}, args.rounds,
                              args.iters, 1)
    mine = h.midi_heuristic(c)
    table = h.note_table(mine, f0)
    m, (_, _, _, pitch) = theirs()
    row = dict(measure.card(), config=f'B={b} T={t}',
               what='midi_heuristic + note_table (mean)', **times,
               mask_frames_differ=int((mine != m).sum()),
               notes=int(table.count.sum()), torch_notes=int(pitch.numel()),
               iters=args.iters, rounds=args.rounds)
    print(json.dumps(row))
    rows.append(row)
  return rows


def reference(args):
  _, hr = mk._load()
  tf = mk.ref_on_shim.tf()
  rows = []
  for b, t in SIZES:
    f0, amps = _inputs(b, t)
    c = {'f0_hz': tf.constant(f0), 'harmonic': {'controls': {'amplitudes': amps}}}
    t0 = time.perf_counter()
    with np.errstate(all='ignore'):
      hr.segment_notes_batch(hr.midi_heuristic, hr.mean_f0, hr.median_amps, c)
    row = dict(device='CPU', config=f'B={b} T={t}',
               what='reference segment_notes_batch(midi_heuristic, mean_f0) on the NumPy shim',
               cpu_ms=(time.perf_counter() - t0) * 1e3)
    print(json.dumps(row))
    rows.append(row)
  return rows


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--reference', action='store_true')
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  rows = reference(args) if args.reference else gpu(args)
  if args.out:
    measure.append_rows(args.out, rows)


if __name__ == '__main__':
  main()
