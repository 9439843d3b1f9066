"""Time of the wavetable kernels (csrc/wavetable.cuh) at B = 32 and 256, F = 1000,
N = 64000: time-varying [B, F, W] tables at W = 1024 and 2048, and a static
[B, 2048] table.  Per shape: the forward, the backward with and without d f0 (all
three gradients / d amplitudes and d wavetables), the backward split into its two
halves (d f0 + d amplitudes: phase passes, frame sums and finalize; d wavetables:
phase passes, scatter and segment reduce), and forward + backward through
`core.wavetable_synthesis`.  Then float32 torch autograd of the reference
formulation (tables resampled to N, [B, N, W + 1] distance and weight tensors) at
the largest B of 1, 2, 4, 8 that fits.

  python tools/wavetable_time.py [--iters 30] [--warmup 5] [--out FILE]

Kernel times are CUDA events over a ring of input sets larger than twice the L2.
Algorithmic bytes, as a share of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s):
forward reads the tables once (4 B F W) and writes the audio (4 B N); the backward
reads the tables and the upstream gradient and writes d wavetables (8 B F W + 4 B N).
Prints the card name and power limit read in the same run."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import _lib  # noqa: E402
from ddsp_b200 import core  # noqa: E402
from tools import measure  # noqa: E402


def _sets(B, F, Fw, W, N, dev):
  n = measure.ring_len(4 * (B * Fw * W + 3 * B * F + B * N))
  g = torch.Generator(dev).manual_seed(0)
  out = []
  for _ in range(n):
    out.append((50.0 + 1000.0 * torch.rand((B, F), device=dev, generator=g),
                torch.rand((B, F), device=dev, generator=g),
                torch.randn((B, Fw, W), device=dev, generator=g),
                torch.randn((B, N), device=dev, generator=g)))
  return out


def _backward_call(s, N, want, ws, nbytes, outs):
  """The backward entry point writing the gradients `want` (a subset of 'fat')."""
  f0, amps, tab, g = s
  B, F = amps.shape
  _, Fw, W = tab.shape
  d_f0, d_amp, d_tab = (o.data_ptr() if c in want else 0 for o, c in zip(outs, 'fat'))
  _lib.check(_lib.load().ddsp_b200_wavetable_backward(
      f0.data_ptr(), amps.data_ptr(), tab.data_ptr(), g.data_ptr(), d_f0, d_amp, d_tab,
      B, F, N, Fw, W, 16000.0, _lib.AMP_WINDOW, ws.data_ptr(), nbytes,
      torch.cuda.current_stream().cuda_stream))


def _shape(B, F, Fw, W, N, iters, warmup, dev):
  sets = _sets(B, F, Fw, W, N, dev)
  lib = _lib.load()
  nbytes = lib.ddsp_b200_wavetable_backward_workspace(B, F, N, Fw, W)
  ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
  outs = (torch.empty((B, F), device=dev), torch.empty((B, F), device=dev),
          torch.empty((B, Fw, W), device=dev))

  def ms(fn):
    return measure.event_ms(fn, iters, warmup, sets)

  fwd = ms(lambda s: core.wavetable_forward(s[0], s[1], s[2], N, 16000.0, 'window'))
  bwd, bwd_nof0, bwd_frames, bwd_table = (
      ms(lambda s, w=w: _backward_call(s, N, w, ws, nbytes, outs))
      for w in ('fat', 'at', 'fa', 't'))

  def step(s):
    x = [t.requires_grad_(True) for t in s[:3]]
    core.wavetable_synthesis(x[0][..., None], x[1][..., None],
                             x[2] if Fw > 1 else x[2][:, 0], n_samples=N).backward(s[3])
    for t in x:
      t.grad = None
      t.requires_grad_(False)
  both = ms(step)
  fb, bb = 4.0 * (B * Fw * W + B * N), 4.0 * (2 * B * Fw * W + B * N)
  return {'B': B, 'F': F, 'Fw': Fw, 'W': W, 'N': N,
          'forward_ms': fwd, 'backward_ms': bwd, 'backward_no_f0_ms': bwd_nof0,
          'backward_f0_amplitudes_ms': bwd_frames, 'backward_wavetables_ms': bwd_table,
          'forward_backward_ms': both,
          'forward_hbm_share': fb / (fwd * 1e-3) / measure.HBM_BYTES_PER_S,
          'backward_hbm_share': bb / (bwd * 1e-3) / measure.HBM_BYTES_PER_S,
          'ring_sets': len(sets)}


def _torch_reference(B, F, W, N, iters, dev):
  """Float32 torch autograd of the reference's formulation, one shape."""
  g = torch.Generator(dev).manual_seed(1)
  f0 = (50.0 + 1000.0 * torch.rand((B, F, 1), device=dev, generator=g)).requires_grad_(True)
  amps = torch.rand((B, F, 1), device=dev, generator=g).requires_grad_(True)
  tab = torch.randn((B, F, W), device=dev, generator=g).requires_grad_(True)
  up = torch.randn((B, N), device=dev, generator=g)

  def step():
    amp = torch.nn.functional.interpolate(amps.transpose(1, 2), size=N, mode='linear',
                                          align_corners=False).transpose(1, 2)[..., 0]
    f = torch.nn.functional.interpolate(f0.transpose(1, 2), size=N, mode='linear',
                                        align_corners=False).transpose(1, 2)
    t = torch.nn.functional.interpolate(tab.transpose(1, 2), size=N, mode='linear',
                                        align_corners=False).transpose(1, 2)
    t = torch.cat([t, t[..., :1]], -1)
    ph = torch.remainder(torch.cumsum(f / 16000.0, 1) - f / 16000.0, 1.0)
    lin = torch.linspace(0.0, 1.0, W + 1, device=dev)
    w = torch.relu(1.0 - torch.abs(ph - lin) * W)
    ((w * t).sum(-1) * amp).backward(up)
  return measure.event_ms(step, iters, 1)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=30)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--out', default=None)
  a = ap.parse_args()
  measure.require_cuda('wavetable_time.py')
  dev = torch.device('cuda', 0)
  res = {'card': measure.card(), 'shapes': []}
  for B in (32, 256):
    for Fw, W in ((1000, 1024), (1000, 2048), (1, 2048)):
      r = _shape(B, 1000, Fw, W, 64000, a.iters, a.warmup, dev)
      print(json.dumps(r), flush=True)
      res['shapes'].append(r)
  res['torch_reference'] = []
  for B in (1, 2, 4, 8):
    try:
      ms = _torch_reference(B, 1000, 1024, 64000, 3, dev)
    except torch.OutOfMemoryError:
      res['torch_reference'].append({'B': B, 'W': 1024, 'forward_backward_ms': None,
                                     'note': 'out of memory'})
      break
    finally:
      torch.cuda.empty_cache()
    res['torch_reference'].append({'B': B, 'W': 1024, 'forward_backward_ms': ms})
    print(json.dumps(res['torch_reference'][-1]), flush=True)
  print(json.dumps(res['card']))
  if a.out:
    measure.append_rows(a.out, [res])


if __name__ == '__main__':
  main()
