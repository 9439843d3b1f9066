"""Times `ddsp_b200_harmonic_backward` (G0 / G1 of the harmonic synthesizer, the transposes
HarmonicSynthesisFn and the decoder's backward train through) in this tree's library against
another build of it, alternated on the same inputs.  The other library is a path, normally
one built from an earlier commit in a worktree of that commit:

  git worktree add /tmp/base <commit>
  (cd /tmp/base && python -c "from ddsp_b200 import build; \\
      build.build(out='$PWD/tools/variants/lib_base.so')")
  python tools/harmonic_backward_time.py tools/variants/lib_base.so [--iters 20] \\
      [--rounds 5] [--out FILE]

Shapes, window amplitudes, 100 harmonics at 16 kHz, f0 of 80 .. 800 Hz with a 5 Hz
vibrato (so most frames' live harmonic count changes inside the frame):
  * hop 64, B = 128, F = 1000 (the C4 training step's shape);
  * hops 128, 256 and 1024 at B = 32 and about 64000 samples (F = 500, 250 and 63);
  * hop 8192, F = 8 at B = 1 and B = 32, and hop 256, F = 250 at B = 1 (small batches
    at large hops).
Each timed call takes the next input set of a ring larger than twice the L2 cache.  Times
are CUDA events, the median of `rounds` alternated rounds.  Each row gives both times and
how the two libraries' outputs differ: whether they are bitwise equal, and the largest
|difference| over the largest |output|.  Prints the card name and power limit read in the
same run."""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import _lib  # noqa: E402
from tools import measure  # noqa: E402

SR = 16000.0
K = 100
SHAPES = [(128, 1000, 64), (32, 500, 128), (32, 250, 256), (32, 63, 1024),
          (1, 8, 8192), (32, 8, 8192), (1, 250, 256)]     # (B, F, hop)


def _f0(B, F, hop, gen):
  base = 80.0 + 720.0 * torch.rand(B, 1, device='cuda', generator=gen)
  ph = 2 * math.pi * torch.rand(B, 1, device='cuda', generator=gen)
  t = torch.arange(F, device='cuda') * (hop / SR)
  return base * (1.0 + 0.03 * torch.sin(2 * math.pi * 5.0 * t + ph))


def _shape(libs, B, F, hop, iters, rounds):
  N = F * hop
  gen = torch.Generator(device='cuda').manual_seed(B * F + hop)
  n = measure.ring_len(4 * (B * F + B * N + 2 * B * F * K))
  f0s = [_f0(B, F, hop, gen) for _ in range(n)]
  gs = [torch.randn(B, N, device='cuda', generator=gen) for _ in range(n)]
  outs = {name: (torch.empty(B, F, K, device='cuda'), torch.empty(B, F, K, device='cuda'))
          for name in libs}

  def call(name, i):
    g0, g1 = outs[name]
    rc = libs[name].ddsp_b200_harmonic_backward(
        f0s[i].data_ptr(), gs[i].data_ptr(), g0.data_ptr(), g1.data_ptr(), B, F, K, N, SR,
        _lib.AMP_WINDOW, torch.cuda.current_stream().cuda_stream)
    if rc:
      raise RuntimeError('%s: harmonic_backward returned %d: %s' % (
          name, rc, libs[name].ddsp_b200_last_error().decode()))

  def timed(name):
    state = {'i': 0}

    def fn():
      call(name, state['i'] % n)
      state['i'] += 1
    return fn

  times = measure.alternate({name: timed(name) for name in libs}, rounds, iters, 2 * n)
  for name in libs:
    call(name, 0)
  torch.cuda.synchronize()
  (a0, a1), (b0, b1) = outs['ours'], outs['base']
  peak = max(b0.abs().max().item(), b1.abs().max().item())
  diff = max((a0 - b0).abs().max().item(), (a1 - b1).abs().max().item())
  bitwise = bool(torch.equal(a0.view(torch.int32), b0.view(torch.int32)) and
                 torch.equal(a1.view(torch.int32), b1.view(torch.int32)))
  return {'B': B, 'F': F, 'hop': hop, 'K': K, 'N': N,
          'ours_ms': times['ours'], 'base_ms': times['base'],
          'ours_over_base': times['ours'] / times['base'],
          'bitwise_equal': bitwise, 'max_abs_diff_over_peak': diff / peak}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('base_lib', help='the library to compare with, e.g. one built from an '
                  'earlier commit')
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('harmonic_backward_time.py')
  libs = {'ours': _lib.load(), 'base': _lib.bind(os.path.abspath(args.base_lib))}
  row = {'card': measure.card(), 'base_lib': os.path.basename(args.base_lib),
         'shapes': [_shape(libs, B, F, hop, args.iters, args.rounds) for B, F, hop in SHAPES]}
  print(json.dumps(row))
  if args.out:
    measure.append_rows(args.out, [row])


if __name__ == '__main__':
  main()
