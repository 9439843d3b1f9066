"""Times harmonic_forward (on controls), the decoder step (raw outputs, get_controls
fused) and the noise kernel alone for each library given on the command line
(variants of libddsp_b200.so built with different -D flags, tools/build_variants.sh).
Each library is loaded with ctypes directly, next to the product library.
usage: python tools/variant_time.py [B=256] lib1.so lib2.so ..."""
import argparse
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ddsp_b200  # noqa: E402
from ddsp_b200 import _lib  # noqa: E402
from tests.util import synth_inputs  # noqa: E402
from tools import measure  # noqa: E402

F, K, NB, N = 1000, 100, 65, 64000


def timed(fn, reps=5, n=24):
  """Median us per call over `reps` runs of n calls fn(i), after 6 warm-up calls."""
  return statistics.median(1e3 * measure.event_ms(fn, n, 6 if r == 0 else 0, range(n))
                           for r in range(reps))


def main():
  ap = argparse.ArgumentParser(description='Times the kernels of each variant library.')
  ap.add_argument('libs', nargs='*', metavar='[B] lib',
                  help='the batch size (default 256), then the variant libraries')
  args = ap.parse_args().libs
  B = int(args.pop(0)) if args and args[0].isdigit() else 256
  measure.require_cuda('variant_time.py')
  sets = []
  for s in range(3):
    inp = synth_inputs(B, F, K, NB, N, seed=1234 + s)
    f = {k: torch.from_numpy(inp[k]).cuda()
         for k in ['amps', 'harmonic_distribution', 'f0_hz', 'noise_magnitudes']}
    ctl = ddsp_b200.Harmonic().get_controls(f['amps'], f['harmonic_distribution'], f['f0_hz'])
    sets.append((f, ctl, torch.empty(B, N, device='cuda')))
  st = torch.cuda.current_stream().cuda_stream

  for path in args:
    lib = _lib.bind(os.path.abspath(path))

    def harm(i):
      f, ctl, out = sets[i % 3]
      rc = lib.ddsp_b200_harmonic_forward(
          ctl['f0_hz'].data_ptr(), ctl['amplitudes'].data_ptr(),
          ctl['harmonic_distribution'].data_ptr(), out.data_ptr(), B, F, K, N, 16000.0, 0, 0, 0,
          st)
      assert rc == 0, lib.ddsp_b200_last_error()

    def noise(i):
      f, ctl, out = sets[i % 3]
      rc = lib.ddsp_b200_filtered_noise_forward(
          f['noise_magnitudes'].data_ptr(), None, 7, i, out.data_ptr(), B, F, NB, N, 0, 1, None,
          0, st)
      assert rc == 0, lib.ddsp_b200_last_error()

    def dec(i):
      f, ctl, out = sets[i % 3]
      rc = lib.ddsp_b200_decoder_forward(
          f['amps'].data_ptr(), f['harmonic_distribution'].data_ptr(), f['f0_hz'].data_ptr(),
          f['noise_magnitudes'].data_ptr(), None, 7, i, out.data_ptr(), B, F, K, NB, N, 16000.0,
          0, 3, 0, -5.0, st)
      assert rc == 0, lib.ddsp_b200_last_error()

    th, tn, td = timed(harm), timed(noise), timed(dec)
    print('%-44s B=%d harmonic(controls) %.1f  noise %.1f  decoder %.1f  (decoder - noise %.1f) us'
          % (os.path.basename(path), B, th, tn, td, td - tn), flush=True)


if __name__ == '__main__':
  main()
