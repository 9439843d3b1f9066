"""Times effects.Reverb-shaped convolutions (48000-tap IR on 64000 samples): the
hand-written partitioned overlap-save kernels vs the framed cuFFT formulation.

  python tools/reverb_time.py"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import core  # noqa: E402
from tools import measure  # noqa: E402


def main():
  argparse.ArgumentParser(description=__doc__.split('\n\n')[0]).parse_args()
  measure.require_cuda('reverb_time.py')
  rng = np.random.default_rng(0)
  for B, shared in ((32, False), (32, True), (256, True)):
    audio = torch.from_numpy(rng.standard_normal((B, 64000)).astype(np.float32)).cuda()
    ir = torch.from_numpy((rng.standard_normal((1 if shared else B, 48000)) *
                           np.exp(-np.arange(48000) / 8000.0)).astype(np.float32)).cuda()

    def ours():
      return core.fft_convolve(audio, ir, padding='same', delay_compensation=0)

    def cufft():
      fft_size = core.get_fft_size(64000, 48000)
      return core._fft_convolve_cufft(audio, ir[:, None, :], 1, 64000, fft_size, 0, 64000)

    for name, fn in (('partitioned overlap-save (ours)', ours), ('framed cuFFT', cufft)):
      print('B=%d shared_ir=%s %-34s %.3f ms' % (B, shared, name, measure.event_ms(fn, 10, 3)),
            flush=True)
    d = (ours() - cufft()).abs().max().item()
    print('  max |ours - cufft| = %.2e' % d)


if __name__ == '__main__':
  main()
