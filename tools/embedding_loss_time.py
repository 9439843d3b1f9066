"""Time of losses.PretrainedCREPE's framing, forward plus backward, at B = 64 items of
64000 samples (4 s at 16 kHz) with centring, against the torch composition of the
reference's ops on the same GPU (F.pad, unfold, tf.nn.moments' mean and population
variance, the division by sqrt(var) + 1e-5, and torch.autograd for the backward):
  * hop 1024, what PretrainedCREPE.call uses: 63 frames per item, no sample in two
    frames (csrc/crepe.cuh's disjoint backward);
  * hop 160: 401 frames per item, each sample in up to 7 (the overlap backward).
Each row prints both times, the largest |difference| of the two audio gradients
relative to the largest gradient, and the time of each CUDA kernel (torch.profiler).

  python tools/embedding_loss_time.py [--iters 20] [--rounds 3] [--out FILE]

Times are CUDA events after warm-up, the median of `rounds` alternated rounds.  Prints
the card name and power limit read in the same run."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import autograd  # noqa: E402
from tools import measure  # noqa: E402

DEV = 'cuda'
B, N = 64, 64000


def torch_frames(audio, hop):
  x = torch.nn.functional.pad(audio, (512, 512))
  f = x.unfold(-1, 1024, hop)
  mu = f.mean(-1, keepdim=True)
  var = ((f - mu.detach()) ** 2).mean(-1, keepdim=True)
  return (f - mu) / (var ** 0.5 + 1e-5)


def _step(frames_fn, audio, grad, hop):
  x = audio.detach().requires_grad_(True)
  frames_fn(x, hop).backward(grad)
  return x.grad


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('embedding_loss_time.py')
  torch.manual_seed(0)
  card = measure.card()
  print(card)
  audio = torch.randn(B, N, device=DEV) * 0.1
  cuda_frames = lambda x, hop: autograd.CrepeLossFramesFn.apply(x, hop, True)
  lines = []
  for hop in (1024, 160):
    f = 1 + N // hop
    grad = torch.randn(B, f, 1024, device=DEV)
    cuda_fn = lambda: _step(cuda_frames, audio, grad, hop)
    torch_fn = lambda: _step(torch_frames, audio, grad, hop)
    t = measure.alternate({'cuda_ms': cuda_fn, 'torch_ms': torch_fn}, args.rounds,
                          args.iters, 1)
    got, want = cuda_fn(), torch_fn()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
      cuda_fn()
      torch.cuda.synchronize()
    kernels = {e.key: round(e.device_time_total / 1e3, 4) for e in prof.key_averages()
               if 'crepe' in e.key}
    line = dict(card, config=f'B={B} N={N} hop={hop} center frames={f}',
                what='frames forward + backward', **t,
                grad_rel_diff=float((got - want).abs().max() / want.abs().max()),
                kernel_ms=kernels,
                iters=args.iters, rounds=args.rounds)
    print(json.dumps(line))
    lines.append(line)
  if args.out:
    measure.append_rows(args.out, lines)


if __name__ == '__main__':
  main()
