"""Time of the three CREPE kernels (csrc/crepe.cuh) at B = 64 items of 4 s at 16 kHz,
hop 64 (250 frames per second) with 'center' padding, so T = 1001 frames each, against
torch compositions of the reference's ops on the same GPU:
  * frames:  pad + frame + normalise (spectral_ops._crepe_frames) against F.pad, unfold
             and float32 mean / population variance;
  * viterbi: PretrainedCREPE.viterbi_decode against the dense 360 x 360 Viterbi step of
             tfp's posterior_mode written in torch (max and argmax over predecessors per
             frame, then a gather per frame to backtrack);
  * decode:  activations_to_f0_and_confidence against its ops in torch.
Each row prints both times and whether the two agree (frames: largest |difference|;
viterbi: the fraction of equal centres; decode: largest relative f0 difference).

  python tools/crepe_time.py [--iters 20] [--rounds 3] [--out FILE]

Times are CUDA events after warm-up, the median of `rounds` alternated rounds.  Prints
the card name and power limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import spectral_ops  # noqa: E402
from tools import measure  # noqa: E402

DEV = 'cuda'
B, SECONDS, SR, HOP = 64, 4, 16000, 64
N = SECONDS * SR
T = 1 + N // HOP


# ---- torch compositions of the reference's ops ----------------------------------------
def torch_frames(audio):
  x = torch.nn.functional.pad(audio, (512, 512))
  f = x.unfold(-1, 1024, HOP).reshape(-1, 1024)
  mu = f.mean(-1, keepdim=True)
  var = ((f - mu) ** 2).mean(-1, keepdim=True)
  std = torch.where(var.abs() > 0, var.sqrt(), torch.full_like(var, 1e-8))
  return (f - mu) / std


def _log_transition():
  bins = torch.arange(360, dtype=torch.float32, device=DEV)
  w = torch.clamp(12 - (bins[None, :] - bins[:, None]).abs(), min=1e-5)
  return torch.log(w / w.sum(1, keepdim=True))        # [from, to]


def torch_viterbi(acts, log_trans):
  b, t, k = acts.shape
  emission = torch.log(torch.eye(k, device=DEV) * 0.1 + 0.9 / k)   # [state, count]
  lp = acts @ emission.T                                            # [B, T, state]
  delta = lp[:, 0] - np.log(k)
  back = torch.empty((t, b, k), dtype=torch.int64, device=DEV)
  for s in range(1, t):
    cand = delta[:, :, None] + log_trans
    delta, back[s] = cand.max(dim=1)
    delta = delta + lp[:, s]
  path = torch.empty((b, t), dtype=torch.int64, device=DEV)
  path[:, -1] = delta.argmax(-1)
  for s in range(t - 1, 0, -1):
    path[:, s - 1] = back[s].gather(1, path[:, s:s + 1])[:, 0]
  return path


def torch_decode(acts):
  cents = (torch.linspace(0, 7180, 360, dtype=torch.float64, device=DEV) +
           1997.3794084376191).to(torch.float32)
  confidence = acts.max(-1, keepdim=True).values
  idx = acts.argmax(-1)[:, None] - 4 + torch.arange(10, device=DEV)[None]
  idx = idx.clamp(0, 359)
  w = acts.gather(1, idx)
  f0_cent = (w * cents[idx]).sum(-1) / w.sum(-1)
  return 10 * 2 ** (f0_cent / 1200.0), confidence


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('crepe_time.py')
  torch.manual_seed(0)
  card = measure.card()
  print(card)
  audio = torch.randn(B, N, device=DEV) * 0.1
  centre = torch.clamp(180 + torch.cumsum(torch.randn(B, T, device=DEV) * 3, -1), 0, 359)
  bins = torch.arange(360, device=DEV)
  acts = 0.9 * torch.exp(-0.5 * ((bins - centre[..., None]) / 2.0) ** 2)
  acts = (acts + 0.05 * torch.rand(B, T, 360, device=DEV)).clamp(0, 1).contiguous()
  rows = acts.reshape(-1, 360)
  model = spectral_ops.PretrainedCREPE(lambda x: x, hop_size=HOP)
  log_trans = _log_transition()

  checks = {
      'frames': lambda: float((spectral_ops._crepe_frames(audio, HOP, 'center')[0] -
                               torch_frames(audio)).abs().max()),
      'viterbi': lambda: float((model.viterbi_decode(acts) ==
                                torch_viterbi(acts, log_trans)).double().mean()),
      'decode': lambda: float(((model.activations_to_f0_and_confidence(rows)[0] -
                                torch_decode(rows)[0]).abs() /
                               torch_decode(rows)[0]).max()),
  }
  cases = {
      'frames': (lambda: spectral_ops._crepe_frames(audio, HOP, 'center'),
                 lambda: torch_frames(audio), args.iters),
      'viterbi': (lambda: model.viterbi_decode(acts),
                  lambda: torch_viterbi(acts, log_trans), max(1, args.iters // 10)),
      'decode': (lambda: model.activations_to_f0_and_confidence(rows),
                 lambda: torch_decode(rows), args.iters),
  }
  lines = []
  with torch.no_grad():
    for what, (cuda_fn, torch_fn, iters) in cases.items():
      t = measure.alternate({'cuda_ms': cuda_fn, 'torch_ms': torch_fn}, args.rounds, iters, 1)
      line = dict(card, config=f'B={B} T={T} hop={HOP} center', what=what, **t,
                  agreement=checks[what](), iters=iters, rounds=args.rounds)
      print(json.dumps(line))
      lines.append(line)
  if args.out:
    measure.append_rows(args.out, lines)


if __name__ == '__main__':
  main()
