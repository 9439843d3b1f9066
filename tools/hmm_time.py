"""Time of losses.HmmTranscriber's HMM (csrc/hmm.cuh) against a float32 torch composition
of tfp's dense HiddenMarkovModel algorithms, run as a step loop.

Shape: the MIDI autoencoder's HMM prior (hmm_prior.gin), T = 1000 steps, K = 128 states,
at B = 16 and 256.  Timed: log_prob; log_prob with its backward to the observations;
Viterbi (posterior_mode).  The composition runs each of the T steps as a K x K
logsumexp (or max / argmax for Viterbi) over [B, K, K], autograd for the backward, and
a gather loop for the backtrack.

  python tools/hmm_time.py [--iters 10] [--rounds 3] [--out FILE]

Times are CUDA events after warm-up, the median of `rounds` alternated rounds; peak
memory is torch.cuda.max_memory_allocated above the inputs.  Prints the card name and
power limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import core, losses  # noqa: E402
from tools import measure  # noqa: E402

DEV = 'cuda'
T, K = 1000, 128


def dense_params(hmm):
  k = hmm.n_pitches
  trans = torch.full((k, k), hmm.other, device=DEV)
  trans.fill_diagonal_(hmm.hold)
  trans = trans / trans.sum(1, keepdim=True)
  return (torch.full((k,), -float(np.log(k)), device=DEV), torch.log(trans),
          torch.as_tensor(hmm.loc, device=DEV), torch.as_tensor(hmm.scale, device=DEV))


def dense_obs(x, loc, scale):
  z = (x[..., None, :] - loc) / scale
  return torch.sum(-0.5 * z * z - torch.log(scale) - 0.5 * float(np.log(2 * np.pi)), -1)


def dense_log_prob(x, log_init, log_trans, loc, scale):
  lp = dense_obs(x, loc, scale)
  alpha = log_init + lp[:, 0]
  for t in range(1, lp.shape[1]):
    alpha = lp[:, t] + torch.logsumexp(alpha[:, :, None] + log_trans, dim=1)
  return torch.logsumexp(alpha, -1)


def dense_viterbi(x, log_init, log_trans, loc, scale):
  lp = dense_obs(x, loc, scale)
  delta = log_init + lp[:, 0]
  back = []
  for t in range(1, lp.shape[1]):
    best, arg = torch.max(delta[:, :, None] + log_trans, dim=1)
    back.append(arg)
    delta = lp[:, t] + best
  s = torch.argmax(delta, -1)
  path = [s]
  for arg in reversed(back):
    s = torch.gather(arg, 1, s[:, None])[:, 0]
    path.append(s)
  return torch.stack(path[::-1], 1)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=10)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('hmm_time.py')
  hmm = losses.HmmTranscriber(n_timesteps=T, n_pitches=K)
  loc, scale = (torch.as_tensor(v, device=DEV) for v in (hmm.loc, hmm.scale))
  dense = dense_params(hmm)
  result = {'card': measure.card(), 'T': T, 'K': K, 'rows': []}
  for b in (16, 256):
    rng = np.random.default_rng(b)
    x = torch.as_tensor(np.stack([rng.integers(1, K, (b, T)) + 0.2 * rng.normal(size=(b, T)),
                                  1.5 + 0.2 * rng.normal(size=(b, T))], -1),
                        dtype=torch.float32, device=DEV)
    xg = x.clone().requires_grad_()

    def cuda_fwd():
      core.hmm_log_prob(x, loc, scale, hmm.hold, hmm.other)

    def cuda_bwd():
      xg.grad = None
      core.hmm_log_prob(xg, loc, scale, hmm.hold, hmm.other).sum().backward()

    def cuda_vit():
      core.hmm_posterior_mode(x, loc, scale, hmm.hold, hmm.other)

    def torch_fwd():
      with torch.no_grad():
        dense_log_prob(x, *dense)

    def torch_bwd():
      xg.grad = None
      dense_log_prob(xg, *dense).sum().backward()

    def torch_vit():
      with torch.no_grad():
        dense_viterbi(x, *dense)

    pairs = {'log_prob': (cuda_fwd, torch_fwd), 'log_prob+backward': (cuda_bwd, torch_bwd),
             'viterbi': (cuda_vit, torch_vit)}
    for name, (c, r) in pairs.items():
      t = measure.alternate({'cuda_ms': c, 'torch_ms': r}, args.rounds,
                            {'cuda_ms': args.iters, 'torch_ms': max(1, args.iters // 5)},
                            {'cuda_ms': 3, 'torch_ms': 1})
      row = {'B': b, 'op': name, **t, 'cuda_peak_MB': measure.peak_bytes(c) / 2**20,
             'torch_peak_MB': measure.peak_bytes(r) / 2**20}
      row['speedup'] = row['torch_ms'] / row['cuda_ms']
      result['rows'].append(row)
      print(json.dumps(row), flush=True)
  lp = core.hmm_log_prob(x, loc, scale, hmm.hold, hmm.other)
  ref = dense_log_prob(x.double(), *(p.double() for p in dense))
  result['log_prob_max_rel_vs_float64'] = float(((lp.double() - ref) / ref).abs().max())
  print(json.dumps({k: v for k, v in result.items() if k != 'rows'}))
  if args.out:
    measure.append_rows(args.out, [result])


if __name__ == '__main__':
  main()
