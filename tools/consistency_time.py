"""Time of the consistency-loss kernels (csrc/consistency.cuh) against a float32
torch composition of the reference formulation.

Configurations (ICML 2020 self-supervised pitch model, 16 kHz):
  * kde:       KDEConsistencyLoss at the pretrain config, B = 32, T = 125 frames,
               100 sinusoids against 100 harmonics; forward, and forward + backward;
  * twm_c1:    TWMLoss.call forward + backward with one candidate per frame (a
               harmonic encoder's f0), B = 32, T = 125, P = 100;
  * twm_c100:  TWMLoss.call forward + backward with the 100 sinusoid frequencies as
               candidates, B = 32, T = 125, C = P = 100;
  * predict:   TWMLoss.predict_f0 as TWMEvaluator calls it (candidates = freqs),
               B = 32, T = 125, C = P = 100.
Each is alternated in the same run with the reference formulation in float32 torch:
the broadcast pairwise Normal log-probs, log_softmax'd weights and torch.logsumexp,
whose peak memory (torch.cuda.max_memory_allocated above the inputs) is reported too.

  python tools/consistency_time.py [--iters 20] [--rounds 3] [--out FILE]

Times are CUDA events after warm-up, the median of `rounds` alternated rounds.
Component evaluations are counted from shapes, as the reference formulation does the
work: KDE 2 B T K^2 per forward; TWM B T C P G (comb) + B T C n_points P (mixture)
per forward; forward + backward counts the forward's twice.  Prints the card name and
power limit read in the same run."""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import losses  # noqa: E402
from tools import measure  # noqa: E402

DEV = 'cuda'
HALF_LOG_2PI = 0.5 * math.log(2 * math.pi)


# ---- the reference formulation, float32 torch ------------------------------------
def _safe_divide(n, d, eps=1e-7):
  return n / torch.where(d == 0.0, torch.full_like(d, eps), d)


def _hz_to_midi(f):
  safe = torch.where(f <= 0.0, torch.full_like(f, 1e-5), f)
  notes = 12.0 * (torch.log(safe) / math.log(2.0) - math.log(440.0) / math.log(2.0)) + 69.0
  return torch.where(f <= 0.0, torch.zeros_like(notes), notes)


def _mixture_log_prob(x, logits, loc, scale):
  lp = -0.5 * ((x[..., None] - loc) / scale)**2 - math.log(scale) - HALF_LOG_2PI
  return torch.logsumexp(lp + torch.log_softmax(logits, -1), -1)


def _probs(amps):
  amps = torch.where(amps == 0.0, torch.full_like(amps, 1e-7), amps)
  return _safe_divide(amps, amps.sum(-1, keepdim=True))


def ref_kde(amps_a, freqs_a, amps_b, freqs_b, scale=0.1):
  def nll(amps, freqs, amps_t, freqs_t):
    x = _hz_to_midi(freqs).permute(2, 0, 1)
    n = -_mixture_log_prob(x, torch.log(_probs(amps_t)), _hz_to_midi(freqs_t), scale)
    return torch.mean(n.permute(1, 2, 0) * _safe_divide(amps, amps.sum(-1, keepdim=True)), -1)
  return (nll(amps_a, freqs_a, amps_b, freqs_b).mean() + nll(amps_b, freqs_b, amps_a, freqs_a).mean()
          + torch.mean(torch.abs(amps_a.mean(-1) - amps_b.mean(-1))))


def ref_twm_tensors(f0, freqs, amps, n_points=10, n_gauss=30):
  g = torch.full((n_gauss,), 1.0 / n_gauss, device=DEV)
  loc = torch.arange(1, n_gauss + 1, dtype=torch.float32, device=DEV)
  ratios = _safe_divide(freqs[:, :, None, :], f0[:, :, :, None])
  a = amps[:, :, None, :]
  s = _safe_divide(torch.sum(-_mixture_log_prob(ratios, g, loc, 0.2) * a, -1), a.sum(-1))
  n = torch.arange(1, n_points + 1, dtype=torch.float32, device=DEV)
  harmonics = _hz_to_midi(f0[:, :, :, None] * n)
  nll_h = -_mixture_log_prob(harmonics.permute(2, 3, 0, 1), torch.log(_probs(amps)),
                             _hz_to_midi(freqs), 0.5).permute(2, 3, 0, 1)
  h = nll_h * torch.linspace(1.0, 1.0 / n_points, n_points, device=DEV)
  mask = (harmonics < _hz_to_midi(torch.tensor(8000.0, device=DEV))).float()
  h = h * _safe_divide(mask, mask.mean(-1, keepdim=True))
  return s, h.mean(-1)


def ref_twm(f0, freqs, amps):
  s, h = ref_twm_tensors(f0, freqs, amps)
  c = s + h
  return torch.mean(c * torch.softmax(-c, -1))


def ref_predict(f0, freqs, amps):
  s, h = ref_twm_tensors(f0, freqs, amps)
  idx = torch.argmin(torch.nan_to_num(s + h, nan=math.inf), -1, keepdim=True)
  return torch.gather(f0, -1, idx)


# ---- inputs ----------------------------------------------------------------------
def _sinusoids(b, t, k, seed):
  rng = np.random.default_rng(seed)
  f0 = np.exp(rng.uniform(np.log(80.0), np.log(400.0), (b, t, 1)))
  n = np.arange(1, k + 1)
  freqs = np.minimum(f0 * n * np.exp(rng.normal(0.0, 0.01, (b, t, k))), 7900.0)
  amps = rng.uniform(0.1, 1.0, (b, t, k)) / n
  cast = lambda v: torch.as_tensor(v, dtype=torch.float32, device=DEV)
  return cast(amps), cast(freqs), cast(f0 * np.exp(rng.uniform(-0.5, 0.5, (b, t, 1))))


def _fwd_bwd(fn, inputs):
  def run():
    for x in inputs:
      x.grad = None
    fn(*inputs).backward()
  return run


def configs():
  b, t, k = 32, 125, 100
  amps_a, freqs_a, _ = _sinusoids(b, t, k, 1)
  amps_b, freqs_b, f0 = _sinusoids(b, t, k, 2)
  kde_in = [x.clone().requires_grad_(True) for x in (amps_a, freqs_a, amps_b, freqs_b)]
  kde = losses.KDEConsistencyLoss()
  twm = losses.TWMLoss()
  c1 = [x.clone().requires_grad_(True) for x in (f0, freqs_b, amps_b)]
  c100 = [x.clone().requires_grad_(True) for x in (freqs_b, freqs_b.clone(), amps_b)]
  evals_kde = 2 * b * t * k * k
  evals_twm = lambda c: b * t * c * k * 30 + b * t * c * 10 * k
  with torch.no_grad():
    kde_plain = [x.detach() for x in kde_in]
    pred_in = [x.detach() for x in c100]
  return [
      ('kde_forward', lambda: kde(*kde_plain), lambda: ref_kde(*kde_plain), evals_kde),
      ('kde_forward_backward', _fwd_bwd(kde, kde_in), _fwd_bwd(ref_kde, kde_in),
       2 * evals_kde),
      ('twm_c1_forward_backward', _fwd_bwd(twm, c1), _fwd_bwd(ref_twm, c1),
       2 * evals_twm(1)),
      ('twm_c100_forward_backward', _fwd_bwd(twm, c100), _fwd_bwd(ref_twm, c100),
       2 * evals_twm(k)),
      ('predict_f0', lambda: twm.predict_f0(*pred_in), lambda: ref_predict(*pred_in),
       evals_twm(k)),
  ]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('consistency_time.py')
  torch.backends.cuda.matmul.allow_tf32 = False
  card = measure.card()
  rows = []
  for name, ours, theirs, evals in configs():
    t = measure.alternate({'ms': ours, 'torch_ms': theirs}, args.rounds,
                          {'ms': args.iters, 'torch_ms': max(2, args.iters // 4)}, 3)
    torch.cuda.empty_cache()
    row = {'config': name, **t, 'peak_mb': measure.peak_bytes(ours) / 2**20,
           'torch_peak_mb': measure.peak_bytes(theirs) / 2**20, 'component_evals': evals}
    row['evals_per_s'] = evals / (row['ms'] * 1e-3)
    row['torch_evals_per_s'] = evals / (row['torch_ms'] * 1e-3)
    row.update(card)
    rows.append(row)
    print(json.dumps(row), flush=True)
    torch.cuda.empty_cache()
  if args.out:
    measure.append_rows(args.out, rows)


if __name__ == '__main__':
  main()
