"""Time of the tone-transfer adjustment on its CUDA kernels (csrc/postprocessing.cuh)
against a numpy composition of the same steps on the CPU:

  * the notebook's adjust step on one 60 s clip at 250 Hz (T = 15000): detect_notes,
    fit_quantile_transform with inv_quantile, get_tuning_factor and auto_tune;
  * compute_dataset_statistics' quantile fit on [1000, 1000].

  python tools/postprocessing_time.py [--iters 10] [--rounds 3] [--out FILE]
  python tools/postprocessing_time.py --reference [--out FILE]   # CPU: the reference on
                                                                 # the NumPy shim

GPU times are CUDA events around `iters` calls (each ends in the host copy the API
makes), the median of `rounds` rounds alternated with the CPU composition, which is
labelled CPU.  Prints the card name and power limit read in the same run, and appends
JSON lines to --out (default tools/results/postprocessing_h100.jsonl)."""
import argparse
import contextlib
import io
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.golden import make_postprocessing_golden as mk  # noqa: E402
from tools import measure  # noqa: E402

T = 15000


def _clip():
  loud, f0, conf = mk.clip(T, 9000)
  f0_midi = (12 * np.log2(np.maximum(f0, 1e-5) / 440.0) + 69).astype(np.float32)
  return loud, f0_midi, conf


def _dataset():
  return np.round(np.random.default_rng(9001).normal(-30, 10, (1000, 1000)) * 4) / 4


# ---- the CPU composition --------------------------------------------------------------
def _np_smooth(x, k):
  w = np.float32(1) / np.float32(k)
  left = (k - 1) // 2
  p = np.concatenate([np.zeros(left, np.float32), x, np.zeros(k - 1 - left, np.float32)])
  return np.convolve(p, np.full(k, w, np.float32), 'valid').astype(np.float32)


def _np_quantiles(x, nq=1000):
  refs = np.linspace(0, 1, min(nq, x.shape[0]))
  return np.maximum.accumulate(np.nanpercentile(x, refs * 100, axis=0)), refs


def _np_adjust(loud, f0_midi, conf):
  ratio = _np_smooth(conf**2, 40) * (loud + 80) / ((np.mean(loud) + 80) * 0.49)
  mask = ratio >= 1.0
  flat = loud[mask][:, None]
  q, refs = _np_quantiles(flat)
  u = np.interp(flat[:, 0], q[:, 0], refs)
  np.interp(u, refs, q[:, 0])
  factors = np.linspace(-0.5, 0.5, 101)
  d = (f0_midi[mask][:, None] - factors[None]) % 1.0
  d[d > 0.5] -= 1.0
  cost = np.mean(conf[mask][:, None] * np.abs(d), axis=0)
  tf = factors[np.argmin(cost)]
  md = (f0_midi - tf) % 1.0
  md[md > 0.5] -= 1.0
  return f0_midi - 0.5 * md


# ---- the CUDA path --------------------------------------------------------------------
def _gpu_adjust(post, cu, loud, f0_midi, conf, inv):
  with contextlib.redirect_stdout(io.StringIO()):
    mask, _ = post.detect_notes(loud, conf)
    post.fit_quantile_transform(loud, mask, inv_quantile=inv)
    tf = cu.get_tuning_factor(f0_midi, conf, mask)
    return cu.auto_tune(f0_midi, tf, mask, amount=0.5)


def _time_cpu(fn, iters):
  t0 = time.perf_counter()
  for _ in range(iters):
    fn()
  return (time.perf_counter() - t0) * 1e3 / iters


def run_gpu(args):
  import torch
  measure.require_cuda('postprocessing_time.py')
  from ddsp_b200 import colab_utils as cu
  from ddsp_b200 import postprocessing as post
  loud, f0_midi, conf = _clip()
  dl, df, dc = (torch.as_tensor(v, device='cuda') for v in (loud, f0_midi, conf))
  inv = post.QuantileTransformer().fit(dl[::2, None])
  data = _dataset()
  dd = torch.as_tensor(data, device='cuda')
  cases = {
      'adjust_T15000': (lambda: _gpu_adjust(post, cu, dl, df, dc, inv),
                        lambda: _np_adjust(loud, f0_midi, conf)),
      'quantile_fit_1000x1000': (lambda: post.QuantileTransformer().fit(dd),
                                 lambda: _np_quantiles(data)),
  }
  rows = []
  for name, (gpu_fn, cpu_fn) in cases.items():
    g, c = [], []
    for _ in range(args.rounds):
      g.append(measure.event_ms(gpu_fn, args.iters, 1))
      c.append(_time_cpu(cpu_fn, max(1, args.iters // 5)))
    rows.append({'case': name, 'cuda_ms': float(np.median(g)),
                 'cpu_numpy_ms': float(np.median(c)), 'label_cpu': 'CPU (numpy)',
                 **measure.card()})
  return rows


def run_reference(args):
  post, cu = mk._load()
  loud, f0_midi, conf = _clip()
  inv = post.QuantileTransformer().fit(loud[::2, None])
  data = _dataset()

  def adjust():
    with contextlib.redirect_stdout(io.StringIO()):
      mask, _ = post.detect_notes(loud, conf)
      post.fit_quantile_transform(loud, mask, inv_quantile=inv)
      tf = cu.get_tuning_factor(f0_midi, conf, mask)
      cu.auto_tune(f0_midi, tf, mask, amount=0.5)

  del args
  with np.errstate(all='ignore'):
    return [{'case': 'adjust_T15000', 'reference_cpu_ms': _time_cpu(adjust, 1),
             'label_cpu': 'CPU (reference on the NumPy shim)'},
            {'case': 'quantile_fit_1000x1000',
             'reference_cpu_ms': _time_cpu(lambda: post.QuantileTransformer().fit(data), 1),
             'label_cpu': 'CPU (reference on the NumPy shim)'}]


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--iters', type=int, default=10)
  p.add_argument('--rounds', type=int, default=3)
  p.add_argument('--reference', action='store_true')
  p.add_argument('--out', default=os.path.join(ROOT, 'tools', 'results',
                                               'postprocessing_h100.jsonl'))
  args = p.parse_args()
  rows = run_reference(args) if args.reference else run_gpu(args)
  for r in rows:
    print(json.dumps(r))
  measure.append_rows(args.out, rows)


if __name__ == '__main__':
  main()
