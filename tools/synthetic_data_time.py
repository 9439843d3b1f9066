"""Times InverseSynthesis's synthetic data (ddsp_b200.synthetic_data) on the GPU and,
for scale, the float64 host restatement and the reference on the NumPy shim (where
the reference sources exist).  CUDA events after a warm-up; one JSON line per
measurement, the card name and power limit in every line.

  python tools/synthetic_data_time.py [--out tools/results/synthetic_data_h100.jsonl]
"""
import argparse
import json
import os
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ddsp_b200 import synthetic_data as sd   # noqa: E402
from tests import synthetic_data_ref as ref  # noqa: E402
from tools import measure  # noqa: E402

T, K, M = 125, 100, 65
# bytes written per example: the kernel's float64 rows and the float32 controls
# (harm_amp, harm_dist, f0_hz, sin_amps, sin_freqs, noise_magnitudes)
F64_BYTES = 8 * (T + T * K + T + T * M + 1)
F32_BYTES = 4 * (T + 3 * T * K + T + T * M)


def gpu_ms(fn, reps):
  """Median and least ms of `reps` calls, each timed on its own after 3 warm-up calls."""
  times = [measure.event_ms(fn, 1, 3 if r == 0 else 0) for r in range(reps)]
  return float(np.median(times)), float(np.min(times))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('synthetic_data_time.py')
  card = measure.card()
  rows = []

  def emit(**kw):
    kw.update(card=card)
    rows.append(kw)
    print(json.dumps(kw), flush=True)

  seeds = sd.example_seeds(16384)
  for b in (64, 1024, 16384):
    s = seeds[:b]
    med, best = gpu_ms(lambda: sd.generate_notes_v2(seeds=s), 10 if b < 16384 else 5)
    emit(what='v2 seeds mode', batch=b, ms_median=med, ms_min=best,
         examples_per_s=b / med * 1e3,
         bytes_per_example=F64_BYTES + F32_BYTES,
         write_gbps=b * (F64_BYTES + F32_BYTES) / med * 1e-6,
         hbm_fraction=b * (F64_BYTES + F32_BYTES) / med * 1e3 / measure.HBM_BYTES_PER_S)
  np.random.seed(0)
  med, best = gpu_ms(lambda: sd.generate_notes_v2(n_batch=64), 5)
  emit(what='v2 state mode', batch=64, ms_median=med, ms_min=best,
       examples_per_s=64 / med * 1e3)
  med, best = gpu_ms(lambda: sd.generate_notes(64, T), 10)
  emit(what='v1 (host draws, GPU render)', batch=64, ms_median=med, ms_min=best,
       examples_per_s=64 / med * 1e3)

  t0 = time.perf_counter()
  for s in range(20):
    ref.seeded_v2(s)
  emit(what='host float64 restatement, one core', ms_per_example=(time.perf_counter() - t0) / 20 * 1e3)
  try:
    from tests.golden import make_synthetic_data_golden as golden
    _, m = golden._load()
    with warnings.catch_warnings():
      warnings.simplefilter('ignore')
      t0 = time.perf_counter()
      for s in range(20):
        np.random.seed(s)
        m.generate_notes_v2()
    emit(what='reference on the NumPy shim, one core',
         ms_per_example=(time.perf_counter() - t0) / 20 * 1e3)
  except Exception as e:  # the reference sources are not everywhere
    print('reference on the shim not timed: %s' % e, file=sys.stderr)
  if args.out:
    measure.append_rows(args.out, rows)


if __name__ == '__main__':
  main()
