"""Shared synthetic inputs for tests and bench (SURVEY.md section 8d)."""
import numpy as np


def synth_inputs(B, F, K, nb, N, seed=1234, sample_rate=16000, f0_lo=80.0,
                 f0_hi=800.0):
  """Raw network-output-like inputs of the decoder, float32 numpy.

  f0: per-item base U[f0_lo, f0_hi] Hz with a 3 % / 5 Hz vibrato, clipped to
  [20, 2000]; amps / harmonic_distribution / noise magnitudes ~ N(0,1) (the
  pre-get_controls distribution of processors_test.py:35-42); noise U[-1,1).
  """
  rng = np.random.default_rng(seed)
  hop = N / F
  t_frame = np.arange(F) * hop / sample_rate
  base = rng.uniform(f0_lo, f0_hi, size=(B, 1))
  ph = rng.uniform(0, 2 * np.pi, size=(B, 1))
  f0 = base * (1.0 + 0.03 * np.sin(2 * np.pi * 5.0 * t_frame[None, :] + ph))
  f0 = np.clip(f0, 20.0, 2000.0)[..., None].astype(np.float32)
  return {
      'f0_hz': f0,
      'amps': rng.standard_normal((B, F, 1)).astype(np.float32),
      'harmonic_distribution': rng.standard_normal((B, F, K)).astype(np.float32),
      'noise_magnitudes': rng.standard_normal((B, F, nb)).astype(np.float32),
      'noise': rng.uniform(-1.0, 1.0, size=(B, N)).astype(np.float32),
  }


def rel_err(a, b):
  """(max-abs error / max-abs reference, relative L2 error)."""
  a = np.asarray(a, np.float64)
  b = np.asarray(b, np.float64)
  peak = max(np.abs(b).max(), 1e-30)
  l2 = np.sqrt(((a - b)**2).sum() / max((b**2).sum(), 1e-60))
  return np.abs(a - b).max() / peak, l2


def linearity(grad, g, oracle_fn, shape, n_dirs=3, seed=0):
  """For an output y linear in the differentiated input x, with upstream gradient
  g and dL/dx = grad: <grad, D> against sum g * oracle_fn(D) in float64 for random
  directions D >= 0, relative to sum |g * oracle_fn(D)| (the inner product without
  cancellation).  oracle_fn(D) is the oracle's output for input D; no restatement
  of the operation is involved."""
  rng = np.random.default_rng(seed)
  gnp = g.double().cpu().numpy()
  grad = grad.double().cpu().numpy()
  for _ in range(n_dirs):
    d = rng.uniform(0.0, 1.0, shape)
    y = oracle_fn(d)
    want = float((gnp * y).sum())
    scale = float(np.abs(gnp * y).sum())
    got = float((grad * d).sum())
    assert abs(got - want) <= 1e-4 * scale, (got, want, scale)


class HostQueriesOnly:
  """Stands in for the loaded library where no device work may happen yet: the
  size and shape queries (ddsp_b200_ir_size, *_workspace, *_takes), which run on
  the host alone, go to the real library; any other entry point fails the test."""

  def __init__(self, real):
    self.real = real

  def __getattr__(self, name):
    if name == 'ddsp_b200_ir_size' or name.endswith(('_workspace', '_takes')):
      return getattr(self.real, name)
    raise AssertionError(f'{name} was looked up before the argument checks')
