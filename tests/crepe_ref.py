"""Float64 restatement of what spectral_ops.PretrainedCREPE (spectral_ops.py:171-220,
432-566) does around its network: pad, batch_frames and normalize_frames; create_hmm's
360-state HMM and HiddenMarkovModel.posterior_mode on it, in the dense 360 x 360
formulation (the band structure csrc/crepe.cuh exploits is deliberately not used); and
activations_to_f0_and_confidence.  Pinned to the unmodified reference by
tests/golden/crepe.npz (tests/golden/make_crepe_golden.py).

`ShimMultinomial` and `ShimHiddenMarkovModel` wrap the same functions for the reference
run on the NumPy TensorFlow shim, which the generator installs there for that run only.
"""
import numpy as np
from scipy.special import gammaln

BINS = 360
FRAME = 1024


# ---- frames ---------------------------------------------------------------------------
def pad(x, frame_size, hop_size, padding='center'):
  """spectral_ops.pad along the last axis of [B, N] (or [N]), constant zeros."""
  x = np.asarray(x, np.float64)
  if padding == 'valid':
    return x
  n = x.shape[-1]
  if padding == 'same':
    n_frames = -(-n // hop_size)
    widths = (0, (n_frames - 1) * hop_size + frame_size - n)
  else:
    widths = (frame_size // 2, frame_size // 2)
  return np.pad(x, [(0, 0)] * (x.ndim - 1) + [widths])


def batch_frames(audio, hop_size):
  """tf.signal.frame(audio, 1024, hop) reshaped to [-1, 1024]; audio of exactly 1024
  samples is returned as it is."""
  audio = np.asarray(audio, np.float64)
  if audio.shape[-1] == FRAME:
    return audio
  n = audio.shape[-1]
  n_frames = max(0, 1 + (n - FRAME) // hop_size)
  idx = np.arange(n_frames)[:, None] * hop_size + np.arange(FRAME)[None, :]
  return audio[..., idx].reshape(-1, FRAME)


def normalize_frames(frames):
  """tf.nn.moments' mean and population variance, std = 1e-8 where the variance is 0."""
  frames = np.asarray(frames, np.float64)
  mu = frames.mean(-1, keepdims=True)
  var = np.mean((frames - mu) ** 2, -1, keepdims=True)
  std = np.where(np.abs(var) > 0, np.sqrt(var), 1e-8)
  return (frames - mu) / std


def frames(audio, hop_size, padding='center'):
  """What the network reads: [B * F, 1024]."""
  audio = np.asarray(audio, np.float64)
  audio = audio[None] if audio.ndim == 1 else audio
  return normalize_frames(batch_frames(pad(audio, FRAME, hop_size, padding), hop_size))


# ---- the HMM --------------------------------------------------------------------------
def create_hmm():
  """(log initial [360], log transition [from, to], emission probs [360, 360]) as
  create_hmm builds them, in float64."""
  bins = np.arange(BINS, dtype=np.float64)
  xx, yy = np.meshgrid(bins, bins)
  transition = np.maximum(12 - np.abs(xx - yy), 1e-5)
  transition = transition / np.sum(transition, axis=1)[:, None]
  emission = np.eye(BINS) * 0.1 + np.ones((BINS, BINS)) * (0.9 / BINS)
  return np.full(BINS, -np.log(BINS)), np.log(transition), emission


def multinomial_log_prob(counts, probs):
  """Multinomial(total_count=1, probs).log_prob(counts) for counts [..., K] under every
  row of probs [S, K]: [..., S].  Counts need not be integers, as in tfp."""
  counts = np.asarray(counts, np.float64)
  n = counts.sum(-1, keepdims=True)
  log_comb = gammaln(n + 1.0) - gammaln(counts + 1.0).sum(-1, keepdims=True)
  return log_comb + counts @ np.log(probs).T


def viterbi(log_init, log_trans, lp):
  """(path [B, T] int64, best log-joint [B]) of emission log-probs lp [B, T, S]; every
  argmax takes the lowest index among equal values (tf.argmax, np.argmax)."""
  b, t, k = lp.shape
  delta = log_init + lp[:, 0]
  back = np.zeros((b, t, k), np.int64)
  for s in range(1, t):
    cand = delta[:, :, None] + log_trans        # [B, from, to]
    back[:, s] = np.argmax(cand, axis=1)
    delta = lp[:, s] + np.max(cand, axis=1)
  path = np.zeros((b, t), np.int64)
  path[:, -1] = np.argmax(delta, axis=-1)
  for s in range(t - 1, 0, -1):
    path[:, s - 1] = back[np.arange(b), s, path[:, s]]
  return path, np.max(delta, axis=-1)


def viterbi_decode(acts):
  """posterior_mode of create_hmm's model for activations [B, T, 360]: (path, score)."""
  log_init, log_trans, emission = create_hmm()
  return viterbi(log_init, log_trans, multinomial_log_prob(acts, emission))


def path_score(path, acts):
  """log p(path, acts) [B] under create_hmm's model."""
  log_init, log_trans, emission = create_hmm()
  lp = multinomial_log_prob(acts, emission)
  path = np.asarray(path)
  b, t = path.shape
  rows = np.arange(b)
  out = log_init[path[:, 0]] + lp[rows, 0, path[:, 0]]
  for s in range(1, t):
    out = out + log_trans[path[:, s - 1], path[:, s]] + lp[rows, s, path[:, s]]
  return out


# ---- f0 and confidence ----------------------------------------------------------------
CENTS = (np.linspace(0, 7180, BINS) + 1997.3794084376191).astype(np.float32).astype(
    np.float64)


def activations_to_f0_and_confidence(acts, centers=None):
  """(f0_hz [M], confidence [M, 1]) in float64 over the float32 cents table."""
  acts = np.asarray(acts, np.float64)
  confidence = acts.max(-1, keepdims=True)
  centers = np.argmax(acts, -1) if centers is None else np.asarray(centers)
  idx = centers.astype(np.int64)[:, None] - 4 + np.arange(10)[None, :]
  idx = np.clip(idx, 0, BINS - 1)
  w = np.take_along_axis(acts, idx, axis=1)
  with np.errstate(invalid='ignore', divide='ignore'):
    f0_cent = np.sum(w * CENTS[idx], -1) / np.sum(w, -1)
  return 10.0 * 2.0 ** (f0_cent / 1200.0), confidence


# ---- the shim's tfp ------------------------------------------------------------------
def _np(x):
  return np.asarray(x.numpy() if hasattr(x, 'numpy') else x, np.float64)


class ShimMultinomial:
  """tfd.Multinomial(total_count, probs=...) as create_hmm builds it."""

  def __init__(self, total_count, probs=None, **_):
    assert float(_np(total_count)) == 1.0, total_count
    self.probs = _np(probs)


class ShimHiddenMarkovModel:
  """tfd.HiddenMarkovModel(Categorical, Categorical, Multinomial, num_steps):
  posterior_mode by the dense Viterbi of this module, returning a shim tensor."""

  def __init__(self, initial_distribution, transition_distribution,
               observation_distribution, num_steps, **_):
    self.initial_distribution = initial_distribution
    self.transition_distribution = transition_distribution
    self.observation_distribution = observation_distribution
    self.num_steps = num_steps

  def posterior_mode(self, x):
    import tensorflow as tf   # the shim, imported by the generator before this call
    probs = self.observation_distribution.probs.reshape(BINS, BINS)
    lp = multinomial_log_prob(_np(x), probs)
    assert lp.shape[1] == self.num_steps
    path, _ = viterbi(self.initial_distribution.log_probs(),
                      self.transition_distribution.log_probs(), lp)
    return tf.constant(path)
