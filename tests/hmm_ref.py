"""Float64 restatement of losses.HmmTranscriber (losses.py:247-345) and of the parts of
tfp it runs on: Categorical, MultivariateNormalDiag and HiddenMarkovModel's log_prob and
posterior_mode, in the dense K x K formulation (the structure the CUDA kernels exploit
is deliberately not used).  Differentiable: the tests take float64 autograd gradients of
`log_prob`.  Pinned two ways: to the unmodified reference by tests/golden/hmm.npz, and
by brute-force enumeration of every path at K <= 3, T <= 7 (tests/test_hmm_transcriber.py).

`ShimCategorical`, `ShimMultivariateNormalDiag` and `ShimHiddenMarkovModel` wrap the same
functions for the reference run on the NumPy TensorFlow shim
(tests/golden/make_hmm_golden.py installs them there for that run only).
"""
import itertools
import math

import numpy as np
import torch

F64 = torch.float64
LOG_2PI = math.log(2.0 * math.pi)


def t64(x):
  return x.to(F64) if torch.is_tensor(x) else torch.as_tensor(np.asarray(x), dtype=F64)


def transcriber_params(avg_length=200, midi_std=0.5, amps_on_center=1.5, amps_on_scale=0.5,
                       amps_off_center=0.0, amps_off_scale=0.1, n_pitches=128, **_):
  """HmmTranscriber.__init__: (log initial [K], log transitions [K, K], loc [K, 2],
  scale [K, 2]), the transition rows normalised as the reference does."""
  k = n_pitches
  hold = 1.0 - 1.0 / avg_length
  other = (1.0 - hold) / (k - 1)
  trans = (hold - other) * torch.eye(k, dtype=F64) + other * torch.ones((k, k), dtype=F64)
  trans = trans / trans.sum(1, keepdim=True)
  loc = torch.stack([torch.cat([torch.tensor([k / 2.0], dtype=F64),
                                torch.arange(1, k, dtype=F64)]),
                     torch.tensor([amps_off_center] + [amps_on_center] * (k - 1),
                                  dtype=F64)], -1)
  scale = torch.stack([torch.tensor([float(k)] + [midi_std] * (k - 1), dtype=F64),
                       torch.tensor([amps_off_scale] + [amps_on_scale] * (k - 1),
                                    dtype=F64)], -1)
  return (torch.full((k,), -math.log(k), dtype=F64), torch.log(trans), loc, scale)


def mvn_diag_log_prob(x, loc, scale):
  """MultivariateNormalDiag(loc, scale).log_prob(x[..., None, :]): [..., K]."""
  z = (t64(x)[..., None, :] - loc) / scale
  return torch.sum(-0.5 * z * z - torch.log(scale) - 0.5 * LOG_2PI, -1)


def log_prob(x, log_init, log_trans, loc, scale):
  """HiddenMarkovModel.log_prob of x [B, T, 2]: the forward algorithm, [B]."""
  lp = mvn_diag_log_prob(x, loc, scale)
  alpha = log_init + lp[:, 0]
  for t in range(1, lp.shape[1]):
    alpha = lp[:, t] + torch.logsumexp(alpha[:, :, None] + log_trans, dim=1)
  return torch.logsumexp(alpha, dim=-1)


def posterior_mode(x, log_init, log_trans, loc, scale):
  """HiddenMarkovModel.posterior_mode of x [B, T, 2] by Viterbi, [B, T] int64; every
  argmax takes the lowest index among equal values (np.argmax)."""
  lp = mvn_diag_log_prob(x, loc, scale).detach().numpy()
  lt = log_trans.detach().numpy()
  b, t, k = lp.shape
  delta = log_init.detach().numpy() + lp[:, 0]
  back = np.zeros((b, t, k), np.int64)
  for s in range(1, t):
    cand = delta[:, :, None] + lt                  # [B, from, to]
    back[:, s] = np.argmax(cand, axis=1)
    delta = lp[:, s] + np.max(cand, axis=1)
  path = np.zeros((b, t), np.int64)
  path[:, -1] = np.argmax(delta, axis=-1)
  for s in range(t - 1, 0, -1):
    path[:, s - 1] = back[np.arange(b), s, path[:, s]]
  return path


def log_joint(path, x, log_init, log_trans, loc, scale):
  """log p(path, x) [B] of state paths [B, T]."""
  lp = mvn_diag_log_prob(x, loc, scale).detach().numpy()
  lt = log_trans.detach().numpy()
  path = np.asarray(path)
  b, t = path.shape
  rows = np.arange(b)
  out = log_init.detach().numpy()[path[:, 0]] + lp[rows, 0, path[:, 0]]
  for s in range(1, t):
    out = out + lt[path[:, s - 1], path[:, s]] + lp[rows, s, path[:, s]]
  return out


def brute_force(x, log_init, log_trans, loc, scale):
  """(log_prob [B], best path [B, T], gap [B]) by enumerating all K^T paths; gap is the
  best log-joint's margin over the second best (the path is unique where it is > 0)."""
  x = t64(x)
  b, t, _ = x.shape
  k = loc.shape[0]
  paths = np.array(list(itertools.product(range(k), repeat=t)), np.int64)
  lps, best, gap = [], [], []
  for i in range(b):
    joint = log_joint(paths, x[i:i + 1].expand(len(paths), t, 2), log_init, log_trans,
                      loc, scale)
    order = np.argsort(-joint, kind='stable')
    lps.append(np.logaddexp.reduce(joint))
    best.append(paths[order[0]])
    gap.append(joint[order[0]] - joint[order[1]])
  return np.array(lps), np.stack(best), np.array(gap)


# ---- the shim's tfp ------------------------------------------------------------------
def _np(x):
  return np.asarray(x.numpy() if hasattr(x, 'numpy') else x, np.float64)


class ShimCategorical:
  """tfd.Categorical(probs=...) or (logits=...); `log_probs()` is log(probs)."""

  def __init__(self, logits=None, probs=None, **_):
    self._logits = None if logits is None else _np(logits)
    self._probs = None if probs is None else _np(probs)

  def log_probs(self):
    if self._logits is not None:
      return self._logits - np.logaddexp.reduce(self._logits, axis=-1, keepdims=True)
    with np.errstate(divide='ignore'):
      return np.log(self._probs)


class ShimMultivariateNormalDiag:

  def __init__(self, loc, scale_diag, **_):
    self.loc = _np(loc)
    self.scale_diag = _np(scale_diag)


class ShimHiddenMarkovModel:
  """tfd.HiddenMarkovModel(Categorical, Categorical, MultivariateNormalDiag, num_steps):
  log_prob and posterior_mode of this module, returning shim tensors."""

  def __init__(self, initial_distribution, transition_distribution,
               observation_distribution, num_steps, name='HiddenMarkovModel', **_):
    self.initial_distribution = initial_distribution
    self.transition_distribution = transition_distribution
    self.observation_distribution = observation_distribution
    self.num_steps = num_steps
    self.name = name

  def _params(self):
    obs = self.observation_distribution
    return (t64(self.initial_distribution.log_probs()),
            t64(self.transition_distribution.log_probs()), t64(obs.loc),
            t64(obs.scale_diag))

  def log_prob(self, x):
    import tensorflow as tf   # the shim, imported by the generator before this call
    return tf.constant(log_prob(t64(_np(x)), *self._params()).numpy())

  def posterior_mode(self, x):
    import tensorflow as tf
    return tf.constant(posterior_mode(t64(_np(x)), *self._params()))
