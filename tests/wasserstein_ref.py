"""Float64 torch restatement of the reference's `losses.wasserstein_distance` and
`losses.WassersteinConsistencyLoss` (losses.py:584-686), step for step: sort the union,
searchsorted(side='right') into each side's sorted values, gather the zero-padded
cumulative weights, and sum delta |U - V|^p.  Its gradients are torch autograd's.  The
sorts are stable, as TensorFlow's -top_k(-x) is, so a tie keeps concat order (u before
v, lower index first) and the value gradients land where the reference's do.  Pinned to
the unmodified reference by tests/golden/wasserstein.npz."""
import numpy as np
import torch


def t64(x):
  if torch.is_tensor(x):
    return x if x.dtype == torch.float64 else x.detach().cpu().double()
  return torch.as_tensor(np.asarray(x, np.float64))


def _cdf(values, weights, points):
  """The cumulative weights of `values` at or below each of `points` (raw, not
  normalised: the reference discards its safe_divide)."""
  sorted_values, sorter = torch.sort(values, dim=-1, stable=True)
  idx = torch.searchsorted(sorted_values.detach().contiguous(), points.detach().contiguous(),
                           right=True)
  cum = torch.cumsum(torch.gather(weights, -1, sorter), dim=-1)
  cum = torch.cat([torch.zeros_like(cum[..., :1]), cum], dim=-1)
  return torch.gather(cum, -1, idx)


def wasserstein_distance(u_values, v_values, u_weights, v_weights, p=1.0):
  u, v, wu, wv = (t64(x) for x in (u_values, v_values, u_weights, v_weights))
  all_values, _ = torch.sort(torch.cat([u, v], dim=-1), dim=-1, stable=True)
  deltas = all_values[..., 1:] - all_values[..., :-1]
  points = all_values[..., :-1]
  u_cdf = _cdf(u, wu, points)
  v_cdf = _cdf(v, wv, points)
  return torch.sum(deltas * torch.abs(u_cdf - v_cdf)**p, dim=-1)**(1.0 / p)


def hz_to_midi(f):
  f = t64(f)
  notes = 12.0 * (torch.log2(torch.where(f <= 0.0, torch.full_like(f, 1e-5), f)) -
                  np.log2(440.0)) + 69.0
  return torch.where(f <= 0.0, torch.zeros_like(notes), notes)


def wasserstein_consistency(amps_a, freqs_a, amps_b, freqs_b, weight=1.0, midi=True):
  if not (weight > 0.0 and midi):
    return torch.tensor(0.0, dtype=torch.float64)
  dist = wasserstein_distance(hz_to_midi(freqs_a), hz_to_midi(freqs_b), t64(amps_a),
                              t64(amps_b), p=1.0)
  return torch.mean(weight * dist)
