"""References for the modulated delay (core.variable_length_delay, core.py:1285-1314 on
core.linear_lookup, 1168-1214; effects.ModDelay.get_signal, effects.py:328-394).

TEST INFRASTRUCTURE.  Two kinds, kept in one place because they restate one formula:

* NumPy (`variable_length_delay`, `mod_delay_get_signal`), in the two modes of
  oracle/ddsp_oracle.py: np.float64, the closed form of the reference's
  interpolation and the arbiter of the parity gate; np.float32, the reference's own
  TF-order arithmetic.  tests/test_mod_delay.py pins both to the unmodified
  reference run on the shim (tests/golden/mod_delay.npz).
* float64 torch (`torch_variable_length_delay`, `torch_mod_delay`), differentiable,
  the reference of the backward kernel ("what TF autodiff gives the reference"),
  pinned to the NumPy closed form at <= 1e-12.
"""
import numpy as np
import torch


def _per_sample(x, shape, dtype):
  """[B, N, 1] / [B, N] / [B, 1, 1] / [B, 1] -> [B, N] (TF's broadcast)."""
  x = np.asarray(x, dtype)
  if x.ndim == 3:
    x = x[..., 0]
  return np.broadcast_to(x, shape)


def variable_length_delay(phase, audio, max_length=512, dtype=np.float64):
  """core.variable_length_delay (core.py:1285-1314) on core.linear_lookup.

  float64: the closed form of the reference's interpolation over the L + 1 reversed
  frame columns (column L is column 0 appended, so it reads x[t]): with
  pos = phase * L, out(t) = (1 - frac) v_j0 + frac v_{j0+1}, v_j = x[t - j] for
  0 <= j < L (0 before the start), v_L = x[t], v_j = 0 outside [0, L].
  float32: TF order - zero pad, frame with step 1, reverse, append the wrap column,
  |phase - linspace(0, 1, L + 1)| * L, relu(1 - .), weighted sum over the L + 1
  columns, every op in float32 with the [B, N, L + 1] intermediates (small shapes
  only)."""
  L = int(max_length)
  x = np.asarray(audio, dtype)
  b, n = x.shape
  ph = _per_sample(phase, (b, n), dtype)
  if dtype == np.float32:
    padded = np.concatenate([np.zeros((b, L - 1), np.float32), x], axis=1)
    idx = np.arange(n)[:, None] + np.arange(L)[None, :]
    frames = padded[:, idx][..., ::-1]
    frames = np.concatenate([frames, frames[..., 0:1]], axis=-1)
    delta = np.float32(1.0) / np.float32(L)
    lin = np.concatenate([delta * np.arange(L, dtype=np.float32),
                          np.ones((1,), np.float32)]).astype(np.float32)
    dist = np.abs(ph[:, :, None] - lin[None, None, :]) * np.float32(L)
    weights = np.maximum(np.float32(1.0) - dist, np.float32(0.0))
    return np.sum(weights * frames, axis=-1).astype(np.float32)
  pos = ph * L
  j0 = np.clip(np.floor(pos), -2, L + 2)
  frac = pos - j0
  t = np.arange(n)[None, :]

  def tap(j):
    src = np.where(j == L, t, t - j)
    ok = (j >= 0) & (j <= L) & (src >= 0)
    return np.where(ok, np.take_along_axis(x, np.clip(src, 0, n - 1).astype(np.int64),
                                           axis=1), 0.0)
  return (1.0 - frac) * tap(j0) + frac * tap(j0 + 1)


def mod_delay_get_signal(audio, gain, phase, center_ms=15.0, depth_ms=10.0,
                         sample_rate=16000, add_dry=True, dtype=np.float64):
  """effects.ModDelay.get_signal (effects.py:368-394) on scaled controls: the phase
  mapping `phase * depth / max + center / max` (float32 ops in float32 mode), the
  delay, the gain (a 3-D gain loses its channel axis) and the dry mix."""
  max_delay_ms = center_ms + depth_ms
  L = int(sample_rate / 1000.0 * max_delay_ms)
  ph = np.asarray(phase, dtype)
  ph = ph * dtype(depth_ms / max_delay_ms) + dtype(center_ms / max_delay_ms)
  x = np.asarray(audio, dtype)
  wet = variable_length_delay(ph, x, L, dtype=dtype)
  g = np.asarray(gain, dtype)
  if g.ndim == 3:
    g = g[..., 0]
  wet = (wet * g).astype(dtype)
  return (wet + x).astype(dtype) if add_dry else wet


def torch_variable_length_delay(phase, audio, max_length):
  """core.variable_length_delay (core.py:1285-1314) in float64 torch ops, phase and
  audio [B, N]: `variable_length_delay`'s closed form, with TensorFlow's
  subgradients - the position's gradient is 0 where phase * L is an integer
  (abs'(0) = relu'(0) = 0 in the reference's relu(1 - |pos - j|))."""
  L = int(max_length)
  b, n = audio.shape
  pos = phase * L
  j0 = torch.clamp(torch.floor(pos.detach()), -2, L + 2)
  frac = pos - j0
  frac = torch.where(frac.detach() == 0, frac.detach(), frac)
  t = torch.arange(n, device=audio.device)[None, :]

  def tap(j):
    j = j.long()
    src = torch.where(j == L, t, t - j)
    ok = (j >= 0) & (j <= L) & (src >= 0)
    v = torch.gather(audio, 1, torch.clamp(src, 0, n - 1))
    return torch.where(ok, v, torch.zeros_like(v))
  return (1.0 - frac) * tap(j0) + frac * tap(j0 + 1)


def torch_mod_delay(audio, gain, phase, max_length, scale=1.0, offset=0.0, add_dry=False):
  """`[add_dry] audio + gain * variable_length_delay(phase * scale + offset)` in
  float64 torch ops (ModDelay.get_signal, effects.py:368-394; gain None = 1).  The
  mapped phase takes the value of the reference's float32 arithmetic (two
  roundings) and the derivative of the exact map: a float64 map would move a
  position across a knot now and then, where the interpolation's gradient jumps."""
  exact = phase * scale + offset
  p32 = phase.detach().to(torch.float32)
  mapped = (p32 * torch.tensor(scale, dtype=torch.float32)
            + torch.tensor(offset, dtype=torch.float32)).to(torch.float64)
  wet = torch_variable_length_delay(exact + (mapped - exact).detach(), audio, max_length)
  if gain is not None:
    wet = wet * gain
  return wet + audio if add_dry else wet
