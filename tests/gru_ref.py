"""Float64 restatement of tf.keras.layers.GRU with TF2's defaults (reset_after=True, gate
columns z | r | h, h0 = 0), differentiable by torch autograd:
  z = sigmoid(x W_z + b_z + h U_z + c_z),  r = sigmoid(x W_r + b_r + h U_r + c_r),
  h~ = tanh(x W_h + b_h + r * (h U_h + c_h)),  h' = z * h + (1 - z) * h~."""
import torch


def gru(x, kernel, recurrent_kernel, bias):
  """Every state [B, T, H] of the GRU over x [B, T, in] (tensors of any float dtype and
  device; float64 for a reference)."""
  h_units = recurrent_kernel.shape[0]
  xw = torch.matmul(x, kernel) + bias[0]
  h = torch.zeros(x.shape[0], h_units, dtype=x.dtype, device=x.device)
  out = []
  for t in range(x.shape[1]):
    hu = h @ recurrent_kernel + bias[1]
    xz, xr, xh = torch.split(xw[:, t], h_units, dim=-1)
    uz, ur, uh = torch.split(hu, h_units, dim=-1)
    z = torch.sigmoid(xz + uz)
    r = torch.sigmoid(xr + ur)
    hc = torch.tanh(xh + r * uh)
    h = z * h + (1.0 - z) * hc
    out.append(h)
  return torch.stack(out, dim=1)


def torch_gru_weights(kernel, recurrent_kernel, bias):
  """The same weights for torch.nn.GRU: its gates are ordered r | z | n, its matrices are
  transposed, and its b_hn sits inside r * (h W_hn + b_hn) as Keras's c_h does."""
  def reorder(m):
    z, r, h = torch.chunk(m, 3, dim=-1)
    return torch.cat([r, z, h], dim=-1)
  return {'weight_ih_l0': reorder(kernel).t(), 'weight_hh_l0': reorder(recurrent_kernel).t(),
          'bias_ih_l0': reorder(bias[0]), 'bias_hh_l0': reorder(bias[1])}


def random_weights(n_in, units, seed, dtype=torch.float64, scale=1.0):
  """Keras-like random weights: glorot-uniform kernel, orthogonal recurrent kernel and a
  non-zero bias, so that every bias term is exercised."""
  g = torch.Generator().manual_seed(seed)
  lim = (6.0 / (n_in + 3 * units))**0.5
  kernel = (torch.rand((n_in, 3 * units), generator=g, dtype=torch.float64) * 2 - 1) * lim
  q, _ = torch.linalg.qr(torch.randn((3 * units, units), generator=g, dtype=torch.float64))
  recurrent_kernel = q.t().contiguous() * scale
  bias = 0.1 * torch.randn((2, 3 * units), generator=g, dtype=torch.float64)
  return kernel.to(dtype), recurrent_kernel.to(dtype), bias.to(dtype)
