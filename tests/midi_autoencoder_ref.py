"""Float64 restatements of nn.DilatedConvStack's pieces (nn.py:1075-1323) for
tests/test_dilated_conv.py: TensorFlow's 'same' dilated convolution along time,
normalize_op, the residual site and the whole stack, plain or conditional, from a
built module's parameters."""
import torch
import torch.nn.functional as F

GROUPS = {'layer': lambda c: 1, 'group': lambda c: 32, 'instance': lambda c: c}


def conv_time(x, kernel, bias, dilation):
  """Conv2D(ch, (k, 1), dilation_rate=(d, 1), padding='same') of x [B, T, C]: kernel
  [k, 1, C, ch]; TensorFlow pads (k - 1) d, the odd element after."""
  k = kernel.shape[0]
  total = (k - 1) * dilation
  xp = F.pad(x.transpose(1, 2), (total // 2, total - total // 2))
  return F.conv1d(xp, kernel[:, 0].permute(2, 1, 0), bias, dilation=dilation).transpose(1, 2)


def normalize(y, norm_type, eps=1e-5):
  """normalize_op of y [B, T, C]; None is y itself."""
  if norm_type is None:
    return y
  b, t, c = y.shape
  g = GROUPS[norm_type](c)
  v = y.reshape(b, t, g, c // g)
  var, mean = torch.var_mean(v, dim=(1, 3), correction=0, keepdim=True)
  return ((v - mean) / torch.sqrt(var + eps)).reshape(b, t, c)


def site(y, x, norm_type, s, h):
  """x + normalize(y) s + h and its ReLU."""
  x_next = x + normalize(y, norm_type) * s + h
  return x_next, torch.relu(x_next)


def film_split(film, c, shift_only):
  return (1.0, film) if shift_only else (film[..., :c], film[..., c:])


def stack(module, x, z=None):
  """nn.DilatedConvStack `module` (built) on float64 x [B, T, C_in] (and z), with its
  parameters as float64 CPU leaves: (output, {parameter name: leaf})."""
  leaves = {n: p.detach().double().cpu().requires_grad_(True)
            for n, p in module.named_parameters()}

  def p(name):
    return leaves[name]

  h = conv_time(x, p('conv_in.kernel'), p('conv_in.bias'), 1)
  c = h.shape[-1]
  if z is not None and z.dim() == 2:
    z = z[:, None, :]
  for i, layer in enumerate(module.layers):
    y = conv_time(torch.relu(h), p(f'layers.{i}.kernel'), p(f'layers.{i}.bias'),
                  layer.dilation_rate[0])
    if module.conditional:
      pre = f'norms.{i}.conditional_scale_and_shift.dense.'
      film = torch.matmul(z, p(pre + 'kernel')) + p(pre + 'bias')
      s, sh = film_split(film, c, module.shift_only)
    else:
      s, sh = p(f'norms.{i}.scale').reshape(c), p(f'norms.{i}.shift').reshape(c)
    h, _ = site(y, h, module.norm_type, s, sh)
  return h, leaves
