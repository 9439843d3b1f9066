"""nn.normalize_relu on the fused kernel of csrc/norm.cuh, the ResNet's layers and the two
inverse-synthesis encoders.  On the CPU: TensorFlow's 'same' padding, the layers' names,
shapes and initialisers, the refusals, and the C ABI's refusals in a process without a
device.  On the GPU: the kernel's forward and every gradient against float64 at every
site shape of the 'small' ResNet and at the edges of its geometry, its determinism and
coverage, and each ResidualLayer and both encoders against the float64 restatement
(tests/inverse_synthesis_ref.py)."""
import json
import os
import subprocess
import sys

import pytest
import torch

from ddsp_b200 import _lib, core, encoders, nn, spectral_ops
from tests import inverse_synthesis_ref as ref
from tests.util import rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu


# ---- CPU ---------------------------------------------------------------------------
# Every (width, kernel, stride) the 'small', 'medium' and 'large' ResNets meet on a
# 229-bin log-mel, with TensorFlow's padding: (pad before, pad after).
SAME = [(229, 7, 2, (3, 3)), (115, 3, 2, (1, 1)), (58, 3, 2, (0, 1)), (29, 3, 2, (1, 1)),
        (15, 3, 2, (1, 1)), (58, 1, 2, (0, 0)), (29, 1, 2, (0, 0)), (15, 1, 2, (0, 0)),
        (125, 7, 1, (3, 3)), (125, 3, 1, (1, 1)), (125, 1, 1, (0, 0)), (58, 3, 1, (1, 1)),
        (8, 1, 1, (0, 0))]


@pytest.mark.parametrize('size,k,s,want', SAME)
def test_same_padding_is_tensorflows(size, k, s, want):
  assert nn.same_padding(size, k, s) == want
  assert ref.tf_same(size, k, s) == want
  out = -(-size // s)
  assert (size + sum(want) - k) // s + 1 == out


@pytest.mark.parametrize('size,k,s,want', SAME)
def test_conv_and_pool_widths_on_the_cpu(size, k, s, want):
  x = torch.randn(1, 2, size, 3)
  conv = nn.Conv2D(5, (1, k), (1, s))
  y = conv(x)
  assert y.shape == (1, 2, -(-size // s), 5) and y.is_contiguous()
  torch.testing.assert_close(y, ref.conv2d(x, conv.kernel, conv.bias, (1, s)))
  pool = nn.MaxPool2D((1, k), (1, s))
  torch.testing.assert_close(pool(x), ref.max_pool(x, (1, k), (1, s)))


def test_conv2d_parameters_and_initialiser():
  conv = nn.Conv2D(64, (7, 7), (1, 2))
  conv(torch.zeros(1, 3, 20, 2))
  assert conv.kernel.shape == (7, 7, 2, 64) and conv.bias.shape == (64,)
  limit = (6.0 / (49 * 2 + 49 * 64))**0.5
  assert conv.kernel.abs().max() <= limit and conv.kernel.abs().max() > 0.9 * limit
  assert not conv.bias.any()
  with pytest.raises(ValueError):
    conv(torch.zeros(1, 3, 20, 5))
  with pytest.raises(NotImplementedError):
    nn.Conv2D(4, 3, padding='valid')


def _small_names():
  names = ['layers.0.kernel', 'layers.0.bias']
  for stack, blocks in (('layers.2.', [2, 3, 4]), ('layers.3.', [3])):
    i = 0
    for n in blocks:
      for j in range(n):
        p = f'{stack}layers.{i}.'
        names += [p + 'norm_input.scale', p + 'norm_input.shift']
        if j == 0:
          names += [p + 'conv_proj.kernel', p + 'conv_proj.bias']
        names += [p + 'bottleneck.0.kernel', p + 'bottleneck.0.bias']
        for b in (1, 2):
          names += [f'{p}bottleneck.{b}.norm.scale', f'{p}bottleneck.{b}.norm.shift',
                    f'{p}bottleneck.{b}.conv.kernel', f'{p}bottleneck.{b}.conv.bias']
        i += 1
    names += [f'{stack}layers.{i}.scale', f'{stack}layers.{i}.shift']
  return names


def test_resnet_structure_names_and_shapes():
  net = nn.ResNet('small')
  # built by hand on the CPU: every lazy layer takes its input width
  assert len(net.layers[2].layers) == 10 and len(net.layers[3].layers) == 4
  norms = [m for m in net.modules() if isinstance(m, nn.NormRelu)]
  assert len(norms) == 3 * 12 + 2
  layer = net.layers[2].layers[2]   # the first layer of the 64-channel block
  assert layer.shortcut and layer.bottleneck[1].conv.strides == (1, 2)
  assert layer.conv_proj.filters == 256 and layer.conv_proj.kernel_size == (1, 1)
  assert not net.layers[2].layers[3].shortcut
  assert net.layers[1].pool_size == (1, 3) and net.layers[1].strides == (1, 2)
  assert [net.layers[3].layers[0].bottleneck[i].conv.filters for i in (1, 2)] == [256, 1024]


def test_resnet_refusals():
  with pytest.raises(KeyError):
    nn.ResNet('tiny')
  with pytest.raises(KeyError):
    encoders.ResnetSinusoidalEncoder()   # the reference's default size 'tiny'
  for cls, args in ((nn.ResNet, ('small',)), (nn.ResidualStack, ([32], [1], [1], 'layer')),
                    (nn.ResidualLayer, (32, 1, True, 'layer'))):
    with pytest.raises(NotImplementedError):
      cls(*args, conditional=True)
  with pytest.raises(NotImplementedError):
    nn.ResidualStack([32], [1], [1], 'layer', nonlinearity='leaky_relu')


def test_normalize_relu_refusals_on_the_cpu():
  x = torch.zeros(1, 2, 3, 8)
  with pytest.raises(ValueError, match='CUDA'):
    nn.normalize_relu(x, torch.ones(8), torch.zeros(8))
  with pytest.raises(ValueError):
    nn.normalize_relu(torch.zeros(2, 8), torch.ones(8), torch.zeros(8))


def test_rnn_sandwich_layers():
  net = nn.RnnSandwich()
  assert isinstance(net[0], nn.FcStack) and isinstance(net[1], nn.Rnn)
  assert isinstance(net[2], nn.FcStack) and net[1].rnn.units == 512
  assert len(net[0]) == 2 and net[0][0][0].units == 256


@pytest.mark.parametrize('c,g', [(c, g) for c in (0, 2, 4, 6, 8, 32, 36, 1024, 2048, 2052)
                                 for g in (0, 1, 3, 4, 32, c)])
def test_takes_query(c, g):
  lib = _lib.load()
  want = c >= 4 and c <= 2048 and c % 4 == 0 and g >= 1 and c % g == 0
  assert lib.ddsp_b200_norm_relu_takes(c, g) == int(want)


def test_inverse_synthesis_bounds_are_taken():
  """InverseSynthesis's FilteredNoise (125 frames, 65 bands, 64000 samples, window 0) and
  its GRU (512 units) train only while their kernels take these shapes."""
  lib = _lib.load()
  assert lib.ddsp_b200_filtered_noise_backward_takes(125, 65, 64000, 0) == 1
  assert lib.ddsp_b200_gru_takes(512) == 1


def _abi_refusals():
  lib = _lib.load()
  calls = {
      'forward_channels': lambda: lib.ddsp_b200_norm_relu_forward(
          16, 16, 16, 1 << 20, 2 << 20, 3 << 20, 2, 3, 6, 1, 1e-5, None),
      'forward_groups': lambda: lib.ddsp_b200_norm_relu_forward(
          16, 16, 16, 1 << 20, 2 << 20, 3 << 20, 2, 3, 8, 3, 1e-5, None),
      'forward_shape': lambda: lib.ddsp_b200_norm_relu_forward(
          16, 16, 16, 1 << 20, 2 << 20, 3 << 20, -1, 3, 8, 1, 1e-5, None),
      'forward_align': lambda: lib.ddsp_b200_norm_relu_forward(
          20, 16, 16, 1 << 20, 2 << 20, 3 << 20, 2, 3, 8, 1, 1e-5, None),
      'forward_null': lambda: lib.ddsp_b200_norm_relu_forward(
          16, None, 16, 1 << 20, 2 << 20, 3 << 20, 2, 3, 8, 1, 1e-5, None),
      'forward_overlap': lambda: lib.ddsp_b200_norm_relu_forward(
          1 << 20, 16, 32, 1 << 20, 2 << 20, 3 << 20, 2, 3, 8, 1, 1e-5, None),
      'backward_workspace': lambda: lib.ddsp_b200_norm_relu_backward(
          1 << 20, 16, 32, 48, 64, 2 << 20, 3 << 20, 4 << 20, 5 << 20, 6 << 20,
          4 * 2 * 8 * 2 * 8 - 4, 2, 3, 8, 1, None),
      'backward_overlap': lambda: lib.ddsp_b200_norm_relu_backward(
          1 << 20, 16, 32, 48, 64, 2 << 20, 1 << 20, 4 << 20, 5 << 20, 6 << 20,
          4 * 2 * 8 * 2 * 8, 2, 3, 8, 1, None),
      'backward_channels': lambda: lib.ddsp_b200_norm_relu_backward(
          1 << 20, 16, 32, 48, 64, 2 << 20, 3 << 20, 4 << 20, 5 << 20, 6 << 20,
          1 << 16, 2, 3, 4096, 1, None),
      'forward_empty': lambda: lib.ddsp_b200_norm_relu_forward(
          None, None, None, None, None, None, 0, 3, 8, 1, 1e-5, None),
  }
  rows = {}
  for name, call in calls.items():
    before = lib.ddsp_b200_launch_count()
    rc = call()
    rows[name] = [rc, lib.ddsp_b200_last_error().decode(), lib.ddsp_b200_launch_count() - before]
  return rows


def test_abi_refusals_without_a_device():
  proc = subprocess.run(
      [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [
          '-c', 'import json; from tests.test_norm_relu import _abi_refusals; '
                'print(json.dumps(_abi_refusals()))'],
      cwd=ROOT, env=dict(os.environ, CUDA_VISIBLE_DEVICES=''), capture_output=True,
      text=True)
  assert proc.returncode == 0, proc.stderr
  rows = json.loads(proc.stdout.strip().splitlines()[-1])
  want = {
      'forward_channels': (_lib.E_UNSUPPORTED, 'C=6 channels in G=1 groups'),
      'forward_groups': (_lib.E_UNSUPPORTED, 'C=8 channels in G=3 groups'),
      'forward_shape': (_lib.E_INVALID, 'norm_relu_forward: bad shape'),
      'forward_align': (_lib.E_INVALID, 'must be 16-byte aligned'),
      'forward_null': (_lib.E_INVALID, 'norm_relu_forward: null pointer'),
      'forward_overlap': (_lib.E_INVALID, 'y must not overlap x'),
      'backward_workspace': (_lib.E_INVALID, 'the workspace has'),
      'backward_overlap': (_lib.E_INVALID, 'dx must not overlap x'),
      'backward_channels': (_lib.E_UNSUPPORTED, 'C=4096'),
      'forward_empty': (0, ''),
  }
  for name, (rc, msg) in want.items():
    assert rows[name][0] == rc, (name, rows[name])
    assert msg in rows[name][1], (name, rows[name])
    assert rows[name][2] == 0, name


# ---- GPU: the kernel ---------------------------------------------------------------
# (H, W, C) of every Normalize -> ReLU site of the 'small' ResNet at T = 125.
SITES = [(125, 58, 64), (125, 58, 32), (125, 58, 128), (125, 29, 64), (125, 29, 256),
         (125, 29, 128), (125, 15, 128), (125, 15, 512), (125, 15, 256), (125, 8, 256),
         (125, 8, 1024)]
EDGES = [(1, 1, 1, 4), (2, 3, 5, 4), (1, 1, 1, 32), (3, 1, 1, 1024), (1, 7, 9, 32),
         (64, 5, 6, 32), (64, 2, 3, 4), (2, 1, 1, 2048), (2, 11, 13, 36), (1, 125, 8, 1024)]
NORMS = ('layer', 'group', 'instance')


def _inputs(b, h, w, c, seed, mean=0.0):
  g = torch.Generator().manual_seed(seed)
  x = mean + torch.randn((b, h, w, c), generator=g, dtype=torch.float64)
  scale = 1.0 + 0.5 * torch.randn(c, generator=g, dtype=torch.float64)
  shift = 0.5 * torch.randn(c, generator=g, dtype=torch.float64)
  up = torch.randn((b, h, w, c), generator=g, dtype=torch.float64)
  x = x.float().double()   # the float32 values both sides see
  return [v.cuda() for v in (x, scale, shift, up)]


def _ours(x, scale, shift, up, norm_type):
  ins = [v.float().requires_grad_(True) for v in (x, scale, shift)]
  y = nn.normalize_relu(*ins, norm_type)
  y.backward(up.float())
  return [y.detach()] + [v.grad for v in ins]


def _float64(x, scale, shift, up, norm_type):
  ins = [v.clone().requires_grad_(True) for v in (x, scale, shift)]
  y = ref.norm_relu(*ins, norm_type)
  y.backward(up)
  return [y.detach()] + [v.grad for v in ins]


def _check(got, want, tol=(1e-4, 1e-5), grad_tol=(2e-3, 1e-4)):
  for name, g, w in zip(('y', 'dx', 'dscale', 'dshift'), got, want):
    emax, el2 = rel_err(g.cpu().numpy(), w.cpu().numpy())
    t = tol if name == 'y' else grad_tol
    assert emax < t[0] and el2 < t[1], (name, emax, el2)


@gpu
@pytest.mark.parametrize('norm_type', NORMS)
@pytest.mark.parametrize('h,w,c', SITES, ids=[f'{h}x{w}x{c}' for h, w, c in SITES])
def test_sites_against_float64(h, w, c, norm_type):
  args = _inputs(2, h, w, c, seed=h + w + c)
  _check(_ours(*args, norm_type), _float64(*args, norm_type))


@gpu
@pytest.mark.parametrize('b,h,w,c', EDGES, ids=[f'B{b}-{h}x{w}x{c}' for b, h, w, c in EDGES])
def test_edges_against_float64(b, h, w, c):
  for norm_type in NORMS:
    if norm_type == 'group' and c % 32:
      continue
    args = _inputs(b, h, w, c, seed=b + h + w + c)
    if h * w * (c // {'layer': c, 'group': 32, 'instance': 1}[norm_type]) == 1:
      continue   # a single element per group: x - mean = 0, nothing to compare but eps
    _check(_ours(*args, norm_type), _float64(*args, norm_type))


@gpu
@pytest.mark.parametrize('norm_type', NORMS)
def test_large_mean_against_float64(norm_type):
  """Inputs of mean 1e3 and std 1: a sum / sum-of-squares variance would lose all of
  its digits here."""
  x, scale, shift, up = _inputs(3, 125, 29, 256, seed=7, mean=1e3)
  # no ReLU input near 0: the float32 input itself rounds x by 6e-5, which would move
  # elements across the ReLU's threshold
  scale = 1.0 + 0.1 * torch.rand_like(scale)
  shift = 10.0 + shift
  args = (x, scale, shift, up)
  _check(_ours(*args, norm_type), _float64(*args, norm_type), tol=(1e-3, 2e-4),
         grad_tol=(5e-3, 1e-3))


@gpu
@pytest.mark.parametrize('norm_type', NORMS)
def test_exact_relu_ties(norm_type):
  """Groups of constant x normalize to exactly 0, and with shift 0 the ReLU's input is
  exactly 0: y = 0 and no gradient passes there, as in torch and TensorFlow."""
  x, scale, shift, up = _inputs(2, 6, 7, 64, seed=3)
  x[0] = 2.5                     # item 0: every group constant
  x[1, ..., :32] = -1.0          # item 1: a constant half (one group, 16 instances)
  shift[:] = 0.0
  got = _ours(x, scale, shift, up, norm_type)
  want = _float64(x, scale, shift, up, norm_type)
  assert not got[0][0].any() and not got[1][0].any()
  _check(got, want)


def _launch(x, scale, shift, groups, up=None, fill=float('nan')):
  """The entry points' own outputs, every one first filled with `fill`."""
  b, h, w, c = x.shape
  y = torch.full_like(x, fill)
  mean = torch.full((b, groups), fill, device='cuda')
  rstd = torch.full_like(mean, fill)
  core._launch('ddsp_b200_norm_relu_forward', x, scale, shift, y, mean, rstd, b, h * w, c,
               groups, 1e-5)
  if up is None:
    return y, mean, rstd
  dx = torch.full_like(x, fill)
  dscale, dshift = torch.full_like(scale, fill), torch.full_like(shift, fill)
  ws = torch.full((2 * _lib.NORM_CLUSTER * b * c,), fill, device='cuda')
  core._launch('ddsp_b200_norm_relu_backward', x, scale, shift, mean, rstd, up, dx, dscale,
               dshift, ws, ws.numel() * 4, b, h * w, c, groups)
  return y, mean, rstd, dx, dscale, dshift


@gpu
@pytest.mark.parametrize('c,groups', [(4, 1), (32, 32), (64, 1), (1024, 32), (36, 9)])
def test_every_output_is_written(c, groups):
  x, scale, shift, up = [v.float().contiguous() for v in _inputs(5, 9, 7, c, seed=c)]
  for out in _launch(x, scale, shift, groups, up):
    assert not torch.isnan(out).any()


@gpu
def test_bitwise_reproducible_and_batch_independent():
  x, scale, shift, up = [v.float().contiguous() for v in _inputs(33, 125, 15, 512, seed=9)]
  first = _launch(x, scale, shift, 32, up)
  second = _launch(x, scale, shift, 32, up)
  for f, s in zip(first, second):
    assert torch.equal(f, s)
  for i in (0, 17, 32):
    alone = _launch(x[i:i + 1].contiguous(), scale, shift, 32, up[i:i + 1].contiguous())
    for k in (0, 1, 2, 3):   # y, mean, rstd, dx
      assert torch.equal(alone[k][0], first[k][i])


@gpu
def test_launches_per_call():
  """One launch forward; the backward's kernel and its parameter reduction."""
  count = _lib.load().ddsp_b200_launch_count
  x, scale, shift, up = _inputs(3, 10, 9, 64, seed=1)
  xf = x.float().requires_grad_(True)
  sf, tf = scale.float().requires_grad_(True), shift.float().requires_grad_(True)
  before = count()
  y = nn.normalize_relu(xf, sf, tf, 'group')
  assert count() - before == 1
  seen = {}
  y.register_hook(lambda g: seen.__setitem__('before', count()))
  xf.register_hook(lambda g: seen.__setitem__('after', count()))
  y.backward(up.float())
  assert seen['after'] - seen['before'] == 2


@gpu
def test_refusals_on_the_gpu():
  x = torch.zeros(2, 3, 4, 6, device='cuda')
  with pytest.raises(NotImplementedError):
    nn.normalize_relu(x, torch.ones(6, device='cuda'), torch.zeros(6, device='cuda'))
  with pytest.raises(ValueError):
    nn.normalize_relu(torch.zeros(2, 3, 4, 8, device='cuda'), torch.ones(8, device='cuda'),
                      torch.zeros(8, device='cuda'), 'group')
  with pytest.raises(KeyError):
    nn.normalize_relu(torch.zeros(2, 3, 4, 8, device='cuda'), torch.ones(8, device='cuda'),
                      torch.zeros(8, device='cuda'), 'batch')


# ---- GPU: layers and encoders against the float64 restatement ---------------------
@pytest.fixture
def no_tf32():
  saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
  torch.backends.cudnn.allow_tf32 = False
  torch.backends.cuda.matmul.allow_tf32 = False
  yield
  torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _randomize(module, seed):
  """Random parameters, so that every scale, shift and bias is exercised."""
  g = torch.Generator().manual_seed(seed)
  with torch.no_grad():
    for name, p in module.named_parameters():
      noise = torch.randn(p.shape, generator=g).to(p.device)
      if name.endswith('scale'):
        p.copy_(1.0 + 0.3 * noise)
      elif name.endswith(('shift', 'bias')):
        p.copy_(0.1 * noise)


def _params64(module):
  return {n: p.detach().double().clone().requires_grad_(True)
          for n, p in module.named_parameters()}


def _compare_grads(module, p64, tol=(2e-3, 5e-4)):
  for name, p in module.named_parameters():
    assert p.grad is not None and p64[name].grad is not None, name
    emax, el2 = rel_err(p.grad.cpu().numpy(), p64[name].grad.cpu().numpy())
    assert emax < tol[0] and el2 < tol[1], (name, emax, el2)


LAYERS = [(32, 1, True, 64, 58), (32, 1, False, 128, 58), (64, 2, True, 128, 58),
          (128, 2, True, 256, 29), (256, 2, True, 512, 15), (256, 1, False, 1024, 8)]


@gpu
@pytest.mark.parametrize('ch,stride,shortcut,c_in,w', LAYERS,
                         ids=[f'ch{c}-s{s}-{"proj" if p else "id"}' for c, s, p, _, _ in LAYERS])
def test_residual_layer_against_float64(no_tf32, ch, stride, shortcut, c_in, w):
  g = torch.Generator().manual_seed(ch + c_in)
  x = torch.randn((2, 20, w, c_in), generator=g, dtype=torch.float64).float().double().cuda()
  up = torch.randn((2, 20, -(-w // stride), 4 * ch), generator=g, dtype=torch.float64).cuda()
  layer = nn.ResidualLayer(ch, stride, shortcut, 'layer')
  xf = x.float().requires_grad_(True)
  layer(xf)
  _randomize(layer, ch)
  p64 = _params64(layer)
  y = layer(xf)
  y.backward(up.float())
  x64 = x.clone().requires_grad_(True)
  y64 = ref.residual_layer(p64, '', x64, stride, shortcut, 'layer')
  y64.backward(up)
  emax, el2 = rel_err(y.detach().cpu().numpy(), y64.detach().cpu().numpy())
  assert emax < 1e-4 and el2 < 1e-5, (emax, el2)
  emax, el2 = rel_err(xf.grad.cpu().numpy(), x64.grad.cpu().numpy())
  assert emax < 2e-3 and el2 < 5e-4, (emax, el2)
  _compare_grads(layer, p64)


def _audio(b, n, seed):
  g = torch.Generator().manual_seed(seed)
  t = torch.arange(n, dtype=torch.float64) / 16000.0
  f0 = 110.0 + 330.0 * torch.rand((b, 1), generator=g, dtype=torch.float64)
  audio = 0.5 * torch.sin(2 * torch.pi * f0 * t) + 0.05 * torch.randn((b, n), generator=g,
                                                                       dtype=torch.float64)
  return audio.float().cuda()


PRETRAIN_SPLITS = (('frequencies', 6400), ('amplitudes', 100), ('noise_magnitudes', 65))


def _logmel(audio):
  return spectral_ops.compute_logmel(audio, lo_hz=0.0, hi_hz=8000.0, bins=229,
                                     fft_size=2048, overlap=0.75, pad_end=True)


@gpu
def test_resnet_sinusoidal_encoder_against_float64(no_tf32):
  """pretrain_model.gin's encoder at 64000 samples: [B, 125, 229] log-mel, ResNet
  output [B, 125, 8, 1024], and every parameter's gradient."""
  enc = encoders.ResnetSinusoidalEncoder(PRETRAIN_SPLITS, spectral_fn=_logmel, size='small')
  audio = _audio(2, 64000, seed=1)
  enc({'audio': audio})
  _randomize(enc, 2)
  p64 = _params64(enc)
  out = enc({'audio': audio})
  assert {k: tuple(v.shape) for k, v in out.items()} == {
      'frequencies': (2, 125, 6400), 'amplitudes': (2, 125, 100),
      'noise_magnitudes': (2, 125, 65)}
  g = torch.Generator().manual_seed(3)
  ups = {k: torch.randn(v.shape, generator=g, dtype=torch.float64).cuda()
         for k, v in out.items()}
  sum((v * ups[k].float()).sum() for k, v in out.items()).backward()
  assert {n for n in p64 if n.startswith('resnet.')} == {'resnet.' + n for n in _small_names()}
  mag = _logmel(audio).double()
  out64 = ref.resnet_sinusoidal(p64, mag, 'small', [k for k, _ in PRETRAIN_SPLITS])
  sum((v * ups[k]).sum() for k, v in out64.items()).backward()
  for k in out:
    emax, el2 = rel_err(out[k].detach().cpu().numpy(), out64[k].detach().cpu().numpy())
    assert emax < 1e-3 and el2 < 1e-4, (k, emax, el2)
  # 38 normalizations deep in float32: the gradients of the first convolution's kernel
  # and of the biases before a normalization are sums with heavy cancellation
  _compare_grads(enc, p64, tol=(2e-2, 1e-2))


@gpu
def test_sinusoidal_to_harmonic_encoder_against_float64(no_tf32):
  enc = encoders.SinusoidalToHarmonicEncoder(net=nn.RnnSandwich())
  g = torch.Generator().manual_seed(4)
  sin_freqs = (20.0 + 7000.0 * torch.rand((3, 125, 100), generator=g,
                                          dtype=torch.float64)).float().double().cuda()
  sin_amps = (0.02 * torch.rand((3, 125, 100), generator=g,
                                dtype=torch.float64)).float().double().cuda()
  enc(sin_freqs.float(), sin_amps.float())
  _randomize(enc, 5)
  p64 = {n: p.detach().double().cpu().clone().requires_grad_(True)
         for n, p in enc.named_parameters()}
  out = enc(sin_freqs.float(), sin_amps.float())
  ups = {k: torch.randn(v.shape, generator=g, dtype=torch.float64) for k, v in out.items()}
  sum((v * ups[k].float().cuda()).sum() for k, v in out.items()).backward()
  out64 = ref.sinusoidal_to_harmonic(p64, sin_freqs.cpu(), sin_amps.cpu())
  sum((v * ups[k]).sum() for k, v in out64.items()).backward()
  for k in out:
    emax, el2 = rel_err(out[k].detach().cpu().numpy(), out64[k].detach().numpy())
    assert emax < 1e-3 and el2 < 1e-4, (k, emax, el2)
  _compare_grads(enc, p64, tol=(5e-3, 1e-3))
