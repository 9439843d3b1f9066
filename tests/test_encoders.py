"""nn.normalize_op, nn.Normalize and encoders.MfccTimeDistributedRnnEncoder: the
normalization against a float64 restatement of the reference (every norm type, ranks 2
to 4, C = 1, 30, 32 and 128, T = 1) and gradcheck; the encoder's refusals, names and
defaults; and on the GPU, z and every parameter's gradient against a float64
composition at every z_time_steps the encoder takes."""
import copy
import pickle
import re

import numpy as np
import pytest
import torch

import ddsp_b200
from ddsp_b200 import encoders, nn
from tests import encoder_ref
from tests import routing_ref
from tests.util import rel_err

gpu = pytest.mark.gpu
NORM_TYPES = ['instance', 'layer', 'group']


def _x(shape, seed, dtype=torch.float32):
  g = torch.Generator().manual_seed(seed)
  return (3.0 * torch.randn(shape, generator=g, dtype=torch.float64) + 1.5).to(dtype)


def _shape(rank, t, c):
  return {2: (3, c), 3: (3, t, c), 4: (3, t, 2, c)}[rank]


@pytest.mark.parametrize('norm_type', NORM_TYPES)
@pytest.mark.parametrize('rank', [2, 3, 4])
@pytest.mark.parametrize('c', [1, 30, 32, 128])
@pytest.mark.parametrize('t', [1, 7])
def test_normalize_against_float64(norm_type, rank, c, t):
  x = _x(_shape(rank, t, c), seed=c + t)
  layer = nn.Normalize(norm_type)
  if norm_type == 'group' and c % 32:
    with pytest.raises(ValueError, match='32 groups'):
      layer(x)
    return
  layer(x)
  with torch.no_grad():
    layer.scale.copy_(_x((1, 1, 1, c), seed=1))
    layer.shift.copy_(_x((1, 1, 1, c), seed=2))
  y = layer(x)
  assert y.shape == x.shape and y.dtype == torch.float32
  want = encoder_ref.normalize(x.double().numpy(), norm_type, layer.scale.detach().double()
                               .numpy(), layer.shift.detach().double().numpy())
  emax, el2 = rel_err(y.detach().numpy(), want)
  assert emax < 1e-5 and el2 < 1e-5, (emax, el2)


@pytest.mark.parametrize('norm_type', NORM_TYPES + [None])
def test_normalize_op_against_float64(norm_type):
  x = _x((2, 9, 3, 64), seed=5)
  y = nn.normalize_op(x, norm_type)
  want = encoder_ref.normalize_op(x.double().numpy(), norm_type)
  emax, el2 = rel_err(y.numpy(), want)
  assert emax < 1e-5 and el2 < 1e-5, (emax, el2)
  if norm_type is None:
    assert y is x


@pytest.mark.parametrize('norm_type', NORM_TYPES)
def test_normalize_gradcheck(norm_type):
  x = _x((2, 3, 2, 32), seed=7, dtype=torch.float64).requires_grad_(True)
  assert torch.autograd.gradcheck(lambda v: nn.normalize_op(v, norm_type), (x,))
  layer = nn.Normalize(norm_type)
  layer(x.detach())
  scale = _x((1, 1, 1, 32), seed=8, dtype=torch.float64).requires_grad_(True)
  shift = _x((1, 1, 1, 32), seed=9, dtype=torch.float64).requires_grad_(True)
  x3 = x.detach()[:, :, 0].requires_grad_(True)
  assert torch.autograd.gradcheck(
      lambda v, s, b: torch.func.functional_call(layer, {'scale': s, 'shift': b}, (v,)),
      (x3, scale, shift))


def test_normalize_names_shapes_and_refusals():
  layer = nn.Normalize()
  assert layer.norm_type == 'layer' and not list(layer.parameters())
  layer(torch.zeros(2, 5, 30))
  assert [(n, tuple(p.shape)) for n, p in layer.named_parameters()] == [
      ('scale', (1, 1, 1, 30)), ('shift', (1, 1, 1, 30))]
  assert layer.scale.eq(1).all() and layer.shift.eq(0).all()
  with pytest.raises(ValueError, match='width 30'):
    layer(torch.zeros(2, 5, 31))
  with pytest.raises(ValueError, match='rank 2, 3 or 4'):
    layer(torch.zeros(5))
  with pytest.raises(ValueError, match='32 groups'):
    nn.normalize_op(torch.zeros(2, 5, 1, 30), 'group')
  with pytest.raises(KeyError):
    nn.normalize_op(torch.zeros(2, 5, 1, 30), 'batch')
  assert nn.ensure_4d(torch.zeros(2, 3)).shape == (2, 1, 1, 3)
  assert nn.ensure_4d(torch.zeros(2, 4, 3)).shape == (2, 4, 1, 3)
  assert nn.inv_ensure_4d(torch.zeros(2, 4, 1, 3), 3).shape == (2, 4, 3)
  assert nn.inv_ensure_4d(torch.zeros(2, 1, 1, 3), 2).shape == (2, 3)


def test_encoder_defaults_refusals_and_names():
  with pytest.raises(ValueError, match=re.escape(
      '`z_time_steps` currently limited to 63,125,250,500 and 1000')):
    encoders.MfccTimeDistributedRnnEncoder(z_time_steps=100)
  with pytest.raises(NotImplementedError, match="rnn_type='gru'"):
    encoders.MfccTimeDistributedRnnEncoder(rnn_type='lstm')
  enc = encoders.MfccTimeDistributedRnnEncoder()
  assert (enc.rnn.rnn.units, enc.dense_out.units) == (512, 32)
  assert (enc.fft_size, enc.overlap) == (1024, 0.75)
  assert enc.z_norm.norm_type == 'instance'
  assert enc.input_keys == ['audio', 'f0_scaled']
  for steps, (fft_size, overlap) in encoder_ref.Z_AUDIO_SPEC.items():
    e = encoders.MfccTimeDistributedRnnEncoder(z_time_steps=steps)
    assert (e.fft_size, e.overlap) == (fft_size, overlap)
    assert e.z_audio_spec[str(steps)] == {'fft_size': fft_size, 'overlap': overlap}
  with pytest.raises(KeyError, match='audio'):
    enc({'f0_scaled': torch.zeros(1, 10, 1)})
  with pytest.raises(KeyError, match='f0_scaled'):
    enc({'audio': torch.zeros(1, 640)})
  assert ddsp_b200.encoders is encoders


class _Identity(encoders.ZEncoder):
  def compute_z(self, x):
    return x


def test_z_encoder_keys_and_time_axis():
  enc = _Identity()
  assert enc.input_keys == ['x', 'f0_scaled']
  z = torch.arange(6.0).reshape(2, 3)
  out = enc(z, torch.zeros(2, 1, 1))
  assert list(out) == ['z'] and torch.equal(out['z'], z[:, None, :])
  same = torch.randn(2, 5, 3)
  assert enc({'x': same, 'f0_scaled': torch.zeros(2, 5, 1)})['z'] is same
  with pytest.raises(ValueError, match='3 inputs'):
    enc(same, same, same)
  with pytest.raises(NotImplementedError):
    encoders.ZEncoder()(torch.zeros(1, 2, 1))


@gpu
@pytest.mark.parametrize('frames,steps', [(1, 1000), (63, 1000), (250, 1000), (125, 250)])
def test_z_encoder_resamples_to_the_time_axis(frames, steps):
  z = torch.randn(2, frames, 16, device='cuda').squeeze(1)
  out = _Identity()(z, torch.zeros(2, steps, 1, device='cuda'))['z']
  want = routing_ref.resample((z if z.dim() == 3 else z[:, None]).double(), steps)
  emax, el2 = rel_err(out.cpu().numpy(), want.cpu().numpy())
  assert out.shape == (2, steps, 16) and emax < 1e-6 and el2 < 1e-6, (emax, el2)


def _audio(b, n, seed):
  """Harmonic tones with gliding pitch and a loudness envelope, plus a little noise, so
  that every MFCC coefficient varies over time."""
  rng = np.random.default_rng(seed)
  t = np.arange(n) / 16000.0
  out = []
  for _ in range(b):
    f0 = rng.uniform(110, 220) * 2.0**(rng.uniform(-1, 1) * t / t[-1])
    phase = 2 * np.pi * np.cumsum(f0) / 16000.0
    env = 0.5 + 0.4 * np.sin(2 * np.pi * rng.uniform(0.5, 2) * t)
    x = sum(np.sin(k * phase) / k for k in range(1, 12)) * env
    out.append(0.3 * x + 0.01 * rng.standard_normal(n))
  return torch.from_numpy(np.stack(out)).float()


@gpu
@pytest.mark.parametrize('z_time_steps,z_dims', [(63, 16), (125, 16), (250, 16),
                                                 (500, 16), (1000, 16), (125, 128)])
def test_encoder_against_float64(z_time_steps, z_dims):
  torch.manual_seed(0)
  b, n, t = 2, 64000, 1000
  enc = encoders.MfccTimeDistributedRnnEncoder(z_dims=z_dims, z_time_steps=z_time_steps)
  audio = _audio(b, n, seed=z_time_steps).cuda()
  f0_scaled = torch.rand(b, t, 1, device='cuda')
  enc({'audio': audio, 'f0_scaled': f0_scaled})      # builds
  with torch.no_grad():   # a non-trivial scale and shift, so both gradients are tested
    enc.z_norm.scale.copy_(1.0 + 0.2 * torch.randn_like(enc.z_norm.scale))
    enc.z_norm.shift.copy_(0.2 * torch.randn_like(enc.z_norm.shift))
  z = enc({'audio': audio, 'f0_scaled': f0_scaled})['z']
  assert z.shape == (b, t, z_dims)
  up = torch.randn(z.shape, generator=torch.Generator().manual_seed(1)).cuda()
  (z * up).sum().backward()
  params = {k: v.detach().double().requires_grad_(True) for k, v in enc.named_parameters()}
  want = encoder_ref.encoder_z(audio.double(), params, z_time_steps, t)
  (want * up.double()).sum().backward()
  emax, el2 = rel_err(z.detach().cpu().numpy(), want.detach().cpu().numpy())
  assert emax < 1e-4 and el2 < 1e-4, (emax, el2)
  for name, v in enc.named_parameters():
    emax, el2 = rel_err(v.grad.cpu().numpy(), params[name].grad.cpu().numpy())
    assert emax < 2e-3 and el2 < 1e-3, (name, emax, el2)


@gpu
def test_encoder_names_shapes_and_copies():
  torch.manual_seed(0)
  enc = encoders.MfccTimeDistributedRnnEncoder(z_dims=16, z_time_steps=125)
  feats = {'audio': _audio(1, 64000, seed=3).cuda(),
           'f0_scaled': torch.zeros(1, 1000, 1, device='cuda')}
  z = enc(feats)['z']
  assert [(n, tuple(p.shape)) for n, p in enc.named_parameters()] == [
      ('z_norm.scale', (1, 1, 1, 30)), ('z_norm.shift', (1, 1, 1, 30)),
      ('rnn.rnn.kernel', (30, 1536)), ('rnn.rnn.recurrent_kernel', (512, 1536)),
      ('rnn.rnn.bias', (2, 1536)), ('dense_out.kernel', (512, 16)),
      ('dense_out.bias', (16,))]
  for other in (copy.deepcopy(enc), pickle.loads(pickle.dumps(enc))):
    assert torch.equal(other(feats)['z'], z)
    assert other.rnn.rnn._handles[z.device] is not enc.rnn.rnn._handles[z.device]
