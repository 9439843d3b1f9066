"""decoders.RnnFcDecoder at the ae.gin (ch=512, 3 layers per stack, 3 inputs) and VST
(ch=256, 1 layer, 2 inputs) configurations: outputs and every parameter's gradient
against a float64 restatement with the same weights, and end to end through the
synthesizers and SpectralLoss."""
import pytest
import torch

import ddsp_b200
from ddsp_b200 import decoders, losses
from tests import gru_ref
from tests.util import rel_err

gpu = pytest.mark.gpu
AE = dict(ch=512, layers_per_stack=3, input_keys=('ld_scaled', 'f0_scaled', 'z'))
VST = dict(ch=256, layers_per_stack=1, input_keys=('pw_scaled', 'f0_scaled'))
WIDTHS = {'ld_scaled': 1, 'f0_scaled': 1, 'z': 16, 'pw_scaled': 1}


def test_refusals_and_keys():
  with pytest.raises(NotImplementedError, match='stateless'):
    decoders.RnnFcDecoder(stateless=True)
  with pytest.raises(NotImplementedError, match="rnn_type='gru'"):
    decoders.RnnFcDecoder(rnn_type='lstm')
  d = decoders.RnnFcDecoder()
  assert d.output_keys == ('amps', 'harmonic_distribution')
  assert ddsp_b200.RnnFcDecoder is decoders.RnnFcDecoder
  with pytest.raises(KeyError, match='z'):
    d({'ld_scaled': torch.zeros(1, 2, 1), 'f0_scaled': torch.zeros(1, 2, 1)})


def _features(keys, b, t, seed, dev='cuda'):
  g = torch.Generator().manual_seed(seed)
  return {k: torch.rand((b, t, WIDTHS[k]), generator=g).to(dev) for k in keys}


def _float64_decoder(dec, feats):
  """The decoder's forward in float64 on copies of its parameters: (outputs, params)."""
  p = {n: v.detach().double().requires_grad_(True) for n, v in dec.named_parameters()}

  def stack(prefix, x, layers):
    for i in range(layers):
      d = x @ p[f'{prefix}.{i}.0.kernel'] + p[f'{prefix}.{i}.0.bias']
      d = torch.nn.functional.layer_norm(d, d.shape[-1:], p[f'{prefix}.{i}.1.gamma'],
                                         p[f'{prefix}.{i}.1.beta'], 1e-3)
      x = torch.nn.functional.leaky_relu(d, 0.2)
    return x

  layers = len(dec.out_stack)
  ins = [stack(f'input_stacks.{i}', feats[k].double(), layers)
         for i, k in enumerate(dec.input_keys)]
  x = gru_ref.gru(torch.cat(ins, -1), p['rnn.rnn.kernel'], p['rnn.rnn.recurrent_kernel'],
                  p['rnn.rnn.bias'])
  x = stack('out_stack', torch.cat(ins + [x], -1), layers)
  return x @ p['dense_out.kernel'] + p['dense_out.bias'], p


@gpu
@pytest.mark.parametrize('config,t', [('ae', 1000), ('vst', 201)])
def test_against_float64(config, t):
  torch.manual_seed(0)
  cfg = AE if config == 'ae' else VST
  dec = decoders.RnnFcDecoder(**cfg)
  feats = _features(cfg['input_keys'], 2, t, seed=1)
  out = dec(feats)
  assert list(out) == ['amps', 'harmonic_distribution']
  assert out['amps'].shape == (2, t, 1) and out['harmonic_distribution'].shape == (2, t, 40)
  y = torch.cat([out['amps'], out['harmonic_distribution']], -1)
  up = torch.randn(y.shape, generator=torch.Generator().manual_seed(2)).cuda()
  (y * up).sum().backward()
  want, params = _float64_decoder(dec, feats)
  (want * up.double()).sum().backward()
  emax, el2 = rel_err(y.detach().cpu().numpy(), want.detach().cpu().numpy())
  assert emax < 1e-4 and el2 < 1e-4, (emax, el2)
  for name, v in dec.named_parameters():
    emax, el2 = rel_err(v.grad.cpu().numpy(), params[name].grad.cpu().numpy())
    assert emax < 2e-3 and el2 < 1e-3, (name, emax, el2)


@gpu
@pytest.mark.parametrize('config', ['ae', 'vst'])
def test_end_to_end_through_synthesis_and_spectral_loss(config):
  torch.manual_seed(0)
  cfg = AE if config == 'ae' else VST
  b, t, n = 2, 250, 64000
  dec = decoders.RnnFcDecoder(
      **cfg, output_splits=(('amps', 1), ('harmonic_distribution', 60),
                            ('noise_magnitudes', 65)))
  feats = _features(cfg['input_keys'], b, t, seed=3)
  out = dec(feats)
  out['f0_hz'] = 110.0 + 330.0 * feats['f0_scaled']
  group = ddsp_b200.ProcessorGroup(dag=[
      (ddsp_b200.Harmonic(n_samples=n), ['amps', 'harmonic_distribution', 'f0_hz']),
      (ddsp_b200.FilteredNoise(n_samples=n), ['noise_magnitudes']),
      (ddsp_b200.Add(), ['filtered_noise/signal', 'harmonic/signal'])])
  audio = group(out, return_outputs_dict=True)['signal']
  target = 0.1 * torch.randn((b, n), generator=torch.Generator().manual_seed(4)).cuda()
  loss = losses.SpectralLoss()(target, audio)
  loss.backward()
  for name, v in dec.named_parameters():
    assert v.grad is not None and torch.isfinite(v.grad).all(), name
    assert v.grad.abs().max() > 0, name
