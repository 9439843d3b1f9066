"""models.InverseSynthesis: its bookkeeping on the CPU with stand-in parts (loss keys of
each call mode, the zipped split, stop_gradient), and on the GPU the pretrain_model.gin
and finetune_model.gin models at B = 4 and 64000 samples on generate_notes_v2's
synthetic notes: every call mode, gradients to every parameter, stop_gradient and one
Adam step."""
import pytest
import torch

import ddsp_b200
from ddsp_b200 import autograd, core, encoders, losses, models, nn, spectral_ops
from ddsp_b200 import synthetic_data

gpu = pytest.mark.gpu


# ---- CPU: bookkeeping with stand-in parts --------------------------------------------
class _Group:
  """A processor group stand-in: audio [B, T] from the controls."""
  processors = []

  def __call__(self, inputs):
    return (inputs['amplitudes'] * inputs['frequencies']).sum(-1) + inputs[
        'noise_magnitudes'].sum(-1)

  def get_controls(self, inputs):
    return {'sinusoidal': {'signal': inputs['amplitudes']}, 'out': {'signal': self(inputs)}}

  def get_signal(self, controls):
    return controls['out']['signal']


class _SinEncoder(torch.nn.Module):
  def __init__(self):
    super().__init__()
    self.w = torch.nn.Parameter(torch.linspace(0.5, 1.5, 6))

  def forward(self, features, training=True):
    a = features['audio'][..., None]
    return {'frequencies': a * self.w[:4], 'amplitudes': a * self.w[4:5] - 1.0,
            'noise_magnitudes': a * self.w[5:] + 0.5}


class _HarmEncoder(torch.nn.Module):
  def __init__(self):
    super().__init__()
    self.w = torch.nn.Parameter(torch.tensor([0.7, 1.3]))
    self.seen = []

  def forward(self, sin_freqs, sin_amps):
    self.seen.append((sin_freqs, sin_amps))
    f0 = (sin_freqs.mean(-1, keepdim=True) * self.w[0]).abs() + 1.0
    amp = sin_amps.mean(-1, keepdim=True) * self.w[1]
    return {'harm_amp': amp, 'harm_dist': torch.softmax(f0.expand(-1, -1, 3), -1),
            'f0_hz': f0}


class _Loss:
  def __init__(self, name, n_args):
    self.name, self.n_args = name, n_args

  def __call__(self, *args):
    assert len(args) == self.n_args
    return sum(a.float().mean() for a in args)

  def get_losses_dict(self, *args):
    return {self.name: self(*args)}


class _HarmConsistency(losses.HarmonicConsistencyLoss):
  def __call__(self, *args):
    assert len(args) == 6
    return {'harm_amp_loss': args[0].mean(), 'harm_dist_loss': args[2].mean(),
            'f0_hz_loss': args[4].mean()}


def _model(monkeypatch, harmonic=True, stop_gradient=True):
  monkeypatch.setattr(core, 'get_harmonic_frequencies',
                      lambda f, n: f * torch.arange(1, n + 1, dtype=f.dtype))
  model = models.InverseSynthesis(
      sinusoidal_encoder=_SinEncoder(), harmonic_encoder=_HarmEncoder() if harmonic else None,
      losses=[_Loss('spectral_loss', 2)],
      sinusoidal_consistency_losses=[_Loss('kde_consistency_loss', 4)],
      harmonic_consistency_losses=[_HarmConsistency(), _Loss('twm', 4)],
      filtered_noise_consistency_loss=_Loss('filtered_noise_consistency_loss', 2),
      twm_loss=_Loss('twm_loss', 3), harmonic_distribution_prior=_Loss('prior', 1),
      freq_scale_fn=lambda x: x * 100.0, reverb=False, stop_gradient=stop_gradient)
  model.processor_group = _Group()
  model.amps_scale_fn = autograd.exp_sigmoid
  return model


def _ss(b, t, seed):
  g = torch.Generator().manual_seed(seed)
  return {'sin_amps': torch.rand((b, t, 4), generator=g),
          'sin_freqs': 100.0 * torch.rand((b, t, 4), generator=g),
          'noise_magnitudes': torch.rand((b, t, 1), generator=g),
          'harm_amp': torch.rand((b, t, 1), generator=g),
          'harm_dist': torch.rand((b, t, 3), generator=g),
          'f0_hz': 100.0 + torch.rand((b, t, 1), generator=g)}


UNSUPERVISED = {'sin_spectral_loss', 'prior', 'harm_spectral_loss', 'kde_consistency_loss',
                'twm_loss'}
SELF_SUPERVISED = {'ss_kde_consistency_loss', 'ss_filtered_noise_consistency_loss',
                   'ss_harm_amp_loss', 'ss_harm_dist_loss', 'ss_f0_hz_loss', 'ss_harm_twm'}


def test_loss_keys_of_each_mode(monkeypatch):
  model = _model(monkeypatch)
  audio = torch.rand(2, 5)
  _, got = model({'audio': audio}, return_losses=True)
  assert set(got) == UNSUPERVISED | {'total_loss'}
  _, got = model(_ss(3, 5, 1), return_losses=True)
  assert set(got) == UNSUPERVISED | SELF_SUPERVISED | {'total_loss'}
  _, got = model((_ss(3, 5, 1), {'audio': audio}), return_losses=True)
  assert set(got) == UNSUPERVISED | SELF_SUPERVISED | {'total_loss'}
  model = _model(monkeypatch, harmonic=False)
  _, got = model({'audio': audio}, return_losses=True)
  assert set(got) == {'sin_spectral_loss', 'twm_loss', 'total_loss'}
  with pytest.raises(KeyError):   # the self-supervised losses need the harmonic outputs
    model(_ss(3, 5, 1))


def test_zipped_split(monkeypatch):
  model = _model(monkeypatch)
  audio, ss = torch.rand(2, 5), _ss(3, 5, 2)
  out = model(({'audio': audio}, ss))
  assert torch.equal(out['audio'], audio)
  assert all(not isinstance(v, dict) for v in out.values())
  assert 'sinusoidal' not in out and out['sin_amps'].shape[0] == 2
  assert torch.equal(ss['audio'], model.generate_synthetic_audio(ss))
  # the same as one call on the concatenated batch
  whole = model.forward({'audio': torch.cat([audio, ss['audio']])})
  for k, v in out.items():
    torch.testing.assert_close(v, whole[k][:2], rtol=0, atol=0)
  assert model.parse_zipped_features([ss, {'audio': audio}])[1] is ss
  assert model.get_audio_from_outputs(out) is out['harm_audio']


@pytest.mark.parametrize('stop_gradient', [True, False])
def test_stop_gradient(monkeypatch, stop_gradient):
  """stop_gradient detaches the harmonic encoder's inputs and the sinusoids of the
  sinusoidal consistency loss, and nothing else."""
  model = _model(monkeypatch, stop_gradient=stop_gradient)
  model.audio_loss_objs = []
  model.twm_loss = None
  model.harmonic_distribution_prior = None
  audio = torch.rand(2, 5)
  _, got = model({'audio': audio}, return_losses=True)
  sin_freqs, sin_amps = model.harmonic_encoder.seen[-1]
  assert sin_freqs.requires_grad != stop_gradient
  assert sin_amps.requires_grad != stop_gradient
  got['kde_consistency_loss'].backward()
  w = model.sinusoidal_encoder.w.grad
  assert (w is None or not w.any()) == stop_gradient
  assert model.harmonic_encoder.w.grad is not None


# ---- GPU: the paper's models --------------------------------------------------------
def _pretrain(finetune=False, reverb=False):
  kde = dict(weight_a=1.0, weight_b=1.0, scale_a=0.1, scale_b=0.1)
  harm = dict(amp_weight=1.0, dist_weight=1.0, f0_weight=1.0)
  spectral = dict(loss_type='L1', mag_weight=0.0, logmag_weight=0.0)
  fn_weight = 1.0
  if finetune:
    spectral.update(mag_weight=1.0, logmag_weight=1.0)
    kde = dict(weight_mean_amp=0.1, weight_a=0.1, weight_b=0.1, scale_a=0.1, scale_b=0.1)
    harm = dict(amp_weight=10.0, dist_weight=100.0, f0_weight=1.0)
    fn_weight = 100.0

  def logmel(audio):
    return spectral_ops.compute_logmel(audio, lo_hz=0.0, hi_hz=8000.0, bins=229,
                                       fft_size=2048, overlap=0.75, pad_end=True)

  return models.InverseSynthesis(
      reverb=reverb,
      sinusoidal_encoder=encoders.ResnetSinusoidalEncoder(
          size='small', spectral_fn=logmel,
          output_splits=(('frequencies', 6400), ('amplitudes', 100),
                         ('noise_magnitudes', 65))),
      harmonic_encoder=encoders.SinusoidalToHarmonicEncoder(net=nn.RnnSandwich()),
      losses=[losses.SpectralLoss(**spectral)],
      sinusoidal_consistency_losses=losses.KDEConsistencyLoss(**kde),
      harmonic_consistency_losses=losses.HarmonicConsistencyLoss(**harm),
      filtered_noise_consistency_loss=losses.FilteredNoiseConsistencyLoss(weight=fn_weight),
      twm_loss=losses.TWMLoss()).cuda()


def _notes(b, seed):
  return synthetic_data.generate_notes_v2(seeds=list(range(seed, seed + b)))


def _audio(b, seed):
  g = torch.Generator().manual_seed(seed)
  t = torch.arange(64000, dtype=torch.float64) / 16000.0
  f0 = 110.0 + 330.0 * torch.rand((b, 1), generator=g, dtype=torch.float64)
  return (0.3 * torch.sin(2 * torch.pi * f0 * t)).float().cuda()


@gpu
@pytest.mark.parametrize('finetune', [False, True], ids=['pretrain', 'finetune'])
def test_every_mode_runs_and_trains(finetune):
  torch.manual_seed(0)
  model = _pretrain(finetune, reverb=finetune)
  out, got = model(_notes(4, 10), return_losses=True)
  assert out['harm_audio'].shape == (4, 64000) and out['f0_hz'].shape == (4, 125, 1)
  assert 'ss_harm_amp_loss' in got and 'ss_kde_consistency_loss' in got
  out, got = model({'audio': _audio(4, 1)}, return_losses=True)
  assert set(got) >= {'sin_spectral_loss', 'harm_spectral_loss', 'kde_consistency_loss',
                      'twm_loss'}
  out, got = model(({'audio': _audio(4, 2)}, _notes(4, 20)), return_losses=True)
  assert out['sin_audio'].shape == (4, 64000)
  total = got['total_loss']
  assert torch.isfinite(total)
  model.zero_grad()
  total.backward()
  params = dict(model.named_parameters())
  assert ('processor_variables.reverb.magnitudes' in params) == finetune
  for name, p in params.items():
    assert p.grad is not None, name
    assert torch.isfinite(p.grad).all() and p.grad.any(), name
  opt = torch.optim.Adam(model.parameters(), lr=1e-3)
  opt.step()
  batch = ({'audio': _audio(4, 2)}, _notes(4, 20))
  _, again = model(batch, return_losses=True)
  assert again['total_loss'].item() != total.item()


@gpu
def test_stop_gradient_keeps_harmonic_losses_off_the_sinusoidal_encoder():
  torch.manual_seed(0)
  model = _pretrain()
  _, got = model({'audio': _audio(2, 3)}, return_losses=True)
  harmonic = (got['harm_spectral_loss'] + got['harm_dist_prior']
              if 'harm_dist_prior' in got else got['harm_spectral_loss'])
  harmonic = harmonic + got['kde_consistency_loss']
  model.zero_grad()
  harmonic.backward()
  for name, p in model.sinusoidal_encoder.named_parameters():
    assert p.grad is None or not p.grad.any(), name
  assert any(p.grad is not None and p.grad.any()
             for p in model.harmonic_encoder.parameters())


def test_package_exports():
  assert ddsp_b200.InverseSynthesis is models.InverseSynthesis
  assert ddsp_b200.ResnetSinusoidalEncoder is encoders.ResnetSinusoidalEncoder
  assert ddsp_b200.SinusoidalToHarmonicEncoder is encoders.SinusoidalToHarmonicEncoder
