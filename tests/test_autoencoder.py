"""models.Model and models.Autoencoder: the losses bookkeeping and the glue on the CPU
with stand-in parts; on the GPU, the reference's five autoencoder configurations
(nsynth_ae, solo_instrument, VST at 16, 32 and 48 kHz) built from their gin values, the
ae.gin model bitwise against the same modules wired by hand, gradients to every
parameter including the trainable reverbs', an optimizer step, and copies."""
import copy
import pickle

import numpy as np
import pytest
import torch

import ddsp_b200
from ddsp_b200 import (core, decoders, effects, encoders, losses, models, preprocessing,
                       processors, synths)

gpu = pytest.mark.gpu


# ---- CPU: bookkeeping and glue with stand-in parts ------------------------------------
class _Loss:
  def __init__(self, name, scale):
    self.name, self.scale = name, scale

  def get_losses_dict(self, target, audio):
    return {self.name: self.scale * (target - audio).abs().mean()}


class _Toy(models.Model):
  def __init__(self, loss_objs):
    super().__init__()
    self.loss_objs = loss_objs

  def call(self, features, training=True):
    outputs = {'audio_synth': 0.5 * features['audio']}
    if training:
      self._update_losses_dict(self.loss_objs, features['audio'], outputs['audio_synth'])
    return outputs


def test_model_losses_bookkeeping():
  model = _Toy([_Loss('a', 1.0), object(), _Loss('b', 3.0)])
  feats = {'audio': torch.ones(2, 8)}
  outputs, loss = model(feats, return_losses=True)
  assert list(outputs) == ['audio_synth']
  assert list(loss) == ['a', 'b', 'total_loss']
  assert float(loss['a']) == 0.5 and float(loss['b']) == 1.5
  assert float(loss['total_loss']) == 2.0
  assert model(feats) is not None and model._losses_dict == {'a': loss['a'], 'b': loss['b']}
  outputs, loss = model(feats, training=False, return_losses=True)
  assert list(loss) == ['total_loss'] and float(loss['total_loss']) == 0.0
  assert list(_Toy(None)(feats, return_losses=True)[1]) == ['total_loss']


def test_model_base_refusals():
  model = models.Model()
  with pytest.raises(NotImplementedError, match='call'):
    model({'audio': torch.zeros(1)})
  with pytest.raises(NotImplementedError, match='get_audio_from_outputs'):
    model.get_audio_from_outputs({})
  with pytest.raises(NotImplementedError, match='state_dict'):
    model.restore('/nonexistent')


class _Variables:
  """A processor with one variable built at its first call, as the trainable reverbs."""
  name = 'reverb'

  def __init__(self):
    self._ir = None

  def named_variables(self):
    return [] if self._ir is None else [('ir', self._ir)]

  def __call__(self, audio):
    if self._ir is None:
      self._ir = torch.nn.Parameter(torch.full((3,), 0.5))
    return audio * self._ir.sum()


class _Group:
  def __init__(self):
    self.reverb = _Variables()
    self.processors = [self.reverb, processors.Add()]

  def __call__(self, features, return_outputs_dict=False):
    signal = self.reverb(features['amps'])
    controls = {'inputs': features, 'reverb': {'signal': signal}, 'out': {'signal': signal}}
    return dict(signal=signal, controls=controls) if return_outputs_dict else signal


class _Scale(torch.nn.Module):
  def __init__(self, key, out_key):
    super().__init__()
    self.key, self.out_key = key, out_key
    self.w = torch.nn.Parameter(torch.tensor(2.0))

  def forward(self, features):
    return {self.out_key: self.w * features[self.key]}


class _Preprocessor:
  def __call__(self, features):
    return {'f0_scaled': features['f0_hz'] / 100.0}


def _toy_autoencoder():
  return models.Autoencoder(preprocessor=_Preprocessor(), encoder=_Scale('f0_scaled', 'z'),
                            decoder=_Scale('z', 'amps'), processor_group=_Group(),
                            losses=_Loss('l1', 1.0))


def test_autoencoder_glue_and_processor_variables():
  model = _toy_autoencoder()
  assert [n for n, _ in model.named_parameters()] == ['encoder.w', 'decoder.w']
  feats = {'f0_hz': torch.full((1, 4), 100.0), 'audio': torch.ones(1, 4)}
  outputs, loss = model(feats, return_losses=True)
  assert list(feats) == ['f0_hz', 'audio', 'f0_scaled', 'z', 'amps']
  assert list(outputs) == ['inputs', 'reverb', 'out', 'audio_synth']
  assert outputs['inputs'] is feats
  assert torch.equal(model.get_audio_from_outputs(outputs), torch.full((1, 4), 6.0))
  assert list(loss) == ['l1', 'total_loss'] and float(loss['total_loss'].detach()) == 5.0
  ir = model.processor_group.reverb._ir
  assert dict(model.named_parameters())['processor_variables.reverb.ir'] is ir
  assert model.state_dict()['processor_variables.reverb.ir'] is not None
  loss['total_loss'].backward()
  assert ir.grad is not None and ir.grad.abs().sum() > 0
  _, loss = model(feats, training=False, return_losses=True)
  assert list(loss) == ['total_loss']
  model(feats, return_losses=True)     # copies leave this call's autograd graph behind
  for other in (copy.deepcopy(model), pickle.loads(pickle.dumps(model))):
    other_ir = other.processor_group.reverb._ir
    assert other_ir is not ir and torch.equal(other_ir, ir)
    assert dict(other.named_parameters())['processor_variables.reverb.ir'] is other_ir


# ---- GPU: the reference's configurations ---------------------------------------------
def _spectral_loss(fft_sizes=(2048, 1024, 512, 256, 128, 64)):
  return losses.SpectralLoss(fft_sizes=fft_sizes, loss_type='L1', mag_weight=1.0,
                             logmag_weight=1.0)


def _ae_group(n_samples=64000, seed=0):
  """ae.gin's ProcessorGroup."""
  return processors.ProcessorGroup(dag=[
      (synths.Harmonic(n_samples=n_samples, sample_rate=16000, normalize_below_nyquist=True,
                       scale_fn=core.exp_sigmoid, name='harmonic'),
       ['amps', 'harmonic_distribution', 'f0_hz']),
      (synths.FilteredNoise(n_samples=n_samples, window_size=0, scale_fn=core.exp_sigmoid,
                            name='filtered_noise', seed=seed), ['noise_magnitudes']),
      (processors.Add(name='add'), ['filtered_noise/signal', 'harmonic/signal'])])


def nsynth_ae():
  """models/ae.gin (papers/iclr2020/nsynth_ae.gin)."""
  return models.Autoencoder(
      preprocessor=preprocessing.F0LoudnessPreprocessor(time_steps=1000),
      encoder=encoders.MfccTimeDistributedRnnEncoder(rnn_channels=512, rnn_type='gru',
                                                     z_dims=16, z_time_steps=125),
      decoder=decoders.RnnFcDecoder(
          rnn_channels=512, rnn_type='gru', ch=512, layers_per_stack=3,
          input_keys=('ld_scaled', 'f0_scaled', 'z'),
          output_splits=(('amps', 1), ('harmonic_distribution', 100),
                         ('noise_magnitudes', 65))),
      processor_group=_ae_group(), losses=[_spectral_loss()])


def solo_instrument():
  """models/solo_instrument.gin: ae.gin without the encoder, a smaller output and a
  trainable 48000-tap Reverb after the Add."""
  group = _ae_group()
  return models.Autoencoder(
      preprocessor=preprocessing.F0LoudnessPreprocessor(time_steps=1000),
      decoder=decoders.RnnFcDecoder(
          rnn_channels=512, rnn_type='gru', ch=512, layers_per_stack=3,
          input_keys=('ld_scaled', 'f0_scaled'),
          output_splits=(('amps', 1), ('harmonic_distribution', 60),
                         ('noise_magnitudes', 65))),
      processor_group=processors.ProcessorGroup(dag=[
          (group.harmonic, ['amps', 'harmonic_distribution', 'f0_hz']),
          (group.filtered_noise, ['noise_magnitudes']),
          (group.add, ['filtered_noise/signal', 'harmonic/signal']),
          (effects.Reverb(name='reverb', reverb_length=48000, trainable=True),
           ['add/signal'])]),
      losses=[_spectral_loss()])


VST = {  # sample rate: (harmonics, noise bands, reverb length, initial bias, FFT sizes)
    16000: (60, 65, 24000, -3.0, (2048, 1024, 512, 256, 128, 64)),
    32000: (100, 98, 48000, -4.0, (4096, 2048, 1024, 512, 256, 128)),
    48000: (100, 98, 72000, -4.0, (6144, 3072, 1536, 768, 384, 192)),
}


def vst(sample_rate):
  """models/vst/vst.gin, vst_32k.gin and vst_48k.gin: power and f0 at 50 frames/s from
  centred frames, one extra frame of synthesis cropped at the end."""
  n_harmonics, n_bands, reverb_length, initial_bias, fft_sizes = VST[sample_rate]
  hop = sample_rate // 50
  n_samples = 4 * sample_rate + hop
  return models.Autoencoder(
      preprocessor=preprocessing.OnlineF0PowerPreprocessor(
          frame_rate=50, frame_size=1024, padding='center', compute_power=True,
          compute_f0=False, crepe_saved_model_path=None),
      decoder=decoders.RnnFcDecoder(
          rnn_channels=512, rnn_type='gru', ch=256, layers_per_stack=1,
          input_keys=('pw_scaled', 'f0_scaled'),
          output_splits=(('amps', 1), ('harmonic_distribution', n_harmonics),
                         ('noise_magnitudes', n_bands))),
      processor_group=processors.ProcessorGroup(dag=[
          (synths.Harmonic(n_samples=n_samples, sample_rate=sample_rate,
                           normalize_below_nyquist=True, scale_fn=core.exp_sigmoid,
                           amp_resample_method='linear',
                           use_angular_cumsum=sample_rate > 16000, name='harmonic'),
           ['amps', 'harmonic_distribution', 'f0_hz']),
          (synths.FilteredNoise(n_samples=n_samples, window_size=0,
                                scale_fn=core.exp_sigmoid, name='filtered_noise'),
           ['noise_magnitudes']),
          (processors.Add(name='add'), ['filtered_noise/signal', 'harmonic/signal']),
          (effects.FilteredNoiseReverb(name='reverb', reverb_length=reverb_length,
                                       n_frames=500, n_filter_banks=32,
                                       initial_bias=initial_bias, trainable=True),
           ['add/signal']),
          (processors.Crop(frame_size=hop, crop_location='back'), ['reverb/signal'])]),
      losses=[_spectral_loss(fft_sizes)])


CONFIGS = {  # name: (builder, sample rate, frame rate, centred)
    'nsynth_ae': (nsynth_ae, 16000, 250, False),
    'solo_instrument': (solo_instrument, 16000, 250, False),
    'vst_16kHz': (lambda: vst(16000), 16000, 50, True),
    'vst_32kHz': (lambda: vst(32000), 32000, 50, True),
    'vst_48kHz': (lambda: vst(48000), 48000, 50, True),
}


def _inputs(name, n_batch=1, tones=False, seed=0):
  """The reference test's inputs (autoencoder_test.py): 4 s of N(0, 1) audio (and its
  16 kHz version), zero f0, loudness and confidence, one more frame when centred.  With
  tones, f0 glides over 110-440 Hz and the audio is a quieter noise, so that every
  parameter of the model receives a gradient."""
  _, sample_rate, frame_rate, centered = CONFIGS[name]
  n_frames = frame_rate * 4 + (1 if centered else 0)
  rng = np.random.default_rng(seed)
  zeros = np.zeros([n_batch, n_frames])
  f0 = zeros
  if tones:
    f0 = 110.0 * 2.0**(2.0 * rng.uniform(size=(n_batch, 1)) * np.linspace(0, 1, n_frames))
  inputs = {'loudness_db': zeros, 'f0_hz': f0, 'f0_confidence': zeros,
            'audio': rng.standard_normal((n_batch, sample_rate * 4)) * (0.1 if tones else 1),
            'audio_16k': rng.standard_normal((n_batch, 16000 * 4))}
  return {k: core.tf_float32(v) for k, v in inputs.items()}


@gpu
@pytest.mark.parametrize('name', list(CONFIGS))
def test_build_model(name):
  torch.manual_seed(0)
  model = CONFIGS[name][0]()
  inputs = _inputs(name)
  with torch.no_grad():   # the reference test runs without a gradient tape
    outputs = model(inputs)
  assert isinstance(outputs, dict)
  audio_gen = model.get_audio_from_outputs(outputs)
  assert list(audio_gen.shape) == list(inputs['audio'].shape)
  assert torch.isfinite(audio_gen).all()


def _assert_nested_equal(a, b, path=''):
  assert type(a) is type(b), path
  if isinstance(a, dict):
    assert list(a) == list(b), path
    for k in a:
      _assert_nested_equal(a[k], b[k], f'{path}/{k}')
  elif torch.is_tensor(a):
    assert torch.equal(a, b), path
  else:
    assert a == b, path


FEATURE_KEYS = ['loudness_db', 'f0_hz', 'f0_confidence', 'audio', 'audio_16k']
AE_FEATURES = FEATURE_KEYS + ['f0_scaled', 'ld_scaled', 'z', 'amps',
                              'harmonic_distribution', 'noise_magnitudes']


@gpu
def test_glue_is_exact():
  torch.manual_seed(0)
  model = nsynth_ae()
  features = _inputs('nsynth_ae', n_batch=2, tones=True)
  feats = dict(features)
  outputs, loss = model(feats, return_losses=True)
  assert list(feats) == AE_FEATURES
  assert list(outputs) == (['inputs'] + AE_FEATURES +
                           ['harmonic', 'filtered_noise', 'add', 'out', 'audio_synth'])
  assert outputs['inputs'] is feats
  assert list(loss) == ['spectral_loss', 'total_loss']

  by_hand = dict(features)
  by_hand.update(model.preprocessor(by_hand))
  by_hand.update(model.encoder(by_hand))
  by_hand.update(model.decoder(by_hand))
  pg_out = _ae_group()(by_hand, return_outputs_dict=True)
  want = dict(pg_out['controls'], audio_synth=pg_out['signal'])
  want_loss = _spectral_loss()(by_hand['audio'], pg_out['signal'])
  assert torch.equal(outputs['audio_synth'], want['audio_synth'])
  for k in outputs:
    if k != 'inputs':
      _assert_nested_equal(outputs[k], want[k], k)
  assert torch.equal(loss['spectral_loss'], want_loss)
  assert torch.equal(loss['total_loss'], want_loss)


def _variable(model):
  holder = model.processor_variables['reverb']
  return dict(holder.named_parameters())


@gpu
@pytest.mark.parametrize('name', ['nsynth_ae', 'solo_instrument', 'vst_16kHz'])
def test_training_reaches_every_parameter(name):
  torch.manual_seed(0)
  model = CONFIGS[name][0]()
  assert not list(model.parameters())
  _, loss = model(_inputs(name, n_batch=2, tones=True), return_losses=True)
  names = dict(model.named_parameters())
  assert all(n.split('.')[0] in ('encoder', 'decoder', 'processor_variables')
             for n in names)
  if name == 'nsynth_ae':
    assert tuple(names['encoder.z_norm.scale'].shape) == (1, 1, 1, 30)
    assert tuple(names['encoder.dense_out.kernel'].shape) == (512, 16)
    assert tuple(names['decoder.dense_out.kernel'].shape) == (512, 166)
    assert not list(model.processor_variables.parameters())
  else:
    reverb = model.processor_group.reverb
    var_name, shape = (('ir', (48000,)) if name == 'solo_instrument' else
                       ('magnitudes', (500, 32)))
    var = getattr(reverb, '_' + var_name)
    assert names[f'processor_variables.reverb.{var_name}'] is var
    assert tuple(var.shape) == shape
    assert model.state_dict()[f'processor_variables.reverb.{var_name}'].data_ptr() == \
        var.data_ptr()
  loss['total_loss'].backward()
  for n, p in model.named_parameters():
    assert p.grad is not None and torch.isfinite(p.grad).all(), n
    assert p.grad.abs().max() > 0, n
  if name != 'nsynth_ae':
    before = var.detach().clone()
    torch.optim.Adam(model.parameters(), lr=1e-3).step()
    assert not torch.equal(var.detach(), before)


@gpu
@pytest.mark.parametrize('name', ['nsynth_ae', 'solo_instrument', 'vst_16kHz'])
def test_copies(name):
  torch.manual_seed(0)
  model = CONFIGS[name][0]()
  features = _inputs(name, tones=True)
  _, loss = model(dict(features), return_losses=True)    # builds
  loss['total_loss'].backward()
  copies = [copy.deepcopy(model), pickle.loads(pickle.dumps(model))]
  want = model(dict(features))['audio_synth']
  gru = (model.decoder.rnn.rnn, model.decoder.rnn.rnn._handles)
  for other in copies:
    assert torch.equal(other(dict(features))['audio_synth'], want)
    assert other.decoder.rnn.rnn._handles[want.device] is not gru[1][want.device]
    if name == 'nsynth_ae':
      enc = other.encoder.rnn.rnn._handles[want.device]
      assert enc is not model.encoder.rnn.rnn._handles[want.device]
    else:
      mine, theirs = _variable(model), _variable(other)
      for k in mine:
        assert theirs[k] is not mine[k] and torch.equal(theirs[k], mine[k])
        assert theirs[k].data_ptr() != mine[k].data_ptr()
        assert getattr(other.processor_group.reverb, '_' + k) is theirs[k]


def test_package_exports():
  assert ddsp_b200.models is models and ddsp_b200.encoders is encoders
