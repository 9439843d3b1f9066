"""models.Model and models.Autoencoder (ddsp/training/models/model.py:26-131,
autoencoder.py:24-74): the model that wires a preprocessor, an encoder, a decoder, a
ProcessorGroup and losses into one training step, as ae.gin, solo_instrument.gin and
the VST configs build it.  models.InverseSynthesis (inverse_synthesis.py:24-330) is
the self-supervised pitch model of pretrain_model.gin and finetune_model.gin.  Each part
runs on its own kernels; this module is Python glue."""
import functools

import torch

from ddsp_b200 import core
from ddsp_b200 import effects
from ddsp_b200 import losses as losses_lib
from ddsp_b200 import processors
from ddsp_b200 import synths


class Model(torch.nn.Module):
  """Base class of the models: call() runs the forward pass and adds its losses to the
  losses dict, which every call resets."""

  def __init__(self):
    super().__init__()
    self._losses_dict = {}

  def __call__(self, *args, return_losses=False, **kwargs):
    """Runs call(*args, **kwargs) and returns its outputs dict, or (outputs, losses)
    with return_losses=True, where losses['total_loss'] is the sum of the scalar
    losses call() added (0 when it added none)."""
    args = [core.copy_if_tf_function(a) if isinstance(a, dict) else a for a in args]
    self._losses_dict = {}
    outputs = self._dispatch(*args, **kwargs)
    if not return_losses:
      return outputs
    self._losses_dict['total_loss'] = self.sum_losses(self._losses_dict)
    return outputs, self._losses_dict

  def __getstate__(self):
    """Copies and pickles leave the last call's losses behind: they belong to that call's
    autograd graph, which cannot be copied, and the next call resets them anyway."""
    state = dict(super().__getstate__())
    state['_losses_dict'] = {}
    return state

  def _dispatch(self, *args, **kwargs):
    """How __call__ reaches call(): through torch's Module call, which runs forward."""
    return super().__call__(*args, **kwargs)

  def forward(self, *args, **kwargs):
    return self.call(*args, **kwargs)

  def sum_losses(self, losses_dict):
    """Sum of the scalar losses of a dict, a 0-d tensor.  A loss given as a number (a
    SpectralLoss whose weights are all 0 gives 0.0) joins on the others' device."""
    values = list(losses_dict.values())
    if not values:
      return torch.zeros(())
    device = next((v.device for v in values if torch.is_tensor(v)), None)
    values = [v if torch.is_tensor(v) else torch.tensor(float(v), device=device)
              for v in values]
    return torch.stack(values).sum()

  def _update_losses_dict(self, loss_objs, *args, **kwargs):
    """Runs each loss object that has get_losses_dict on args and adds its losses."""
    for loss_obj in core.make_iterable(loss_objs):
      if hasattr(loss_obj, 'get_losses_dict'):
        self._losses_dict.update(loss_obj.get_losses_dict(*args, **kwargs))

  def restore(self, checkpoint_path, verbose=True, restore_keys=None):
    """The reference restores TensorFlow checkpoints; this model does not read them."""
    raise NotImplementedError(
        'Model.restore reads TensorFlow checkpoints, which this library does not; save '
        'and load the model with torch.save(model.state_dict()) and '
        'model.load_state_dict() after a first call has built it')

  def get_audio_from_outputs(self, outputs):
    """Extract audio output tensor from outputs dict of call()."""
    raise NotImplementedError('Must implement `self.get_audio_from_outputs()`.')

  def _register_processor_variables(self):
    """Registers the variables the processors of self.processor_group have built since
    the last call, in self.processor_variables (a ModuleDict the subclass creates), as
    processor_variables.<processor name>.<variable>.  The processor keeps the registered
    Parameter itself, so the gradients land on the tensor an optimizer updates."""
    for proc in self.processor_group.processors:
      if not hasattr(proc, 'named_variables'):
        continue
      for name, variable in proc.named_variables():
        if proc.name not in self.processor_variables:
          self.processor_variables[proc.name] = torch.nn.Module()
        holder = self.processor_variables[proc.name]
        if getattr(holder, name, None) is not variable:
          holder.register_parameter(name, variable)

  def call(self, *args, training=False, **kwargs):
    """Runs the forward pass, adds the losses to self._losses_dict and returns a dict
    of the relevant output tensors."""
    raise NotImplementedError('Must implement a `self.call()` method.')


class Autoencoder(Model):
  """Preprocessor -> encoder -> decoder -> processor group, with losses between the
  features' 'audio' and the synthesized audio.

  As Keras does, call() adds the preprocessor's, encoder's and decoder's outputs to the
  caller's features dict.  The preprocessor and encoder may be None.  Losses are
  computed only when training is true.

  Parameters are created at the first call, as every lazy layer here creates its own:
  the encoder's and decoder's, and the trainable variables of the processor group's
  processors (the impulse response of Reverb(trainable=True), the magnitudes of
  FilteredNoiseReverb, the gain and decay of ExpDecayReverb).  Those are registered
  as this model's parameters under processor_variables.<processor name>.<variable>, so
  build an optimizer from model.parameters() after the first call, and the state_dict
  holds them from then on."""

  def __init__(self, preprocessor=None, encoder=None, decoder=None, processor_group=None,
               losses=None):
    super().__init__()
    self.preprocessor = preprocessor
    self.encoder = encoder
    self.decoder = decoder
    self.processor_group = processor_group
    self.loss_objs = list(core.make_iterable(losses))
    self.processor_variables = torch.nn.ModuleDict()

  def encode(self, features, training=True):
    """Get conditioning by preprocessing then encoding."""
    if self.preprocessor is not None:
      features.update(self.preprocessor(features))
    if self.encoder is not None:
      features.update(self.encoder(features))
    return features

  def decode(self, features, training=True):
    """Get generated audio by decoding then processing."""
    features.update(self.decoder(features))
    audio = self.processor_group(features)
    self._register_processor_variables()
    return audio

  def get_audio_from_outputs(self, outputs):
    """Extract audio output tensor from outputs dict of call()."""
    return outputs['audio_synth']

  def call(self, features, training=True):
    """Run the core of the network, get predictions and loss."""
    features = self.encode(features, training=training)
    features.update(self.decoder(features))
    pg_out = self.processor_group(features, return_outputs_dict=True)
    self._register_processor_variables()
    outputs = pg_out['controls']
    outputs['audio_synth'] = pg_out['signal']
    if training:
      self._update_losses_dict(self.loss_objs, features['audio'], outputs['audio_synth'])
    return outputs



class InverseSynthesis(Model):
  """The inverse-synthesis model (DDSP-INV, ICML 2020): audio -> sinusoids ->
  harmonics -> sinusoids -> audio.

  sinusoidal_encoder (e.g. encoders.ResnetSinusoidalEncoder) maps the features to raw
  'frequencies', 'amplitudes' and 'noise_magnitudes'; frequencies go through
  freq_scale_fn (frequencies_softmax, depth 64) and both amplitude kinds through
  exp_sigmoid.  A Sinusoidal and a FilteredNoise synthesizer (window_size 0), added and,
  with reverb=True, through a trainable FilteredNoiseReverb (2 s, 500 frames, 16 banks),
  make 'sin_audio'.  harmonic_encoder (e.g. encoders.SinusoidalToHarmonicEncoder, or
  None) maps the sinusoids to a harmonic model, synthesized as sinusoids at f0 [1..K]
  by the same processor group: 'harm_audio'.  With stop_gradient the harmonic branch
  sees the sinusoid controls detached, and so do the sinusoidal consistency losses.

  call() takes plain features (losses sin_*, the harmonic prior, harm_*, the
  consistency and TWM losses), a self-supervised dict that has 'sin_amps' (its audio is
  synthesized from the controls; the same losses plus ss_* against the true controls),
  or a (features, ss_features) pair in either order, run as one batch and split at the
  first one's batch size; the zipped outputs drop nested dicts, as the reference does.

  The reverb's magnitudes are created at the first call and registered then as
  processor_variables.reverb.magnitudes, as Autoencoder registers its processors'
  variables: build an optimizer from model.parameters() after the first call."""

  def __init__(self,
               sinusoidal_encoder=None,
               harmonic_encoder=None,
               losses=None,
               sinusoidal_consistency_losses=None,
               harmonic_consistency_losses=None,
               filtered_noise_consistency_loss=None,
               twm_loss=None,
               harmonic_distribution_prior=None,
               freq_scale_fn=None,
               reverb=True,
               n_samples=64000,
               sample_rate=16000,
               stop_gradient=True):
    super().__init__()
    self.sinusoidal_encoder = sinusoidal_encoder
    self.harmonic_encoder = harmonic_encoder
    self.audio_loss_objs = list(core.make_iterable(losses))
    self.sinusoidal_consistency_losses = list(core.make_iterable(
        sinusoidal_consistency_losses))
    self.harmonic_consistency_losses = list(core.make_iterable(harmonic_consistency_losses))
    self.filtered_noise_consistency_loss = filtered_noise_consistency_loss
    self.twm_loss = twm_loss
    self.harmonic_distribution_prior = harmonic_distribution_prior
    self.stop_gradient = stop_gradient

    self.n_samples = n_samples
    self.sample_rate = sample_rate
    self.amps_scale_fn = core.exp_sigmoid
    self.freq_scale_fn = freq_scale_fn or functools.partial(core.frequencies_softmax,
                                                            depth=64)
    self.sinusoidal_synth = synths.Sinusoidal(
        n_samples=self.n_samples, sample_rate=self.sample_rate, amp_scale_fn=None,
        freq_scale_fn=None, name='sinusoidal')
    self.filtered_noise_synth = synths.FilteredNoise(
        n_samples=self.n_samples, window_size=0, scale_fn=None, name='filtered_noise')
    dag = [
        (self.sinusoidal_synth, ['amplitudes', 'frequencies']),
        (self.filtered_noise_synth, ['noise_magnitudes']),
        (processors.Add(), [f'{self.filtered_noise_synth.name}/signal',
                            f'{self.sinusoidal_synth.name}/signal']),
    ]
    if reverb:
      self.reverb = effects.FilteredNoiseReverb(
          reverb_length=int(self.sample_rate * 2), window_size=257, n_frames=500,
          n_filter_banks=16, trainable=True, name='reverb')
      dag.append((self.reverb, ['add/signal']))
    self.processor_group = processors.ProcessorGroup(dag=dag)
    self.processor_variables = torch.nn.ModuleDict()

  def _dispatch(self, *args, **kwargs):
    # forward() is the reference's model pass, so calls go to call() directly.
    return self.call(*args, **kwargs)

  def generate_synthetic_audio(self, features):
    """Convert synthetic controls into audio."""
    audio = self.processor_group({
        'amplitudes': features['sin_amps'],
        'frequencies': features['sin_freqs'],
        'noise_magnitudes': features['noise_magnitudes']
    })
    self._register_processor_variables()
    return audio

  def parse_zipped_features(self, features):
    """(features, self-supervised features) of a pair in either order: the one whose
    'sin_amps' is not None is the self-supervised one."""
    assert len(features) == 2
    ss_idx = int(features[1].get('sin_amps') is not None)
    s_idx = int(not ss_idx)
    return features[s_idx], features[ss_idx]

  def get_audio_from_outputs(self, outputs):
    """Extract audio output tensor from outputs dict of call()."""
    return (outputs['sin_audio'] if self.harmonic_encoder is None else
            outputs['harm_audio'])

  def call(self, features, training=True):
    """Run the core of the network, get predictions and loss."""
    if isinstance(features, (list, tuple)):
      features, ss_features = self.parse_zipped_features(features)
      ss_features = core.copy_if_tf_function(ss_features)
      ss_features['audio'] = self.generate_synthetic_audio(ss_features)
      batch_size = features['audio'].shape[0]
      inputs = {'audio': torch.cat([features['audio'], ss_features['audio']], dim=0)}
      all_outputs = self.forward(inputs, training)
      outputs = {k: v[:batch_size] for k, v in all_outputs.items()
                 if not isinstance(v, dict)}
      ss_outputs = {k: v[batch_size:] for k, v in all_outputs.items()
                    if not isinstance(v, dict)}
      self.append_losses(outputs)
      self.append_losses(ss_outputs, ss_features)
    elif features.get('sin_amps') is not None:
      ss_features = core.copy_if_tf_function(features)
      ss_features['audio'] = self.generate_synthetic_audio(ss_features)
      outputs = self.forward(ss_features, training)
      self.append_losses(outputs)
      self.append_losses(outputs, ss_features)
    else:
      outputs = self.forward(features, training)
      self.append_losses(outputs)
    return outputs

  def append_losses(self, outputs, self_supervised_features=None):
    """Compute losses from outputs and append to self._losses_dict."""
    o = outputs
    f = self_supervised_features
    if f is None:
      for loss_obj in self.audio_loss_objs:
        self._losses_dict['sin_{}'.format(loss_obj.name)] = loss_obj(o['audio'],
                                                                     o['sin_audio'])
      if self.harmonic_encoder is not None:
        self._update_losses_dict(self.harmonic_distribution_prior, o['harm_dist'])
        for loss_obj in self.audio_loss_objs:
          self._losses_dict['harm_{}'.format(loss_obj.name)] = loss_obj(o['audio'],
                                                                        o['harm_audio'])
        if self.sinusoidal_consistency_losses:
          sin_amps = o['sin_amps']
          sin_freqs = o['sin_freqs']
          if self.stop_gradient:
            sin_amps = sin_amps.detach()
            sin_freqs = sin_freqs.detach()
          self._update_losses_dict(self.sinusoidal_consistency_losses,
                                   sin_amps, sin_freqs, o['harm_amps'], o['harm_freqs'])
      if self.twm_loss is not None:
        f0_c = o['sin_freqs'] if self.harmonic_encoder is None else o['f0_hz']
        self._update_losses_dict(self.twm_loss, f0_c, o['sin_freqs'], o['sin_amps'])
    else:
      for loss_obj in self.sinusoidal_consistency_losses:
        self._losses_dict['ss_' + loss_obj.name] = loss_obj(
            o['sin_amps'], o['sin_freqs'], f['sin_amps'], f['sin_freqs'])
      fncl = self.filtered_noise_consistency_loss
      if fncl is not None:
        self._losses_dict['ss_' + fncl.name] = fncl(o['noise_magnitudes'],
                                                    f['noise_magnitudes'])
      for loss_obj in self.harmonic_consistency_losses:
        if isinstance(loss_obj, losses_lib.HarmonicConsistencyLoss):
          harm_losses = loss_obj(o['harm_amp'], f['harm_amp'], o['harm_dist'],
                                 f['harm_dist'], o['f0_hz'], f['f0_hz'])
          self._losses_dict.update({'ss_' + k: v for k, v in harm_losses.items()})
        else:
          self._losses_dict['ss_harm_' + loss_obj.name] = loss_obj(
              o['harm_amp'], o['f0_hz'], f['harm_amp'], f['f0_hz'])

  def forward(self, features, training=True):
    """Run forward pass of model (no losses) on a dictionary of features."""
    audio = features['audio']
    pg_in = self.sinusoidal_encoder(features, training=training)
    sin_freqs = self.freq_scale_fn(pg_in['frequencies'])
    sin_amps = self.amps_scale_fn(pg_in['amplitudes'])
    noise_magnitudes = self.amps_scale_fn(pg_in['noise_magnitudes'])
    pg_in['frequencies'] = sin_freqs
    pg_in['amplitudes'] = sin_amps
    pg_in['noise_magnitudes'] = noise_magnitudes

    controls = self.processor_group.get_controls(pg_in)
    sin_audio = self.processor_group.get_signal(controls)
    self._register_processor_variables()
    outputs = {
        'audio': audio,
        'noise_magnitudes': noise_magnitudes,
        'sin_audio': sin_audio,
        'sin_amps': sin_amps,
        'sin_freqs': sin_freqs,
    }
    outputs.update(controls)

    if self.stop_gradient:
      sin_freqs = sin_freqs.detach()
      sin_amps = sin_amps.detach()
      noise_magnitudes = noise_magnitudes.detach()

    if self.harmonic_encoder is not None:
      h_out = self.harmonic_encoder(sin_freqs, sin_amps)
      harm_amp, harm_dist, f0_hz = [h_out[k] for k in ['harm_amp', 'harm_dist', 'f0_hz']]
      n_harmonics = int(harm_dist.shape[-1])
      harm_freqs = core.get_harmonic_frequencies(f0_hz, n_harmonics)
      harm_amps = harm_amp * harm_dist
      pg_in['frequencies'] = harm_freqs
      pg_in['amplitudes'] = harm_amps
      pg_in['noise_magnitudes'] = noise_magnitudes
      harm_audio = self.processor_group(pg_in)
      outputs.update({
          'harm_audio': harm_audio,
          'harm_amp': harm_amp,
          'harm_dist': harm_dist,
          'f0_hz': f0_hz,
          'harm_freqs': harm_freqs,
          'harm_amps': harm_amps,
      })
    return outputs
