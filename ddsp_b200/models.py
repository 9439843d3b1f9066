"""models.Model and models.Autoencoder (ddsp/training/models/model.py:26-131,
autoencoder.py:24-74): the model that wires a preprocessor, an encoder, a decoder, a
ProcessorGroup and losses into one training step, as ae.gin, solo_instrument.gin and
the VST configs build it.  models.InverseSynthesis (inverse_synthesis.py:24-330) is
the self-supervised pitch model of pretrain_model.gin and finetune_model.gin.
models.MidiAutoencoder and models.ZMidiAutoencoder (midi_autoencoder.py:28-615) are the
MIDI autoencoders of midiae.gin and z_midiae.gin.  Each part runs on its own kernels;
this module is Python glue."""
import functools

import torch

from ddsp_b200 import core
from ddsp_b200 import effects
from ddsp_b200 import losses as losses_lib
from ddsp_b200 import nn
from ddsp_b200 import preprocessing
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


class MidiAutoencoder(Model):
  """An autoencoder with a MIDI representation at its bottleneck, in two branches.  The
  synthcoder branch: preprocessor -> synthcoder (e.g. decoders.DilatedConvDecoder) ->
  Harmonic + FilteredNoise (-> a trainable FilteredNoiseReverb of 24000 taps, 500 frames
  and 32 banks, with reverb) -> 'synth_audio'.  The MIDI branch: the synthcoder's
  controls (in dB; detached with sg_before_midiae) -> midi_encoder (e.g.
  encoders.HarmonicToMidiEncoder), quantized to integers by the straight-through
  estimator -> midi_decoder (decoders.MidiToHarmonicDecoder) -> the same processor group
  -> 'midi_audio'.  With midi_encoder None, the MIDI comes from the features'
  'note_active_velocities' piano roll, and with mask_f0_loss the f0 loss is weighted to
  frames within 2 semitones of it.

  The db key is 'power_db' for a preprocessing.F0PowerPreprocessor, else 'loudness_db'.
  The synthcoder branch passes the preprocessor no audio, so a preprocessor that computes
  loudness from audio fails there, as it does in the reference.  Loss objects
  (qpitch_f0rec_loss, pitch_f0rec_loss, pitch_qpitch_loss) are anything
  _update_losses_dict takes; midi_slowness_loss is called as loss(z_pitch, mask) and
  named by its `name`.  Losses are computed only when training is true.
  midi_decoder=None raises ValueError (the reference fails at its first call).

  The reverb's magnitudes are created at the first call and registered then as
  processor_variables.reverb.magnitudes: build an optimizer from model.parameters() after
  the first call."""

  def __init__(self, synthcoder=None, midi_encoder=None, midi_decoder=None,
               sg_before_midiae=True, reverb=True, preprocessor=None,
               reconstruction_losses=None, qpitch_f0rec_loss=None, pitch_f0rec_loss=None,
               pitch_qpitch_loss=None, midi_slowness_loss=None, mask_f0_loss=True):
    super().__init__()
    if midi_decoder is None:
      raise ValueError(f'{type(self).__name__}: midi_decoder=None; the model needs a MIDI '
                       'decoder (the reference fails at its first call without one)')
    self.synthcoder = synthcoder
    self.midi_encoder = midi_encoder
    self.midi_decoder = midi_decoder
    self.reconstruction_losses = reconstruction_losses
    self.mask_f0_loss = mask_f0_loss
    self.qpitch_f0rec_loss = qpitch_f0rec_loss
    self.pitch_f0rec_loss = pitch_f0rec_loss
    self.pitch_qpitch_loss = pitch_qpitch_loss
    self.slowness_loss = midi_slowness_loss
    self.sg_before_midiae = sg_before_midiae
    self.preprocessor = preprocessor
    if isinstance(self.preprocessor, preprocessing.F0PowerPreprocessor):
      self.db_key = 'power_db'
    else:
      self.db_key = 'loudness_db'
    dag = [
        (synths.Harmonic(), ['amplitudes', 'harmonic_distribution', 'f0_hz']),
        (synths.FilteredNoise(), ['magnitudes']),
        (processors.Add(), ['filtered_noise/signal', 'harmonic/signal']),
    ]
    if reverb:
      dag.append((effects.FilteredNoiseReverb(trainable=True, reverb_length=24000,
                                              n_frames=500, n_filter_banks=32,
                                              name='reverb'), ['add/signal']))
    self.processor_group = processors.ProcessorGroup(dag=dag)
    self.processor_variables = torch.nn.ModuleDict()

  def _controls_and_signal(self, pg_in):
    controls = self.processor_group.get_controls(pg_in)
    audio = self.processor_group.get_signal(controls)
    self._register_processor_variables()
    return controls, audio

  def encode_to_midi(self, *args):
    """Encodes *args (f0, amps, hd, noise) into MIDI with a network."""
    if self.sg_before_midiae:
      args = [arg.detach() for arg in args]
    z_pitch, z_vel = self.midi_encoder(*args).values()
    q_pitch = nn.straight_through_int_quantization(z_pitch)
    z_vel = z_vel * 0.0
    q_vel = z_vel
    return z_pitch, q_pitch, z_vel, q_vel

  def synthesize_audio(self, f0_hz, db, z=None, training=False, return_params=False):
    """Run synthcoder and processor group."""
    features = {'f0_hz': f0_hz, self.db_key: db}
    if z is not None:
      features['z'] = z
    features.update(self.preprocessor(features))
    features.update(self.synthcoder(features, training=training))
    synth_params, audio = self._controls_and_signal(features)
    return (audio, synth_params) if return_params else audio

  @staticmethod
  def extract_harm_controls(synth_params, log_scale=True, stop_gradient=False):
    """Get harmonic synth controls from the outputs of the processor group."""
    amps = synth_params['harmonic']['controls']['amplitudes']
    hd = synth_params['harmonic']['controls']['harmonic_distribution']
    noise = synth_params['filtered_noise']['controls']['magnitudes']
    if log_scale:
      amps = core.amplitude_to_db(amps, use_tf=True)
      noise = core.amplitude_to_db(noise, use_tf=True)
    if stop_gradient:
      amps, hd, noise = amps.detach(), hd.detach(), noise.detach()
    return amps, hd, noise

  @staticmethod
  def pianoroll_to_midi(pianoroll):
    """Converts a piano roll into conditioning format for the decoder: the argmax key
    (the first of ties) and the largest velocity of each frame, [B, T, 1] each."""
    notes = torch.argmax(pianoroll, dim=-1).to(torch.float32)[:, :, None]
    velocities = torch.amax(pianoroll, dim=-1)[:, :, None]
    return notes, velocities

  @staticmethod
  def midi_to_pianoroll(q_pitch, q_vel, piano_keys=128, thresh=20.0):
    """One-hot piano roll [..., piano_keys] of the quantized pitch with every axis of
    length 1 squeezed out, as tf.squeeze does (so B = 1 drops the batch axis).  Pitches
    at or below thresh (when thresh > 0) give key 0; a pitch truncated to an integer
    outside [0, piano_keys) gives a zero row, as tf.one_hot does."""
    midi_space = torch.squeeze(q_pitch.detach())
    if thresh > 0.0:
      midi_space = midi_space * (midi_space > thresh).to(midi_space.dtype)
    keys = torch.trunc(midi_space).to(torch.int64)
    inside = (keys >= 0) & (keys < piano_keys)
    roll = torch.nn.functional.one_hot(torch.where(inside, keys, 0), piano_keys)
    return (roll * inside[..., None]).to(torch.float32)

  def add_closeness_loss(self, loss_obj, f0, pitch, tag=''):
    """Applies loss_obj on abs(f0 - pitch)."""
    self._update_losses_dict(loss_obj, torch.abs(pitch - f0))

  def add_slowness_loss(self, loss_obj, z_pitch, q_pitch, tag=''):
    """Applies slowness loss to pitch encoding for short notes: the frames of notes
    shorter than 40 frames with a pitch above 0.  (The reference passes the first note's
    length alone, [B], which broadcasts against the [B, notes] pitches only at B = 1;
    this passes every note's length.)"""
    if loss_obj is not None:
      note_mask = nn.get_note_mask(q_pitch, note_on_only=False)
      note_lengths = nn.get_note_lengths(note_mask)
      note_pitches = nn.get_note_moments(q_pitch, note_mask, return_std=False)
      loss_mask = nn.get_short_note_loss_mask(note_mask, note_lengths,
                                              note_pitches[..., 0], min_length=40)
      self._losses_dict[f'{loss_obj.name}{tag}'] = self.slowness_loss(z_pitch, loss_mask)

  def add_zpitch_losses(self, z_pitch, q_pitch, f0_midi_pred):
    """Helper function to update pitch encoder losses (if z_pitch available)."""
    if z_pitch is not None:
      self.add_slowness_loss(self.slowness_loss, z_pitch, q_pitch)
      self._update_losses_dict(self.pitch_qpitch_loss, z_pitch, q_pitch)
      self.add_closeness_loss(self.pitch_f0rec_loss, f0_midi_pred, z_pitch)

  def midi_to_audio(self, q_pitch, q_vel, z=None, return_synth_params=False):
    """Decode midi or piano roll to audio."""
    midi_synth_params, midi_audio = self._controls_and_signal(
        self.midi_decoder(q_pitch, q_vel, z))
    return (midi_audio, midi_synth_params) if return_synth_params else midi_audio

  def get_audio_from_outputs(self, outputs):
    """Extract audio output tensor from outputs dict of call()."""
    return outputs['synth_audio']

  def preprocess(self, features):
    """Run preprocessor and add extra keys to `features`."""
    features.update(self.preprocessor(features))
    features['f0_midi'] = core.hz_to_midi(features['f0_hz'])
    features['db'] = features[self.db_key]
    return features

  def synthcoder_branch(self, features, training=True, z=None):
    """Wrapper to run the synthcoder branch."""
    return self.synthesize_audio(features['f0_hz'], features['db'], z=z, training=training,
                                 return_params=True)

  def get_gt_midi(self, features):
    """Prepare the ground truth MIDI."""
    q_pitch, q_vel = self.pianoroll_to_midi(features['note_active_velocities'])
    q_vel = q_vel * 0.0   # velocities are not used
    f0_loss_weights = None
    if self.mask_f0_loss:
      f0_loss_weights = (torch.abs(features['f0_midi'] - q_pitch) < 2.0).to(torch.float32)
    return q_pitch, q_vel, f0_loss_weights

  def _midi_pitch(self, features, amps, hd, noise):
    """(z_pitch, q_pitch, q_vel, f0_loss_weights) from the MIDI encoder, or from the
    ground-truth piano roll without one (z_pitch None)."""
    if self.midi_encoder is not None:
      f0_midi = features['f0_midi']
      z_pitch, q_pitch, _, q_vel = self.encode_to_midi(f0_midi, amps, hd, noise)
      return z_pitch, q_pitch, q_vel, torch.ones_like(f0_midi)
    q_pitch, q_vel, f0_loss_weights = self.get_gt_midi(features)
    return None, q_pitch, q_vel, f0_loss_weights

  def _finish(self, outputs, features, synth_params, training):
    """The reference's outputs dict, without the None entries, with the features and
    synth_params added; the reconstruction losses when training."""
    outputs = {k: v for k, v in outputs.items() if v is not None}
    outputs.update({k: v for k, v in features.items() if k not in outputs})
    outputs.update(synth_params)
    if training and self.reconstruction_losses is not None:
      self._losses_dict.update(self.reconstruction_losses(outputs))
    return outputs

  def _outputs(self, synth_params, synth_audio, midi_synth_params, midi_audio, q_pitch,
               q_vel, f0_midi_pred, amps, hd, noise, features, f0_loss_weights, **extra):
    amps_pred, hd_pred, noise_pred = self.extract_harm_controls(midi_synth_params)
    outputs = {
        'synth_params': synth_params,
        'synth_audio': synth_audio,
        'midi_synth_params': midi_synth_params,
        'midi_audio': midi_audio,
        'q_pitch': q_pitch,
        'q_vel': q_vel,
        **extra,
        'pianoroll': self.midi_to_pianoroll(q_pitch, q_vel),
        'f0_midi_pred': f0_midi_pred,
        'f0_hz_pred': core.midi_to_hz(f0_midi_pred),
        'amps': amps,
        'hd': hd,
        'noise': noise,
        'amps_pred': amps_pred,
        'hd_pred': hd_pred,
        'noise_pred': noise_pred,
        'f0_loss_weights': f0_loss_weights,
        f'{self.db_key}_pred': features['db'],
    }
    return outputs

  def call(self, features, training=True):
    """Run the network to get a prediction and optionally get losses."""
    features = self.preprocess(features)
    synth_audio, synth_params = self.synthcoder_branch(features, training)
    amps, hd, noise = self.extract_harm_controls(synth_params)
    z_pitch, q_pitch, q_vel, f0_loss_weights = self._midi_pitch(features, amps, hd, noise)

    pg_in = self.midi_decoder(q_pitch, q_vel)
    f0_midi_pred = pg_in['f0_midi']
    midi_synth_params, midi_audio = self._controls_and_signal(pg_in)
    if training:
      self.add_zpitch_losses(z_pitch, q_pitch, f0_midi_pred)
      self.add_closeness_loss(self.qpitch_f0rec_loss, f0_midi_pred, q_pitch)

    outputs = self._outputs(synth_params, synth_audio, midi_synth_params, midi_audio,
                            q_pitch, q_vel, f0_midi_pred, amps, hd, noise, features,
                            f0_loss_weights, z_pitch=z_pitch)
    return self._finish(outputs, features, synth_params, training)


class ZMidiAutoencoder(MidiAutoencoder):
  """A MidiAutoencoder with latents besides the MIDI: z_synth_encoders' z (concatenated)
  condition the synthcoder; z_global_encoders' z and, through z_note_encoder, a per-note
  latent pooled over the notes of q_pitch (nn.get_note_mask, nn.pool_over_notes) are
  concatenated, through z_preconditioning_stack (e.g. nn.FcStackOut) if given, and
  condition the MIDI decoder.  z_global_prior and z_note_prior add their losses and
  replace the latents by what they return.  The synthcoder's controls (in dB) join the
  features as 'amps_scaled', 'hd_scaled' and 'noise_scaled' for the z encoders."""

  def __init__(self, synthcoder=None, midi_encoder=None, midi_decoder=None,
               sg_before_midiae=True, reverb=True, preprocessor=None,
               reconstruction_losses=None, qpitch_f0rec_loss=None, pitch_f0rec_loss=None,
               pitch_qpitch_loss=None, midi_slowness_loss=None, mask_f0_loss=True,
               z_synth_encoders=None, z_global_encoders=None, z_note_encoder=None,
               z_preconditioning_stack=None, z_global_prior=None, z_note_prior=None):
    super().__init__(synthcoder=synthcoder, midi_encoder=midi_encoder,
                     midi_decoder=midi_decoder, sg_before_midiae=sg_before_midiae,
                     reverb=reverb, preprocessor=preprocessor,
                     reconstruction_losses=reconstruction_losses,
                     qpitch_f0rec_loss=qpitch_f0rec_loss, pitch_f0rec_loss=pitch_f0rec_loss,
                     pitch_qpitch_loss=pitch_qpitch_loss,
                     midi_slowness_loss=midi_slowness_loss, mask_f0_loss=mask_f0_loss)
    self.z_synth_encoders = (None if z_synth_encoders is None else
                             torch.nn.ModuleList(z_synth_encoders))
    self.z_global_encoders = (None if z_global_encoders is None else
                              torch.nn.ModuleList(z_global_encoders))
    self.z_note_encoder = z_note_encoder
    self.z_preconditioning_stack = z_preconditioning_stack
    self.z_global_prior = z_global_prior
    self.z_note_prior = z_note_prior

  def z_synth_encode(self, features):
    """Encode other latents besides pitch and velocity."""
    if self.z_synth_encoders is None:
      return None
    return torch.cat([enc(features)['z'] for enc in self.z_synth_encoders], dim=-1)

  def z_global_encode(self, features):
    """Encode other latents besides pitch and velocity."""
    if self.z_global_encoders is None:
      return None
    return torch.cat([enc(features)['z'] for enc in self.z_global_encoders], dim=-1)

  def z_note_encode(self, features, q_pitch):
    """Encode latents per a note with local pooling: each frame gets its note's mean of
    the z_note_encoder's z.  (The reference concatenates pool_over_notes's (mean, std)
    pair with the global latent, which TensorFlow cannot do; the mean is the pooled
    latent.)"""
    if self.z_note_encoder is None:
      return None
    z_notes = self.z_note_encoder(features)['z']
    return nn.pool_over_notes(z_notes, nn.get_note_mask(q_pitch), return_std=False)

  def call(self, features, training=True):
    """Run the network to get a prediction and optionally get losses."""
    features = self.preprocess(features)
    z_synth = self.z_synth_encode(features)
    synth_audio, synth_params = self.synthcoder_branch(features, training, z_synth)
    amps, hd, noise = self.extract_harm_controls(synth_params)
    features['amps_scaled'] = amps
    features['hd_scaled'] = hd
    features['noise_scaled'] = noise
    z_pitch, q_pitch, q_vel, f0_loss_weights = self._midi_pitch(features, amps, hd, noise)
    z_vel = None

    z_global = self.z_global_encode(features)
    z_notes = self.z_note_encode(features, q_pitch)
    if self.z_global_prior is not None:
      self._update_losses_dict(self.z_global_prior, z_global)
      z_global = self.z_global_prior(z_global)
    if self.z_note_prior is not None:
      self._update_losses_dict(self.z_note_prior, z_notes)
      z_notes = self.z_note_prior(z_notes)
    z_midi_decoder = z_global if z_notes is None else torch.cat([z_global, z_notes], dim=-1)
    if self.z_preconditioning_stack is not None:
      z_midi_decoder = self.z_preconditioning_stack(z_midi_decoder)

    pg_in = self.midi_decoder(q_pitch, q_vel, z_midi_decoder)
    f0_midi_pred = pg_in['f0_midi']
    midi_synth_params, midi_audio = self._controls_and_signal(pg_in)
    if training:
      self.add_closeness_loss(self.qpitch_f0rec_loss, f0_midi_pred, q_pitch)
      self.add_zpitch_losses(z_pitch, q_pitch, f0_midi_pred)

    outputs = self._outputs(synth_params, synth_audio, midi_synth_params, midi_audio,
                            q_pitch, q_vel, f0_midi_pred, amps, hd, noise, features,
                            f0_loss_weights, z_pitch=z_pitch, z_vel=z_vel,
                            z_global=z_global, z_notes=z_notes)
    return self._finish(outputs, features, synth_params, training)
