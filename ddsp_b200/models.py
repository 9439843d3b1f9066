"""models.Model and models.Autoencoder (ddsp/training/models/model.py:26-131,
autoencoder.py:24-74): the model that wires a preprocessor, an encoder, a decoder, a
ProcessorGroup and losses into one training step, as ae.gin, solo_instrument.gin and
the VST configs build it.  Each part runs on its own kernels; this module is Python
glue."""
import torch

from ddsp_b200 import core


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
    outputs = super().__call__(*args, **kwargs)
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

  def forward(self, *args, **kwargs):
    return self.call(*args, **kwargs)

  def sum_losses(self, losses_dict):
    """Sum of the scalar losses of a dict, a 0-d tensor."""
    values = list(losses_dict.values())
    return torch.stack(values).sum() if values else torch.zeros(())

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

  def _register_processor_variables(self):
    """Registers the variables the processors have built since the last call.  The
    processor keeps the registered Parameter itself, so the gradients land on the tensor
    an optimizer updates."""
    for proc in self.processor_group.processors:
      if not hasattr(proc, 'named_variables'):
        continue
      for name, variable in proc.named_variables():
        if proc.name not in self.processor_variables:
          self.processor_variables[proc.name] = torch.nn.Module()
        holder = self.processor_variables[proc.name]
        if getattr(holder, name, None) is not variable:
          holder.register_parameter(name, variable)
