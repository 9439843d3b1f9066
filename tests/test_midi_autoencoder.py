"""models.MidiAutoencoder and models.ZMidiAutoencoder.  On the CPU: the model's
bookkeeping (piano rolls, ground-truth MIDI, the MIDI encoder's stop-gradient and
quantization, the db key, the refusals).  On the GPU: midiae.gin and z_midiae.gin built
as the configs wire them, trained one step end to end, copied and reloaded."""
import copy

import pytest
import torch

from ddsp_b200 import core, decoders, encoders, losses, models, nn, preprocessing

gpu = pytest.mark.gpu


class _Decoder(torch.nn.Module):
  def forward(self, q_pitch, q_vel=None, z=None):
    return {'f0_midi': q_pitch}


def _model(cls=models.MidiAutoencoder, **kw):
  return cls(synthcoder=None, midi_decoder=_Decoder(),
             preprocessor=preprocessing.F0LoudnessPreprocessor(compute_loudness=False),
             **kw)


# ---- CPU ---------------------------------------------------------------------------
def test_refusals_and_db_key():
  with pytest.raises(ValueError, match='midi_decoder'):
    models.MidiAutoencoder(midi_decoder=None)
  with pytest.raises(ValueError, match='midi_decoder'):
    models.ZMidiAutoencoder()
  assert _model().db_key == 'loudness_db'
  power = models.MidiAutoencoder(midi_decoder=_Decoder(),
                                 preprocessor=preprocessing.F0PowerPreprocessor())
  assert power.db_key == 'power_db'
  reverb = _model().processor_group.processors[-1]
  assert reverb.name == 'reverb' and reverb.trainable
  assert reverb._n_frames == 500 and reverb._n_filter_banks == 32
  assert len(_model(reverb=False).processor_group.processors) == 3


@pytest.mark.parametrize('b', [1, 3])
def test_midi_to_pianoroll(b):
  q = torch.tensor([[60.0, 61.7, 20.0, 19.0, 127.0, 128.0]] * b)[:, :, None]
  roll = models.MidiAutoencoder.midi_to_pianoroll(q, None)
  want_shape = (6, 128) if b == 1 else (b, 6, 128)   # tf.squeeze drops B = 1
  assert roll.shape == want_shape
  roll = roll.reshape(b, 6, 128)
  assert roll.sum(-1).tolist() == [[1.0, 1.0, 1.0, 1.0, 1.0, 0.0]] * b
  assert roll.argmax(-1)[0, :5].tolist() == [60, 61, 0, 0, 127]
  assert models.MidiAutoencoder.midi_to_pianoroll(q, None, thresh=0.0).reshape(
      b, 6, 128).argmax(-1)[0, 2:4].tolist() == [20, 19]


def test_ground_truth_midi_and_loss_weights():
  pr = torch.zeros(2, 4, 128)
  pr[0, :, 60] = 0.5
  pr[1, :2, 64] = 1.0
  pr[1, :2, 40] = 1.0   # a tie: the first key wins
  f0_midi = torch.tensor([[60.5, 63.0, 58.5, 60.0], [40.0, 41.0, 0.0, 0.5]])[:, :, None]
  m = _model()
  q_pitch, q_vel, w = m.get_gt_midi({'note_active_velocities': pr, 'f0_midi': f0_midi})
  assert q_pitch[..., 0].tolist() == [[60.0] * 4, [40.0, 40.0, 0.0, 0.0]]
  assert not q_vel.any() and q_vel.shape == (2, 4, 1)
  assert w[..., 0].tolist() == [[1.0, 0.0, 1.0, 1.0], [1.0, 1.0, 1.0, 1.0]]
  assert _model(mask_f0_loss=False).get_gt_midi(
      {'note_active_velocities': pr, 'f0_midi': f0_midi})[2] is None
  notes, vel = m.pianoroll_to_midi(pr)
  assert vel[0, 0, 0] == 0.5 and notes.dtype == torch.float32


class _Encoder(torch.nn.Module):
  def forward(self, f0_midi, amps, hd, noise):
    return {'z_pitch': f0_midi * 1.3 + amps, 'z_vel': amps + 1.0}


@pytest.mark.parametrize('sg', [True, False])
def test_encode_to_midi(sg):
  m = _model(midi_encoder=_Encoder(), sg_before_midiae=sg)
  f0 = torch.tensor([[[40.2], [41.6]]], requires_grad=True)
  amps = torch.zeros(1, 2, 1, requires_grad=True)
  z_pitch, q_pitch, z_vel, q_vel = m.encode_to_midi(f0, amps, amps, amps)
  assert q_pitch[..., 0].tolist() == [[52.0, 54.0]]
  assert not z_vel.any() and q_vel is z_vel
  assert q_pitch.requires_grad == (not sg)
  if not sg:
    (g,) = torch.autograd.grad(q_pitch.sum(), [f0])   # straight-through
    torch.testing.assert_close(g, torch.full_like(f0, 1.3))


def test_closeness_loss_hooks():
  class Loss:
    name = 'l'

    def get_losses_dict(self, x):
      return {'closeness': x.sum()}

  m = _model()
  m._losses_dict = {}
  m.add_closeness_loss(Loss(), torch.tensor([1.0, 2.0]), torch.tensor([2.0, 0.0]))
  assert m._losses_dict['closeness'] == 3.0
  m.add_closeness_loss(None, torch.zeros(1), torch.zeros(1))
  m.add_zpitch_losses(None, None, None)
  assert list(m._losses_dict) == ['closeness']


# ---- GPU: the configs end to end ------------------------------------------------------
B, N, T = 4, 64000, 1000
RECON_KEYS = ['spectral_loss_synth', 'f0_reconstruction', 'amplitude_reconstruction',
              'harmonic_distribution_reconstruction', 'noise_reconstruction']


def _recon_losses():
  return losses.LossGroup(
      dag=[['synth_spectral_loss', ['audio', 'synth_audio']],
           ['f0_loss', ['f0_midi', 'f0_midi_pred', 'f0_loss_weights']],
           ['amps_loss', ['amps', 'amps_pred']],
           ['hd_loss', ['hd', 'hd_pred']],
           ['noise_loss', ['noise', 'noise_pred']]],
      amps_loss=losses.ParamLoss(weight=0.5, loss_type='L1', name='amplitude_reconstruction'),
      f0_loss=losses.ParamLoss(weight=50.0, loss_type='L2', name='f0_reconstruction'),
      hd_loss=losses.ParamLoss(weight=500.0, loss_type='L1',
                               name='harmonic_distribution_reconstruction'),
      noise_loss=losses.ParamLoss(weight=0.5, loss_type='L1', name='noise_reconstruction'),
      synth_spectral_loss=losses.SpectralLoss(loss_type='L1', mag_weight=1.0,
                                              logmag_weight=1.0, name='spectral_loss_synth'))


def _synthcoder(conditional):
  return decoders.DilatedConvDecoder(
      ch=128, layers_per_stack=9, norm_type='layer', input_keys=('ld_scaled', 'f0_scaled'),
      stacks=2, conditioning_keys=('z',) if conditional else None, precondition_stack=None,
      output_splits=(('amplitudes', 1), ('harmonic_distribution', 60), ('magnitudes', 65)))


def _midi_decoder(conditional):
  return decoders.MidiToHarmonicDecoder(
      f0_residual=True, norm=True,
      output_splits=(('f0_midi', 1), ('amplitudes', 1), ('harmonic_distribution', 60),
                     ('magnitudes', 65)),
      net=nn.DilatedConvStack(ch=128, layers_per_stack=5, stacks=4, norm_type='layer',
                              conditional=conditional))


def build_midiae():
  """midiae.gin.  Its synthcoder branch passes the preprocessor no audio, so loudness is
  read from the features rather than computed."""
  return models.MidiAutoencoder(
      preprocessor=preprocessing.F0LoudnessPreprocessor(time_steps=T, compute_loudness=False),
      synthcoder=_synthcoder(False), sg_before_midiae=True, midi_encoder=None,
      midi_decoder=_midi_decoder(False), reconstruction_losses=_recon_losses())


def build_z_midiae():
  """z_midiae.gin."""
  z_stack = lambda: nn.DilatedConvStack(ch=128, layers_per_stack=5, stacks=4,
                                        norm_type='layer', conditional=False)
  expression = lambda pool: encoders.ExpressionEncoder(
      input_keys=('f0_scaled', 'amps_scaled', 'hd_scaled', 'noise_scaled'), z_dims=128,
      pool_time=pool, net=z_stack())
  one_hot = lambda: encoders.OneHotEncoder(one_hot_key='instrument_id', vocab_size=13,
                                           n_dims=128, skip_expand=False)
  return models.ZMidiAutoencoder(
      preprocessor=preprocessing.F0LoudnessPreprocessor(time_steps=T, compute_loudness=False),
      z_synth_encoders=[one_hot(), encoders.MfccTimeDistributedRnnEncoder(
          rnn_channels=512, rnn_type='gru', z_dims=128, z_time_steps=1000)],
      synthcoder=_synthcoder(True), sg_before_midiae=True, midi_encoder=None,
      z_global_encoders=[one_hot(), expression(True)], z_note_encoder=expression(False),
      z_preconditioning_stack=nn.FcStackOut(ch=512, layers=5, n_out=256),
      midi_decoder=_midi_decoder(True), reconstruction_losses=_recon_losses())


def features(b=B, seed=0):
  g = torch.Generator().manual_seed(seed)
  t = torch.arange(N) / 16000.0
  f0 = 220.0 * 2 ** (torch.randint(0, 12, (b, 1), generator=g) / 12.0)
  audio = 0.3 * torch.sin(2 * torch.pi * f0 * t) + 0.01 * torch.randn(b, N, generator=g)
  f0_hz = f0[:, :, None].expand(b, T, 1) * (1 + 0.01 * torch.randn(b, T, 1, generator=g))
  ld = -30.0 + 5 * torch.randn(b, T, 1, generator=g)
  keys = (69 + 12 * torch.log2(f0 / 440.0)).round().long()
  pr = torch.zeros(b, T, 128)
  pr[torch.arange(b)[:, None], torch.arange(T)[None, :], keys.expand(b, T)] = 0.8
  pr[:, :50] = 0.0
  feats = {'audio': audio, 'f0_hz': f0_hz, 'loudness_db': ld, 'note_active_velocities': pr,
           'instrument_id': torch.randint(0, 13, (b,), generator=g)}
  return {k: v.cuda() for k, v in feats.items()}


@gpu
@pytest.mark.parametrize('build', [build_midiae, build_z_midiae])
def test_config_trains_end_to_end(build):
  torch.manual_seed(0)
  model = build()
  outputs, loss = model(features(), training=True, return_losses=True)
  assert set(RECON_KEYS + ['total_loss']) == set(loss)
  for key in ('synth_audio', 'midi_audio', 'pianoroll', 'f0_hz_pred', 'amps_pred',
              'loudness_db_pred', 'f0_loss_weights', 'q_pitch'):
    assert key in outputs, key
  assert outputs['synth_audio'].shape == (B, N) and outputs['pianoroll'].shape == (B, T, 128)
  if build is build_z_midiae:
    assert outputs['z_global'].shape == (B, T, 256) and outputs['z_notes'].shape == (B, T, 128)
  loss['total_loss'].backward()
  named = dict(model.named_parameters())
  assert 'processor_variables.reverb.magnitudes' in named
  for name, p in named.items():
    assert p.grad is not None, name
    assert torch.isfinite(p.grad).all() and p.grad.abs().max() > 0, name
  before = {n: p.detach().clone() for n, p in named.items()}
  torch.optim.Adam(model.parameters(), lr=1e-3).step()
  for name, p in named.items():
    assert not torch.equal(before[name], p.detach()), name


@gpu
@pytest.mark.parametrize('build', [build_midiae, build_z_midiae])
def test_copies_and_state_dict(build):
  torch.manual_seed(1)
  model = build()
  feats = features(b=2, seed=3)
  with torch.no_grad():
    out = model(dict(feats), training=False)
    twin = copy.deepcopy(model)
    fresh = build()
    fresh(dict(feats), training=False)   # builds the lazy layers
    fresh.load_state_dict(model.state_dict())
    for other in (twin, fresh):
      got = other(dict(feats), training=False)
      # the audio carries each call's own filtered noise; the controls do not
      for key in ('f0_midi_pred', 'amps', 'hd', 'noise', 'amps_pred', 'hd_pred',
                  'noise_pred'):
        assert torch.equal(got[key], out[key]), key


# ---- GPU: the MIDI encoder branch and the loss hooks ------------------------------
# Notes of each item, (MIDI pitch, frames): items differ, so the short-note mask of one
# item can only come from that item's own note lengths.
NOTES = [[(60, 30), (62, 200), (64, 10), (65, 760)],
         [(50, 300), (0, 20), (55, 35), (57, 645)],
         [(70, 39), (72, 40), (74, 921)]]


class _Synthcoder(torch.nn.Module):
  """Controls from ld_scaled, f0_scaled (and z) through one Dense layer."""

  def __init__(self):
    super().__init__()
    self.dense = nn.Dense(18)

  def forward(self, features, training=True):
    x = [features['ld_scaled'], features['f0_scaled']] + (
        [features['z']] if 'z' in features else [])
    return nn.split_to_dict(self.dense(torch.cat(x, -1)), (('amplitudes', 1),
                                                           ('harmonic_distribution', 8),
                                                           ('magnitudes', 9)))


class _MidiEncoder(torch.nn.Module):
  """z_pitch = f0_midi + a learned offset (0 at first), z_vel from the amplitudes."""

  def __init__(self):
    super().__init__()
    self.offset = torch.nn.Parameter(torch.zeros(()))

  def forward(self, f0_midi, amps, hd, noise):
    return {'z_pitch': f0_midi + self.offset, 'z_vel': amps}


class _ZEncoder(torch.nn.Module):
  def __init__(self):
    super().__init__()
    self.dense = nn.Dense(4)

  def forward(self, features):
    return {'z': self.dense(features['f0_scaled'])}


class _Loss:
  """A loss object with get_losses_dict, keeping its arguments."""

  def __init__(self, name):
    self.name = name
    self.seen = None

  def get_losses_dict(self, *args):
    self.seen = args
    return {self.name: sum(torch.mean(torch.abs(a)) for a in args)}


class _Slowness:
  name = 'slowness'

  def __init__(self):
    self.mask = None

  def __call__(self, z_pitch, mask):
    self.mask = mask
    return torch.sum(z_pitch[..., 0] * mask) / 1e3


class _Prior(_Loss):
  """A prior: a loss on the latent, and the latent it samples (half the input)."""

  def __call__(self, z):
    return 0.5 * z


def _notes_features():
  f0_midi = torch.cat([torch.cat([torch.full((n,), float(p)) for p, n in item])[None]
                       for item in NOTES])[:, :, None]
  b = f0_midi.shape[0]
  g = torch.Generator().manual_seed(4)
  return {'audio': 0.1 * torch.randn(b, 64000, generator=g).cuda(),
          'f0_hz': core.midi_to_hz(f0_midi, midi_zero_silence=True).cuda(),
          'loudness_db': (-40.0 + torch.randn(b, 1000, 1, generator=g)).cuda()}


def _midi_decoder_small(conditional):
  return decoders.MidiToHarmonicDecoder(
      net=nn.DilatedConvStack(ch=16, layers_per_stack=2, stacks=1, norm_type='layer',
                              conditional=conditional),
      output_splits=(('f0_midi', 1), ('amplitudes', 1), ('harmonic_distribution', 8),
                     ('magnitudes', 9)))


def _encoder_branch(cls, midi_encoder, **kw):
  hooks = {'qpitch_f0rec_loss': _Loss('qpitch_f0rec'),
           'pitch_f0rec_loss': _Loss('pitch_f0rec'),
           'pitch_qpitch_loss': _Loss('pitch_qpitch'),
           'midi_slowness_loss': _Slowness()}
  model = cls(synthcoder=_Synthcoder(), midi_encoder=midi_encoder,
              midi_decoder=_midi_decoder_small(cls is models.ZMidiAutoencoder),
              preprocessor=preprocessing.F0LoudnessPreprocessor(compute_loudness=False),
              reconstruction_losses=lambda o: {'recon': torch.mean(torch.abs(
                  o['synth_audio'] - o['audio']))}, reverb=False, **hooks, **kw)
  return model, hooks


def _expected_slowness_mask(q_pitch):
  """Frames of each item's notes shorter than 40 frames with a pitch above 0."""
  mask = torch.zeros(q_pitch.shape[:2])
  for b, item in enumerate(NOTES):
    t = 0
    for pitch, n in item:
      if n < 40 and pitch > 0:
        mask[b, t:t + n] = 1.0
      t += n
  return mask


@gpu
@pytest.mark.parametrize('cls', [models.MidiAutoencoder, models.ZMidiAutoencoder])
def test_midi_encoder_branch_and_loss_hooks(cls):
  torch.manual_seed(5)
  z_kw = {}
  if cls is models.ZMidiAutoencoder:
    z_kw = dict(z_global_encoders=[_ZEncoder()], z_note_encoder=_ZEncoder(),
                z_global_prior=_Prior('global_kl'), z_note_prior=_Prior('note_kl'))
  model, hooks = _encoder_branch(cls, _MidiEncoder(), **z_kw)
  outputs, loss = model(_notes_features(), training=True, return_losses=True)
  want = {'slowness', 'pitch_qpitch', 'pitch_f0rec', 'qpitch_f0rec', 'recon', 'total_loss'}
  if cls is models.ZMidiAutoencoder:
    want |= {'global_kl', 'note_kl'}
  assert set(loss) == want

  # the encoder's pitch, quantized; the closeness losses see |f0 - pitch|
  q_pitch, z_pitch, f0_pred = outputs['q_pitch'], outputs['z_pitch'], outputs['f0_midi_pred']
  assert torch.equal(q_pitch, torch.round(z_pitch)) and 'z_pitch' in outputs
  assert torch.equal(hooks['pitch_qpitch_loss'].seen[0], z_pitch)
  assert torch.equal(hooks['pitch_qpitch_loss'].seen[1], q_pitch)
  assert torch.equal(hooks['pitch_f0rec_loss'].seen[0], torch.abs(z_pitch - f0_pred))
  assert torch.equal(hooks['qpitch_f0rec_loss'].seen[0], torch.abs(q_pitch - f0_pred))
  assert not outputs['q_vel'].any()
  assert torch.equal(outputs['f0_loss_weights'], torch.ones_like(outputs['f0_midi']))

  # the slowness mask: every note's own length, at B = 3
  mask = hooks['midi_slowness_loss'].mask
  note_mask = nn.get_note_mask(q_pitch, note_on_only=False)
  lib = nn.get_short_note_loss_mask(note_mask, nn.get_note_lengths(note_mask),
                                    nn.get_note_moments(q_pitch, note_mask,
                                                        return_std=False)[..., 0])
  assert torch.equal(mask, lib)
  assert torch.equal(mask.cpu(), _expected_slowness_mask(q_pitch))

  if cls is models.ZMidiAutoencoder:
    # the priors' samples replace the latents the MIDI decoder sees
    g, n = model.z_global_prior.seen[0], model.z_note_prior.seen[0]
    assert g.shape == (3, 1000, 4) and n.shape == (3, 1000, 4)
    assert torch.equal(outputs['z_global'], 0.5 * g)
    assert torch.equal(outputs['z_notes'], 0.5 * n)

  loss['total_loss'].backward()
  # the stop-gradient before the MIDI encoder leaves the synthcoder to the other losses;
  # the straight-through quantization trains the encoder
  assert model.midi_encoder.offset.grad is not None and model.midi_encoder.offset.grad != 0
  assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.grad is not None)


@gpu
@pytest.mark.parametrize('cls', [models.MidiAutoencoder, models.ZMidiAutoencoder])
def test_loss_keys_without_midi_encoder_and_in_evaluation(cls):
  torch.manual_seed(6)
  z_kw = {}
  if cls is models.ZMidiAutoencoder:
    z_kw = dict(z_global_encoders=[_ZEncoder()], z_note_encoder=_ZEncoder())
  model, hooks = _encoder_branch(cls, None, **z_kw)
  feats = _notes_features()
  roll = torch.zeros(3, 1000, 128, device='cuda')
  roll[..., 60] = 1.0
  feats['note_active_velocities'] = roll
  outputs, loss = model(dict(feats), training=True, return_losses=True)
  assert set(loss) == {'qpitch_f0rec', 'recon', 'total_loss'}
  assert 'z_pitch' not in outputs and hooks['midi_slowness_loss'].mask is None
  _, loss = model(dict(feats), training=False, return_losses=True)
  assert set(loss) == {'total_loss'}
