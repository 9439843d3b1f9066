"""The training preprocessors of training/preprocessing.py (preprocessing.py:28-244):
torch compositions of compute_loudness, compute_power, core.resample and
PretrainedCREPE, which run on CUDA kernels.  Each preprocessor's __call__(features)
reads its call()'s arguments from the features dict by name, as nn.DictLayer does, and
returns a dict of its output keys."""
import inspect

from ddsp_b200 import core
from ddsp_b200 import spectral_ops

F0_RANGE = spectral_ops.F0_RANGE
DB_RANGE = spectral_ops.DB_RANGE


# ---- helpers (preprocessing.py:28-54) -------------------------------------------------
def at_least_3d(x):
  """Adds time, batch, then channel dimensions: [] -> [1, 1, 1], [T] -> [1, T, 1],
  [B, T] -> [B, T, 1]."""
  x = core._as_f32(x) if not hasattr(x, 'dim') else x
  x = x[None] if x.dim() == 0 else x
  x = x[None, :] if x.dim() == 1 else x
  x = x[:, :, None] if x.dim() == 2 else x
  return x


def scale_db(db):
  """Scales [-DB_RANGE, 0] to [0, 1]."""
  return (db / DB_RANGE) + 1.0


def inv_scale_db(db_scaled):
  """Scales [0, 1] to [-DB_RANGE, 0]."""
  return (db_scaled - 1.0) * DB_RANGE


def scale_f0_hz(f0_hz):
  """Scales [0, Nyquist] Hz to [0, 1.0] MIDI-scaled."""
  return core.hz_to_midi(f0_hz) / F0_RANGE


def inv_scale_f0_hz(f0_scaled):
  """Scales [0, 1.0] MIDI-scaled to [0, Nyquist] Hz."""
  return core.midi_to_hz(f0_scaled * F0_RANGE)


def _call_on_dict(call, features, output_keys):
  """nn.DictLayer.__call__ on one features dict: call()'s arguments looked up by name
  (a missing one without a default raises KeyError), its outputs named by output_keys."""
  kwargs = {}
  for name, p in inspect.signature(call).parameters.items():
    if name in features:
      kwargs[name] = features[name]
    elif p.default is inspect.Parameter.empty:
      raise KeyError(f'{type(call.__self__).__name__} needs the input {name!r}; the '
                     f'features have {sorted(features)}')
  return dict(zip(output_keys, call(**kwargs)))


# ---- preprocessors (preprocessing.py:57-244) ------------------------------------------
class F0LoudnessPreprocessor:
  """Resamples and scales 'f0_hz' and 'loudness_db' features."""

  output_keys = ('f0_hz', 'loudness_db', 'f0_scaled', 'ld_scaled')

  def __init__(self, time_steps=1000, frame_rate=250, sample_rate=16000,
               compute_loudness=True):
    self.time_steps = time_steps
    self.frame_rate = frame_rate
    self.sample_rate = sample_rate
    self.compute_loudness = compute_loudness

  def __call__(self, features):
    return _call_on_dict(self.call, features, self.output_keys)

  def call(self, loudness_db, f0_hz, audio=None):
    if self.compute_loudness:
      loudness_db = spectral_ops.compute_loudness(
          audio, sample_rate=self.sample_rate, frame_rate=self.frame_rate)
    f0_hz = self.resample(f0_hz)
    loudness_db = self.resample(loudness_db)
    f0_scaled = scale_f0_hz(f0_hz)
    ld_scaled = scale_db(loudness_db)
    return f0_hz, loudness_db, f0_scaled, ld_scaled

  @staticmethod
  def invert_scaling(f0_scaled, ld_scaled):
    """Puts scaled f0 and loudness back to Hz and dB."""
    return inv_scale_f0_hz(f0_scaled), inv_scale_db(ld_scaled)

  def resample(self, x):
    return core.resample(at_least_3d(x), self.time_steps)


class F0PowerPreprocessor(F0LoudnessPreprocessor):
  """Resamples and scales 'f0_hz', and 'power_db' taken from the features or computed
  from 'audio'."""

  output_keys = ('f0_hz', 'pw_db', 'f0_scaled', 'pw_scaled')

  def __init__(self, time_steps=1000, frame_rate=250, sample_rate=16000, frame_size=64):
    super().__init__(time_steps)
    self.frame_rate = frame_rate
    self.sample_rate = sample_rate
    self.frame_size = frame_size

  def call(self, f0_hz, power_db=None, audio=None):
    f0_hz = self.resample(f0_hz)
    f0_scaled = scale_f0_hz(f0_hz)
    if power_db is not None:
      pw_db = power_db
    elif audio is not None:
      pw_db = spectral_ops.compute_power(audio, sample_rate=self.sample_rate,
                                         frame_rate=self.frame_rate,
                                         frame_size=self.frame_size)
    else:
      raise ValueError('Power preprocessing requires either '
                       '"power_db" or "audio" keys to be provided '
                       'in the dataset.')
    pw_db = self.resample(pw_db)
    pw_scaled = scale_db(pw_db)
    return f0_hz, pw_db, f0_scaled, pw_scaled

  @staticmethod
  def invert_scaling(f0_scaled, pw_scaled):
    """Puts scaled f0 and power back to Hz and dB."""
    return inv_scale_f0_hz(f0_scaled), inv_scale_db(pw_scaled)


class OnlineF0PowerPreprocessor:
  """Computes 'pw_db' and 'f0_hz' (with 'f0_confidence') from 16 kHz audio, framed with
  `padding`.  crepe_saved_model_path is PretrainedCREPE's model_size_or_path (a network
  or a TorchScript path; the default 'full' names weights that are not shipped and
  raises NotImplementedError) or None for no network.  f0 and its confidence carry no
  gradient, as in the reference."""

  output_keys = ('f0_hz', 'pw_db', 'f0_scaled', 'pw_scaled', 'f0_confidence')

  def __init__(self, frame_rate=250, frame_size=1024, padding='center', compute_power=True,
               compute_f0=True, crepe_saved_model_path='full', viterbi=False):
    self.sample_rate = spectral_ops.CREPE_SAMPLE_RATE
    self.frame_rate = frame_rate
    self.frame_size = frame_size
    self.hop_size = self.sample_rate // frame_rate
    self.compute_f0 = compute_f0
    self.compute_power = compute_power
    self.padding = padding
    if crepe_saved_model_path:
      self.crepe_model = spectral_ops.PretrainedCREPE(
          model_size_or_path=crepe_saved_model_path, hop_size=self.hop_size)
    self.viterbi = viterbi

  def __call__(self, features):
    return _call_on_dict(self.call, features, self.output_keys)

  def call(self, audio, f0_hz=None, f0_confidence=None, audio_16k=None, pw_db=None):
    if audio_16k is not None:
      audio = audio_16k
    if self.compute_power:
      pw_db = spectral_ops.compute_power(audio, sample_rate=self.sample_rate,
                                         frame_rate=self.frame_rate,
                                         frame_size=self.frame_size, padding=self.padding)
    if self.compute_f0:
      f0_hz, f0_confidence = self.crepe_model.predict_f0_and_confidence(
          audio, viterbi=self.viterbi, padding=self.padding)
    elif f0_hz is None or f0_confidence is None:
      raise ValueError('Preprocessor must either have `compute_f0=True`, or'
                       '__call__ must be supplied 3 arguments, '
                       '[audio, f0_hz, and f0_confidence].')

    pw_db = at_least_3d(pw_db)
    f0_hz = at_least_3d(f0_hz)
    pw_scaled = scale_db(pw_db)
    f0_scaled = scale_f0_hz(f0_hz)

    # the frame count the configuration gives, so that a wrong frame_rate or padding
    # shows here and not as a shape error in the model
    n_t = audio.shape[1]
    time_steps, _ = spectral_ops.get_framed_lengths(n_t, self.frame_size, self.hop_size,
                                                    self.padding)
    for k, output in {'f0_hz': f0_hz, 'pw_db': pw_db, 'f0_scaled': f0_scaled,
                      'pw_scaled': pw_scaled, 'f0_confidence': f0_confidence}.items():
      if output.shape[1] != time_steps:
        raise ValueError(
            f'OnlineF0PowerPreprocessor output: ({k}) does not have '
            f'{time_steps} timesteps. Output shape: {tuple(output.shape)}. '
            f'\nInputs: seconds ({n_t / self.sample_rate}), '
            f'frame_rate ({self.frame_rate}), '
            f'padding ("{self.padding}").')
    return f0_hz, pw_db, f0_scaled, pw_scaled, f0_confidence
