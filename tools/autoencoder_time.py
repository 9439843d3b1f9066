"""Time of one models.Autoencoder training step (forward, losses and backward, no optimizer
step) at the reference's default batch, B = 32 items of 4 s at 16 kHz (N = 64000) with
1000 frames:
  * ae.gin (nsynth_ae): F0LoudnessPreprocessor, MfccTimeDistributedRnnEncoder,
    RnnFcDecoder, Harmonic + FilteredNoise + Add and SpectralLoss;
  * solo_instrument.gin: no encoder, and a trainable 48000-tap Reverb after the Add.
Each model is timed against itself with torch.nn.GRU (cuDNN, the same weights) in place
of every GRU, in alternated rounds; torch.backends.cudnn.allow_tf32 is recorded in each
row.  Each row also gives the time of each stage (preprocessor, encoder, decoder,
processor group, loss, backward) from CUDA events recorded around it, the peak device
memory of a step, and the largest |difference| of the decoder's harmonic distribution
between the two GRUs relative to its largest value.

  python tools/autoencoder_time.py [--rounds 3] [--out FILE]

Times are CUDA events after warm-up, the median of `rounds` alternated rounds.  Prints
the card name and power limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import gru_ref  # noqa: E402
from tests.test_autoencoder import nsynth_ae, solo_instrument  # noqa: E402
from tools import measure  # noqa: E402

DEV = 'cuda'
B, N, FRAMES = 32, 64000, 1000
STAGES = ('preprocessor', 'encoder', 'decoder', 'processor_group', 'loss', 'backward')


def _features(seed=0):
  """Harmonic tones of gliding pitch over quiet noise, with their f0."""
  rng = np.random.default_rng(seed)
  f0 = 110.0 * 2.0**(2.0 * rng.uniform(size=(B, 1)) * np.linspace(0, 1, FRAMES))
  f0_audio = np.repeat(f0, N // FRAMES, axis=1)
  phase = 2 * np.pi * np.cumsum(f0_audio, axis=1) / 16000.0
  audio = sum(np.sin(k * phase) / k for k in range(1, 8)) * 0.2
  audio = audio + 0.01 * rng.standard_normal((B, N))
  return {k: torch.tensor(v, dtype=torch.float32, device=DEV) for k, v in
          {'audio': audio, 'f0_hz': f0, 'loudness_db': np.zeros((B, FRAMES))}.items()}


def _step(model, features):
  model.zero_grad(set_to_none=True)
  outputs, loss = model(dict(features), return_losses=True)
  loss['total_loss'].backward()
  return outputs


def _cudnn_for(rnn):
  """torch.nn.GRU with the weights of an nn.Rnn that has been built."""
  g = rnn.rnn
  cudnn = torch.nn.GRU(g.input_width, g.units, batch_first=True).to(DEV)
  cudnn.load_state_dict({k: v.float() for k, v in gru_ref.torch_gru_weights(
      g.kernel.detach(), g.recurrent_kernel.detach(), g.bias.detach()).items()})
  return cudnn


class _Rnns:
  """Switches every GRU of a model between the library's and cuDNN's."""

  def __init__(self, model):
    self.rnns = [m.rnn for m in (model.encoder, model.decoder) if m is not None]
    self.cudnn = [_cudnn_for(r) for r in self.rnns]

  def use_cudnn(self, on):
    for rnn, cudnn in zip(self.rnns, self.cudnn):
      if on:
        rnn.forward = lambda x, c=cudnn: c(x)[0]
      else:
        rnn.__dict__.pop('forward', None)


class _Timed:
  """A stand-in for a plain-object stage of the model that records its calls as a stage
  of `events`."""

  def __init__(self, inner, name, events):
    self.inner, self.name, self.events = inner, name, events

  def _run(self, fn, args, kwargs):
    self.events.begin(self.name)
    out = fn(*args, **kwargs)
    self.events.end(self.name)
    return out

  def __call__(self, *args, **kwargs):
    return self._run(self.inner, args, kwargs)

  def get_losses_dict(self, *args, **kwargs):
    return self._run(self.inner.get_losses_dict, args, kwargs)

  def __getattr__(self, name):
    return getattr(self.inner, name)


def stage_ms(model, features, iters, warmup):
  """{stage: mean ms per step} from CUDA events around each stage of a training step."""
  events = measure.StageEvents()
  saved = (model.preprocessor, model.processor_group, model.loss_objs)
  model.preprocessor = _Timed(model.preprocessor, 'preprocessor', events)
  model.processor_group = _Timed(model.processor_group, 'processor_group', events)
  model.loss_objs = [_Timed(l, 'loss', events) for l in model.loss_objs]
  hooks = []
  for name in ('encoder', 'decoder'):
    module = getattr(model, name)
    if module is not None:
      hooks += [module.register_forward_pre_hook(lambda *_, n=name: events.begin(n)),
                module.register_forward_hook(lambda *_, n=name: events.end(n))]
  try:
    for i in range(warmup + iters):
      if i == warmup:
        events.clear()
      model.zero_grad(set_to_none=True)
      _, loss = model(dict(features), return_losses=True)
      events.begin('backward')
      loss['total_loss'].backward()
      events.end('backward')
    ms = events.mean_ms(iters)
  finally:
    for h in hooks:
      h.remove()
    model.preprocessor, model.processor_group, model.loss_objs = saved
  return {s: ms[s] for s in STAGES if s in ms}


def row(name, build, rounds):
  torch.manual_seed(0)
  model = build()
  features = _features()
  _step(model, features)                 # builds every lazy layer
  rnns = _Rnns(model)

  def run(on):
    def fn():
      rnns.use_cudnn(on)
      try:
        return _step(model, features)
      finally:
        rnns.use_cudnn(False)
    return fn

  ms = measure.alternate({'ours': run(False), 'cudnn': run(True)}, rounds, 5, 2)
  stages = {}
  for label, on in (('ours', False), ('cudnn', True)):
    rnns.use_cudnn(on)
    try:
      stages[label] = stage_ms(model, features, 5, 2)
    finally:
      rnns.use_cudnn(False)
  # the decoder's output, which both GRUs reach and the noise does not
  a, c = run(False)()['harmonic_distribution'], run(True)()['harmonic_distribution']
  out = {'workload': name, 'B': B, 'N': N, 'frames': FRAMES, 'ms': ms,
         'speedup_vs_cudnn': ms['cudnn'] / ms['ours'], 'stages_ms': stages,
         'peak_mb': measure.peak_bytes(run(False)) / 2**20,
         'cudnn_peak_mb': measure.peak_bytes(run(True)) / 2**20,
         'cudnn_allow_tf32': torch.backends.cudnn.allow_tf32,
         'max_rel_diff_vs_cudnn': ((a - c).abs().max() / c.abs().max()).item()}
  print(json.dumps(out), flush=True)
  return out


def main():
  ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('autoencoder_time.py')
  card = measure.card()
  print(json.dumps({'card': card}), flush=True)
  rows = [row('ae_train_step', nsynth_ae, args.rounds),
          row('solo_instrument_train_step', solo_instrument, args.rounds)]
  if args.out:
    measure.append_rows(args.out, [dict(r, card=card) for r in rows])


if __name__ == '__main__':
  main()
