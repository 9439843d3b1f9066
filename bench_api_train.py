#!/usr/bin/env python
"""bench_api_train.py - one training step of the `ae.gin` decoder, written two ways.

  python bench_api_train.py [--steps K] [--warmup W] [--rounds R] [--batch B] [--out DIR]

BASELINE.json configs[3] (B = 128, F = 1000, K = 100, 65 noise bands, N = 64000 @16 kHz,
forward + backward through the multi-scale SpectralLoss) through
  (a) `autograd.decoder_train`: one autograd node, controls never leave the chip;
  (b) `group(features, return_outputs_dict=True)`: the Processor API, node by node, as
      the reference's models call it - both control tensors and three [B, N] signals
      are materialised, every node has its own backward.
The two alternate in one process, R rounds of W warm-up and K timed steps each (bench.py
--config c4's counts by default), on a ring of three input sets, eager autograd, timed
with CUDA events.  Both see the same Philox stream (same seed, offset = step), so the
last timed step is compared as well: the audio, and the gradients both decoders return
for ONE upstream gradient, dL/d audio of (a)'s loss.  (Each path's own float32 loss
gradient is not a yardstick for the other: L1 of log magnitudes has gradient sign / |X|
per bin, and the bins where the spectrum nearly cancels turn a 1e-7 difference in the
audio into a different gradient.)

One JSON line on stdout: ms per step and launches per step of each, the differences,
and the card's name and enforced power limit read in the same run.  --out DIR also
writes it to DIR/bench_api_train.json.  There is no CPU path.
"""
import argparse
import itertools
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

N_SAMPLES, N_FRAMES, N_HARM, N_BANDS, SAMPLE_RATE = 64000, 1000, 100, 65, 16000
GRAD_KEYS = ('amps', 'harmonic_distribution', 'noise_magnitudes')


def card(index):
  """Name and enforced power limit (W) of the device: NVML, else nvidia-smi's query."""
  import torch
  name, limit = torch.cuda.get_device_name(index), None
  try:
    import pynvml
    pynvml.nvmlInit()
    try:
      h = pynvml.nvmlDeviceGetHandleByUUID(
          'GPU-' + str(torch.cuda.get_device_properties(index).uuid))
    except Exception:  # pylint: disable=broad-except
      h = pynvml.nvmlDeviceGetHandleByIndex(index)
    limit = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
  except Exception:  # pylint: disable=broad-except
    try:
      out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit',
                            '--format=csv,noheader,nounits', '-i', str(index)],
                           capture_output=True, text=True, timeout=30).stdout
      limit = float(out.strip().splitlines()[0])
    except Exception:  # pylint: disable=broad-except
      limit = None
  return name, limit


def rel_diff(a, b):
  """(max-abs difference / max-abs of b, relative L2 difference)."""
  a, b = a.double(), b.double()
  return (float((a - b).abs().max() / b.abs().max().clamp_min(1e-30)),
          float((a - b).norm() / b.norm().clamp_min(1e-30)))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=10)
  ap.add_argument('--warmup', type=int, default=10)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--batch', type=int, default=128)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  import torch
  if not torch.cuda.is_available():
    raise SystemExit('bench_api_train.py needs a CUDA device; there is no CPU path.')
  import ddsp_b200
  from ddsp_b200 import _lib, autograd as ag, core, losses
  from tests.util import synth_inputs
  torch.cuda.set_device(0)
  dev = torch.device('cuda', 0)
  lib = _lib.load()
  torch.manual_seed(4321)
  B = args.batch
  host = synth_inputs(B, N_FRAMES, N_HARM, N_BANDS, N_SAMPLES, seed=55)
  sets = []
  for s in range(3):                       # inputs + targets of three sets > 2x L2
    d = {k: torch.from_numpy(host[k]).to(dev) for k in GRAD_KEYS + ('f0_hz',)}
    if s:
      d['amps'] = d['amps'] + 0.01 * s
    for k in GRAD_KEYS:
      d[k].requires_grad_(True)
    d['target'] = 0.1 * torch.randn(B, N_SAMPLES, device=dev)
    sets.append(d)
  loss_obj = losses.SpectralLoss(mag_weight=1.0, logmag_weight=1.0)
  harm = ddsp_b200.Harmonic(n_samples=N_SAMPLES, sample_rate=SAMPLE_RATE)
  noise = ddsp_b200.FilteredNoise(n_samples=N_SAMPLES, window_size=0, seed=1)
  group = ddsp_b200.ProcessorGroup(dag=[
      (harm, ['amps', 'harmonic_distribution', 'f0_hz']),
      (noise, ['noise_magnitudes']),
      (ddsp_b200.Add(), ['filtered_noise/signal', 'harmonic/signal'])])

  def step_fused(i):
    d = sets[i % 3]
    for k in GRAD_KEYS:
      d[k].grad = None
    audio = ag.decoder_train(d['amps'], d['harmonic_distribution'], d['f0_hz'],
                             d['noise_magnitudes'], n_samples=N_SAMPLES, window_size=0,
                             seed=1, offset=i)
    loss_obj(d['target'], audio).backward()

  def step_api(i):
    d = sets[i % 3]
    for k in GRAD_KEYS:
      d[k].grad = None
    noise._calls = itertools.count(i)      # this step's Philox offset, as (a)'s
    out = group({k: d[k] for k in GRAD_KEYS + ('f0_hz',)}, return_outputs_dict=True)
    loss_obj(d['target'], out['signal']).backward()

  def timed(fn):
    for i in range(args.warmup):
      fn(i)
    torch.cuda.synchronize()
    c0 = lib.ddsp_b200_launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
      fn(args.warmup + i)
    e1.record()
    torch.cuda.synchronize()
    return (e0.elapsed_time(e1) / args.steps,
            (lib.ddsp_b200_launch_count() - c0) / args.steps)

  name, limit = card(0)
  ms = {'fused': [], 'api': []}
  launches = {}
  for _ in range(args.rounds):
    for key, fn in (('fused', step_fused), ('api', step_api)):
      t, n = timed(fn)
      ms[key].append(t)
      launches[key] = n

  # the last timed step of each, on the same inputs and the same noise, driven by the
  # same upstream gradient
  i = args.warmup + args.steps - 1
  d = sets[i % 3]
  feats = {k: d[k] for k in GRAD_KEYS + ('f0_hz',)}
  audio_a = ag.decoder_train(d['amps'], d['harmonic_distribution'], d['f0_hz'],
                             d['noise_magnitudes'], n_samples=N_SAMPLES, window_size=0,
                             seed=1, offset=i)
  g_audio, = torch.autograd.grad(loss_obj(d['target'], audio_a), audio_a, retain_graph=True)
  want = dict(zip(GRAD_KEYS, torch.autograd.grad(audio_a, [d[k] for k in GRAD_KEYS], g_audio)))
  want['audio'] = audio_a.detach()
  noise._calls = itertools.count(i)
  audio_b = group(feats, return_outputs_dict=True)['signal']
  got = dict(zip(GRAD_KEYS, torch.autograd.grad(audio_b, [d[k] for k in GRAD_KEYS], g_audio)))
  got['audio'] = audio_b.detach()
  torch.cuda.synchronize()
  diffs = {k: dict(zip(('max_rel', 'l2_rel'), rel_diff(got[k], want[k]))) for k in want}

  # the get_controls vector-Jacobian product alone: three reads and one write of
  # [B, F, K] against the time HBM needs for them at the data-sheet rate
  d = sets[0]
  up_a, up_h = torch.randn_like(d['amps']), torch.randn_like(d['harmonic_distribution'])
  o_a, o_h = torch.empty_like(up_a), torch.empty_like(up_h)

  def vjp():
    core._launch('ddsp_b200_harmonic_controls_vjp', d['amps'].detach(),
                 d['harmonic_distribution'].detach(), d['f0_hz'], up_a, up_h, o_a, o_h, B,
                 N_FRAMES, N_HARM, float(SAMPLE_RATE), _lib.CTL_SCALE | _lib.CTL_NYQUIST)
  for _ in range(5):
    vjp()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(50):
    vjp()
  e1.record()
  torch.cuda.synchronize()
  vjp_bytes = 4 * 4 * B * N_FRAMES * N_HARM
  vjp_ms = e0.elapsed_time(e1) / 50

  line = {
      'metric': 'ms per training step (decoder forward + backward through SpectralLoss)',
      'gpu': name, 'power_limit_w': limit,
      'config': {'batch': B, 'n_frames': N_FRAMES, 'n_harmonics': N_HARM,
                 'n_bands': N_BANDS, 'n_samples': N_SAMPLES, 'steps': args.steps,
                 'warmup': args.warmup, 'rounds': args.rounds,
                 'timing': 'CUDA events around the timed steps of each round, eager '
                           'autograd, the two paths alternating'},
      'decoder_train': {'ms_per_step': min(ms['fused']), 'ms_per_step_rounds': ms['fused'],
                        'library_launches_per_step': launches['fused']},
      'processor_api': {'ms_per_step': min(ms['api']), 'ms_per_step_rounds': ms['api'],
                        'library_launches_per_step': launches['api']},
      'processor_api_vs_decoder_train': diffs,
      'harmonic_controls_vjp': {
          'ms': vjp_ms, 'bytes_four_passes': vjp_bytes,
          'GBps_four_passes': vjp_bytes / (vjp_ms * 1e-3) / 1e9,
          'ms_at_3350_GBps_datasheet': vjp_bytes / 3350e9 * 1e3,
          'note': 'operands of 51 MB each stay partly in the 50 MB L2 between launches'},
  }
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'bench_api_train.json'), 'w') as f:
      json.dump(line, f, indent=1)
  print(json.dumps(line), flush=True)


if __name__ == '__main__':
  main()
