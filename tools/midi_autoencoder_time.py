"""Times of models.MidiAutoencoder and ZMidiAutoencoder and of their residual site:
  * nn.norm_residual forward + backward ('layer', B = 32, T = 1000, C = 128) against the
    torch composition x + normalize_op(y) s + h (and its ReLU) with autograd, in every
    variant the configs run: per-channel scale and shift with the ReLU output, the
    stack's last layer (no ReLU output), and FiLM (scale and shift read per row from
    the Dense output).  Beside the autograd call, the two entry points alone (launched
    directly on preallocated buffers), with their nominal traffic in GB/s and as a share
    of the data sheet's HBM bandwidth;
  * one midiae.gin and one z_midiae.gin training step (B = 32, 64000 samples, 1000
    frames): forward, losses and backward, no optimizer step.  CUDA events around the
    step, its forward and its backward give the step time; in further steps, events
    around every convolution and residual site split the forward (the rest: encoders'
    Dense and GRU layers, synthesis and losses), with the step timed again in the same
    steps.

  python tools/midi_autoencoder_time.py [--rounds 3] [--out FILE]

Times are CUDA events after warm-up: the site rows are the median of `rounds` alternated
rounds, the step rows means over `rounds` x 2 steps.  Prints the card name and power limit
read in the same run."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import _lib, core, nn  # noqa: E402
from tests.test_midi_autoencoder import build_midiae, build_z_midiae, features  # noqa: E402
from tools import measure  # noqa: E402

B, T, C = 32, 1000, 128


def _site_rows(rounds):
  rows = []
  for variant in ('channel_relu', 'channel_last', 'film_relu'):
    g = torch.Generator(device='cuda').manual_seed(len(variant))
    y = torch.randn((B, T, C), device='cuda', generator=g).requires_grad_(True)
    x = torch.randn((B, T, C), device='cuda', generator=g).requires_grad_(True)
    relu = variant != 'channel_last'
    if variant == 'film_relu':
      params = [torch.randn((B, T, 2 * C), device='cuda', generator=g).requires_grad_(True)]
    else:
      params = [(1.0 + 0.1 * torch.randn(C, device='cuda', generator=g)).requires_grad_(True),
                (0.1 * torch.randn(C, device='cuda', generator=g)).requires_grad_(True)]
    ups = [torch.randn((B, T, C), device='cuda', generator=g) for _ in range(2)]
    leaves = [y, x] + params

    def fused():
      if variant == 'film_relu':
        out = nn.norm_residual(y, x, 'layer', film=params[0], relu=relu)
      else:
        out = nn.norm_residual(y, x, 'layer', *params, relu=relu)
      outs = out if relu else (out,)
      torch.autograd.grad(outs, leaves, ups[:len(outs)])

    def composition():
      yh = nn.normalize_op(y[:, :, None, :], 'layer')[:, :, 0, :]
      if variant == 'film_relu':
        s, h = params[0][..., :C], params[0][..., C:]
      else:
        s, h = params
      x_next = x + yh * s + h
      outs = (x_next, torch.relu(x_next)) if relu else (x_next,)
      torch.autograd.grad(outs, leaves, ups[:len(outs)])

    kernels, nbytes = _kernels(variant, y.detach(), x.detach(), [p.detach() for p in params],
                               [u for u in ups])
    t = measure.alternate({'fused': fused, 'composition': composition, 'kernels': kernels},
                          rounds, 20, 5)
    rows.append({'site': variant, 'shape': [B, T, C], 'fused_ms': t['fused'],
                 'composition_ms': t['composition'],
                 'speedup': t['composition'] / t['fused'], 'kernels_ms': t['kernels'],
                 'nominal_bytes': nbytes,
                 'kernels_nominal_GBps': nbytes / t['kernels'] / 1e6,
                 'kernels_of_hbm_peak': nbytes / t['kernels'] / 1e-3 / measure.HBM_BYTES_PER_S})
  return rows


def _kernels(variant, y, x, params, ups):
  """The site's forward and backward entry points on preallocated buffers, and their
  nominal traffic in bytes: forward, y twice (statistics, then the epilogue), x, x_next
  and r; backward, y, gx, gr, x_next and dx (first pass) and y, dx and dy (second); per
  row also the Dense output's scale and shift columns forward, its scale columns twice and
  both gradient columns backward."""
  relu = variant != 'channel_last'
  per_row = variant == 'film_relu'
  x_next, r = torch.empty_like(y), torch.empty_like(y) if relu else None
  mean, rstd = torch.empty(B, 1, device='cuda'), torch.empty(B, 1, device='cuda')
  dy, dx = torch.empty_like(y), torch.empty_like(y)
  gx, gr = ups[0], ups[1] if relu else None
  if per_row:
    film = params[0]
    dfilm = torch.empty_like(film)
    s, h, ds, dh, ld = (film.data_ptr(), film.data_ptr() + 4 * C, dfilm.data_ptr(),
                        dfilm.data_ptr() + 4 * C, 2 * C)
    ws = (None, 0)
  else:
    (s, h), ld = params, 0
    ds, dh = torch.empty_like(s), torch.empty_like(h)
    ws = core._workspace(4 * 2 * _lib.NORM_CLUSTER * B * C, y.device)

  def run():
    core._launch('ddsp_b200_norm_residual_forward', y, x, s, h, ld, x_next, r, mean, rstd,
                 B, T, C, 1, 1e-5)
    core._launch('ddsp_b200_norm_residual_backward', y, s if per_row else params[0], ld,
                 x_next, mean, rstd, gx, gr, dy, dx, ds, dh, *ws, B, T, C, 1)

  passes = (3 + 1 + int(relu)) + (3 + 2 * int(relu) + 3)
  if per_row:
    passes += 2 + 2 + 2
  return run, passes * 4 * y.numel()


def _stage_hooks(model, stages):
  for m in model.modules():
    if isinstance(m, nn.Conv2D):
      m.register_forward_pre_hook(lambda *a: stages.begin('convolutions'))
      m.register_forward_hook(lambda *a: stages.end('convolutions'))
  original = nn.norm_residual

  def timed(*args, **kwargs):
    stages.begin('residual_sites')
    out = original(*args, **kwargs)
    stages.end('residual_sites')
    return out

  nn.norm_residual = timed


def _step_rows(rounds):
  rows = []
  for name, build in (('midiae', build_midiae), ('z_midiae', build_z_midiae)):
    torch.manual_seed(0)
    model = build()
    batch = features(b=B)
    stages = measure.StageEvents()

    def step():
      stages.begin('step')
      model.zero_grad(set_to_none=True)
      stages.begin('forward_and_losses')
      _, losses = model(dict(batch), training=True, return_losses=True)
      stages.end('forward_and_losses')
      stages.begin('backward')
      losses['total_loss'].backward()
      stages.end('backward')
      stages.end('step')

    def mean_ms(steps):
      stages.clear()
      for _ in range(steps):
        step()
      return stages.mean_ms(steps)

    for _ in range(2):
      step()
    plain = mean_ms(2 * rounds)
    original = nn.norm_residual
    _stage_hooks(model, stages)
    try:
      split = mean_ms(2 * rounds)
    finally:
      nn.norm_residual = original
    split['synthesis_losses_and_rest'] = split['forward_and_losses'] - split[
        'convolutions'] - split['residual_sites']
    rows.append({'step': name, 'batch': B, 'step_ms': plain['step'],
                 'forward_and_losses_ms': plain['forward_and_losses'],
                 'backward_ms': plain['backward'], 'stages_ms': split,
                 'cudnn_allow_tf32': torch.backends.cudnn.allow_tf32,
                 'matmul_allow_tf32': torch.backends.cuda.matmul.allow_tf32})
  return rows


def main():
  parser = argparse.ArgumentParser()
  parser.add_argument('--rounds', type=int, default=3)
  parser.add_argument('--out', default=None)
  args = parser.parse_args()
  measure.require_cuda('midi_autoencoder_time.py')
  card = measure.card()
  print(json.dumps(card))
  rows = [dict(r, kind='norm_residual', **card) for r in _site_rows(args.rounds)]
  rows += [dict(r, kind='step', **card) for r in _step_rows(args.rounds)]
  for r in rows:
    print(json.dumps(r))
  if args.out:
    measure.append_rows(args.out, rows)


if __name__ == '__main__':
  main()
