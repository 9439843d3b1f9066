"""Times of models.InverseSynthesis and of its fused normalize-ReLU:
  * nn.normalize_relu forward + backward ('layer', as the model runs it) at every site
    shape of the 'small' ResNet at B = 32 and T = 125, against the torch composition
    relu(normalize_op(x) * scale + shift) with autograd, with the fused kernel's
    nominal traffic (3 passes over x forward, 5 backward) in GB/s;
  * one pretrain_model.gin training step (B = 32, 64000 samples, self-supervised
    synthetic notes) and one finetune_model.gin step (zipped, 32 + 32): forward, losses
    and backward, no optimizer step, with the forward split into stages (log-mel, ResNet
    convolutions and pooling, ResNet norms, frequency head, RnnSandwich, synthesis,
    losses) by CUDA events around each stage, and the backward as one stage.

  python tools/inverse_synthesis_time.py [--rounds 3] [--out FILE]

Times are CUDA events after warm-up, the median of `rounds` alternated rounds.  Prints
the card name and power limit read in the same run."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import nn, synthetic_data  # noqa: E402
from tests.test_inverse_synthesis import _audio, _pretrain  # noqa: E402
from tests.test_norm_relu import SITES  # noqa: E402
from tools import measure  # noqa: E402

B = 32


def _site_rows(rounds):
  rows = []
  for h, w, c in SITES:
    g = torch.Generator(device='cuda').manual_seed(c)
    x = torch.randn((B, h, w, c), device='cuda', generator=g).requires_grad_(True)
    scale = (1.0 + 0.1 * torch.randn(c, device='cuda', generator=g)).requires_grad_(True)
    shift = (0.1 * torch.randn(c, device='cuda', generator=g)).requires_grad_(True)
    up = torch.randn((B, h, w, c), device='cuda', generator=g)

    def fused():
      torch.autograd.grad(nn.normalize_relu(x, scale, shift, 'layer'), (x, scale, shift), up)

    def composition():
      y = torch.relu(nn.normalize_op(x, 'layer') * scale + shift)
      torch.autograd.grad(y, (x, scale, shift), up)

    t = measure.alternate({'fused': fused, 'composition': composition}, rounds, 20, 5)
    nbytes = 8 * 4 * x.numel()
    rows.append({'site': [B, h, w, c], 'fused_ms': t['fused'],
                 'composition_ms': t['composition'],
                 'speedup': t['composition'] / t['fused'],
                 'fused_nominal_GBps': nbytes / t['fused'] / 1e6,
                 'of_hbm_peak': nbytes / t['fused'] / 1e-3 / measure.HBM_BYTES_PER_S})
  return rows


def _stage_hooks(model, stages):
  """CUDA events around each forward stage of the model."""
  def around(module, name):
    module.register_forward_pre_hook(lambda *a: stages.begin(name))
    module.register_forward_hook(lambda *a: stages.end(name))

  enc = model.sinusoidal_encoder
  fn = enc.spectral_fn

  def spectral(audio):
    stages.begin('logmel')
    out = fn(audio)
    stages.end('logmel')
    return out

  enc.spectral_fn = spectral
  for m in enc.resnet.modules():
    if isinstance(m, (nn.Conv2D, nn.MaxPool2D)):
      around(m, 'resnet_convs')
    elif isinstance(m, nn.NormRelu):
      around(m, 'resnet_norms')
  around(enc.dense_outs[0], 'frequency_head')
  around(model.harmonic_encoder.net, 'rnn_sandwich')


def _step_rows(rounds):
  rows = []
  for name, finetune in (('pretrain', False), ('finetune', True)):
    torch.manual_seed(0)
    model = _pretrain(finetune)
    notes = synthetic_data.generate_notes_v2(seeds=list(range(B)))
    batch = ({'audio': _audio(B, 1)}, notes) if finetune else notes
    stages = measure.StageEvents()

    def step():
      model.zero_grad(set_to_none=True)
      feats = (dict(batch[0]), dict(batch[1])) if finetune else dict(batch)
      stages.begin('forward_and_losses')
      _, losses = model(feats, return_losses=True)
      stages.end('forward_and_losses')
      stages.begin('backward')
      losses['total_loss'].backward()
      stages.end('backward')

    step()
    t = measure.alternate({name: step}, rounds, 5, 2)[name]
    _stage_hooks(model, stages)
    stages.clear()
    for _ in range(3):
      step()
    split = stages.mean_ms(3)
    split['synthesis_and_losses_and_rest'] = split['forward_and_losses'] - sum(
        split[k] for k in ('logmel', 'resnet_convs', 'resnet_norms', 'frequency_head',
                           'rnn_sandwich'))
    rows.append({'step': name, 'batch': B * (2 if finetune else 1), 'step_ms': t,
                 'stages_ms': split,
                 'cudnn_allow_tf32': torch.backends.cudnn.allow_tf32,
                 'matmul_allow_tf32': torch.backends.cuda.matmul.allow_tf32})
  return rows


def main():
  parser = argparse.ArgumentParser()
  parser.add_argument('--rounds', type=int, default=3)
  parser.add_argument('--out', default=None)
  args = parser.parse_args()
  measure.require_cuda('inverse_synthesis_time.py')
  card = measure.card()
  print(json.dumps(card))
  rows = [dict(r, kind='norm_relu', **card) for r in _site_rows(args.rounds)]
  rows += [dict(r, kind='step', **card) for r in _step_rows(args.rounds)]
  for r in rows:
    print(json.dumps(r))
  if args.out:
    measure.append_rows(args.out, rows)


if __name__ == '__main__':
  main()
