"""Time of the GRU recurrence (csrc/gru.cuh through autograd.GruFn) against
torch.nn.GRU (cuDNN) with the same weights, on the same GPU:
  * B = 32, T = 1000, H = 512, input widths 1536 (ae.gin) and 1024
    (solo_instrument.gin), forward and forward + backward;
  * B = 32, T = 201, width 512 (the VST configs), forward and forward + backward;
  * B = 1, T = 45000 (3 minutes at 250 frames/s), forward (inference);
  * decoders.RnnFcDecoder at ae.gin's shape (B = 32, T = 1000), forward + backward, with
    its GRU or with cuDNN's in its place.
cuDNN runs twice: as torch runs it by default (torch.backends.cudnn.allow_tf32, recorded
in each row, is True unless changed, so its GEMMs may use TF32) and with TF32 off
(`cudnn_fp32_*`).  Each row gives the times, the per-step time of ours, the largest
|difference| of our output from each cuDNN output relative to the largest output, and the
active-cluster count the library queried for the launch.

  python tools/gru_time.py [--rounds 3] [--out FILE]

Times are CUDA events after warm-up, the median of `rounds` alternated rounds.  Prints
the card name and power limit read in the same run."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import _lib, autograd, decoders  # noqa: E402
from tests import gru_ref  # noqa: E402
from tools import measure  # noqa: E402

DEV = 'cuda'
H = 512


def _cudnn(n_in, kernel, rk, bias):
  g = torch.nn.GRU(n_in, H, batch_first=True).to(DEV)
  g.load_state_dict({k: v.float().to(DEV) for k, v in
                     gru_ref.torch_gru_weights(kernel, rk, bias).items()})
  return g


def _rel(a, b):
  return ((a - b).abs().max() / b.abs().max()).item()


def gru_rows(rounds):
  rows = []
  for name, b, t, n_in, train in [('ae', 32, 1000, 1536, True), ('solo', 32, 1000, 1024, True),
                                  ('vst', 32, 201, 512, True), ('inference_3min', 1, 45000, 1536, False)]:
    kernel, rk, bias = gru_ref.random_weights(n_in, H, seed=0)
    params = [v.float().to(DEV).requires_grad_(train) for v in (kernel, rk, bias)]
    x = torch.randn((b, t, n_in), device=DEV).requires_grad_(train)
    up = torch.randn((b, t, H), device=DEV)
    handle = autograd.GruHandle(H, DEV)
    cudnn = _cudnn(n_in, kernel, rk, bias)
    cudnn.requires_grad_(train)

    def ours_fwd():
      with torch.no_grad():
        return autograd.GruFn.apply(x, *params, handle, False)

    def theirs_fwd():
      with torch.no_grad():
        return cudnn(x)[0]

    def fp32(fn):
      def run():
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
          return fn()
      return run

    fns = {'ours_forward': ours_fwd, 'cudnn_forward': theirs_fwd,
           'cudnn_fp32_forward': fp32(theirs_fwd)}
    if train:
      fns['ours_train'] = lambda: autograd.GruFn.apply(x, *params, handle, True).backward(up)
      fns['cudnn_train'] = lambda: cudnn(x)[0].backward(up)
      fns['cudnn_fp32_train'] = fp32(lambda: cudnn(x)[0].backward(up))
    iters = 2 if t > 10000 else 5
    ms = measure.alternate(fns, rounds, iters, 2)
    lib = _lib.load()
    row = {'workload': name, 'B': b, 'T': t, 'H': H, 'input_width': n_in,
           'ms': ms, 'us_per_step_forward': 1e3 * ms['ours_forward'] / t,
           'speedup_forward': ms['cudnn_forward'] / ms['ours_forward'],
           'clusters_forward': lib.ddsp_b200_gru_clusters(handle.ptr, b, 0),
           'clusters_backward': lib.ddsp_b200_gru_clusters(handle.ptr, b, 1),
           'cudnn_allow_tf32': torch.backends.cudnn.allow_tf32,
           'max_rel_diff_vs_cudnn': _rel(ours_fwd(), theirs_fwd()),
           'max_rel_diff_vs_cudnn_fp32': _rel(ours_fwd(), fp32(theirs_fwd)())}
    if train:
      row['us_per_step_train'] = 1e3 * ms['ours_train'] / t
      row['speedup_train'] = ms['cudnn_train'] / ms['ours_train']
    rows.append(row)
    print(json.dumps(row), flush=True)
  return rows


def decoder_row(rounds):
  b, t = 32, 1000
  torch.manual_seed(0)
  dec = decoders.RnnFcDecoder()
  feats = {'ld_scaled': torch.rand(b, t, 1, device=DEV), 'f0_scaled': torch.rand(b, t, 1, device=DEV),
           'z': torch.randn(b, t, 16, device=DEV)}
  dec(feats)   # builds
  g = dec.rnn.rnn
  cudnn = _cudnn(g.input_width, g.kernel.detach().double().cpu(),
                 g.recurrent_kernel.detach().double().cpu(), g.bias.detach().double().cpu())

  def step(use_cudnn):
    orig = dec.rnn.forward
    if use_cudnn:
      dec.rnn.forward = lambda x: cudnn(x)[0]
    try:
      out = dec(feats)
      (out['amps'].sum() + out['harmonic_distribution'].sum()).backward()
      return out
    finally:
      dec.rnn.forward = orig

  ms = measure.alternate({'ours_train': lambda: step(False),
                          'cudnn_train': lambda: step(True)}, rounds, 5, 2)
  with torch.no_grad():
    a = dec(feats)['harmonic_distribution']
    orig = dec.rnn.forward
    dec.rnn.forward = lambda x: cudnn(x)[0]
    c = dec(feats)['harmonic_distribution']
    dec.rnn.forward = orig
  row = {'workload': 'decoder_ae', 'B': b, 'T': t, 'ms': ms,
         'cudnn_allow_tf32': torch.backends.cudnn.allow_tf32,
         'speedup_train': ms['cudnn_train'] / ms['ours_train'],
         'max_rel_diff_vs_cudnn': _rel(a, c)}
  print(json.dumps(row), flush=True)
  return [row]


def main():
  ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  measure.require_cuda('gru_time.py')
  card = measure.card()
  print(json.dumps({'card': card}), flush=True)
  rows = gru_rows(args.rounds) + decoder_row(args.rounds)
  if args.out:
    measure.append_rows(args.out, [dict(r, card=card) for r in rows])


if __name__ == '__main__':
  main()
