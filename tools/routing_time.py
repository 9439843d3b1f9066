"""Time of the routing kernels (csrc/routing.cuh) at B = 32 and 256, N = 64000, each
against float32 torch autograd of the reference formulas on the same GPU:

  * Mix forward and backward (C = 1, the mix level [B, N, 1]);
  * the resample backward of a [B, 1000, 1] mix level to N samples ('linear');
  * the ExpDecayReverb impulse response, forward and backward, at L = 48000 (one row
    per item, in-kernel Philox noise);
  * the whole ExpDecayReverb (L = 48000, add_dry) forward + backward, gradients to
    audio, gain and decay.

  python tools/routing_time.py [--iters 50] [--warmup 10]

Kernel times are CUDA events over a ring of input sets larger than twice the L2.
Each kernel's algorithmic bytes over its time are reported as a share of the H100
SXM data-sheet HBM bandwidth (3.35 TB/s): Mix forward 16 B per sample (read s1, s2,
m; write out), Mix backward 28 (read s1, s2, m, g; write three gradients), resample
backward 4 per sample + 4 per frame, IR forward 4 per tap (write), IR backward 4 per
tap (read).  Prints the card name and power limit read in the same run."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import _lib  # noqa: E402
from ddsp_b200 import core  # noqa: E402
from ddsp_b200 import effects  # noqa: E402
from tools import measure  # noqa: E402


def _linear_taps(F, N, device):
  """resample 'linear' (add_endpoint) sample -> frame taps in TF's float32 math."""
  scale = torch.tensor(F / N, dtype=torch.float32)
  src = torch.arange(N, dtype=torch.float32) * scale
  fl = torch.floor(src)
  lo = fl.long().clamp(0, F - 1)
  hi = torch.ceil(src).long().clamp(max=F - 1)
  return lo.to(device), hi.to(device), (src - fl).to(device)


def _entry(ms, nbytes, torch_ms):
  sec = ms * 1e-3
  return {'us': ms * 1e3, 'bytes': nbytes, 'achieved_TBps': nbytes / sec / 1e12,
          'fraction_of_hbm_peak': nbytes / sec / measure.HBM_BYTES_PER_S,
          'torch_us': torch_ms * 1e3, 'speedup_vs_torch': torch_ms / ms}


def run(B, N, F, L, iters, warmup):
  lib = _lib.load()
  st = torch.cuda.current_stream().cuda_stream
  n_sets = measure.ring_len(4 * 4 * B * N)
  gen = torch.Generator(device='cuda').manual_seed(B)
  sets = []
  for _ in range(n_sets):
    s1, s2, g = (torch.randn((B, N, 1), device='cuda', generator=gen) for _ in range(3))
    m = torch.rand((B, N, 1), device='cuda', generator=gen)
    sets.append((s1, s2, m, g))
  out = torch.empty((B, N, 1), device='cuda')
  d = [torch.empty((B, N, 1), device='cuda') for _ in range(3)]
  res = {'B': B, 'N': N, 'input_sets': n_sets}

  def ms(fn, inputs):
    return measure.event_ms(fn, iters, warmup, inputs)

  def mix_f(s):
    _lib.check(lib.ddsp_b200_mix_forward(s[0].data_ptr(), s[1].data_ptr(), s[2].data_ptr(),
                                         out.data_ptr(), B, N, 1, st))

  def mix_b(s):
    _lib.check(lib.ddsp_b200_mix_backward(
        s[0].data_ptr(), s[1].data_ptr(), s[2].data_ptr(), s[3].data_ptr(), d[0].data_ptr(),
        d[1].data_ptr(), d[2].data_ptr(), B, N, 1, st))

  def torch_mix(s):
    return torch.sqrt(torch.abs(s[2])) * s[0] + (1.0 - torch.sqrt(torch.abs(s[2] - 1.0))) * s[1]

  def torch_mix_f(s):
    torch_mix(s)

  tsets = [tuple(v.clone().requires_grad_(True) for v in s[:3]) + (s[3],) for s in sets]

  def torch_mix_b(s):
    torch.autograd.grad(torch_mix(s), s[:3], s[3])

  samples = B * N
  res['mix_forward'] = _entry(ms(mix_f, sets), 16 * samples, ms(torch_mix_f, sets))
  res['mix_backward'] = _entry(ms(mix_b, sets), 28 * samples, ms(torch_mix_b, tsets))

  # resample backward of a [B, F, 1] mix level
  lo, hi, frac = _linear_taps(F, N, 'cuda')
  levels = [torch.rand((B, F, 1), device='cuda', generator=gen).requires_grad_(True)
            for _ in range(n_sets)]
  rsets = [(levels[i], sets[i][3]) for i in range(n_sets)]
  d_in = torch.empty((B, F, 1), device='cuda')

  def rs_b(s):
    _lib.check(lib.ddsp_b200_resample_backward(s[1].data_ptr(), d_in.data_ptr(), B, F, 1, N,
                                               1, 1, st))

  def torch_rs_b(s):
    x = s[0]
    top, bot = x[:, lo], x[:, hi]
    y = top + (bot - top) * frac[None, :, None]
    torch.autograd.grad(y, x, s[1])

  res['resample_backward'] = _entry(ms(rs_b, rsets), 4 * (samples + B * F),
                                    ms(torch_rs_b, rsets))

  # ExpDecayReverb impulse response, one row per item
  gains = [torch.rand((B,), device='cuda', generator=gen) for _ in range(n_sets)]
  decays = [torch.rand((B,), device='cuda', generator=gen) * 4.0 for _ in range(n_sets)]
  gir = [torch.randn((B, L), device='cuda', generator=gen) for _ in range(n_sets)]
  isets = list(zip(gains, decays, gir))
  ir = torch.empty((B, L), device='cuda')
  dg, dd = torch.empty((B,), device='cuda'), torch.empty((B,), device='cuda')

  def ir_f(s):
    _lib.check(lib.ddsp_b200_exp_decay_ir(s[0].data_ptr(), s[1].data_ptr(), None, 1, 0,
                                          ir.data_ptr(), B, L, st))

  def ir_b(s):
    _lib.check(lib.ddsp_b200_exp_decay_ir_backward(
        s[0].data_ptr(), s[1].data_ptr(), None, 1, 0, s[2].data_ptr(), dg.data_ptr(),
        dd.data_ptr(), B, L, st))

  time = torch.linspace(0.0, 1.0, L, device='cuda')[None, :]
  noise = core.uniform_noise(1, L, seed=1, offset=0)

  def torch_ir(g, dcy):
    return g[:, None] * torch.exp(-(2.0 + torch.exp(dcy[:, None])) * time) * noise

  def torch_ir_f(s):
    torch_ir(s[0], s[1])

  tisets = [(a.clone().requires_grad_(True), b.clone().requires_grad_(True), c)
            for a, b, c in isets]

  def torch_ir_b(s):
    torch.autograd.grad(torch_ir(s[0], s[1]), s[:2], s[2])

  res['ir_forward'] = _entry(ms(ir_f, isets), 4 * B * L, ms(torch_ir_f, isets))
  res['ir_backward'] = _entry(ms(ir_b, isets), 4 * B * L, ms(torch_ir_b, tisets))

  # the whole ExpDecayReverb, forward + backward
  audio = [s[0][:, :, 0].clone().requires_grad_(True) for s in sets]
  gsets = [(audio[i], gains[i][:, None].clone().requires_grad_(True),
            decays[i][:, None].clone().requires_grad_(True), sets[i][3][:, :, 0])
           for i in range(n_sets)]
  rev = effects.ExpDecayReverb(reverb_length=L, seed=1)

  def reverb(s):
    out = rev(s[0], s[1], s[2])
    torch.autograd.grad(out, s[:3], s[3])

  def torch_reverb(s):
    ir_ = 2.0 * torch.sigmoid(s[1])**2.302585092994046 + 1e-7
    ir_ = torch_ir(ir_[:, 0], s[2][:, 0])
    ir_ = torch.cat([torch.zeros_like(ir_[:, :1]), ir_[:, 1:]], 1)
    m = N + L - 1
    wet = torch.fft.irfft(torch.fft.rfft(s[0], m) * torch.fft.rfft(ir_, m), m)[:, :N]
    torch.autograd.grad(wet + s[0], s[:3], s[3])

  t_ours = measure.event_ms(reverb, max(iters // 5, 3), 3, gsets)
  t_torch = measure.event_ms(torch_reverb, max(iters // 5, 3), 3, gsets)
  res['exp_decay_reverb_fwd_bwd'] = {'ms': t_ours, 'torch_ms': t_torch,
                                     'speedup_vs_torch': t_torch / t_ours}
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--n', type=int, default=64000)
  ap.add_argument('--frames', type=int, default=1000)
  ap.add_argument('--reverb-length', type=int, default=48000)
  ap.add_argument('--iters', type=int, default=50)
  ap.add_argument('--warmup', type=int, default=10)
  args = ap.parse_args()
  measure.require_cuda('routing_time.py')
  out = {'card': measure.card(), 'runs': []}
  for B in (32, 256):
    out['runs'].append(run(B, args.n, args.frames, args.reverb_length, args.iters,
                           args.warmup))
    torch.cuda.empty_cache()
  print(json.dumps(out))


if __name__ == '__main__':
  main()
