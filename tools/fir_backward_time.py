"""Times the backward of the time-varying FIR (`FIRFilter`, `core.frequency_filter`,
`core.fft_convolve` under 2048 taps; csrc/fir_backward.cuh) at
  (a) FIRFilter at the decoder size: B = 32 and 256, N = 64000, F = 1000, nb = 65,
      window 257 (S = 128), with both d magnitudes routes;
  (b) nb = 1025, window 257 (S = 257), B = 32;
  (c) the longest direct-form Reverb: one 2047-tap impulse response per item,
      B = 32, N = 64000.
Per shape: the forward, each backward kernel through its entry point, the whole
`.backward()`, and float32 torch autograd of the reference's framed-FFT formulation.
CUDA events over --iters launches after warm-up; every launch reads its own copy of
the inputs, with enough copies that together they exceed L2.  Prints the card name and
power limit read in the same run.

  python tools/fir_backward_time.py [--iters 50]"""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddsp_b200 import _lib, core  # noqa: E402
from tools import measure  # noqa: E402

SAME = _lib.PAD_SAME


def _torch_filter32(x, mags, ws):
  """frequency_filter as float32 torch ops in the reference's formulation (irfft,
  Hann window, causal crop; framed rfft / multiply / irfft / overlap-add, crop)."""
  ir = torch.fft.irfft(mags.to(torch.complex64))
  s0 = ir.shape[-1]
  if ws <= 0 or ws > s0:
    ws = s0
  k = torch.arange(ws, device=x.device, dtype=torch.float32)
  d = ws if ws % 2 == 0 else ws - 1
  win = 0.5 - 0.5 * torch.cos(2 * math.pi * k / d)
  if ws < s0:
    half = (ws + 1) // 2
    win = torch.cat([win[half:], win.new_zeros(s0 - ws), win[:half]])
    ir = ir * win
    ir = torch.cat([ir[..., s0 - half + 2:], ir[..., :half + 1]], dim=-1)
  else:
    ir = torch.fft.fftshift(ir * torch.fft.fftshift(win), dim=-1)
  return _torch_convolve32(x, ir.reshape(x.shape[0], -1, ir.shape[-1]), -1)


def _torch_convolve32(x, ir, delay):
  b, n = x.shape
  f, s = ir.shape[1], ir.shape[2]
  frame = -(-n // f)
  frames = torch.nn.functional.pad(x, (0, f * frame - n)).reshape(b, f, frame)
  nfft = 1 << (s + frame - 2).bit_length()
  y = torch.fft.irfft(torch.fft.rfft(frames, nfft) * torch.fft.rfft(ir, nfft), nfft)
  if f == 1:
    out = y[:, 0]
  else:
    out = torch.nn.functional.fold(y.transpose(1, 2), output_size=((f - 1) * frame + nfft, 1),
                                   kernel_size=(nfft, 1), stride=(frame, 1))[:, 0, :, 0]
  start = (s - 1) // 2 - 1 if delay < 0 else delay
  return out[:, start:start + n]


def _filter_shape(label, B, F, nb, ws, iters):
  N = 64000
  lib = _lib.load()
  st = torch.cuda.current_stream().cuda_stream
  S = core._ir_size(nb, ws)
  per_set = 4 * (2 * B * N + B * F * nb + B * F * S)
  R = measure.ring_len(per_set)
  xs = [torch.randn(B, N, device='cuda') for _ in range(R)]
  ms = [torch.rand(B, F, nb, device='cuda') + 0.05 for _ in range(R)]
  gs = [torch.randn(B, N, device='cuda') for _ in range(R)]
  irs = [core.frequency_impulse_response(m, ws) for m in ms]
  d_audio = torch.empty(B, N, device='cuda')
  d_mags = torch.empty(B, F, nb, device='cuda')
  d_ir = torch.empty(B, F, S, device='cuda')
  print('%s: B=%d N=%d F=%d nb=%d window %d (S=%d), %d input copies' %
        (label, B, N, F, nb, ws, S, R), flush=True)

  ring, warmup = range(R), max(3, R)     # warm-up touches every input set

  def fwd(i):
    with torch.no_grad():
      return core.frequency_filter(xs[i], ms[i], window_size=ws)
  t_fwd = measure.event_ms(fwd, iters, warmup, ring)
  print('  forward (IR + FIR)                     %8.3f ms' % t_fwd, flush=True)

  def k_audio(i):
    _lib.check(lib.ddsp_b200_fir_time_varying_backward(
        xs[i].data_ptr(), irs[i].data_ptr(), gs[i].data_ptr(), d_audio.data_ptr(),
        None, B, N, F, S, B, SAME, -1, None, 0, st))
  nbytes = lib.ddsp_b200_fir_time_varying_backward_workspace(B, N, F, S, B)
  wsb = torch.empty(max(nbytes, 1), dtype=torch.uint8, device='cuda')

  def k_ir(i):
    _lib.check(lib.ddsp_b200_fir_time_varying_backward(
        xs[i].data_ptr(), irs[i].data_ptr(), gs[i].data_ptr(), None,
        d_ir.data_ptr(), B, N, F, S, B, SAME, -1, wsb.data_ptr(), nbytes, st))

  def k_irb(i):
    _lib.check(lib.ddsp_b200_frequency_impulse_response_backward(
        d_ir.data_ptr(), d_mags.data_ptr(), B * F, nb, ws, st))
  fnbytes = lib.ddsp_b200_frequency_filter_backward_workspace(B, F, nb, N, B, ws, SAME)
  fwsb = torch.empty(max(fnbytes, 1), dtype=torch.uint8, device='cuda')

  def k_mags(i):        # the entry point's own d magnitudes route
    _lib.check(lib.ddsp_b200_frequency_filter_backward(
        xs[i].data_ptr(), irs[i].data_ptr(), gs[i].data_ptr(), None,
        d_mags.data_ptr(), B, F, nb, N, B, ws, SAME, fwsb.data_ptr(), fnbytes, st))
  route = 'fused noise_backward_kernel' if fnbytes == 0 else 'd IR + IR adjoint'
  t_a, t_ir, t_irb, t_m = (measure.event_ms(k, iters, warmup, ring)
                           for k in (k_audio, k_ir, k_irb, k_mags))
  fma = B * N * S
  print('  d audio   fir_adjoint_kernel           %8.3f ms  (%.1f TFMA/s)' %
        (t_a, fma / t_a / 1e9))
  print('  d IR      fir_dir_kernel (+ reduce)    %8.3f ms  (%.1f TFMA/s, %d MB d IR)' %
        (t_ir, fma / t_ir / 1e9, B * F * S * 4 >> 20))
  print('  d mags    ir_backward_kernel           %8.3f ms' % t_irb)
  print('  d mags    kernels 2 + 3                %8.3f ms' % (t_ir + t_irb))
  print('  d mags    entry point (%s) %8.3f ms' % (route, t_m), flush=True)

  x1s = [x.clone().requires_grad_(True) for x in xs]
  m1s = [m.clone().requires_grad_(True) for m in ms]

  def fwd_bwd(i):
    x1, m1 = x1s[i], m1s[i]
    x1.grad = m1.grad = None
    core.frequency_filter(x1, m1, window_size=ws).backward(gs[i])
  t_fb = measure.event_ms(fwd_bwd, iters, warmup, ring)
  print('  forward + .backward()                  %8.3f ms   backward %.3f ms' %
        (t_fb, t_fb - t_fwd), flush=True)
  del x1s, m1s

  def torch_fb():
    x1 = xs[0].clone().requires_grad_(True)
    m1 = ms[0].clone().requires_grad_(True)
    _torch_filter32(x1, m1, ws).backward(gs[0])
  print('  float32 torch autograd                 %8.3f ms' % measure.event_ms(torch_fb, 5, 1),
        flush=True)
  torch.cuda.empty_cache()


def _reverb_shape(B, S, iters):
  N = 64000
  lib = _lib.load()
  st = torch.cuda.current_stream().cuda_stream
  R = measure.ring_len(4 * (2 * B * N + B * S))
  ring, warmup = range(R), max(3, R)     # warm-up touches every input set
  xs = [torch.randn(B, N, device='cuda') for _ in range(R)]
  hs = [torch.randn(B, S, device='cuda') / 45.0 for _ in range(R)]
  gs = [torch.randn(B, N, device='cuda') for _ in range(R)]
  d_audio = torch.empty(B, N, device='cuda')
  d_ir = torch.empty(B, S, device='cuda')
  nbytes = lib.ddsp_b200_fir_time_varying_backward_workspace(B, N, 1, S, B)
  wsb = torch.empty(max(nbytes, 1), dtype=torch.uint8, device='cuda')
  print('(c) direct-form Reverb: B=%d N=%d one %d-tap IR per item, %d input copies, '
        '%d MB workspace' % (B, N, S, R, nbytes >> 20), flush=True)

  def fwd(i):
    with torch.no_grad():
      return core.fft_convolve(xs[i], hs[i], delay_compensation=0)

  def k_audio(i):
    _lib.check(lib.ddsp_b200_fir_time_varying_backward(
        xs[i].data_ptr(), hs[i].data_ptr(), gs[i].data_ptr(), d_audio.data_ptr(),
        None, B, N, 1, S, B, SAME, 0, None, 0, st))

  def k_ir(i):
    _lib.check(lib.ddsp_b200_fir_time_varying_backward(
        xs[i].data_ptr(), hs[i].data_ptr(), gs[i].data_ptr(), None,
        d_ir.data_ptr(), B, N, 1, S, B, SAME, 0, wsb.data_ptr(), nbytes, st))
  fma = B * N * S
  t_f, t_a, t_ir = (measure.event_ms(k, iters, warmup, ring) for k in (fwd, k_audio, k_ir))
  print('  forward (fir_kernel)                   %8.3f ms  (%.1f TFMA/s)' % (t_f, fma / t_f / 1e9))
  print('  d audio   fir_adjoint_kernel           %8.3f ms  (%.1f TFMA/s)' % (t_a, fma / t_a / 1e9))
  print('  d IR      fir_dir_kernel + reduce      %8.3f ms  (%.1f TFMA/s)' % (t_ir, fma / t_ir / 1e9))
  x1s = [x.clone().requires_grad_(True) for x in xs]
  h1s = [h.clone().requires_grad_(True) for h in hs]

  def fwd_bwd(i):
    x1, h1 = x1s[i], h1s[i]
    x1.grad = h1.grad = None
    core.fft_convolve(x1, h1, delay_compensation=0).backward(gs[i])
  t_fb = measure.event_ms(fwd_bwd, iters, warmup, ring)
  print('  forward + .backward()                  %8.3f ms   backward %.3f ms' %
        (t_fb, t_fb - t_f), flush=True)
  del x1s, h1s

  def torch_fb():
    x1 = xs[0].clone().requires_grad_(True)
    h1 = hs[0].clone().requires_grad_(True)
    _torch_convolve32(x1, h1[:, None, :], 0).backward(gs[0])
  print('  float32 torch autograd                 %8.3f ms' % measure.event_ms(torch_fb, 5, 1),
        flush=True)
  torch.cuda.empty_cache()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=50)
  args = ap.parse_args()
  measure.require_cuda('fir_backward_time.py')
  print(json.dumps(measure.card()), flush=True)
  torch.manual_seed(0)
  _filter_shape('(a) FIRFilter', 32, 1000, 65, 257, args.iters)
  _filter_shape('(a) FIRFilter', 256, 1000, 65, 257, args.iters)
  _filter_shape('(b) FIRFilter', 32, 1000, 1025, 257, args.iters)
  _reverb_shape(32, 2047, args.iters)


if __name__ == '__main__':
  main()
