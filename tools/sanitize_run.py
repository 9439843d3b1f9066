"""Small end-to-end run for compute-sanitizer (memcheck / racecheck / synccheck).

  compute-sanitizer --tool memcheck  python tools/sanitize_run.py
  compute-sanitizer --tool racecheck python tools/sanitize_run.py
  compute-sanitizer --tool synccheck python tools/sanitize_run.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ddsp_b200  # noqa: E402
from ddsp_b200 import autograd as ag, core  # noqa: E402
from tests.util import synth_inputs  # noqa: E402

B, F, K, nb, N = 3, 70, 100, 65, 70 * 64      # 3 tiles per item, edges included
inp = synth_inputs(B, F, K, nb, N, seed=1)
feats = {k: torch.from_numpy(inp[k]).cuda() for k in
         ['amps', 'harmonic_distribution', 'f0_hz', 'noise_magnitudes']}
harm = ddsp_b200.Harmonic(n_samples=N)
noise = ddsp_b200.FilteredNoise(n_samples=N, window_size=0)
group = ddsp_b200.ProcessorGroup(dag=[
    (harm, ['amps', 'harmonic_distribution', 'f0_hz']),
    (noise, ['noise_magnitudes']),
    (ddsp_b200.Add(), ['filtered_noise/signal', 'harmonic/signal'])])
a = group(feats)                                 # decoder_forward (fast + pipelined)
outs = group.get_controls(feats)                 # per-processor kernels + Add
b = core.filtered_noise(outs['filtered_noise']['controls']['magnitudes'][:, :, :33]
                        .contiguous(), N, window_size=0)          # generic fused kernel
c = core.frequency_filter(torch.rand(2, 1000).cuda(), torch.rand(2, 13, 513).cuda(),
                          window_size=257)       # generic ir + fir kernels
d, ph = core.streaming_harmonic_synthesis(feats['f0_hz'][:, :2], torch.rand(B, 2, 1).cuda(),
                                          torch.rand(B, 2, K).cuda(), n_samples=320)
raw = {k: feats[k].clone().requires_grad_(True) for k in
       ['amps', 'harmonic_distribution', 'noise_magnitudes']}
audio = ag.decoder_train(raw['amps'], raw['harmonic_distribution'], feats['f0_hz'],
                         raw['noise_magnitudes'], n_samples=N, window_size=0)
audio.square().mean().backward()
# fused spectral-loss pieces, host-buffer pipeline, Sinusoidal, Reverb (cuFFT route)
from ddsp_b200 import losses, host
tgt = 0.1 * torch.randn(B, N, device='cuda')
aud = (0.1 * torch.randn(B, N, device='cuda')).requires_grad_(True)
losses.SpectralLoss(fft_sizes=(256, 64), mag_weight=1.0, logmag_weight=1.0)(tgt, aud).backward()
dec = ddsp_b200.HostDecoder(group, B, F, K, nb, n_chunks=2)
e = dec({k: host.pin(inp[k]) for k in ['amps', 'harmonic_distribution', 'f0_hz',
                                        'noise_magnitudes']})
dec.close()
f = ddsp_b200.Sinusoidal(n_samples=640)(torch.randn(2, 10, 6), torch.randn(2, 10, 6))
g = ddsp_b200.Reverb()(torch.randn(2, 3000).cuda(), 0.01 * torch.randn(2, 2500).cuda())
# round-2 kernels: harmonic_shifts / fused sinusoidal bank, cubic + 4-D resample,
# angular_cumsum (exact and TF order), tf_sequential bank, long-IR convolution forward
# and backward, d f0, f0 < 1 Hz frames
shifts = 0.01 * torch.randn(B, F, K, device='cuda')
h2 = core.harmonic_synthesis(feats['f0_hz'], outs['harmonic']['controls']['amplitudes'],
                             harmonic_shifts=shifts,
                             harmonic_distribution=outs['harmonic']['controls']['harmonic_distribution'],
                             n_samples=N)
r4 = core.resample(torch.randn(2, 9, 3, 2), 37, method='cubic', add_endpoint=False)
om = 0.3 * torch.rand(2, 2300, 3, device='cuda')
pc = core.angular_cumsum(om); ps = core.angular_cumsum(om, tf_sequential=True)
ob = core.oscillator_bank(200 + 3000 * torch.rand(2, 700, 4, device='cuda'),
                          torch.rand(2, 700, 4, device='cuda'), phase_mode='tf_sequential',
                          use_angular_cumsum=True)
xa = torch.randn(2, 5000, device='cuda', requires_grad=True)
hi = (0.02 * torch.randn(1, 4500, device='cuda')).requires_grad_(True)
core.fft_convolve(xa, hi, padding='same', delay_compensation=0).square().mean().backward()
f0g = feats['f0_hz'].clone()
f0g[:, 5:9] = 0.3
f0g.requires_grad_(True)
ag.decoder_train(feats['amps'], feats['harmonic_distribution'], f0g,
                 feats['noise_magnitudes'], n_samples=N, window_size=0).abs().mean().backward()
# windowed-sinc filters: impulse response and its backward, the fused filter forward
# and backward (ragged frames, a shared cutoff, frames split into segments)
sc = (0.5 * torch.rand(2, 7, 1, device='cuda')).requires_grad_(True)
core.sinc_impulse_response(sc, window_size=64, high_pass=True).square().mean().backward()
xs = torch.randn(2, 3000, device='cuda', requires_grad=True)
core.sinc_filter(xs, sc, window_size=64).square().mean().backward()
scs = (0.5 * torch.rand(1, 1, 1, device='cuda')).requires_grad_(True)
core.sinc_filter(xs, scs, window_size=512, padding='valid').square().mean().backward()
# sinusoidal_to_harmonic forward and backward: two harmonic chunks, both normalize modes
sa = torch.rand(2, 5, 37, device='cuda', requires_grad=True)
sfq = (4000.0 * torch.rand(2, 5, 37, device='cuda')).requires_grad_(True)
sf0 = (80.0 + 300.0 * torch.rand(2, 5, 1, device='cuda')).requires_grad_(True)
for norm in (False, True):
  ha, hd = core.sinusoidal_to_harmonic(sa, sfq, sf0, n_harmonics=300, normalize=norm)
  (ha.sum() + hd.square().sum()).backward()
# oscillator_bank backward (both sum_sinusoids values, N past the 128 time segments)
# and angular_cumsum backward
obf = (200 + 9000 * torch.rand(2, 700, 37, device='cuda')).requires_grad_(True)
oba = torch.rand(2, 700, 37, device='cuda', requires_grad=True)
for ss in (True, False):
  core.oscillator_bank(obf, oba, sum_sinusoids=ss).square().mean().backward()
omg = om.clone().requires_grad_(True)
core.angular_cumsum(omg).square().mean().backward()
torch.cuda.synchronize()
assert torch.isfinite(obf.grad).all() and torch.isfinite(oba.grad).all()
assert torch.isfinite(omg.grad).all()
assert torch.isfinite(sc.grad).all() and torch.isfinite(scs.grad).all()
assert torch.isfinite(sa.grad).all() and torch.isfinite(sf0.grad).all()
assert torch.isfinite(h2).all() and torch.isfinite(r4).all() and torch.isfinite(ob).all()
assert torch.isfinite(xa.grad).all() and torch.isfinite(hi.grad).all() and torch.isfinite(f0g.grad).all()
assert torch.isfinite(e).all() and torch.isfinite(f).all() and torch.isfinite(g).all()
# HmmTranscriber: log_prob with its backward (a partial last segment) and Viterbi
hmm = losses.HmmTranscriber(n_timesteps=37, n_pitches=45)
hp = (45.0 * torch.rand(2, 37, 1, device='cuda')).requires_grad_(True)
ha = 1.5 * torch.rand(2, 37, 1, device='cuda')
hmm.nll(hp, ha).backward()
hq = hmm.predict_midi(hp, ha)
torch.cuda.synchronize()
assert torch.isfinite(hp.grad).all() and bool(((hq >= 0) & (hq < 45)).all())
# wasserstein_distance: unequal sides with ties, forward and backward
wx = [torch.round(4.0 * torch.rand(3, n, device='cuda')).requires_grad_(True) for n in (37, 70)]
ww = [torch.rand(3, n, device='cuda').requires_grad_(True) for n in (37, 70)]
losses.wasserstein_distance(wx[0], wx[1], ww[0], ww[1]).sum().backward()
torch.cuda.synchronize()
assert all(torch.isfinite(t.grad).all() for t in wx + ww)
print('sanitize_run ok', float(a.abs().mean()), float(b.abs().mean()),
      float(c.abs().mean()), float(d.abs().mean()),
      float(raw['harmonic_distribution'].grad.abs().mean()))
