"""Forward synthesis kernels at every hop, band count, frame size, window and tile
count they accept, against float64.

  * noise_fused_kernel (noise_fused.cuh): band counts 3 .. 129, frames 16 .. 512,
    padded and clamped windows, ragged last frames, persistent CTAs that walk
    many tiles (prefetch, per-tile re-zeroing, impulse-response rows left from
    the previous tile), accumulate, in-kernel Philox over interior and boundary
    tiles, and a random sweep against the unspecialised IR + FIR kernels;
  * harmonic_v4_kernel (harmonic_v4.cuh): hops 64 .. 8192, K 1 .. 1024, every tile
    width FW, TMA against LDG staging of the frame slab, long items;
  * decoder_forward and HostDecoder at shapes other than the ring shape;
  * the streaming bank (harmonic_generic_kernel) several tiles wide in F.

The route of every case is tabled in tests/grad_ref.py and pinned without a GPU by
tests/test_forward_routing.py; each noise case here also asserts it against the
library's routing on the device, each harmonic case its restated tile width.
Shapes whose [B, N, K] would be large for the NumPy oracle are checked against
grad_ref's float64 restatements on the GPU (pinned to the oracle at <= 1e-12).
"""
import numpy as np
import pytest
import torch

import ddsp_b200
from ddsp_b200 import _lib
from ddsp_b200 import core
from ddsp_b200 import host
from oracle import ddsp_oracle as o
from tests import grad_ref
from tests.util import rel_err, synth_inputs

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')
TOL = 1e-4
ORACLE_ELEMS = 4_000_000        # largest [B, N, K] handed to the NumPy oracle
CHUNK_ELEMS = 20_000_000        # per batch chunk of the float64 GPU reference


def _np(x):
  return x.detach().cpu().numpy()


def _gate(got, want, tol=TOL):
  got = _np(got) if isinstance(got, torch.Tensor) else got
  want = _np(want) if isinstance(want, torch.Tensor) else want
  assert np.isfinite(got).all()
  emax, el2 = rel_err(got, want)
  assert emax < tol and el2 < tol, (emax, el2)


def _n_sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------
# float64 references
# ---------------------------------------------------------------------------
def _harmonic_ref(f0, amp, hd, N, sr, method):
  """[B, N] float64 harmonic synthesis: the NumPy oracle for small shapes,
  grad_ref.harmonic on the GPU in batch chunks otherwise.  Both take the Nyquist
  decision in float32, as the reference does."""
  B, _, K = hd.shape
  if B * N * K <= ORACLE_ELEMS:
    return torch.from_numpy(o.harmonic_synthesis(
        _np(f0), _np(amp), harmonic_distribution=_np(hd), n_samples=N, sample_rate=sr,
        amp_resample_method=method)).to(DEV)
  step = max(1, CHUNK_ELEMS // (N * K))
  return torch.cat([grad_ref.harmonic(f0[i:i + step], amp[i:i + step], hd[i:i + step], N,
                                      sr, method) for i in range(0, B, step)])


def _noise_ref(noise, mags, ws):
  """[B, N] float64 core.frequency_filter: the oracle for small shapes,
  grad_ref.frequency_filter on the GPU otherwise."""
  if noise.numel() <= 1_000_000:
    return torch.from_numpy(o.frequency_filter(_np(noise).astype(np.float64), _np(mags),
                                               window_size=ws)).to(DEV)
  return grad_ref.frequency_filter(noise.to(DEV).double(), mags.to(DEV).double(), ws)


def _philox(B, N, seed, offset):
  return torch.from_numpy(o.philox_uniform_noise(B, N, seed, offset)).to(DEV)


# ---------------------------------------------------------------------------
# A. noise_fused_kernel
# ---------------------------------------------------------------------------
def _assert_noise_route(B, F, nb, N, ws, route):
  """The library's own routing (workspace 0 <=> fused) agrees with the table."""
  kind = 'generic' if route == 'generic' else 'fused'
  assert grad_ref.noise_route(F, nb, N, ws) == kind
  ws_bytes = _lib.load().ddsp_b200_filtered_noise_workspace(B, F, nb, N, ws)
  assert (ws_bytes == 0) == (kind == 'fused'), (route, ws_bytes)
  if kind == 'fused':
    geo = grad_ref.noise_fused_geometry(F, nb, N, ws)
    assert geo['ctas_per_sm'] == int(route[-1])
    return geo
  return None


def _noise_inputs(B, F, nb, N, seed):
  gen = torch.Generator(device='cpu').manual_seed(seed)
  mags = torch.rand(B, F, nb, generator=gen) + 0.02
  noise = torch.rand(B, N, generator=gen) * 2 - 1
  return mags.to(DEV), noise.to(DEV)


@pytest.mark.parametrize('B,F,nb,frame,ws,r,route', grad_ref.FWD_NOISE_CASES)
def test_filtered_noise_every_band_count_frame_and_window(B, F, nb, frame, ws, r, route):
  """core.filtered_noise with injected noise against float64 at band counts 3 ..
  129, frames 16 .. 512, windows 3 .. 257 (odd / even padded, clamped to the IR),
  ragged last frames, and each fused shape's declined neighbour."""
  N = F * frame - r
  _assert_noise_route(B, F, nb, N, ws, route)
  mags, noise = _noise_inputs(B, F, nb, N, seed=nb * 1000 + frame + ws)
  got = core.filtered_noise(mags, N, window_size=ws, noise=noise)
  _gate(got, _noise_ref(noise, mags, ws))


@pytest.mark.parametrize('B,F,nb,frame,ws,r,route', grad_ref.FWD_NOISE_MANY_TILES)
def test_filtered_noise_many_tiles_per_cta(B, F, nb, frame, ws, r, route):
  """Persistent CTAs walking >= 3 tiles each: the cp.async prefetch of the next
  tile's magnitudes, the per-tile re-zeroing of the overlap-add buffer and the
  impulse-response rows that stay in shared memory between tiles.  Injected noise
  against float64, then in-kernel Philox (interior and boundary tiles, the ragged
  tail) against the same Philox stream injected."""
  N = F * frame - r
  geo = _assert_noise_route(B, F, nb, N, ws, route)
  n_tiles = B * geo['tiles_per_item']
  assert n_tiles >= 3 * _n_sms() * geo['ctas_per_sm'], n_tiles
  gen = torch.Generator(device='cpu').manual_seed(F + nb)
  mags = (torch.rand(B, F, nb, generator=gen) + 0.02).to(DEV)
  seed, offset = 1234 + nb, 7
  nz = _philox(B, N, seed, offset)
  got = core.filtered_noise(mags, N, window_size=ws, noise=nz)
  _gate(got, _noise_ref(nz, mags, ws))
  in_kernel = core.filtered_noise(mags, N, window_size=ws, seed=seed, offset=offset)
  assert torch.isfinite(in_kernel).all()
  assert float((in_kernel - got).abs().max()) <= 1e-6 * float(got.abs().max())


@pytest.mark.parametrize('B,F,nb,frame,ws,r,seed,offset', [
    (2, 40, 65, 64, 101, 0, 42, 3),
    (2, 50, 17, 48, 0, 47, 5, 0),        # frame 48: the divide path of the quad index
    (1, 1001, 33, 64, 0, 33, 2**40 + 3, 11),   # 64031 samples: interior tiles, ragged tail
    (3, 45, 33, 80, 31, 40, 9, 1),
    (2, 30, 65, 128, 0, 1, 77, 2**33),
])
def test_filtered_noise_in_kernel_philox(B, F, nb, frame, ws, r, seed, offset):
  """The in-kernel Philox stream (seed, offset) equals the oracle's
  philox_uniform_noise injected, to 1e-6 of the peak, and both match float64."""
  N = F * frame - r
  assert grad_ref.noise_route(F, nb, N, ws) == 'fused'
  gen = torch.Generator(device='cpu').manual_seed(seed % 1000)
  mags = (torch.rand(B, F, nb, generator=gen) + 0.02).to(DEV)
  got = core.filtered_noise(mags, N, window_size=ws, seed=seed, offset=offset)
  nz = _philox(B, N, seed, offset)
  inj = core.filtered_noise(mags, N, window_size=ws, noise=nz)
  assert float((got - inj).abs().max()) <= 1e-6 * float(inj.abs().max())
  _gate(got, _noise_ref(nz, mags, ws))


@pytest.mark.parametrize('B,F,nb,frame,ws,r,misaligned', [
    (3, 40, 33, 64, 0, 0, False),     # TFo * frame <= 3072: the prefetched += operand
    (3, 40, 33, 64, 0, 0, True),
    (2, 45, 33, 64, 31, 2, False),    # N % 4 == 2: rows 1.. misaligned (scalar stores)
    (3, 30, 63, 128, 0, 0, False),    # frame >= 128: the direct read
    (3, 30, 63, 128, 0, 0, True),
    (2, 35, 65, 128, 101, 5, True),
])
def test_filtered_noise_accumulate(B, F, nb, frame, ws, r, misaligned):
  """accumulate=True onto a random base, with rows 16-byte aligned or not (a view
  4 bytes into a larger buffer): base + filtered noise against float64."""
  N = F * frame - r
  assert grad_ref.noise_route(F, nb, N, ws) == 'fused'
  mags, noise = _noise_inputs(B, F, nb, N, seed=N)
  base = 0.5 * torch.randn(B, N, device=DEV, generator=torch.Generator(device=DEV)
                           .manual_seed(N))
  if misaligned:
    flat = torch.zeros(B * N + 1, device=DEV)
    out = flat[1:].view(B, N)
    assert out.data_ptr() % 16 != 0
  else:
    out = torch.empty(B, N, device=DEV)
  out.copy_(base)
  core.filtered_noise(mags, N, window_size=ws, noise=noise, out=out, accumulate=True)
  want = _noise_ref(noise, mags, ws)
  _gate(out.double() - base.double(), want)


def test_filtered_noise_random_shapes_against_the_generic_path():
  """~100 random shapes the fused kernel accepts (fixed seed), with and without
  accumulate, against the unspecialised path - impulse responses to HBM, then the
  plain time-varying FIR kernel - to 2e-5 of the peak, and each bit for bit against
  one repeat of the same launch."""
  lib = _lib.load()
  rng = np.random.default_rng(4096)
  st = torch.cuda.current_stream().cuda_stream
  done = 0
  while done < 100:
    nb = int(rng.choice([3, 5, 9, 17, 31, 33, 63, 65, 101, 127, 129]))
    frame = 16 * int(rng.integers(1, 33))
    F = int(rng.choice([1, 2, 7, 16, 29, 31, 33, 64, 97])) if rng.random() < 0.5 \
        else int(rng.integers(1, 200))
    B = int(rng.integers(1, 7))
    s0 = 2 * (nb - 1)
    ws = int(rng.choice([0, rng.integers(3, s0 + 1), s0 + 1 + int(rng.integers(0, 50))]))
    r = int(rng.integers(0, min(F, frame))) if rng.random() < 0.5 else 0
    N = F * frame - r
    if grad_ref.noise_route(F, nb, N, ws) != 'fused':
      continue
    done += 1
    acc = bool(rng.random() < 0.4)
    mags = torch.rand((B, F, nb), device=DEV) * 1.5
    noise = torch.rand((B, N), device=DEV) * 2 - 1
    base = torch.randn((B, N), device=DEV) if acc else None
    outs = []
    for _ in range(2):
      out = base.clone() if acc else torch.empty((B, N), device=DEV)
      _lib.check(lib.ddsp_b200_filtered_noise_forward(
          mags.data_ptr(), noise.data_ptr(), 0, 0, out.data_ptr(), B, F, nb, N, ws,
          int(acc), None, 0, st))
      outs.append(out)
    assert torch.equal(outs[0], outs[1]), (B, F, nb, frame, ws, r, acc)
    ir = core.frequency_impulse_response(mags, ws)
    want = base.clone() if acc else torch.empty((B, N), device=DEV)
    _lib.check(lib.ddsp_b200_fir_time_varying(
        noise.data_ptr(), ir.data_ptr(), want.data_ptr(), B, N, F, ir.shape[-1], B,
        _lib.PAD_SAME, -1, int(acc), st))
    got = outs[0] - base if acc else outs[0]
    ref = want - base if acc else want
    assert torch.isfinite(got).all()
    err = float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-20))
    assert err < 2e-5, (B, F, nb, frame, ws, r, acc, err)


# ---------------------------------------------------------------------------
# B. harmonic_v4_kernel
# ---------------------------------------------------------------------------
def _harmonic_inputs(B, F, K, sr, regime, seed):
  f0 = grad_ref.low_f0_regime(regime, B, F, sr, seed=seed).to(DEV)
  gen = torch.Generator(device='cpu').manual_seed(seed)
  amp = (torch.rand(B, F, 1, generator=gen) + 0.2).to(DEV)
  hd = torch.rand(B, F, K, generator=gen)
  hd = (hd / hd.sum(-1, keepdim=True)).to(DEV)
  return f0, amp, hd


@pytest.mark.parametrize('B,F,K,hop,sr,method,regime,acc,fw', grad_ref.FWD_HARMONIC_CASES)
def test_harmonic_v4_every_hop_k_and_tile_width(B, F, K, hop, sr, method, regime, acc, fw):
  """core.harmonic_synthesis(phase_mode='recurrence') against float64 at hops 64 ..
  8192 (and 8256, generic), K 1 .. 1024 (and 1025, generic), every tile width FW,
  both amplitude methods, 16 / 44.1 / 48 kHz, every f0 regime, F not a multiple
  of the tile and F = 1, accumulate onto a base.  The launcher's choice of
  kernel and FW is restated in grad_ref.harmonic_v4_tile_width (the library has
  no query for it)."""
  assert grad_ref.harmonic_v4_tile_width(B, F, K, hop, _n_sms()) == fw
  N = F * hop
  f0, amp, hd = _harmonic_inputs(B, F, K, sr, regime, seed=K + hop + F)
  base = None
  if acc:
    base = 0.5 * torch.randn(B, N, device=DEV,
                             generator=torch.Generator(device=DEV).manual_seed(hop))
  out = base.clone() if acc else None
  got = core.harmonic_synthesis(f0, amp, harmonic_distribution=hd, n_samples=N,
                                sample_rate=sr, amp_resample_method=method, out=out,
                                accumulate=acc, phase_mode='recurrence')
  want = _harmonic_ref(f0, amp, hd, N, sr, method)
  _gate(got.double() - base.double() if acc else got, want)


@pytest.mark.parametrize('B,F,K,hop,method', [(2, 40, 64, 256, 'window'),
                                              (3, 33, 100, 64, 'linear'),
                                              (1, 9, 1024, 512, 'window')])
def test_harmonic_v4_tma_and_ldg_staging_agree(B, F, K, hop, method):
  """The frame slab is staged by one TMA bulk copy when harmonic_distribution is
  16-byte aligned and K % 4 == 0, by LDG otherwise.  The same values from an
  aligned tensor and from a view 4 bytes into a larger buffer give bit-identical
  audio, and both match float64."""
  assert K % 4 == 0
  N = F * hop
  f0, amp, hd = _harmonic_inputs(B, F, K, 16000, 'glide', seed=K)
  assert hd.data_ptr() % 16 == 0
  flat = torch.zeros(hd.numel() + 1, device=DEV)
  hd_off = flat[1:].view(B, F, K)
  hd_off.copy_(hd)
  assert hd_off.is_contiguous() and hd_off.data_ptr() % 16 == 4
  tma = core.harmonic_synthesis(f0, amp, harmonic_distribution=hd, n_samples=N,
                                amp_resample_method=method)
  ldg = core.harmonic_synthesis(f0, amp, harmonic_distribution=hd_off, n_samples=N,
                                amp_resample_method=method)
  assert torch.equal(tma, ldg)
  _gate(tma, _harmonic_ref(f0, amp, hd, N, 16000, method))


@pytest.mark.parametrize('hop', [128, 256, 512])
def test_harmonic_v4_long_item(hop):
  """One 64000-sample item: the closed-form tile phase (tile_phase_base) far from
  frame 0 at hops other than 64, against float64 on the GPU."""
  N, K = 64000, 60
  F = N // hop
  inp = synth_inputs(1, F, K, 3, N, seed=hop, f0_lo=60.0, f0_hi=400.0)
  f0 = torch.from_numpy(inp['f0_hz']).to(DEV)
  gen = torch.Generator(device='cpu').manual_seed(hop)
  amp = (torch.rand(1, F, 1, generator=gen) + 0.2).to(DEV)
  hd = torch.rand(1, F, K, generator=gen)
  hd = (hd / hd.sum(-1, keepdim=True)).to(DEV)
  assert grad_ref.harmonic_v4_tile_width(1, F, K, hop, _n_sms()) is not None
  got = core.harmonic_synthesis(f0, amp, harmonic_distribution=hd, n_samples=N)
  _gate(got, grad_ref.harmonic(f0, amp, hd, N, 16000, 'window'))


# ---------------------------------------------------------------------------
# C. decoder_forward and HostDecoder off the ring shape
# ---------------------------------------------------------------------------
def _decoder_ref(inp, N, sr, nyq, ws, bias, noise):
  """harmonic_get_controls -> harmonic_get_signal + noise_get_controls(bias) ->
  noise_get_signal in float64 (the signal stages on the GPU for large shapes)."""
  hc = o.harmonic_get_controls(inp['amps'], inp['harmonic_distribution'], inp['f0_hz'],
                               sample_rate=sr, normalize_below_nyquist=nyq)
  mags = o.noise_get_controls(inp['noise_magnitudes'], initial_bias=bias)['magnitudes']
  f0 = torch.from_numpy(inp['f0_hz']).to(DEV)
  harm = _harmonic_ref(f0, torch.from_numpy(hc['amplitudes']).to(DEV),
                       torch.from_numpy(hc['harmonic_distribution']).to(DEV), N, sr,
                       'window')
  return harm + _noise_ref(noise, torch.from_numpy(mags), ws)


@pytest.mark.parametrize('B,F,K,nb,hop,sr,nyq,ws,bias,noise,route',
                         grad_ref.FWD_DECODER_CASES)
def test_decoder_forward_off_the_ring_shape(B, F, K, nb, hop, sr, nyq, ws, bias, noise,
                                            route):
  """core.decoder_forward from raw network outputs (exp_sigmoid with
  initial_bias fused into noise_fused_kernel's staging) at hops 128 .. 256, 33 /
  65 / 129 bands, padded windows, 44.1 kHz, with and without Nyquist
  normalisation, injected and in-kernel noise."""
  N = F * hop
  _assert_noise_route(B, F, nb, N, ws, route)
  inp = synth_inputs(B, F, K, nb, N, seed=F + K + nb, sample_rate=sr, f0_hi=1500.0)
  seed, offset = 3 + B, 5
  if noise == 'injected':
    nz = torch.from_numpy(inp['noise']).to(DEV)
  else:
    nz = _philox(B, N, seed, offset)
  dev = {k: torch.from_numpy(inp[k]).to(DEV) for k in
         ('amps', 'harmonic_distribution', 'f0_hz', 'noise_magnitudes')}
  got = core.decoder_forward(
      dev['amps'], dev['harmonic_distribution'], dev['f0_hz'], dev['noise_magnitudes'],
      N, sample_rate=sr, normalize_below_nyquist=nyq, window_size=ws,
      initial_bias=bias, noise=nz if noise == 'injected' else None, seed=seed,
      offset=offset)
  _gate(got, _decoder_ref(inp, N, sr, nyq, ws, bias, nz))


def _group(N, seed):
  harm = ddsp_b200.Harmonic(n_samples=N)
  noise = ddsp_b200.FilteredNoise(n_samples=N, window_size=0, seed=seed)
  return ddsp_b200.ProcessorGroup(dag=[
      (harm, ['amps', 'harmonic_distribution', 'f0_hz']),
      (noise, ['noise_magnitudes']),
      (ddsp_b200.Add(), ['filtered_noise/signal', 'harmonic/signal'])])


@pytest.mark.parametrize('chunks', [1, 3, 7])
def test_host_decoder_off_the_ring_shape(chunks):
  """HostDecoder at 33 bands and hop 128 (noise_fused_kernel, not the ring): every
  chunk after the first runs with a non-zero Philox item offset (item_base), and
  the audio is bit-equal to the device ProcessorGroup call and matches float64."""
  B, F, K, nb, hop = 7, 60, 40, 33, 128
  N = F * hop
  _assert_noise_route(B, F, nb, N, 0, 'fused2')
  inp = synth_inputs(B, F, K, nb, N, seed=chunks)
  keys = ['amps', 'harmonic_distribution', 'f0_hz', 'noise_magnitudes']
  feats = {k: inp[k] for k in keys}
  want = _group(N, seed=9)({k: torch.from_numpy(v).to(DEV) for k, v in feats.items()})
  dec = ddsp_b200.HostDecoder(_group(N, seed=9), max_batch=B, n_frames=F, n_harmonics=K,
                              n_bands=nb, n_chunks=chunks)
  got = dec({k: host.pin(v) for k, v in feats.items()})
  dec.close()
  assert torch.equal(got, want.cpu())
  inp['noise'] = _np(_philox(B, N, 9, 0))
  _gate(got.numpy(), _decoder_ref(inp, N, 16000, True, 0, -5.0,
                                  torch.from_numpy(inp['noise']).to(DEV)))


# ---------------------------------------------------------------------------
# D. streaming bank
# ---------------------------------------------------------------------------
def _streaming_inputs(B, F, K, seed):
  rng = np.random.default_rng(seed)
  f0 = rng.uniform(100, 900, (B, F, 1)).astype(np.float32)
  amp = rng.uniform(0.1, 1.0, (B, F, 1)).astype(np.float32)
  hd = rng.uniform(0.0, 1.0, (B, F, K)).astype(np.float32)
  return f0, amp, hd


def _phase_err(got, want):
  """Largest distance between two phases on the circle (the kernel returns the
  wrapped phase plus the initial one, the oracle its running sum)."""
  d = np.mod(_np(got).astype(np.float64) - want, 2 * np.pi)
  return np.minimum(d, 2 * np.pi - d).max()


@pytest.mark.parametrize('B,F,K,hop,method,init', [
    (2, 48, 30, 160, 'linear', 'near0'),
    (3, 41, 12, 160, 'window', 'near2pi'),
    (1, 128, 400, 16, 'linear', 'random'),    # 129 x 400 floats > 200 KB: the tile halves
])
def test_streaming_harmonic_several_tiles_wide(B, F, K, hop, method, init):
  """core.streaming_harmonic_synthesis with the grid several tiles wide in F (the
  last tile writes final_phase), the 160-sample half-hop, a K whose tile halves to
  fit shared memory, and initial phases near 0 and near 2 pi, against the oracle."""
  N = F * hop
  f0, amp, hd = _streaming_inputs(B, F, K, seed=F + K)
  ft0 = min(F, 2048 // hop)           # frames per tile before fit_tile (harmonic.cu)
  ft = ft0
  while ft > 1 and 8 * (3 * ft + 8) + 4 * (2 * (ft + 1) + (ft + 1) * ((K + 3) & ~3)) > \
      200 * 1024:                      # harm_smem_bytes > kMaxDynSmem
    ft = (ft + 1) // 2
  assert -(-F // ft) >= 2 and (ft < ft0) == (K == 400)
  phase = {'near0': np.full((B, 1, 1), 1e-3), 'near2pi': np.full((B, 1, 1), 2 * np.pi - 1e-3),
           'random': np.random.default_rng(K).uniform(0, 2 * np.pi, (B, 1, 1))}[init]
  phase = phase.astype(np.float32)
  want_a, want_p = o.streaming_harmonic_synthesis(f0, amp, hd, phase, n_samples=N,
                                                  amp_resample_method=method)
  got_a, got_p = core.streaming_harmonic_synthesis(f0, amp, hd, phase, n_samples=N,
                                                   amp_resample_method=method)
  _gate(got_a, want_a)
  assert got_p.shape == (B, 1, 1)
  assert _phase_err(got_p, want_p) < 1e-4


def test_streaming_harmonic_eight_chained_calls():
  """Eight hop-by-hop calls that carry final_phase into the next initial_phase
  equal the oracle's eight chained calls, audio and phase."""
  B, F, K, hop, calls = 2, 6, 24, 160, 8
  N = F * hop
  f0, amp, hd = _streaming_inputs(B, F * calls, K, seed=8)
  got, want = [], []
  p_got = p_want = np.full((B, 1, 1), 6.2, np.float32)
  for c in range(calls):
    sl = slice(c * F, (c + 1) * F)
    a, p_got = core.streaming_harmonic_synthesis(f0[:, sl], amp[:, sl], hd[:, sl], p_got,
                                                 n_samples=N)
    w, p_want = o.streaming_harmonic_synthesis(f0[:, sl], amp[:, sl], hd[:, sl], p_want,
                                               n_samples=N)
    got.append(_np(a))
    want.append(w)
  _gate(np.concatenate(got, 1), np.concatenate(want, 1))
  assert _phase_err(p_got, p_want) < 1e-4
