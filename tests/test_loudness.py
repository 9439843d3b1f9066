"""A-weighted loudness and RMS power (csrc/loudness.cuh, spectral_ops.compute_loudness /
compute_power / compute_rms_energy, SpectralLoss's loudness term): argument checks and
the float64 restatement on the CPU; forward, gradients, the loss, reproducibility and
CUDA-graph capture on the GPU.  Reference: tests/loudness_ref.py, pinned to the
unmodified reference by tests/golden/loudness.npz.

Forward tolerance.  The kernel frames, windows and transforms in float32: a radix-2
FFT of M = n_fft / 2 points has log2(M) <= 13 rounding stages, the split step and the
|X|^2 w_k products two more, so each bin carries a relative error of order
(log2 M + 3) * 2^-24 ~ 1e-6 of the frame's energy, and the weighted power sum (which
is dominated by the large bins) the same.  10 log10 turns a relative error e into
4.34 e dB: ~5e-6 dB.  Even a 20 Hz tone, whose weighted power sits ~50 dB below its
unweighted power, only meets the FFT's noise floor (~1e-7 of the peak magnitude per
bin, 1e-14 of its power) at the well-weighted bins, 1e-9 of the weighted total.  The
dB conversion runs in double.  1e-3 dB leaves a 100x margin; the clamped values are
exact."""
import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, core, losses, spectral_ops
from tests import loudness_ref as ref
from tests.golden import make_loudness_golden as mg

P = 0x1000        # a device pointer the library never dereferences on the host
E_INVALID, E_UNSUPPORTED = _lib.E_INVALID, _lib.E_UNSUPPORTED
CENTER, SAME, VALID = _lib.PAD_CENTER, _lib.PAD_SAME, _lib.PAD_VALID
DEV = 'cuda'
TOL_DB = 1e-3

_F, _B, _R = 'loudness_forward', 'loudness_backward', 'rms_power'


def _fwd(a=P, w=P, out=P, B=1, N=4000, T=63, n_fft=512, hop=64, pad=CENTER):
  return (a, w, out, B, N, T, n_fft, hop, pad, 80.0, 0.0, None)


def _bwd(a=P, w=P, g=P, d=P, B=1, N=4000, T=63, n_fft=512, hop=64, pad=CENTER):
  return (a, w, g, d, B, N, T, n_fft, hop, pad, 80.0, 0.0, None)


def _rms(a=P, out=P, B=1, N=4000, T=63, frame=512, hop=64, pad=CENTER, db=1):
  return (a, out, B, N, T, frame, hop, pad, db, 80.0, 0.0, None)


_ABI_CASES = [
    ('f-null-audio', _F, _fwd(a=None), E_INVALID, b'loudness_forward: null pointer'),
    ('f-null-weights', _F, _fwd(w=None), E_INVALID, b'loudness_forward: null pointer'),
    ('f-null-out', _F, _fwd(out=None), E_INVALID, b'loudness_forward: null pointer'),
    ('f-B', _F, _fwd(B=-1), E_INVALID, b'loudness_forward: bad shape B=-1 N=4000 T=63 frame=512 hop=64'),
    ('f-N', _F, _fwd(N=0), E_INVALID, b'loudness_forward: bad shape B=1 N=0 T=63 frame=512 hop=64'),
    ('f-hop', _F, _fwd(hop=0), E_INVALID, b'loudness_forward: bad shape B=1 N=4000 T=63 frame=512 hop=0'),
    ('f-padding', _F, _fwd(pad=3), E_INVALID, b'loudness_forward: bad padding 3'),
    ('f-hop-center', _F, _fwd(n_fft=64, hop=96), E_INVALID, b'loudness_forward: frame_size (64) must be greater than hop_size (96)'),
    ('f-hop-same', _F, _fwd(n_fft=64, hop=96, pad=SAME), E_INVALID, b'loudness_forward: frame_size (64) must be greater than hop_size (96)'),
    ('f-T', _F, _fwd(T=62), E_INVALID, b'loudness_forward: n_frames=62, the padding gives 63'),
    ('f-T-same', _F, _fwd(T=62, pad=SAME), E_INVALID, b'loudness_forward: n_frames=62, the padding gives 63'),
    ('f-T-valid', _F, _fwd(pad=VALID), E_INVALID, b'loudness_forward: n_frames=63, the padding gives 55'),
    ('f-pow2', _F, _fwd(n_fft=500), E_INVALID, b'loudness_forward: n_fft (500) must be a power of two'),
    ('f-one', _F, _fwd(n_fft=1, hop=1, T=4000), E_INVALID, b'loudness_forward: n_fft (1) must be a power of two'),
    ('f-max', _F, _fwd(n_fft=32768), E_UNSUPPORTED, b'loudness_forward: n_fft=32768 exceeds the 16384 supported'),
    ('f-B-grid', _F, _fwd(B=65536), E_INVALID, b'loudness_forward: B=65536 exceeds the 65535 grid limit'),
    ('f-B0', _F, _fwd(B=0), 0, None),
    ('f-T0', _F, _fwd(N=300, T=0, pad=VALID), 0, None),
    ('f-T0-no-out', _F, _fwd(out=None, N=300, T=0, pad=VALID), 0, None),
    ('f-valid-hop', _F, _fwd(B=0, n_fft=64, hop=176, N=1000, T=6, pad=VALID), 0, None),
    ('b-null-grad', _B, _bwd(g=None), E_INVALID, b'loudness_backward: null pointer'),
    ('b-null-d', _B, _bwd(d=None), E_INVALID, b'loudness_backward: null pointer'),
    ('b-shape', _B, _bwd(T=-1), E_INVALID, b'loudness_backward: bad shape B=1 N=4000 T=-1 frame=512 hop=64'),
    ('b-T', _B, _bwd(T=64), E_INVALID, b'loudness_backward: n_frames=64, the padding gives 63'),
    ('b-pow2', _B, _bwd(n_fft=768), E_INVALID, b'loudness_backward: n_fft (768) must be a power of two'),
    ('b-max', _B, _bwd(n_fft=32768), E_UNSUPPORTED, b'loudness_backward: n_fft=32768 exceeds the 16384 supported'),
    ('b-B-grid', _B, _bwd(B=70000), E_INVALID, b'loudness_backward: B=70000 exceeds the 65535 grid limit'),
    ('b-B0', _B, _bwd(B=0), 0, None),
    ('r-null', _R, _rms(out=None), E_INVALID, b'rms_power: null pointer'),
    ('r-frame', _R, _rms(frame=0), E_INVALID, b'rms_power: bad shape B=1 N=4000 T=63 frame=0 hop=64'),
    ('r-padding', _R, _rms(pad=-1), E_INVALID, b'rms_power: bad padding -1'),
    ('r-hop', _R, _rms(frame=64, hop=96, pad=SAME), E_INVALID, b'rms_power: frame_size (64) must be greater than hop_size (96)'),
    ('r-T-odd', _R, _rms(frame=1001, T=64), E_INVALID, b'rms_power: n_frames=64, the padding gives 63'),
    ('r-B-grid', _R, _rms(B=65536), E_INVALID, b'rms_power: B=65536 exceeds the 65535 grid limit'),
    ('r-B0', _R, _rms(B=0, frame=1000, T=63), 0, None),
    ('r-T0', _R, _rms(N=100, T=0, pad=VALID), 0, None),
]


@pytest.mark.parametrize('fn,args,want,msg', [c[1:] for c in _ABI_CASES],
                         ids=[c[0] for c in _ABI_CASES])
def test_loudness_abi_check_table(fn, args, want, msg):
  """Every check of the three entry points: the status and the full message come
  back before any CUDA call, and nothing is launched."""
  lib = _lib.load()
  launches = lib.ddsp_b200_launch_count()
  assert getattr(lib, 'ddsp_b200_' + fn)(*args) == want
  assert lib.ddsp_b200_launch_count() == launches
  if msg is not None:
    assert lib.ddsp_b200_last_error() == msg


def test_value_errors_before_device_work(monkeypatch):
  def fail(*a, **k):
    raise AssertionError('device work before the argument checks')
  monkeypatch.setattr(_lib, 'load', fail)
  monkeypatch.setattr(core, 'torch_float32', fail)
  z = np.zeros((2, 4000), np.float32)
  so = spectral_ops
  with pytest.raises(ValueError, match=r"`padding` must be one of"):
    so.compute_loudness(z, padding='reflect')
  with pytest.raises(ValueError, match=r'frame_size \(512\) must be greater than hop_size \(1000\)'):
    so.compute_loudness(z, frame_rate=16, padding='center')
  with pytest.raises(ValueError, match=r'frame_size \(512\) must be greater than hop_size \(1000\)'):
    so.compute_loudness(z, frame_rate=16, padding='same')
  # the reference's pad() checks the hop before the padding name
  with pytest.raises(ValueError, match=r'must be greater than hop_size'):
    so.compute_loudness(z, frame_rate=16, padding='reflect')
  with pytest.raises(ValueError, match=r'n_fft \(1000\) must be a power of two'):
    so.compute_loudness(z, n_fft=1000)
  for bad in (np.zeros((2, 3, 4), np.float32), np.zeros((), np.float32),
              np.zeros((1, 2, 3, 4), np.float32), torch.zeros(2, 0)):
    with pytest.raises(ValueError, match='audio must be'):
      so.compute_loudness(bad)
    with pytest.raises(ValueError, match='audio must be'):
      so.compute_power(bad)
  with pytest.raises(ValueError, match=r'frame_size \(64\) must be greater than hop_size \(96\)'):
    so.compute_power(z, sample_rate=24000, frame_size=64)
  with pytest.raises(ValueError, match=r"`padding` must be one of"):
    so.compute_rms_energy(z, padding='full')


def test_output_lengths_follow_get_framed_lengths():
  """_framing's frame counts are get_framed_lengths' for even frames; 'valid' on audio
  shorter than a frame gives 0 frames (where get_framed_lengths goes negative, as the
  reference's does)."""
  for n in (1, 63, 64, 65, 511, 512, 513, 4000, 4001, 64000):
    for frame, hop in ((512, 64), (2048, 64), (64, 64), (1024, 176), (1000, 100)):
      for padding in ('center', 'same', 'valid'):
        _, _, _, t, _ = spectral_ops._framing(np.zeros((2, n)), frame, hop, padding)
        want, padded = spectral_ops.get_framed_lengths(n, frame, hop, padding)
        assert t == max(0, want), (n, frame, hop, padding)
        assert padded == {'center': n + frame, 'valid': n,
                          'same': (want - 1) * hop + frame}[padding]
  assert spectral_ops.get_framed_lengths(100, 512, 64, 'valid')[0] < 0
  # odd frames under 'center' pad frame // 2 on each side, one less than frame
  _, _, _, t, _ = spectral_ops._framing(np.zeros(4000), 1001, 64, 'center')
  assert t == 1 + (4000 + 1000 - 1001) // 64


def test_stft_step_is_the_hop():
  """compute_loudness hands stft overlap = 1 - hop / n_fft, and stft's step is
  int(n_fft * (1 - overlap)): equal to the hop for every power-of-two n_fft and every
  hop the kernels take (hop <= n_fft)."""
  for log2 in range(1, 15):
    n_fft = 1 << log2
    for hop in sorted({1, 2, 3, 7, 64, 96, 147, 176, 192, 441, n_fft // 2, n_fft - 1, n_fft}):
      if 1 <= hop <= n_fft:
        assert int(n_fft * (1.0 - (1.0 - hop / n_fft))) == hop, (n_fft, hop)


def test_spectral_loss_takes_a_loudness_weight():
  loss = losses.SpectralLoss(loudness_weight=1.0)
  assert loss.loudness_weight == 1.0


def test_restatement_matches_the_reference():
  """tests/loudness_ref.py against the unmodified reference run wide on the shim, at
  <= 1e-10 dB, over every padding, rate, n_fft and frame size of the fixture."""
  want = np.load(mg.PATH)
  for i, (sr, n_fft, padding, _, _) in enumerate(mg.LOUD):
    got = ref.compute_loudness(torch.from_numpy(mg.loud_input(i)), sample_rate=sr,
                               n_fft=n_fft, padding=padding).numpy()
    w = want['loudness_%02d' % i]
    assert got.shape == w.shape and np.abs(got - w).max() <= 1e-10, mg.LOUD[i]
  for i, (sr, frame, padding, _, _) in enumerate(mg.POWER):
    got = ref.compute_power(torch.from_numpy(mg.power_input(i)), sample_rate=sr,
                            frame_size=frame, padding=padding).numpy()
    w = want['power_%02d' % i]
    assert got.shape == w.shape and np.abs(got - w).max() <= 1e-10, mg.POWER[i]


def test_restated_loss_matches_the_reference():
  from tests import grad_ref
  target, audio = (torch.from_numpy(v).double() for v in mg.loss_inputs())
  got = grad_ref.spectral_loss(target, audio, mag_weight=1.0, logmag_weight=1.0) + (
      ref.compute_loudness(target, n_fft=2048) - ref.compute_loudness(audio, n_fft=2048)
  ).abs().mean()
  want = float(np.load(mg.PATH)['spectral_loss'])
  assert abs(float(got) - want) <= 1e-10 * want


def test_fixture_regenerates():
  """Where the reference is checked out, the fixture is what it computes."""
  from oracle import ref_on_shim
  try:
    ref_on_shim.load()
  except Exception as e:  # pylint: disable=broad-except
    pytest.skip('reference sources not available: %s' % e)
  from tests.golden.make_golden import compare
  compare('loudness', mg.loudness(), np.load(mg.PATH))


# ---- GPU ----------------------------------------------------------------------
def _wide(audio, **kw):
  return ref.compute_loudness(torch.as_tensor(audio).double().cpu(), **kw).numpy()


def _assert_db_close(got, want, range_db=80.0, tol=TOL_DB):
  got = np.asarray(got, np.float64)
  assert got.shape == want.shape, (got.shape, want.shape)
  err = np.abs(got - want)
  assert err.max() <= tol, (err.max(), np.unravel_index(err.argmax(), err.shape))


@pytest.mark.gpu
@pytest.mark.parametrize('i', range(len(mg.LOUD)), ids=[str(c) for c in mg.LOUD])
def test_forward_matches_the_fixture(i):
  sr, n_fft, padding, _, _ = mg.LOUD[i]
  got = spectral_ops.compute_loudness(mg.loud_input(i), sample_rate=sr, n_fft=n_fft,
                                      padding=padding)
  _assert_db_close(got.cpu().numpy(), np.load(mg.PATH)['loudness_%02d' % i])


def _signals(n, sr, seed):
  """[rows, n] float32: white noise at four levels, 20 Hz and 2.5 kHz tones,
  silence, a row fading from silence to full scale (it crosses both clamps), and a
  noise burst between silent stretches."""
  rng = np.random.default_rng(seed)
  t = np.arange(n) / sr
  rows = [rng.uniform(-1, 1, n) * lvl for lvl in (1.0, 0.1, 1e-3, 3e-5)]
  rows += [0.5 * np.sin(2 * np.pi * 20.0 * t), 0.5 * np.sin(2 * np.pi * 2500.0 * t + 0.3),
           np.zeros(n), rng.uniform(-1, 1, n) * np.logspace(-7, 0, n)]
  burst = np.zeros(n)
  burst[n // 3: 2 * n // 3] = rng.standard_normal(2 * n // 3 - n // 3)
  rows.append(burst)
  return np.stack(rows).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize('sr,n_fft,padding,range_db,ref_db', [
    (16000, 2048, 'center', 80.0, 0.0), (16000, 512, 'center', 80.0, 0.0),
    (16000, 512, 'same', 60.0, 20.0), (44100, 1024, 'valid', 100.0, -20.0),
    (48000, 4096, 'center', 80.0, 10.0), (16000, 64, 'same', 40.0, 0.0)])
def test_forward_signals_match_float64(sr, n_fft, padding, range_db, ref_db):
  x = _signals(12000, sr, seed=n_fft)
  kw = dict(sample_rate=sr, n_fft=n_fft, padding=padding, range_db=range_db,
            ref_db=ref_db)
  got = spectral_ops.compute_loudness(x, **kw).cpu().numpy()
  want = _wide(x, **kw)
  _assert_db_close(got, want)
  assert got.min() >= np.float32(-range_db)
  if ref_db >= 0:   # below 0, ref_db lifts the silent floor above -range_db
    assert (got[6] == np.float32(-range_db)).all()
  if n_fft >= 2048:
    # the tones: the A-weighting peak is ~50 dB above 20 Hz (shorter windows leak
    # the 20 Hz tone into better-weighted bins)
    assert np.median(got[5]) - np.median(got[4]) > 40.0


@pytest.mark.gpu
@pytest.mark.parametrize('n_fft', [2 ** k for k in range(1, 15)])
def test_every_supported_n_fft(n_fft):
  """Every power of two from 2 to the 16384 cap, forward and backward, on noise, a
  tone and silence (hop n_fft / 8 above 2048 keeps the float64 reference small)."""
  hop = min(n_fft, 64) if n_fft <= 2048 else n_fft // 8
  sr = hop * 250
  n = max(3 * n_fft, 2000)
  x = _signals(n, sr, seed=7)[[0, 2, 5, 6]]
  got = spectral_ops.compute_loudness(x, sample_rate=sr, n_fft=n_fft)
  _assert_db_close(got.cpu().numpy(), _wide(x, sample_rate=sr, n_fft=n_fft))
  _check_grad(x, dict(sample_rate=sr, n_fft=n_fft), seed=n_fft)


@pytest.mark.gpu
def test_above_the_cap_is_not_implemented():
  with pytest.raises(NotImplementedError, match='n_fft=32768 exceeds the 16384 supported'):
    spectral_ops.compute_loudness(np.zeros((1, 40000), np.float32), n_fft=32768)


@pytest.mark.gpu
def test_shapes_and_use_tf():
  x = _signals(4000, 16000, 3)
  l2 = spectral_ops.compute_loudness(x)
  l1 = spectral_ops.compute_loudness(x[0])
  l3 = spectral_ops.compute_loudness(x[:, :, None])
  assert l2.shape == (x.shape[0], 63) and l1.shape == (63,) and l3.shape == l2.shape
  assert torch.equal(l1, l2[0]) and torch.equal(l3, l2)
  npy = spectral_ops.compute_loudness(x, use_tf=False)
  assert isinstance(npy, np.ndarray) and np.array_equal(npy, l2.cpu().numpy())
  a = torch.from_numpy(x[:, :300]).to(DEV).requires_grad_(True)
  v = spectral_ops.compute_loudness(a, padding='valid')
  assert v.shape == (x.shape[0], 0)
  v.sum().backward()
  assert torch.equal(a.grad, torch.zeros_like(a))
  assert spectral_ops.compute_power(x[:, :300], padding='valid').shape == (x.shape[0], 0)


def _check_grad(x, kw, seed, tol=(1e-4, 2e-5)):
  """d audio of sum(g * loudness) against float64 autograd of the restatement."""
  x = np.asarray(x, np.float32)
  a = torch.from_numpy(x).to(DEV).requires_grad_(True)
  out = spectral_ops.compute_loudness(a, **kw)
  g = torch.randn(out.shape, generator=torch.Generator().manual_seed(seed)).to(DEV)
  out.backward(g)
  b = torch.from_numpy(x).double().requires_grad_(True)
  want = ref.compute_loudness(b, **kw)
  want.backward(g.double().cpu())
  got, w = a.grad.double().cpu(), b.grad
  peak = w.abs().max()
  if peak == 0:
    assert torch.equal(got, torch.zeros_like(got))
    return
  emax = float((got - w).abs().max() / peak)
  el2 = float((got - w).norm() / w.norm())
  assert emax <= tol[0] and el2 <= tol[1], (emax, el2)


@pytest.mark.gpu
@pytest.mark.parametrize('sr,n_fft,padding,range_db,ref_db,n', [
    (16000, 2048, 'center', 80.0, 0.0, 12000), (16000, 512, 'center', 80.0, 0.0, 6001),
    (16000, 512, 'same', 60.0, 20.0, 6000), (24000, 1024, 'valid', 80.0, -20.0, 7000),
    (44100, 64, 'valid', 80.0, 0.0, 3000), (48000, 256, 'same', 80.0, 0.0, 5000),
    (16000, 8192, 'center', 80.0, 0.0, 20000)])
def test_gradient_matches_float64_autograd(sr, n_fft, padding, range_db, ref_db, n):
  """Random upstream gradients over noise, tones, silence and rows that cross the
  clamps (ref_db moves the -range_db clamp away from the pmin clamp); 44.1 kHz with
  n_fft = 64 under 'valid' has hop 176 > n_fft, so samples between frames get 0."""
  x = _signals(n, sr, seed=n)
  _check_grad(x, dict(sample_rate=sr, n_fft=n_fft, padding=padding, range_db=range_db,
                      ref_db=ref_db), seed=n_fft)


@pytest.mark.gpu
def test_silence_gives_minus_range_and_zero_gradient():
  a = torch.zeros((2, 8000), device=DEV, requires_grad=True)
  out = spectral_ops.compute_loudness(a, n_fft=2048, range_db=70.0)
  assert torch.equal(out, torch.full_like(out, -70.0))
  out.backward(torch.randn_like(out))
  assert torch.equal(a.grad, torch.zeros_like(a.grad))


def _loss_ref(target, audio, loss_type, fft_sizes):
  from tests import grad_ref
  t, v = target.double(), audio.double()
  if loss_type == 'L1':
    spec = grad_ref.spectral_loss(t, v, fft_sizes, mag_weight=1.0, logmag_weight=0.0)
    d = lambda a, b: (a - b).abs().mean()  # noqa: E731
  else:
    spec = 0.0
    for size in fft_sizes:
      mt = torch.fft.rfft(grad_ref.stft_frames(t, size), dim=-1).abs()
      mv = torch.fft.rfft(grad_ref.stft_frames(v, size), dim=-1).abs()
      spec = spec + ((mt - mv) ** 2).mean()
    d = lambda a, b: ((a - b) ** 2).mean()  # noqa: E731
  return spec + 0.5 * d(ref.compute_loudness(t, n_fft=2048),
                        ref.compute_loudness(v, n_fft=2048))


@pytest.mark.gpu
@pytest.mark.parametrize('loss_type,fused', [('L1', True), ('L1', False), ('L2', False)])
def test_spectral_loss_with_loudness(loss_type, fused):
  """SpectralLoss(mag, loudness) on the fused kernels (CUDA, L1) and on the torch path
  (weights given, or L2): value and d audio against float64."""
  fft_sizes = (2048, 512, 128)
  gen = torch.Generator().manual_seed(5)
  target = (torch.rand((2, 8000), generator=gen) * 2 - 1) * 0.5
  audio = (0.7 * target + 0.05 * torch.randn((2, 8000), generator=gen)).float()
  loss_obj = losses.SpectralLoss(fft_sizes=fft_sizes, loss_type=loss_type, mag_weight=1.0,
                                 loudness_weight=0.5)
  a = audio.to(DEV).requires_grad_(True)
  t = target.to(DEV)
  weights = None if fused or loss_type == 'L2' else 1.0
  assert loss_obj._fusable(t, a, weights) == fused
  loss = loss_obj(t, a, weights=weights)
  loss.backward()
  b = audio.double().requires_grad_(True)
  want = _loss_ref(target, b, loss_type, fft_sizes)
  want.backward()
  lv, rv = float(loss.detach()), float(want.detach())
  assert abs(lv - rv) <= 1e-4 * rv, (lv, rv)
  emax = float((a.grad.double().cpu() - b.grad).abs().max() / b.grad.abs().max())
  assert emax <= 2e-3, emax


@pytest.mark.gpu
def test_loudness_only_loss_matches_the_fixture():
  target, audio = mg.loss_inputs()
  loss = losses.SpectralLoss(mag_weight=1.0, logmag_weight=1.0, loudness_weight=1.0)
  got = float(loss(torch.from_numpy(target).to(DEV), torch.from_numpy(audio).to(DEV)))
  want = float(np.load(mg.PATH)['spectral_loss'])
  assert abs(got - want) <= 1e-4 * want, (got, want)


@pytest.mark.gpu
def test_decoder_to_loudness_loss_chain():
  """Harmonic synthesis -> SpectralLoss(mag, logmag, loudness) trains: the gradient
  w.r.t. amplitudes and harmonic distribution is the library's spectral-only gradient
  plus the float64 loudness term's gradient through the float64 synthesis."""
  from ddsp_b200 import autograd as ag
  from tests import grad_ref
  from tests.util import synth_inputs
  B, F, K, N = 2, 50, 20, 3200
  inp = synth_inputs(B, F, K, 65, N, seed=4)
  f0 = torch.from_numpy(inp['f0_hz']).to(DEV)
  gen = torch.Generator().manual_seed(2)
  amp = (torch.rand((B, F, 1), generator=gen) + 0.2).to(DEV)
  hd = torch.rand((B, F, K), generator=gen).to(DEV)
  hd = hd / hd.sum(-1, keepdim=True)
  target = (torch.randn((B, N), generator=gen) * 0.1).to(DEV)
  sizes = (1024, 256, 64)

  def grads(loudness_weight):
    x = [amp.clone().requires_grad_(True), hd.clone().requires_grad_(True)]
    audio = ag.HarmonicSynthesisFn.apply(f0, x[0], x[1], N, 16000, 'window')
    loss = losses.SpectralLoss(fft_sizes=sizes, mag_weight=1.0, logmag_weight=1.0,
                               loudness_weight=loudness_weight)(target, audio)
    loss.backward()
    return float(loss), [v.grad.double().cpu() for v in x]

  l_full, g_full = grads(1.0)
  l_spec, g_spec = grads(0.0)
  y = [amp.double().cpu().requires_grad_(True), hd.double().cpu().requires_grad_(True)]
  audio64 = grad_ref.harmonic(f0.double().cpu(), y[0], y[1], N)
  loud = (ref.compute_loudness(target.double().cpu(), n_fft=2048) -
          ref.compute_loudness(audio64, n_fft=2048)).abs().mean()
  loud.backward()
  assert abs((l_full - l_spec) - float(loud)) <= 1e-4 * float(loud) + 1e-5
  for got, spec, want in zip(g_full, g_spec, [v.grad for v in y]):
    err = float((got - spec - want).abs().max() / want.abs().max())
    assert err <= 2e-3, err


@pytest.mark.gpu
def test_full_size_bit_reproducible():
  """B = 128, N = 64000, n_fft = 2048: two forwards and two backwards are
  bit-identical (no atomics; every d-audio sample sums its frames in order)."""
  gen = torch.Generator(DEV).manual_seed(3)
  x = torch.rand((128, 64000), device=DEV, generator=gen) * 2 - 1
  x[:4, 20000:30000] = 0.0
  g = torch.randn((128, 1001), device=DEV, generator=gen)
  runs = []
  for _ in range(2):
    a = x.clone().requires_grad_(True)
    out = spectral_ops.compute_loudness(a, n_fft=2048)
    out.backward(g)
    runs.append((out.detach(), a.grad))
  assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
  # and the values are right at that size
  rows = [0, 1, 77]
  _assert_db_close(runs[0][0][rows].cpu().numpy(), _wide(x[rows], n_fft=2048))


@pytest.mark.gpu
def test_cuda_graph_capture_equals_eager():
  """A training step of the loss with a loudness term has no host synchronisation:
  it captures in a CUDA graph, and the replay equals eager."""
  gen = torch.Generator(DEV).manual_seed(8)
  target = torch.rand((4, 16000), device=DEV, generator=gen) * 2 - 1
  audio = torch.rand((4, 16000), device=DEV, generator=gen) * 2 - 1
  loss_obj = losses.SpectralLoss(mag_weight=1.0, logmag_weight=1.0, loudness_weight=1.0)
  a = audio.clone().requires_grad_(True)

  def step():
    a.grad = None
    loss = loss_obj(target, a)
    loss.backward()
    return loss

  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    for _ in range(2):
      eager = step().detach().clone()
      eager_grad = a.grad.clone()
  torch.cuda.current_stream().wait_stream(s)
  graph = torch.cuda.CUDAGraph()
  a.grad = None
  with torch.cuda.graph(graph):
    static_loss = loss_obj(target, a)
    static_loss.backward()
  graph.replay()
  torch.cuda.synchronize()
  # the spectral terms sum in double atomics, so the loss may differ in its last bit
  assert torch.allclose(static_loss, eager, rtol=1e-6, atol=0.0)
  assert torch.equal(a.grad, eager_grad)


@pytest.mark.gpu
@pytest.mark.parametrize('i', range(len(mg.POWER)), ids=[str(c) for c in mg.POWER])
def test_power_matches_the_fixture(i):
  sr, frame, padding, _, _ = mg.POWER[i]
  got = spectral_ops.compute_power(mg.power_input(i), sample_rate=sr, frame_size=frame,
                                   padding=padding)
  _assert_db_close(got.cpu().numpy(), np.load(mg.PATH)['power_%02d' % i])


@pytest.mark.gpu
@pytest.mark.parametrize('sr,frame,padding,range_db,ref_db', [
    (16000, 64, 'center', 80.0, 0.0), (16000, 1024, 'same', 60.0, 20.0),
    (44100, 1000, 'valid', 80.0, -10.0), (48000, 1001, 'center', 80.0, 0.0),
    (16000, 1, 'valid', 80.0, 0.0), (16000, 4096, 'center', 120.0, 0.0)])
def test_power_and_rms_match_float64(sr, frame, padding, range_db, ref_db):
  x = _signals(9000, sr, seed=frame)
  got = spectral_ops.compute_power(x, sample_rate=sr, frame_size=frame, padding=padding,
                                   range_db=range_db, ref_db=ref_db).cpu().numpy()
  want = ref.compute_power(torch.from_numpy(x), sample_rate=sr, frame_size=frame,
                           padding=padding, range_db=range_db, ref_db=ref_db).numpy()
  _assert_db_close(got, want)
  rms = spectral_ops.compute_rms_energy(x, sample_rate=sr, frame_size=frame,
                                        padding=padding).cpu().numpy()
  fr = ref.frames(torch.from_numpy(x).double(), frame, sr // 250, padding)
  want_rms = (fr ** 2).mean(-1).sqrt().numpy()
  assert rms.shape == want_rms.shape
  assert np.abs(rms - want_rms).max() <= 1e-5 * max(1e-30, np.abs(want_rms).max())


@pytest.mark.gpu
def test_power_refuses_grad():
  a = torch.zeros((1, 4000), device=DEV, requires_grad=True)
  with pytest.raises(RuntimeError, match='compute_power'):
    spectral_ops.compute_power(a)
  with pytest.raises(RuntimeError, match='compute_rms_energy'):
    spectral_ops.compute_rms_energy(a)
  with torch.no_grad():
    assert spectral_ops.compute_power(a).shape == (1, 63)
