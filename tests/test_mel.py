"""Mel, log-mel and MFCC features (csrc/mel.cuh, spectral_ops.compute_mel /
compute_logmel / compute_mfcc) and compute_logmag: argument checks and the float64
restatement on the CPU; forward, gradients, reproducibility and CUDA-graph capture on
the GPU.  Reference: tests/mel_ref.py, pinned to the unmodified reference by
tests/golden/mel.npz.

Forward tolerance.  The kernel frames, windows and transforms in float32.  A radix-2
FFT of M = L / 2 points has log2(M) rounding stages, and the split step and the
magnitude add about three more, so every bin carries an absolute error of about
e_L = (log2 L + 3) 2^-24 times the frame's peak magnitude max_k |X_k|, whatever its own
size.  Band j sums W_kj |X_k|, so its error is at most e_L max|X| sum_k W_kj (the
summation's own rounding, relative 2^-24 per term, is below that).  The mel domain is
therefore compared against 4 e_L max|X| sum_k W_kj, everywhere.  The log turns that
into e_L max|X| sum_k W_kj / mel_j: for broadband input mel_j is of order
max|X| sum_k W_kj / 10, so log-mel is good to ~1e-5 and 2e-4 absolute leaves a
margin for bands of one or two bins whose magnitudes happen to be small.  The MFCC's
DCT rows have an l2 norm of sqrt(2), so the same 2e-4 holds there, plus the DCT's own
float32 sum of `bins` terms, allowed 1e-5 of the coefficient (c0 is the largest: -184
for a silent frame at 128 bins, where one float32 ulp is 1.5e-5).  For tones,
bands far from the tone hold only leakage and the FFT's floor, so log-mel is not
meaningful there; tones are compared in the mel domain only.  Silent and padded
frames are exact: mel == 0 and log-mel == float32(log 1e-5)."""
import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, core, spectral_ops
from tests import mel_ref as ref
from tests.golden import make_mel_golden as mg

P = 0x1000        # a device pointer the library never dereferences on the host
E_INVALID, E_UNSUPPORTED = _lib.E_INVALID, _lib.E_UNSUPPORTED
MEL, LOGMEL, MFCC = _lib.MEL, _lib.LOGMEL, _lib.MFCC
DEV = 'cuda'
TOL_LOG = 2e-4
LOG_EPS = np.float32(np.log(1e-5))

_F, _B = 'mel_forward', 'mel_backward'


def _fwd(a=P, w=P, tab=P, out=P, B=1, N=8000, T=16, fft=1024, L=1024, hop=512, pad=1,
         bins=128, n_out=30, mode=MFCC):
  return (a, w, tab, out, B, N, T, fft, L, hop, pad, bins, n_out, mode, None)


def _bwd(a=P, w=P, tab=P, g=P, d=P, B=1, N=8000, T=16, fft=1024, L=1024, hop=512, pad=1,
         bins=128, n_out=30, mode=MFCC):
  return (a, w, tab, g, d, B, N, T, fft, L, hop, pad, bins, n_out, mode, None)


_ABI_CASES = [
    ('f-null-audio', _F, _fwd(a=None), E_INVALID, b'mel_forward: null pointer'),
    ('f-null-window', _F, _fwd(w=None), E_INVALID, b'mel_forward: null pointer'),
    ('f-null-table', _F, _fwd(tab=None), E_INVALID, b'mel_forward: null pointer'),
    ('f-null-out', _F, _fwd(out=None), E_INVALID, b'mel_forward: null pointer'),
    ('f-B', _F, _fwd(B=-1), E_INVALID, b'mel_forward: bad shape B=-1 N=8000 T=16 fft_size=1024 hop=512'),
    ('f-N', _F, _fwd(N=0), E_INVALID, b'mel_forward: bad shape B=1 N=0 T=16 fft_size=1024 hop=512'),
    ('f-fft', _F, _fwd(fft=0), E_INVALID, b'mel_forward: bad shape B=1 N=8000 T=16 fft_size=0 hop=512'),
    ('f-hop', _F, _fwd(hop=0), E_INVALID, b'mel_forward: bad shape B=1 N=8000 T=16 fft_size=1024 hop=0'),
    ('f-pad', _F, _fwd(pad=2), E_INVALID, b'mel_forward: bad pad_end 2'),
    ('f-mode', _F, _fwd(mode=3), E_INVALID, b'mel_forward: bad mode 3'),
    ('f-bins', _F, _fwd(bins=0, n_out=0), E_INVALID, b'mel_forward: bad bins=0 n_out=0 for mode 2'),
    ('f-n-out', _F, _fwd(n_out=129), E_INVALID, b'mel_forward: bad bins=128 n_out=129 for mode 2'),
    ('f-n-out-neg', _F, _fwd(n_out=-1), E_INVALID, b'mel_forward: bad bins=128 n_out=-1 for mode 2'),
    ('f-n-out-mel', _F, _fwd(mode=MEL), E_INVALID, b'mel_forward: bad bins=128 n_out=30 for mode 0'),
    ('f-pow2', _F, _fwd(L=1000), E_INVALID, b'mel_forward: fft_length (1000) must be a power of two'),
    ('f-L0', _F, _fwd(L=0), E_INVALID, b'mel_forward: fft_length (0) must be a power of two'),
    ('f-max', _F, _fwd(fft=20000, L=32768, hop=10000, T=1), E_UNSUPPORTED, b'mel_forward: fft_length=32768 is outside the 2..16384 supported'),
    ('f-one', _F, _fwd(fft=1, L=1, hop=1, T=8000), E_UNSUPPORTED, b'mel_forward: fft_length=1 is outside the 2..16384 supported'),
    ('f-crop', _F, _fwd(fft=1024, L=512), E_INVALID, b'mel_forward: fft_size (1024) exceeds fft_length (512)'),
    ('f-bins-max', _F, _fwd(bins=1025, n_out=1025, mode=LOGMEL), E_UNSUPPORTED, b'mel_forward: bins=1025 exceeds the 1024 supported'),
    ('f-T', _F, _fwd(T=15), E_INVALID, b'mel_forward: n_frames=15, the padding gives 16'),
    ('f-T-valid', _F, _fwd(pad=0), E_INVALID, b'mel_forward: n_frames=16, the padding gives 14'),
    ('f-T-short', _F, _fwd(N=1000, pad=0, T=1), E_INVALID, b'mel_forward: n_frames=1, the padding gives 0'),
    ('f-B-grid', _F, _fwd(B=65536), E_INVALID, b'mel_forward: B=65536 exceeds the 65535 grid limit'),
    ('f-B0', _F, _fwd(B=0), 0, None),
    ('f-T0', _F, _fwd(N=1000, pad=0, T=0), 0, None),
    ('f-T0-no-out', _F, _fwd(out=None, N=1000, pad=0, T=0), 0, None),
    ('f-C0', _F, _fwd(out=None, n_out=0), 0, None),
    ('f-bins-1024', _F, _fwd(B=0, fft=16384, L=16384, hop=4096, T=2, bins=1024, n_out=1024), 0, None),
    ('f-step-gt-fft', _F, _fwd(B=0, fft=64, L=64, hop=96, T=84), 0, None),
    ('f-L-above', _F, _fwd(B=0, fft=1000, L=2048, hop=500, T=16), 0, None),
    ('b-null-grad', _B, _bwd(g=None), E_INVALID, b'mel_backward: null pointer'),
    ('b-null-d', _B, _bwd(d=None), E_INVALID, b'mel_backward: null pointer'),
    ('b-null-table', _B, _bwd(tab=None), E_INVALID, b'mel_backward: null pointer'),
    ('b-shape', _B, _bwd(T=-1), E_INVALID, b'mel_backward: bad shape B=1 N=8000 T=-1 fft_size=1024 hop=512'),
    ('b-mode', _B, _bwd(mode=-1), E_INVALID, b'mel_backward: bad mode -1'),
    ('b-T', _B, _bwd(T=17), E_INVALID, b'mel_backward: n_frames=17, the padding gives 16'),
    ('b-pow2', _B, _bwd(L=768, fft=768, hop=384, T=21), E_INVALID, b'mel_backward: fft_length (768) must be a power of two'),
    ('b-max', _B, _bwd(fft=16385, L=32768, hop=8192, T=1), E_UNSUPPORTED, b'mel_backward: fft_length=32768 is outside the 2..16384 supported'),
    ('b-bins-max', _B, _bwd(bins=2048, n_out=13), E_UNSUPPORTED, b'mel_backward: bins=2048 exceeds the 1024 supported'),
    ('b-B-grid', _B, _bwd(B=70000), E_INVALID, b'mel_backward: B=70000 exceeds the 65535 grid limit'),
    ('b-B0', _B, _bwd(B=0), 0, None),
    ('b-T0', _B, _bwd(N=1000, pad=0, T=0, g=None), 0, None),
]


@pytest.mark.parametrize('fn,args,want,msg', [c[1:] for c in _ABI_CASES],
                         ids=[c[0] for c in _ABI_CASES])
def test_mel_abi_check_table(fn, args, want, msg):
  """Every check of the two entry points: the status and the full message come back
  before any CUDA call, and nothing is launched."""
  lib = _lib.load()
  launches = lib.ddsp_b200_launch_count()
  assert getattr(lib, 'ddsp_b200_' + fn)(*args) == want
  assert lib.ddsp_b200_launch_count() == launches
  if msg is not None:
    assert lib.ddsp_b200_last_error() == msg


def test_errors_before_device_work(monkeypatch):
  def fail(*a, **k):
    raise AssertionError('device work before the argument checks')
  monkeypatch.setattr(_lib, 'load', fail)
  monkeypatch.setattr(core, 'torch_float32', fail)
  z = np.zeros((2, 4000), np.float32)
  so = spectral_ops
  cases = [
      (ValueError, r'num_mel_bins must be positive. Got: 0', lambda: so.compute_mel(z, bins=0)),
      (ValueError, r'num_mel_bins must be positive. Got: -3',
       lambda: so.compute_mfcc(z, mel_bins=-3)),
      (ValueError, r'lower_edge_hertz must be non-negative. Got: -1.0',
       lambda: so.compute_logmel(z, lo_hz=-1.0)),
      (ValueError, r'lower_edge_hertz 8000.0 >= upper_edge_hertz 8000.0',
       lambda: so.compute_mel(z, lo_hz=8000.0)),
      (ValueError, r'sample_rate must be positive. Got: 0',
       lambda: so.compute_mel(z, sample_rate=0)),
      (ValueError, r'upper_edge_hertz must not be larger than the Nyquist frequency '
                   r'\(sample_rate / 2\). Got 8000.5 for sample_rate: 16000',
       lambda: so.compute_mfcc(z, hi_hz=8000.5)),
      (ValueError, 'audio must be', lambda: so.compute_mel(np.zeros((2, 3, 4), np.float32))),
      (ValueError, 'audio must be', lambda: so.compute_mfcc(torch.zeros(2, 0))),
      (ValueError, 'audio must be', lambda: so.compute_logmel(np.zeros((), np.float32))),
      (ValueError, 'frame_step', lambda: so.compute_mel(z, overlap=1.0)),
      (ValueError, 'fft_size must be positive', lambda: so.compute_mel(z, fft_size=0)),
      (NotImplementedError, r'compute_mel: fft_size=20000 gives fft_length=32768, outside '
                            r'the 2..16384 supported',
       lambda: so.compute_mel(z, fft_size=20000)),
      (NotImplementedError, r'compute_mfcc: fft_size=1 gives fft_length=1',
       lambda: so.compute_mfcc(z, fft_size=1, overlap=0.0)),
      (NotImplementedError, r'compute_logmel: bins=1025 exceeds the 1024 supported',
       lambda: so.compute_logmel(z, bins=1025)),
  ]
  for exc, msg, call in cases:
    with pytest.raises(exc, match=msg):
      call()


def test_output_shapes_follow_the_reference(monkeypatch):
  """Frame counts and column counts (mfcc_bins with Python's slice rules) of every
  fixture case, with the kernel replaced by a stand-in that returns its shape."""
  def fake(x, window, table, meta):
    t, _, fft_length, _, _, bins, n_out, _ = meta
    assert window.shape == (meta[1],)
    assert table.shape == (3 * (fft_length // 2 + 1) + 2 * bins,)
    return torch.zeros((x.shape[0], t, n_out))
  monkeypatch.setattr(spectral_ops.MelFn, 'apply', fake)
  monkeypatch.setattr(spectral_ops, '_audio_2d',
                      lambda a, b, n: torch.as_tensor(np.asarray(a)).reshape(b, n))
  want = np.load(mg.PATH)
  for i, (fn, _, _, kw) in enumerate(mg.CASES):
    if fn == 'compute_logmag':
      continue
    got = getattr(spectral_ops, fn)(mg.mel_input(i), **kw)
    assert tuple(got.shape) == want['%s_%02d' % (fn, i)].shape, mg.CASES[i]


def test_restatement_matches_the_reference():
  """tests/mel_ref.py against the unmodified reference run wide on the shim, at
  <= 1e-10, over every case of the fixture."""
  want = np.load(mg.PATH)
  for i, (fn, _, _, kw) in enumerate(mg.CASES):
    got = getattr(ref, fn)(torch.from_numpy(mg.mel_input(i)), **kw).numpy()
    w = want['%s_%02d' % (fn, i)]
    assert got.shape == w.shape, mg.CASES[i]
    assert w.size == 0 or np.abs(got - w).max() <= 1e-10, mg.CASES[i]


def test_fixture_regenerates():
  """Where the reference is checked out, the fixture is what it computes."""
  from oracle import ref_on_shim
  try:
    ref_on_shim.load()
  except Exception as e:  # pylint: disable=broad-except
    pytest.skip('reference sources not available: %s' % e)
  from tests.golden.make_golden import compare
  compare('mel', mg.mel(), np.load(mg.PATH))


def test_dct_matches_scipy():
  import scipy.fft
  rng = np.random.default_rng(0)
  for bins in (1, 2, 13, 64, 128, 229):
    x = rng.standard_normal((5, bins))
    want = scipy.fft.dct(x, type=2, axis=-1) / np.sqrt(2.0 * bins)
    got = ref.mfccs_from_log_mel_spectrograms(torch.from_numpy(x)).numpy()
    assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())
    assert np.abs(ref.mfccs_from_log_mel_spectrograms(x) - want).max() <= 1e-12 * max(
        1.0, np.abs(want).max())


@pytest.mark.parametrize('bins,k,sr,lo,hi', [
    (64, 1025, 16000, 0.0, 8000.0), (128, 513, 16000, 20.0, 8000.0),
    (229, 1025, 16000, 0.0, 8000.0), (1, 33, 48000, 100.0, 24000.0),
    (128, 33, 16000, 0.0, 8000.0), (80, 1025, 22050, 80.0, 7600.0)])
def test_mel_matrix_properties(bins, k, sr, lo, hi):
  """The restated W: DC row zero, at most two nonzeros per row in adjacent bands,
  rising + falling weights summing to 1 strictly inside (lo, hi) wherever two bands
  meet, nothing outside [lo, hi]; and the library's sparse table is the same W."""
  w = ref.linear_to_mel_weight_matrix(bins, k, sr, lo, hi)
  assert w.shape == (k, bins) and (w[0] == 0).all() and (w >= 0).all()
  f = np.linspace(0.0, sr / 2.0, k)
  nz = w != 0
  assert (nz.sum(1) <= 2).all()
  for row in np.flatnonzero(nz.sum(1) == 2):
    a, b = np.flatnonzero(nz[row])
    assert b == a + 1
  m = ref.hertz_to_mel(f)
  edges = np.linspace(ref.hertz_to_mel(lo), ref.hertz_to_mel(hi), bins + 2)
  inner = (m > edges[1]) & (m < edges[-2])
  inner[0] = False
  assert not inner.any() or np.abs(w[inner].sum(1) - 1.0).max() <= 1e-12
  outside = (f <= lo) | (f >= hi)
  assert (w[outside] == 0).all()
  # the kernel's sparse form holds the same weights (as float32)
  words = spectral_ops.mel_table(bins, k, sr, lo, hi, 'cpu').numpy()
  pair = words[:2 * k].view(np.float32).reshape(k, 2).astype(np.float64)
  band = words[2 * k:3 * k]
  blo, bhi = words[3 * k:3 * k + bins], words[3 * k + bins:]
  dense = np.zeros((k, bins))
  for j in range(bins):
    for kk in range(blo[j], bhi[j]):
      assert band[kk] in (j - 1, j)
      dense[kk, j] = pair[kk, 0] if band[kk] == j else pair[kk, 1]
  assert np.abs(dense - w.astype(np.float32)).max() == 0.0
  for kk in range(k):    # the transpose view: every weight of the row, once
    row = np.zeros(bins)
    if band[kk] >= 0:
      row[band[kk]] += pair[kk, 0]
    if 0 <= band[kk] + 1 < bins:
      row[band[kk] + 1] += pair[kk, 1]
    assert np.array_equal(row, w[kk].astype(np.float32).astype(np.float64))
  assert np.allclose(spectral_ops.linear_to_mel_weight_matrix(bins, k, sr, lo, hi), w,
                     rtol=0, atol=0)


# ---- GPU ----------------------------------------------------------------------
def _kw_mel(fn, kw):
  """(fft_size, overlap, pad_end, bins, sample_rate, lo, hi) of a call's arguments."""
  import inspect
  sig = inspect.signature(getattr(ref, fn))
  a = {k: v.default for k, v in sig.parameters.items() if k != 'audio'}
  a.update(kw)
  bins = a.get('bins', a.get('mel_bins'))
  return a['fft_size'], a['overlap'], a['pad_end'], bins, a['sample_rate'], a['lo_hz'], \
      a['hi_hz']


def _mel_bound(x, fn, kw):
  """4 e_L max_k|X_k| sum_k W_kj per [.., T, bins]: the float32 FFT's error in mel."""
  fft_size, overlap, pad_end, bins, sr, lo, hi = _kw_mel(fn, kw)
  spec = ref.stft(torch.as_tensor(np.asarray(x)), fft_size, overlap, pad_end).abs()
  L = 1 << (int(fft_size) - 1).bit_length()
  w = ref.linear_to_mel_weight_matrix(bins, L // 2 + 1, sr, lo, hi)
  e = (np.log2(L) + 3) * 2.0 ** -24
  peak = spec.amax(-1, keepdim=True).numpy() if spec.shape[-2] else np.zeros(
      spec.shape[:-1] + (1,))
  return 4 * e * peak * w.sum(0)


def _mfcc_slack(fn, want):
  """The DCT's float32 sum of `bins` terms: 1e-5 of the coefficient (c0 of a silent
  frame is -184 at 128 bins, where a float32 ulp is 1.5e-5)."""
  return 1e-5 * np.abs(want) if fn == 'compute_mfcc' else 0.0


def _check_forward(x, fn, kw, log_tol=TOL_LOG):
  got = getattr(spectral_ops, fn)(x, **kw).cpu().numpy().astype(np.float64)
  xt = torch.as_tensor(np.asarray(x))
  want = getattr(ref, fn)(xt, **kw).numpy()
  assert got.shape == want.shape
  if want.size == 0:
    return got
  if fn == 'compute_mel':
    bound = _mel_bound(x, fn, kw)
    assert (np.abs(got - want) <= bound + 1e-30).all(), np.abs(got - want).max()
  else:
    err = np.abs(got - want) - _mfcc_slack(fn, want)
    assert err.max() <= log_tol, (fn, kw, err.max(), np.unravel_index(err.argmax(), err.shape))
  return got


@pytest.mark.gpu
@pytest.mark.parametrize('i', range(len(mg.CASES)),
                         ids=['%02d-%s' % (i, c[0]) for i, c in enumerate(mg.CASES)])
def test_forward_matches_the_fixture(i):
  fn, _, _, kw = mg.CASES[i]
  x = mg.mel_input(i)
  arg = torch.from_numpy(x).to(DEV) if fn == 'compute_logmag' else x
  got = getattr(spectral_ops, fn)(arg, **kw).cpu().numpy().astype(np.float64)
  want = np.load(mg.PATH)['%s_%02d' % (fn, i)]
  assert got.shape == want.shape
  if want.size == 0:
    return
  if fn == 'compute_mel':
    assert (np.abs(got - want) <= _mel_bound(x, fn, kw) + 1e-30).all()
  elif fn == 'compute_logmag':   # torch / cuFFT float32: compare magnitudes
    peak = np.exp(want).max(-1, keepdims=True)
    assert (np.abs(np.exp(got) - np.exp(want)) <= 1e-5 * peak).all()
  else:
    err = np.abs(got - want) - _mfcc_slack(fn, want)
    assert err.max() <= TOL_LOG, err.max()


def _signals(n, sr, seed):
  """[rows, n] float32: noise at 1, 3e-2 and 1e-4 of full scale, a noise row with a
  silent stretch, a 440 Hz + 3 kHz tone pair and silence."""
  rng = np.random.default_rng(seed)
  t = np.arange(n) / sr
  rows = [rng.uniform(-1, 1, n) * lvl for lvl in (1.0, 3e-2, 1e-4)]
  gap = rng.uniform(-1, 1, n)
  gap[n // 4: n // 2] = 0.0
  rows += [gap, 0.5 * np.sin(2 * np.pi * 440.0 * t) + 0.2 * np.sin(2 * np.pi * 3000.0 * t),
           np.zeros(n)]
  return np.stack(rows).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize('fft_length', [2 ** k for k in range(1, 15)])
def test_every_fft_length(fft_length):
  """Every fft_length from 2 to 16384 in all three modes: noise rows in the log
  domains, the tones in the mel domain, silence exact."""
  fft_size = fft_length if fft_length < 64 else fft_length - fft_length // 8
  n = max(3 * fft_length, 2000)
  x = _signals(n, 16000, seed=fft_length)
  kw = dict(fft_size=fft_size, overlap=0.5, bins=40, lo_hz=0.0, hi_hz=8000.0)
  mel = _check_forward(x, 'compute_mel', kw)
  assert (mel[5] == 0).all()
  logmel = _check_forward(x[:4], 'compute_logmel', kw)
  kw_mfcc = dict(fft_size=fft_size, overlap=0.5, mel_bins=40, mfcc_bins=20, lo_hz=0.0)
  _check_forward(x[:4], 'compute_mfcc', kw_mfcc)
  # empty bands (few bins at small fft_length) are exactly 0 / log(1e-5)
  w = ref.linear_to_mel_weight_matrix(40, fft_length // 2 + 1, 16000, 0.0, 8000.0)
  empty = w.sum(0) == 0
  assert (mel[..., empty] == 0).all()
  assert (logmel[..., empty] == LOG_EPS).all()


@pytest.mark.gpu
def test_silence_padding_and_empty_bands_are_exact():
  """Silent rows, the zero padding past the end and bands with no bins give mel == 0
  and log-mel == float32(log 1e-5) exactly; fft_size 64 with 128 bands leaves most
  bands without a bin."""
  x = np.zeros((2, 3000), np.float32)
  x[1, :1000] = np.random.default_rng(1).uniform(-1, 1, 1000)
  kw = dict(fft_size=64, overlap=0.5, bins=128, lo_hz=0.0, hi_hz=8000.0)
  mel = spectral_ops.compute_mel(x, **kw).cpu().numpy()
  logmel = spectral_ops.compute_logmel(x, **kw).cpu().numpy()
  w = ref.linear_to_mel_weight_matrix(128, 33, 16000, 0.0, 8000.0)
  empty = w.sum(0) == 0
  assert empty.sum() > 50
  assert (mel[0] == 0).all() and (logmel[0] == LOG_EPS).all()
  assert (mel[1][:, empty] == 0).all() and (logmel[1][:, empty] == LOG_EPS).all()
  silent = np.arange(mel.shape[1]) * 32 >= 1000
  assert silent.sum() > 10
  assert (mel[1][silent] == 0).all() and (logmel[1][silent] == LOG_EPS).all()
  assert (mel[1][~silent][:, ~empty] > 0).all()
  kw_mfcc = dict(fft_size=64, overlap=0.5, mel_bins=128, mfcc_bins=13, lo_hz=0.0)
  mf = spectral_ops.compute_mfcc(x[:1], **kw_mfcc).cpu().numpy()
  want = ref.compute_mfcc(torch.zeros(1, 3000, dtype=torch.float64), **kw_mfcc).numpy()
  assert (np.abs(mf - want) <= 1e-6 + _mfcc_slack('compute_mfcc', want)).all()


@pytest.mark.gpu
def test_tones_in_the_mel_domain():
  sr = 16000
  t = np.arange(16000) / sr
  x = np.stack([np.sin(2 * np.pi * f * t + 0.1) for f in (55.0, 440.0, 1234.5, 7000.0)])
  x = x.astype(np.float32)
  for kw in (dict(), dict(fft_size=1024, overlap=0.5, bins=128, lo_hz=20.0),
             dict(fft_size=1001, overlap=0.75, bins=229, pad_end=False)):
    _check_forward(x, 'compute_mel', kw)


@pytest.mark.gpu
def test_shapes_and_layouts():
  x = _signals(4000, 16000, 3)
  m2 = spectral_ops.compute_mfcc(x)
  m1 = spectral_ops.compute_mfcc(x[0])
  m3 = spectral_ops.compute_mfcc(x[:, :, None])
  assert m2.shape == (6, 16, 13) and m1.shape == (16, 13) and m3.shape == m2.shape
  assert torch.equal(m1, m2[0]) and torch.equal(m3, m2)
  a = torch.from_numpy(x[:, :500]).to(DEV).requires_grad_(True)
  v = spectral_ops.compute_logmel(a, pad_end=False)
  assert v.shape == (6, 0, 64)
  v.sum().backward()
  assert torch.equal(a.grad, torch.zeros_like(a))
  e = spectral_ops.compute_mfcc(x, mel_bins=20, mfcc_bins=-20)
  assert e.shape == (6, 16, 0)
  lm = spectral_ops.compute_logmag(torch.from_numpy(x).to(DEV))
  assert lm.shape == (6, 8, 1025)


def _check_grad(x, fn, kw, seed, tol=(1e-3, 1e-4)):
  """d audio of sum(g * feature) against float64 autograd of the restatement; the
  forward values do not depend on requires_grad."""
  x = np.asarray(x, np.float32)
  a = torch.from_numpy(x).to(DEV).requires_grad_(True)
  out = getattr(spectral_ops, fn)(a, **kw)
  with torch.no_grad():
    plain = getattr(spectral_ops, fn)(a, **kw)
  assert torch.equal(out.detach(), plain)
  g = torch.randn(out.shape, generator=torch.Generator().manual_seed(seed)).to(DEV)
  out.backward(g)
  b = torch.from_numpy(x).double().requires_grad_(True)
  want = getattr(ref, fn)(b, **kw)
  want.backward(g.double().cpu())
  got, w = a.grad.double().cpu(), b.grad
  peak = w.abs().max()
  if peak == 0:
    assert torch.equal(got, torch.zeros_like(got))
    return
  emax = float((got - w).abs().max() / peak)
  el2 = float((got - w).norm() / w.norm())
  assert emax <= tol[0] and el2 <= tol[1], (emax, el2)


_GRAD_CASES = [
    ('compute_mfcc', 8000, 16000, dict(fft_size=1024, overlap=0.5, mel_bins=128,
                                       mfcc_bins=30)),
    ('compute_logmel', 6001, 22050, dict(fft_size=1001, overlap=0.75, bins=64, lo_hz=0.0,
                                         hi_hz=11025.0, pad_end=False, sample_rate=22050)),
    ('compute_mel', 3000, 16000, dict(fft_size=64, overlap=-0.5, bins=32, lo_hz=0.0)),
    ('compute_logmel', 40000, 16000, dict(fft_size=16384, overlap=0.75, bins=128,
                                          lo_hz=0.0, hi_hz=8000.0)),
    ('compute_mfcc', 9000, 48000, dict(fft_size=2048, overlap=0.75, mel_bins=229,
                                       mfcc_bins=-3, sample_rate=48000)),
    ('compute_mel', 7000, 44100, dict(fft_size=768, overlap=0.0, bins=40, pad_end=False,
                                      hi_hz=22050.0, sample_rate=44100)),
    ('compute_logmel', 5000, 16000, dict(fft_size=512, overlap=0.5, bins=64, lo_hz=0.0,
                                         hi_hz=8000.0)),
    ('compute_mfcc', 4000, 16000, dict(fft_size=96, overlap=0.5, mel_bins=48, mfcc_bins=13,
                                       lo_hz=0.0, hi_hz=8000.0)),
]


@pytest.mark.gpu
@pytest.mark.parametrize('fn,n,sr,kw', _GRAD_CASES,
                         ids=['%d-%s-%d' % (i, c[0], c[3].get('fft_size'))
                              for i, c in enumerate(_GRAD_CASES)])
def test_gradient_matches_float64_autograd(fn, n, sr, kw):
  """Broadband rows (noise at three levels, noise with a silent stretch: the mel <= 0
  and |X| = 0 branches, silence) in every mode.  Tones are left out: most of their bins
  sit at the float32 FFT's floor, where the direction X_k / |X_k| that d|X_k| is applied
  along is noise, yet d|X_k| itself is of order one, so even the mel gradient of a tone
  is not defined to float32 accuracy (TensorFlow's float32 gradient has the same
  limit)."""
  x = _signals(n, sr, seed=n)
  _check_grad(x[[0, 1, 2, 3, 5]], fn, kw, seed=n)


@pytest.mark.gpu
def test_full_size_bit_reproducible():
  """B = 128, N = 64000 with the ae.gin MFCC: two forwards and two backwards are
  bit-identical (no atomics; every d-audio sample sums its frames in order)."""
  gen = torch.Generator(DEV).manual_seed(3)
  x = torch.rand((128, 64000), device=DEV, generator=gen) * 2 - 1
  x[:4, 20000:30000] = 0.0
  kw = dict(fft_size=1024, overlap=0.5, mel_bins=128, mfcc_bins=30)
  g = torch.randn((128, 125, 30), device=DEV, generator=gen)
  runs = []
  for _ in range(2):
    a = x.clone().requires_grad_(True)
    out = spectral_ops.compute_mfcc(a, **kw)
    out.backward(g)
    runs.append((out.detach(), a.grad))
  assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
  rows = [0, 1, 77]
  want = ref.compute_mfcc(x[rows].double().cpu(), **kw).numpy()
  err = np.abs(runs[0][0][rows].cpu().numpy() - want) - _mfcc_slack('compute_mfcc', want)
  assert err.max() <= TOL_LOG


@pytest.mark.gpu
def test_cuda_graph_capture_equals_eager():
  gen = torch.Generator(DEV).manual_seed(8)
  audio = torch.rand((4, 16000), device=DEV, generator=gen) * 2 - 1
  target = torch.randn((4, 32, 64), device=DEV, generator=gen)
  a = audio.clone().requires_grad_(True)

  def step():
    a.grad = None
    loss = (spectral_ops.compute_logmel(a) - target).abs().mean()
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
    static_loss = (spectral_ops.compute_logmel(a) - target).abs().mean()
    static_loss.backward()
  graph.replay()
  torch.cuda.synchronize()
  assert torch.equal(static_loss, eager)
  assert torch.equal(a.grad, eager_grad)


@pytest.mark.gpu
def test_decoder_to_logmel_chain():
  """decoder_train audio -> compute_logmel -> L1 against a target: the gradients reach
  the raw decoder controls and are finite."""
  from ddsp_b200 import autograd as ag
  from tests.util import synth_inputs
  B, F, K, nb, N = 2, 125, 100, 65, 8000
  inp = synth_inputs(B, F, K, nb, N, seed=3)
  raw = {k: torch.from_numpy(inp[k]).to(DEV).requires_grad_(True)
         for k in ['amps', 'harmonic_distribution', 'noise_magnitudes']}
  f0 = torch.from_numpy(inp['f0_hz']).to(DEV)
  audio = ag.decoder_train(raw['amps'], raw['harmonic_distribution'], f0,
                           raw['noise_magnitudes'], n_samples=N, window_size=0, seed=1,
                           offset=0)
  target = torch.randn((B, 16, 64), device=DEV)
  loss = (spectral_ops.compute_logmel(audio) - target).abs().mean()
  loss.backward()
  assert torch.isfinite(loss)
  for v in raw.values():
    assert v.grad is not None and torch.isfinite(v.grad).all() and v.grad.abs().sum() > 0
