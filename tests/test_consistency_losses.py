"""Consistency losses (csrc/consistency.cuh, losses.KDEConsistencyLoss / TWMLoss and
the torch-only consistency losses, core.harmonic_to_sinusoidal): argument checks, the
float64 restatement and the ported core tests on the CPU; forwards, gradients,
predict_f0, reproducibility, CUDA-graph capture and memory on the GPU.  Reference:
tests/consistency_ref.py, pinned to the unmodified reference by
tests/golden/consistency.npz.

Tolerances.  Two sources of error are separated.

* The kernels against float64 on the same float32 inputs (`test_mixture_kernel_*`,
  `test_comb_kernel_*`).  Every exponent of the shifted logsumexp is formed as a
  product of two differences, so it carries a relative error of a few 2^-24 of its
  own value, and the largest term is exactly 1; the NLL's shift term lw* - z*^2/2 is
  one float32 rounding of a value of size |nll|.  Staging mu / s and x / s rounds
  each by 2^-24 relative, which moves z by up to 2^-23 max(|x|, |mu|) / s and the NLL
  by |z| times that.  So mode A is compared against
  4 (2^-23 m / s)(1 + sqrt(2 |nll|)) + 2^-20 |nll| + 1e-5, m the largest |x|, |mu|.
  Mode B: the ratio q = f / f0 is one rounding, so nu moves by |nu'(q)| q 2^-24 with
  |nu'(q)| <= sqrt(2 nu) / s; the window's omitted terms are below 2^-25 of the sum
  (DESIGN §3.17).  It is compared against 2^-21 q_max / s sqrt(2 |nu|) + 2^-20 |nu| +
  1e-5, on the amplitude-weighted mean, which the per-term bound bounds too (sqrt is
  concave).
* The losses against the float64 restatement from hertz.  hz_to_midi in float32 is a
  chain of five roundings: up to 16 ulp, 1.2e-4, at MIDI 128 (the harmonics formed as
  hz_to_midi(f0) + 12 log2 n add two).  A distance error of d = 2.4e-4 MIDI (both
  ends) moves z by d / s and the NLL by |z| d / s <= sqrt(2 |nll| + 2) d / s.  So
  NLL-level outputs are compared against (d / s)(1 + sqrt(2 |want|)) + 2^-20 |want| +
  1e-5, with s the smallest scale in play.  TWM's softmin S = sum_c w_c L_c moves by
  sum_c w_c (1 + |L_c - S| / T) tol(L_c) per frame when each L_c moves by tol(L_c)
  (`_softmin_tol`).
* Gradients: every gradient is a responsibility-weighted sum of z / s terms, so the
  errors above scale them relatively; float32 responsibilities add a few 2^-24.  Each
  gradient tensor is compared normwise, max |got - want| <= 5e-3 max |want|, and
  elementwise within 5e-3 |want| + 1e-3 max |want|.
"""
import math

import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, autograd, core, losses
from tests import consistency_ref as ref
from tests.golden import make_consistency_golden as cg

P = 0x1000        # a device pointer the library never dereferences on the host
E_INVALID, E_UNSUPPORTED = _lib.E_INVALID, _lib.E_UNSUPPORTED
DEV = 'cuda'
D_MIDI = 2.4e-4


def _mf(x=P, mu=P, lw=P, out=P, B=2, T=3, Q=10, J=10, s=0.1):
  return (x, mu, lw, out, B, T, Q, J, s, None)


def _mb(x=P, mu=P, lw=P, g=P, dx=P, dmu=P, dlw=P, B=2, T=3, Q=10, J=10, s=0.1):
  return (x, mu, lw, g, dx, dmu, dlw, B, T, Q, J, s, None)


def _cf(f0=P, f=P, a=P, out=P, B=2, T=3, C=10, Pn=10, G=30, s=0.2):
  return (f0, f, a, out, B, T, C, Pn, G, s, None)


def _cb(f0=P, f=P, a=P, g=P, d0=P, df=P, da=P, B=2, T=3, C=10, Pn=10, G=30, s=0.2):
  return (f0, f, a, g, d0, df, da, B, T, C, Pn, G, s, None)


_MF, _MB, _CF, _CB = ('mixture_nll_forward', 'mixture_nll_backward', 'comb_nll_forward',
                      'comb_nll_backward')
_ABI_CASES = [
    ('mf-null-x', _MF, _mf(x=None), E_INVALID, b'mixture_nll_forward: null pointer'),
    ('mf-null-mu', _MF, _mf(mu=None), E_INVALID, b'mixture_nll_forward: null pointer'),
    ('mf-null-lw', _MF, _mf(lw=None), E_INVALID, b'mixture_nll_forward: null pointer'),
    ('mf-null-out', _MF, _mf(out=None), E_INVALID, b'mixture_nll_forward: null pointer'),
    ('mf-B', _MF, _mf(B=-1), E_INVALID, b'mixture_nll_forward: bad shape B=-1 T=3 Q=10 J=10'),
    ('mf-T', _MF, _mf(T=-2), E_INVALID, b'mixture_nll_forward: bad shape B=2 T=-2 Q=10 J=10'),
    ('mf-Q', _MF, _mf(Q=-1), E_INVALID, b'mixture_nll_forward: bad shape B=2 T=3 Q=-1 J=10'),
    ('mf-J', _MF, _mf(J=-1), E_INVALID, b'mixture_nll_forward: bad shape B=2 T=3 Q=10 J=-1'),
    ('mf-scale0', _MF, _mf(s=0.0), E_INVALID, b'mixture_nll_forward: scale must be positive and finite, got 0'),
    ('mf-scale-neg', _MF, _mf(s=-0.5), E_INVALID, b'mixture_nll_forward: scale must be positive and finite, got -0.5'),
    ('mf-scale-nan', _MF, _mf(s=math.nan), E_INVALID, b'mixture_nll_forward: scale must be positive and finite, got nan'),
    ('mf-scale-inf', _MF, _mf(s=math.inf), E_INVALID, b'mixture_nll_forward: scale must be positive and finite, got inf'),
    ('mf-J-max', _MF, _mf(J=4097), E_UNSUPPORTED, b'mixture_nll_forward: J=4097 components exceed the 4096 supported'),
    ('mf-grid', _MF, _mf(B=65536, T=32768), E_INVALID, b'mixture_nll_forward: B*T=2147483648 exceeds the 2^31 - 1 grid limit'),
    ('mf-B0', _MF, _mf(B=0), 0, None),
    ('mf-T0', _MF, _mf(T=0), 0, None),
    ('mf-Q0', _MF, _mf(Q=0), 0, None),
    ('mf-J0', _MF, _mf(J=0), 0, None),
    ('mf-J-4096', _MF, _mf(B=0, J=4096), 0, None),
    ('mf-empty-null', _MF, _mf(x=None, mu=None, lw=None, out=None, T=0), 0, None),
    ('mb-null-x', _MB, _mb(x=None), E_INVALID, b'mixture_nll_backward: null pointer'),
    ('mb-null-g', _MB, _mb(g=None), E_INVALID, b'mixture_nll_backward: null pointer'),
    ('mb-null-dx', _MB, _mb(dx=None), E_INVALID, b'mixture_nll_backward: null pointer'),
    ('mb-null-dmu', _MB, _mb(dmu=None), E_INVALID, b'mixture_nll_backward: null pointer'),
    ('mb-null-dlw', _MB, _mb(dlw=None), E_INVALID, b'mixture_nll_backward: null pointer'),
    ('mb-Q', _MB, _mb(Q=-3), E_INVALID, b'mixture_nll_backward: bad shape B=2 T=3 Q=-3 J=10'),
    ('mb-scale', _MB, _mb(s=-1.0), E_INVALID, b'mixture_nll_backward: scale must be positive and finite, got -1'),
    ('mb-J-max', _MB, _mb(J=5000), E_UNSUPPORTED, b'mixture_nll_backward: J=5000 components exceed the 4096 supported'),
    ('mb-grid', _MB, _mb(B=1 << 20, T=1 << 12), E_INVALID, b'mixture_nll_backward: B*T=4294967296 exceeds the 2^31 - 1 grid limit'),
    ('mb-B0', _MB, _mb(B=0), 0, None),
    ('mb-J0', _MB, _mb(J=0), 0, None),
    ('cf-null-f0', _CF, _cf(f0=None), E_INVALID, b'comb_nll_forward: null pointer'),
    ('cf-null-f', _CF, _cf(f=None), E_INVALID, b'comb_nll_forward: null pointer'),
    ('cf-null-a', _CF, _cf(a=None), E_INVALID, b'comb_nll_forward: null pointer'),
    ('cf-null-out', _CF, _cf(out=None), E_INVALID, b'comb_nll_forward: null pointer'),
    ('cf-B', _CF, _cf(B=-1), E_INVALID, b'comb_nll_forward: bad shape B=-1 T=3 C=10 P=10 G=30'),
    ('cf-C', _CF, _cf(C=-1), E_INVALID, b'comb_nll_forward: bad shape B=2 T=3 C=-1 P=10 G=30'),
    ('cf-P', _CF, _cf(Pn=-1), E_INVALID, b'comb_nll_forward: bad shape B=2 T=3 C=10 P=-1 G=30'),
    ('cf-G', _CF, _cf(G=0), E_INVALID, b'comb_nll_forward: bad shape B=2 T=3 C=10 P=10 G=0'),
    ('cf-scale', _CF, _cf(s=0.0), E_INVALID, b'comb_nll_forward: scale must be positive and finite, got 0'),
    ('cf-C-max', _CF, _cf(C=4097), E_UNSUPPORTED, b'comb_nll_forward: C=4097 candidates or P=10 points exceed the 4096 supported'),
    ('cf-P-max', _CF, _cf(Pn=4097), E_UNSUPPORTED, b'comb_nll_forward: C=10 candidates or P=4097 points exceed the 4096 supported'),
    ('cf-grid', _CF, _cf(B=65536, T=65536), E_INVALID, b'comb_nll_forward: B*T=4294967296 exceeds the 2^31 - 1 grid limit'),
    ('cf-B0', _CF, _cf(B=0), 0, None),
    ('cf-T0', _CF, _cf(T=0), 0, None),
    ('cf-C0', _CF, _cf(C=0), 0, None),
    ('cf-P0', _CF, _cf(Pn=0), 0, None),
    ('cb-null-g', _CB, _cb(g=None), E_INVALID, b'comb_nll_backward: null pointer'),
    ('cb-null-d0', _CB, _cb(d0=None), E_INVALID, b'comb_nll_backward: null pointer'),
    ('cb-null-df', _CB, _cb(df=None), E_INVALID, b'comb_nll_backward: null pointer'),
    ('cb-null-da', _CB, _cb(da=None), E_INVALID, b'comb_nll_backward: null pointer'),
    ('cb-G', _CB, _cb(G=-4), E_INVALID, b'comb_nll_backward: bad shape B=2 T=3 C=10 P=10 G=-4'),
    ('cb-scale', _CB, _cb(s=math.inf), E_INVALID, b'comb_nll_backward: scale must be positive and finite, got inf'),
    ('cb-P-max', _CB, _cb(Pn=8192), E_UNSUPPORTED, b'comb_nll_backward: C=10 candidates or P=8192 points exceed the 4096 supported'),
    ('cb-T0', _CB, _cb(T=0), 0, None),
    ('cb-P0', _CB, _cb(Pn=0), 0, None),
    ('cb-empty-null', _CB, _cb(f0=None, f=None, a=None, g=None, d0=None, df=None, da=None, B=0), 0, None),
]


@pytest.mark.parametrize('fn,args,want,msg', [c[1:] for c in _ABI_CASES],
                         ids=[c[0] for c in _ABI_CASES])
def test_consistency_abi_check_table(fn, args, want, msg):
  """Every check of the four entry points: the status and the full message come back
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
  z = np.zeros((2, 3, 4), np.float32)
  z5 = np.zeros((2, 3, 5), np.float32)
  kde, twm = losses.KDEConsistencyLoss(), losses.TWMLoss()
  cases = [
      ('amps_a, freqs_a must be two', lambda: kde(z, z5, z, z)),
      ('amps_b, freqs_b must be two', lambda: kde(z, z, z[0], z[0])),
      (r'amps_b, freqs_b has \[batch, time\] \(2, 4\)',
       lambda: kde(z, z, np.zeros((2, 4, 4)), np.zeros((2, 4, 4)))),
      ('scale_b must be positive and finite, got 0',
       lambda: losses.KDEConsistencyLoss(scale_b=0.0)(z, z, z, z)),
      ('scale_a must be positive and finite, got -1',
       lambda: losses.KDEConsistencyLoss(scale_a=-1.0)(z, z, z, z)),
      ('scale_target must be positive and finite, got nan',
       lambda: kde.nll(z, z, z, z, math.nan)),
      ('amps_target, freqs_target must be two', lambda: kde.nll(z, z, z, z5, 0.1)),
      ('amps, freqs must be two', lambda: twm(z, z, z5)),
      ('f0_candidates must be', lambda: twm(z[0], z, z)),
      ('f0_candidates must be', lambda: twm(np.zeros((2, 4, 1)), z, z)),
      ('n_harmonic_points', lambda: losses.TWMLoss(n_harmonic_points=0)(z, z, z)),
      ('n_harmonic_gaussians', lambda: losses.TWMLoss(n_harmonic_gaussians=0)(z, z, z)),
      ('harmonics_scale must be positive and finite, got 0',
       lambda: losses.TWMLoss(harmonics_scale=0.0)(z, z, z)),
      ('sinusoids_scale must be positive and finite, got inf',
       lambda: losses.TWMLoss(sinusoids_scale=math.inf).predict_f0(z, z, z)),
      ('amps, freqs must be two', lambda: twm.get_loss_tensors(z, z5, z)),
  ]
  for msg, call in cases:
    with pytest.raises(ValueError, match=msg):
      call()


def test_names_follow_keras():
  assert losses.KDEConsistencyLoss().name == 'kde_consistency_loss'
  assert losses.TWMLoss().name == 'twm_loss'
  assert losses.HarmonicConsistencyLoss().name == 'harmonic_consistency_loss'
  assert losses.FilteredNoiseConsistencyLoss().name == 'filtered_noise_consistency_loss'
  assert losses.ParamLoss(name='midi').name == 'midi'


# ---- core.harmonic_to_sinusoidal: core_test.py:94-142 ------------------------------
def _close(a, b):
  np.testing.assert_allclose(np.asarray(a), np.asarray(b), rtol=1e-6, atol=1e-6)


def test_harmonic_to_sinusoidal():
  f0_hz = core.midi_to_hz([80, 81, 82, 81, 80])[np.newaxis, :, np.newaxis]
  harm_amps = np.ones(shape=(1, 5, 3))
  harm_amps /= np.sum(harm_amps, axis=-1, keepdims=True)
  amps, sin_freqs = core.harmonic_to_sinusoidal(10, harm_amps, f0_hz)
  sin_freqs = np.squeeze(sin_freqs.numpy())
  f0_hz = np.squeeze(f0_hz.numpy())
  _close(amps, harm_amps * 10)
  _close(sin_freqs[..., 0], f0_hz)
  _close(sin_freqs[..., 1], f0_hz * 2)
  _close(sin_freqs[..., 2], f0_hz * 3)


def test_harmonic_to_sinusoidal_removes_nyquist_f0():
  f0_hz = np.asarray([200, 400, 8001])[np.newaxis, :, np.newaxis]
  harm_amps = np.ones(shape=(1, 3, 3))
  harm_amps /= np.sum(harm_amps, axis=-1, keepdims=True)
  amps, sin_freqs = core.harmonic_to_sinusoidal(10, harm_amps, f0_hz)
  sin_freqs = np.squeeze(sin_freqs.numpy())
  f0_hz = np.squeeze(f0_hz)
  expected_amps_f0 = harm_amps[..., 0] * 10
  expected_amps_f0[:, 2] = 0
  _close(amps[..., 0], expected_amps_f0)
  _close(sin_freqs[..., 0], f0_hz)
  _close(sin_freqs[..., 1], f0_hz * 2)
  _close(sin_freqs[..., 2], f0_hz * 3)


def test_harmonic_to_sinusoidal_removes_nyquist_harmonics():
  f0_hz = np.asarray([50, 3001, 4001, 3001, 50])[np.newaxis, :, np.newaxis]
  orig_harm_amps = np.ones(shape=(1, 5, 3))
  harm_amps = orig_harm_amps / np.sum(orig_harm_amps, axis=-1, keepdims=True)
  amps, sin_freqs = core.harmonic_to_sinusoidal(10, harm_amps, f0_hz)
  sin_freqs = np.squeeze(sin_freqs.numpy())
  f0_hz = np.squeeze(f0_hz)
  expected_amps = orig_harm_amps * 10
  expected_amps[:, 2, 1] = 0          # f1 > nyquist
  expected_amps[:, 1:4, 2] = 0        # f2 > nyquist
  expected_amps[:, 0] /= 3
  expected_amps[:, 1] /= 2
  expected_amps[:, 3] /= 2
  expected_amps[:, 4] /= 3
  for k in range(3):
    _close(amps[..., k], expected_amps[..., k])
    _close(sin_freqs[..., k], f0_hz * (k + 1))


# ---- the restatement and the fixture ------------------------------------------------
def _rel_close(got, want, rtol=1e-9):
  got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
  assert got.shape == want.shape, (got.shape, want.shape)
  assert np.all(np.abs(got - want) <= rtol * (1.0 + np.abs(want))), (got, want)


def test_restatement_matches_the_reference():
  """tests/consistency_ref.py against the unmodified reference run wide on the shim,
  at 1e-9 relative, over every case of the fixture."""
  want = np.load(cg.PATH)
  for i, (name, *_, kw) in enumerate(cg.KDE_CASES):
    x = cg.kde_inputs(i)
    _rel_close(ref.kde_loss(*x, **kw).numpy(), want[name + '_call'])
    scale_b = kw.get('scale_b', 0.1)
    _rel_close(ref.kde_nll(*x, scale_b).numpy(), want[name + '_nll'])
  for i, (name, *_, kw) in enumerate(cg.TWM_CASES):
    x = cg.twm_inputs(i)
    _rel_close(ref.twm_loss(*x, **kw).numpy(), want[name + '_call'])
    s, h = ref.twm_loss_tensors(*x, **kw)
    _rel_close(s.numpy(), want[name + '_sinusoids'])
    _rel_close(h.numpy(), want[name + '_harmonics'])
    _rel_close(ref.twm_predict_f0(*x, **kw), want[name + '_f0'])
  harm_amp, harm_dist, f0 = cg.harmonic_inputs()
  t = cg.harmonic_consistency_targets()
  got = ref.harmonic_consistency(harm_amp, t[0], harm_dist, t[1], f0, t[2], amp_weight=0.5,
                                 dist_weight=2.0, f0_weight=1.5)
  for k, v in got.items():     # the shim's float32 weights: 1e-8
    _rel_close(v.numpy(), want['harmonic_consistency_' + k], rtol=1e-8)
  amps, freqs = ref.harmonic_to_sinusoidal(harm_amp, harm_dist, f0)
  _rel_close(amps.numpy(), want['h2s_amps'])
  _rel_close(freqs.numpy(), want['h2s_freqs'])


def test_fixture_regenerates():
  """Where the reference is checked out, the fixture is what it computes."""
  from oracle import ref_on_shim
  try:
    ref_on_shim.load()
  except Exception as e:  # pylint: disable=broad-except
    pytest.skip('reference sources not available: %s' % e)
  from tests.golden.make_golden import compare
  compare('consistency', cg.consistency(), np.load(cg.PATH))


# ---- GPU: helpers -------------------------------------------------------------------
def _cuda(*xs, grad=False):
  return [torch.as_tensor(np.asarray(x, np.float32), device=DEV).requires_grad_(grad)
          for x in xs]


def _nll_tol(want, s):
  want = np.abs(np.asarray(want, np.float64))
  return (D_MIDI / s) * (1.0 + np.sqrt(2.0 * want)) + 2.0**-20 * want + 1e-5


def _check_nll(got, want, s):
  got = got.detach().cpu().numpy().astype(np.float64) if torch.is_tensor(got) else got
  want = want.detach().numpy() if torch.is_tensor(want) else np.asarray(want)
  assert got.shape == want.shape, (got.shape, want.shape)
  both_nan = np.isnan(got) & np.isnan(want)
  err = np.where(both_nan, 0.0, np.abs(got - want))
  tol = _nll_tol(want, s)
  assert np.all(err <= tol), (np.max(err - tol), got.ravel()[:8], want.ravel()[:8])


def _check_grad(got, want, name='', atol=0.0):
  got = got.detach().cpu().numpy().astype(np.float64)
  want = want.detach().numpy()
  scale = np.max(np.abs(want)) if want.size else 0.0
  err = np.abs(got - want)
  assert np.all(np.isfinite(got)) or not np.all(np.isfinite(want)), name
  assert np.all(err <= 5e-3 * np.abs(want) + 1e-3 * scale + atol + 1e-12), (
      name, np.max(err), scale)


def _normalisation_atol(amps, freqs, amps_t, freqs_t, scale, weight):
  """d amps through KDE's source weights a_k / sum a: autograd forms
  nll_k / s - sum_j nll_j a_j / s^2, which cancels (exactly, at K = 1) in float32 and
  leaves a few 2^-24 of max |nll| / s; scaled by the loss's mean over B T K."""
  x = ref.hz_to_midi(freqs)[..., None]
  lp = (ref.normal_log_prob(x, ref.hz_to_midi(freqs_t)[:, :, None, :], scale) +
        torch.log_softmax(torch.log(ref._amps_probs(ref.t64(amps_t))), -1)[:, :, None, :])
  nll = torch.logsumexp(lp, -1).abs().numpy()
  s = np.abs(np.sum(amps, -1, keepdims=True, dtype=np.float64))
  b, t, k = amps.shape
  return 2.0**-20 * weight * np.max(nll, -1, keepdims=True) / (np.maximum(s, 1e-7) * k * b * t)


def _softmin_tol(loss, sinusoids, harmonics, s):
  """The bound on TWMLoss.call from the per-candidate bounds: the softmin's value
  S = sum_c w_c L_c moves by sum_c w_c (1 + |L_c - S| / T) tol(L_c) per frame."""
  combined = loss.sinusoids_weight * sinusoids + loss.harmonics_weight * harmonics
  temp = loss.softmin_temperature
  w = np.exp(-(combined - np.min(combined, -1, keepdims=True)) / temp)
  w /= np.sum(w, -1, keepdims=True)
  soft = np.sum(w * combined, -1, keepdims=True)
  per = np.where(w > 0, w * (1 + np.abs(combined - soft) / temp), 0.0) * _nll_tol(
      np.where(w > 0, combined, 0.0), s)
  return float(np.mean(np.sum(per, -1)))


# ---- GPU: the kernels on their own ---------------------------------------------------
def _mix_ref(x, mu, lw, s):
  return -torch.logsumexp(lw[..., None, :] + ref.normal_log_prob(x[..., None], mu[..., None, :], s),
                          dim=-1)


@pytest.mark.gpu
@pytest.mark.parametrize('b,t,q,j,s', [(2, 3, 10, 10, 0.1), (3, 5, 1, 1, 0.1),
                                       (2, 4, 37, 5, 0.5), (1, 2, 1300, 700, 0.05),
                                       (2, 2, 5, 4096, 1.0)])
def test_mixture_kernel_against_float64(b, t, q, j, s):
  """Mode A alone, on float32 inputs that the float64 reference reads as they are:
  queries spread over 20 .. 140 MIDI, some 60 MIDI (600 s at s = 0.1) from every
  component, and unnormalised log-weights."""
  rng = np.random.default_rng(q * 7 + j)
  x = rng.uniform(20.0, 140.0, (b, t, q)).astype(np.float32)
  mu = rng.uniform(60.0, 90.0, (b, t, j)).astype(np.float32)
  lw = rng.normal(-3.0, 2.0, (b, t, j)).astype(np.float32)
  xg, mug, lwg = _cuda(x, mu, lw, grad=True)
  nll = autograd.MixtureNLLFn.apply(xg, mug, lwg, s)
  x64, mu64, lw64 = (torch.from_numpy(v).double().requires_grad_(True) for v in (x, mu, lw))
  want = _mix_ref(x64, mu64, lw64, s)
  m = float(np.max(np.abs(np.concatenate([x.ravel(), mu.ravel()]))))
  w = np.abs(want.detach().numpy())
  tol = 4 * (2.0**-23 * m / s) * (1 + np.sqrt(2 * w)) + 2.0**-20 * w + 1e-5
  assert np.all(np.abs(nll.detach().cpu().numpy() - want.detach().numpy()) <= tol)
  g = np.random.default_rng(1).normal(size=(b, t, q))
  nll.backward(torch.as_tensor(g, dtype=torch.float32, device=DEV))
  want.backward(torch.from_numpy(g))
  for name, a, e in (('dx', xg, x64), ('dmu', mug, mu64), ('dlw', lwg, lw64)):
    _check_grad(a.grad, e.grad, name)


@pytest.mark.gpu
def test_mixture_kernel_far_queries_stay_finite():
  """Queries 1000 MIDI from the components at s = 0.01: NLLs of 5e9, finite and to
  float32's relative resolution."""
  x = np.full((1, 1, 3), 1100.0, np.float32)
  mu = np.array([[[60.0, 61.0, 100.0]]], np.float32)
  lw = np.log(np.array([[[0.2, 0.3, 0.5]]], np.float32))
  nll = autograd.MixtureNLLFn.apply(*_cuda(x, mu, lw), 0.01).cpu().numpy()
  want = _mix_ref(*(torch.from_numpy(v).double() for v in (x, mu, lw)), 0.01).numpy()
  assert np.all(np.isfinite(nll)) and np.all(want > 4e9)
  assert np.all(np.abs(nll - want) <= 1e-6 * want)


def _comb_ref(f0, f, a, g_count, s):
  r = ref.safe_divide(f[:, :, None, :], f0[:, :, :, None])
  nu = -ref.mixture_log_prob(r, torch.full((g_count,), 1.0 / g_count, dtype=torch.float64),
                             torch.arange(1, g_count + 1, dtype=torch.float64), s)
  a4 = a[:, :, None, :]
  return ref.safe_divide(torch.sum(nu * a4, -1), torch.sum(a4, -1))


@pytest.mark.gpu
@pytest.mark.parametrize('b,t,c,p,g,s', [(2, 3, 10, 10, 30, 0.2), (2, 3, 1, 8, 30, 0.2),
                                         (1, 2, 100, 100, 30, 0.2), (2, 2, 7, 5, 12, 0.05),
                                         (2, 2, 6, 9, 5, 2.0), (1, 3, 3, 4, 1, 0.3)])
def test_comb_kernel_against_float64(b, t, c, p, g, s):
  """Mode B alone: harmonic points, candidates around f0 and at 0, frequencies <= 0,
  exact zero amplitudes and an all-zero row; window widths from 1 (s = 0.05) to the
  whole comb (s = 2)."""
  rng = np.random.default_rng(c * 13 + p)
  amps, freqs, f0 = cg.harmonic_sinusoids(rng, b, t, p)
  cands = (f0 * np.exp(rng.uniform(-0.8, 0.8, (b, t, c)))).astype(np.float32)
  cands[0, 0, 0] = 0.0
  freqs[-1, -1, 0] = 0.0
  freqs[0, -1, -1] = -20.0
  amps[0, 0, ::2] = 0.0
  amps[-1, -1, :] = 0.0
  cg_, fg, ag = _cuda(cands, freqs, amps, grad=True)
  out = autograd.CombNLLFn.apply(cg_, fg, ag, g, s)
  c64, f64, a64 = (torch.from_numpy(v).double().requires_grad_(True)
                   for v in (cands, freqs, amps))
  want = _comb_ref(c64, f64, a64, g, s)
  q_max = np.max(np.abs(freqs)) / np.min(np.where(cands == 0, 1e-7, np.abs(cands)))
  w = np.abs(want.detach().numpy())
  tol = 2.0**-21 * q_max / s * np.sqrt(2 * w) + 2.0**-20 * w + 1e-5
  assert np.all(np.abs(out.detach().cpu().numpy() - want.detach().numpy()) <= tol)
  gr = np.random.default_rng(2).normal(size=(b, t, c))
  out.backward(torch.as_tensor(gr, dtype=torch.float32, device=DEV))
  want.backward(torch.from_numpy(gr))
  for name, x, e in (('d_f0', cg_, c64), ('d_f', fg, f64), ('d_a', ag, a64)):
    _check_grad(x.grad, e.grad, name)
  assert cg_.grad[0, 0, 0].item() == 0.0          # no gradient to a zero f0


# ---- GPU: the losses ----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('i', range(len(cg.KDE_CASES)), ids=[c[0] for c in cg.KDE_CASES])
def test_kde_fixture_cases(i):
  name, *_, kw = cg.KDE_CASES[i]
  want = np.load(cg.PATH)
  x = cg.kde_inputs(i)
  loss = losses.KDEConsistencyLoss(**kw)
  s = min(loss.scale_a, loss.scale_b)
  _check_nll(loss(*x), want[name + '_call'], s)
  _check_nll(loss.nll(*x, loss.scale_b), want[name + '_nll'], loss.scale_b)


@pytest.mark.gpu
@pytest.mark.parametrize('i', range(len(cg.TWM_CASES)), ids=[c[0] for c in cg.TWM_CASES])
def test_twm_fixture_cases(i):
  name, *_, kw = cg.TWM_CASES[i]
  want = np.load(cg.PATH)
  x = cg.twm_inputs(i)
  loss = losses.TWMLoss(**kw)
  s = min(loss.sinusoids_scale, loss.harmonics_scale)
  sl, hl = loss.get_loss_tensors(*x)
  _check_nll(sl, want[name + '_sinusoids'], s)
  _check_nll(hl, want[name + '_harmonics'], s)
  got = float(loss(*x))
  tol = _softmin_tol(loss, want[name + '_sinusoids'], want[name + '_harmonics'], s)
  assert abs(got - want[name + '_call']) <= tol, (got, want[name + '_call'], tol)


def _kde_case(b, t, ka, kb, seed, kw):
  rng = np.random.default_rng(seed)
  amps_a, freqs_a = cg.sinusoids(rng, b, t, ka)
  amps_b, freqs_b = cg.sinusoids(rng, b, t, kb, 'zeros' if b > 1 else None)
  return (amps_a, freqs_a, amps_b, freqs_b), kw


_KDE_GRAD_CASES = {
    'pretrain': (32, 125, 100, 100, {}),
    'k1': (3, 4, 1, 1, {}),
    'ka-ne-kb': (2, 5, 30, 7, dict(weight_a=0.5, weight_b=2.0, weight_mean_amp=3.0,
                                   scale_a=0.3, scale_b=0.07)),
    't1': (4, 1, 12, 12, {}),
}


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(_KDE_GRAD_CASES))
def test_kde_forward_and_gradients(case):
  """KDEConsistencyLoss.call and the gradients of all four inputs against float64
  autograd of the restatement."""
  b, t, ka, kb, kw = _KDE_GRAD_CASES[case]
  x, kw = _kde_case(b, t, ka, kb, 40 + ka, kw)
  xs = _cuda(*x, grad=True)
  loss = losses.KDEConsistencyLoss(**kw)
  got = loss(*xs)
  x64 = [torch.from_numpy(v).double().requires_grad_(True) for v in x]
  want = ref.kde_loss(*x64, **kw)
  _check_nll(got, want, min(loss.scale_a, loss.scale_b))
  got.backward()
  want.backward()
  atol = {
      'amps_a': _normalisation_atol(x[0], x[1], x[2], x[3], loss.scale_b, loss.weight_a),
      'amps_b': _normalisation_atol(x[2], x[3], x[0], x[1], loss.scale_a, loss.weight_b)}
  for n, a, e in zip(('amps_a', 'freqs_a', 'amps_b', 'freqs_b'), xs, x64):
    _check_grad(a.grad, e.grad, n, atol.get(n, 0.0))


def _twm_case(b, t, c, p, seed, edges=False):
  rng = np.random.default_rng(seed)
  amps, freqs, f0 = cg.harmonic_sinusoids(rng, b, t, p)
  if c == 0:
    cands = freqs.copy()
  else:
    cands = (f0 * np.exp(rng.uniform(-0.7, 0.7, (b, t, c)))).astype(np.float32)
  if edges:
    cands[0, 0, 0] = 0.0
    cands[-1, -1, -1] = 12000.0
    freqs[0, -1, 0] = 0.0
    amps[0, 0, ::2] = 0.0
    amps[-1, -1, :] = 0.0
  return cands, freqs, amps


_TWM_GRAD_CASES = {
    'c1': (4, 25, 1, 100, {}, False),
    'c-eq-p-100': (2, 6, 0, 100, {}, False),
    't1': (3, 1, 5, 20, {}, True),
    'args': (2, 3, 7, 11, dict(sinusoids_weight=0.6, harmonics_weight=1.7,
                               sinusoids_scale=0.3, harmonics_scale=0.1, n_harmonic_points=6,
                               n_harmonic_gaussians=12, softmin_temperature=3.0,
                               sample_rate=22050), True),
}


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(_TWM_GRAD_CASES))
def test_twm_forward_and_gradients(case):
  """TWMLoss's two loss tensors and call, and the gradients of f0_candidates (the
  self-supervised pitch gradient), freqs and amps against float64 autograd."""
  b, t, c, p, kw, edges = _TWM_GRAD_CASES[case]
  x = _twm_case(b, t, c, p, 50 + p, edges)
  xs = _cuda(*x, grad=True)
  loss = losses.TWMLoss(**kw)
  s = min(loss.sinusoids_scale, loss.harmonics_scale)
  x64 = [torch.from_numpy(v).double().requires_grad_(True) for v in x]
  sl, hl = loss.get_loss_tensors(*xs)
  ws, wh = ref.twm_loss_tensors(*x64, **kw)
  _check_nll(sl, ws, s)
  _check_nll(hl, wh, s)
  got = loss(*xs)
  want = ref.twm_loss(*x64, **kw)
  tol = _softmin_tol(loss, ws.detach().numpy(), wh.detach().numpy(), s)
  assert abs(got.item() - want.item()) <= tol, (got.item(), want.item(), tol)
  got.backward()
  want.backward()
  for n, a, e in zip(('f0_candidates', 'freqs', 'amps'), xs, x64):
    _check_grad(a.grad, e.grad, n)


@pytest.mark.gpu
def test_zero_sizes():
  kde, twm = losses.KDEConsistencyLoss(), losses.TWMLoss()
  for b, t in ((0, 5), (3, 0)):
    x = [np.zeros((b, t, 4), np.float32) + 100.0] * 4
    assert kde.nll(*x, 0.1).shape == (b, t)
    s, h = twm.get_loss_tensors(*x[:3])
    assert s.shape == (b, t, 4) and h.shape == (b, t, 4)
  # no sinusoids at all: means over nothing, as in the restatement
  e = np.zeros((2, 3, 0), np.float32)
  got = kde.nll(e, e, e, e, 0.1).cpu().numpy()
  want = ref.kde_nll(e, e, e, e, 0.1).numpy()
  assert got.shape == want.shape and np.all(np.isnan(got) == np.isnan(want))
  f0 = np.full((2, 3, 2), 200.0, np.float32)
  s, h = twm.get_loss_tensors(f0, e, e)
  ws, wh = ref.twm_loss_tensors(f0, e, e)
  assert np.array_equal(s.cpu().numpy(), ws.numpy())
  assert np.array_equal(np.isinf(h.cpu().numpy()), np.isinf(wh.numpy()))
  # no queries but components (Q = 0 < J): the mixture's gradients are exactly 0.
  # Freed NaN memory first, so that gradients left unwritten come back as NaN.
  torch.full((1 << 16,), math.nan, device=DEV)
  x = torch.zeros((2, 3, 0), device=DEV, requires_grad=True)
  mu, lw = _cuda(np.full((2, 3, 5), 60.0), np.full((2, 3, 5), -1.6), grad=True)
  nll = autograd.MixtureNLLFn.apply(x, mu, lw, 0.1)
  assert nll.shape == (2, 3, 0)
  nll.sum().backward()
  assert torch.equal(mu.grad, torch.zeros_like(mu)), mu.grad
  assert torch.equal(lw.grad, torch.zeros_like(lw)), lw.grad


@pytest.mark.gpu
def test_predict_f0_is_the_argmin():
  """Harmonic sinusoids of f0 against candidates f0 / 3 .. 3 f0 (and a NaN loss from a
  NaN candidate): the restatement's minimum is separated from the runner-up by far
  more than the tolerance, and predict_f0 picks it, on the inputs' device."""
  rng = np.random.default_rng(77)
  b, t, p = 4, 30, 20
  amps, freqs, f0 = cg.harmonic_sinusoids(rng, b, t, p)
  ratios = np.array([1 / 3, 0.5, 2 / 3, 1.0, 1.5, 2.0, 3.0])
  cands = (f0 * ratios).astype(np.float32)
  cands[0, 0, 1] = np.nan
  loss = losses.TWMLoss()
  got = loss.predict_f0(*_cuda(cands, freqs, amps))
  assert got.device.type == 'cuda' and got.shape == (b, t, 1)
  want = ref.twm_predict_f0(cands, freqs, amps)
  s, h = ref.twm_loss_tensors(cands, freqs, amps)
  total = np.sort(np.nan_to_num((s + h).numpy(), nan=np.inf), axis=-1)
  assert np.all(total[..., 1] - total[..., 0] > 10 * _nll_tol(total[..., 1], 0.2))
  np.testing.assert_array_equal(got.cpu().numpy(), want.astype(np.float32))
  fixture = np.load(cg.PATH)
  for i, (name, *_, kw) in enumerate(cg.TWM_CASES):
    got = losses.TWMLoss(**kw).predict_f0(*_cuda(*cg.twm_inputs(i))).cpu().numpy()
    np.testing.assert_array_equal(got, fixture[name + '_f0'].astype(np.float32))


@pytest.mark.gpu
def test_torch_consistency_losses():
  want = np.load(cg.PATH)
  harm_amp, harm_dist, f0 = cg.harmonic_inputs()
  t = cg.harmonic_consistency_targets()
  hc = losses.HarmonicConsistencyLoss(amp_weight=0.5, dist_weight=2.0, f0_weight=1.5)
  got = hc.get_losses_dict(harm_amp, t[0], harm_dist, t[1], f0, t[2])
  assert list(got) == ['harmonic_consistency_loss']
  for k, v in got['harmonic_consistency_loss'].items():
    np.testing.assert_allclose(float(v), want['harmonic_consistency_' + k], rtol=1e-5)
  amps, freqs = core.harmonic_to_sinusoidal(*_cuda(harm_amp, harm_dist, f0))
  np.testing.assert_allclose(amps.cpu().numpy(), want['h2s_amps'], rtol=1e-6, atol=1e-7)
  np.testing.assert_allclose(freqs.cpu().numpy(), want['h2s_freqs'], rtol=1e-6)
  rng = np.random.default_rng(5)
  a, b_ = rng.uniform(0, 2, (2, 3, 7)), rng.uniform(0, 2, (2, 3, 7))
  a[0, 0, 0] = 0.0
  w = (rng.uniform(size=(2, 3, 7)) > 0.3).astype(np.float32)
  for log in (False, True):
    np.testing.assert_allclose(float(losses.amp_loss(a, b_, 'L2', log=log)),
                               float(ref.amp_loss(a, b_, 'L2', log=log)), rtol=1e-5)
  np.testing.assert_allclose(
      float(losses.freq_loss(a * 500, b_ * 500, weights=torch.as_tensor(w, device=DEV))),
      float(ref.freq_loss(a * 500, b_ * 500, weights=torch.from_numpy(w).double())),
      rtol=1e-5)
  np.testing.assert_allclose(
      float(losses.FilteredNoiseConsistencyLoss(weight=3.0)(a, b_)),
      3.0 * float(ref.amp_loss(a, b_)), rtol=1e-5)
  pl = losses.ParamLoss(weight=0.5, loss_type='L2', name='p')
  assert list(pl.get_losses_dict(a, b_)) == ['p']
  np.testing.assert_allclose(float(pl(a, b_)), 0.5 * float(ref.amp_loss(a, b_, 'L2')),
                             rtol=1e-5)


def _twm_step(xs, loss):
  for x in xs:
    x.grad = None
  out = loss(*xs)
  out.backward()
  return out.detach().clone(), [x.grad.clone() for x in xs]


@pytest.mark.gpu
def test_backward_is_bit_reproducible():
  x = _twm_case(8, 125, 0, 100, 9)
  xs = _cuda(*x, grad=True)
  loss = losses.TWMLoss()
  first = _twm_step(xs, loss)
  second = _twm_step(xs, loss)
  assert torch.equal(first[0], second[0])
  for a, b in zip(first[1], second[1]):
    assert torch.equal(a, b)
  k = _kde_case(8, 125, 100, 100, 3, {})[0]
  ks = _cuda(*k, grad=True)
  kde = losses.KDEConsistencyLoss()
  first, second = _twm_step(ks, kde), _twm_step(ks, kde)
  assert torch.equal(first[0], second[0])
  for a, b in zip(first[1], second[1]):
    assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize('which', ['twm', 'kde'])
def test_cuda_graph_capture_equals_eager(which):
  if which == 'twm':
    xs = _cuda(*_twm_case(4, 50, 0, 60, 12), grad=True)
    loss = losses.TWMLoss()
  else:
    xs = _cuda(*_kde_case(4, 50, 60, 40, 13, {})[0], grad=True)
    loss = losses.KDEConsistencyLoss()
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    for _ in range(2):
      eager, eager_grads = _twm_step(xs, loss)
  torch.cuda.current_stream().wait_stream(s)
  graph = torch.cuda.CUDAGraph()
  for x in xs:
    x.grad = None
  with torch.cuda.graph(graph):
    static_loss = loss(*xs)
    static_loss.backward()
  graph.replay()
  torch.cuda.synchronize()
  assert torch.equal(static_loss, eager)
  for x, g in zip(xs, eager_grads):
    assert torch.equal(x.grad, g)


@pytest.mark.gpu
def test_twm_memory_has_no_pairwise_tensors():
  """B = 32, T = 125, C = P = 100: the [B, T, C, n_harmonic_points] tensors autograd
  keeps are 16 MB each; the reference's pairwise tensors would be 4.8 GB + 1.6 GB."""
  x = _twm_case(32, 125, 0, 100, 21)
  xs = _cuda(*x, grad=True)
  loss = losses.TWMLoss()
  torch.cuda.synchronize()
  base = torch.cuda.memory_allocated()
  torch.cuda.reset_peak_memory_stats()
  out = loss(*xs)
  out.backward()
  torch.cuda.synchronize()
  rise = torch.cuda.max_memory_allocated() - base
  assert rise < 256 * 2**20, rise / 2**20
  assert all(torch.isfinite(v.grad).all() for v in xs)
