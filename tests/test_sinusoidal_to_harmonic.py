"""core.sinusoidal_to_harmonic (core.py:733-781; csrc/consistency.cuh, mode C): the
float64 restatement against the unmodified reference's fixture, the C ABI's checks, the
Python errors and the zero-size shapes (CPU); the kernels and their gradients against
float64, a known-answer round trip, zero sizes, reproducibility, CUDA-graph capture,
memory, a loss chain and poisoned allocations (GPU).

Tolerances.  Every comparison is elementwise against a bound computed in float64 from
the inputs by running error analysis (`_bounds`), with u = 2^-24 and n-term sums
bounded by n u of the sum of magnitudes.  Per pair (k, s):
  * hf = f0 k is one rounding, |d hf| <= u |f0| k; f - hf and the division by den add
    one each, so q = (f - hf) / den is off by dq <= u (k |f0| / |den| + 3 |q|): the
    harmonic's rounding is relative to f0 k, not to the (small) difference.
  * r = |q| / width and the argument r^2 then carry 2 r dq / |width| + 3 u r^2.  The
    exponent is at most ~104 before exp underflows in float32, so the argument alone
    adds up to ~104 * 3 u relative; expf adds 2 ulp.  So w_ks is within
    eps_ks = 2 r dq / |width| + 3 u r^2 + 2 u relative, plus 3e-45 absolute (a float32
    denormal's spacing, twice).
  * The sums over s and over k, the normalisation, D and the divisions by D add their
    n u terms and the propagated errors of their operands; the gradients repeat the
    same propagation through alpha_k, beta_k and q (see the header comment of mode C).
  * A rounding whose result is a denormal is off by up to 2^-149 absolute, not u
    relative: each product, sum and quotient adds that too.  Pairs whose float32 weight
    is 0 are skipped by the backward; the float64 gradient keeps their (tiny) terms,
    which the 3e-45 absolute error of w covers.
  * The kernels evaluate width as a float32; its representation error rho enters the
    argument as 2 rho r^2 and the gradients' 2 / width^2 as 2 rho.
No factor is fitted to the results: a kernel that passes is within the float32
rounding of the reference's own formula.
"""
import math

import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, autograd, core, losses
from oracle import ref_on_shim
from tests import consistency_ref as cref
from tests import sinusoidal_to_harmonic_ref as ref
from tests.golden import make_sinusoidal_to_harmonic_golden as mg

U = 2.0**-24
TINY = 2.0**-149      # the spacing of float32 denormals: an absolute rounding error
DEN0 = float(np.float32(1e-7))
DEV = 'cuda'


def _fixture():
  return np.load(mg.PATH)


def _case_kw(i):
  _, _, _, _, k, width, sr, norm = mg.CASES[i]
  return dict(harmonic_width=width, n_harmonics=k, sample_rate=sr, normalize=norm)


# ---- CPU ---------------------------------------------------------------------
def test_restatement_matches_the_reference():
  """tests/sinusoidal_to_harmonic_ref.py against the reference run wide on the shim."""
  want = _fixture()
  for i, (name, *_) in enumerate(mg.CASES):
    amp, dist = ref.sinusoidal_to_harmonic(*mg.inputs(i), **_case_kw(i))
    for got, key in ((amp, '_amp_wide'), (dist, '_dist_wide')):
      w = want[name + key]
      assert got.shape == w.shape, name
      assert np.abs(got.numpy() - w).max() <= 1e-12 * max(1.0, np.abs(w).max()), name


@pytest.mark.skipif(not ref_on_shim.available(), reason='reference sources absent')
def test_fixture_regenerates_from_reference():
  mg.compare('sinusoidal_to_harmonic', mg.sinusoidal_to_harmonic(), _fixture())


def test_value_errors_before_device_work(monkeypatch):
  """Shapes, n_harmonics and a zero width raise ValueError and too many sinusoids
  NotImplementedError, before any tensor is moved or the library is loaded."""
  def touched(*a, **k):
    raise AssertionError('device work before the argument checks')
  monkeypatch.setattr(core, 'torch_float32', touched)
  monkeypatch.setattr(core._lib, 'load', touched)
  z = np.zeros((2, 3, 4), np.float32)
  f0 = np.zeros((2, 3, 1), np.float32)
  s2h = core.sinusoidal_to_harmonic
  for call in (lambda: s2h(z, np.zeros((2, 3, 5)), f0),
               lambda: s2h(z[0], z[0], f0[0]),
               lambda: s2h(z, z, np.zeros((2, 3))),
               lambda: s2h(z, z, np.zeros((1, 3, 1))),     # no broadcasting
               lambda: s2h(z, z, np.zeros((2, 3, 4)))):
    with pytest.raises(ValueError, match='must both be'):
      call()
  for bad in (-1, 2.5, True):
    with pytest.raises(ValueError, match='n_harmonics'):
      s2h(z, z, f0, n_harmonics=bad)
  for width in (0.0, -0.0, 1e-50):
    with pytest.raises(ValueError, match='harmonic_width must be nonzero'):
      s2h(z, z, f0, harmonic_width=width)
  big = np.zeros((1, 2, 4097), np.float32)
  with pytest.raises(NotImplementedError, match='4097 sinusoids'):
    s2h(big, big, np.zeros((1, 2, 1)))
  with pytest.raises(ValueError):   # under grad too
    s2h(torch.zeros((2, 3, 4), requires_grad=True), z, np.zeros((2, 3, 2)))


@pytest.mark.parametrize('b,t,s,k', [(0, 3, 4, 5), (2, 0, 4, 5), (2, 3, 0, 5),
                                     (2, 3, 4, 0), (0, 0, 0, 0)])
def test_zero_size_shapes(b, t, s, k):
  """The reference's output shapes, [B, T, 1] and [B, T, K], from static shapes."""
  z = np.zeros((b, t, s), np.float32)
  f0 = np.full((b, t, 1), 200.0, np.float32)
  assert core._sinusoidal_to_harmonic_shapes(z, z, f0, 0.1, k) == (b, t, s, k)
  amp, dist = ref.sinusoidal_to_harmonic(z, z, f0, n_harmonics=k)
  assert tuple(amp.shape) == (b, t, 1) and tuple(dist.shape) == (b, t, k)
  assert not amp.numpy().any() and not dist.numpy().any()


P = 0x1000        # a device pointer the library never dereferences on the host
E_INVALID, E_UNSUPPORTED = _lib.E_INVALID, _lib.E_UNSUPPORTED


def _fwd(a=P, f=P, f0=P, amp=P, dist=P, B=2, T=3, S=5, K=8, w=0.1, sr=16000.0, norm=0):
  return (a, f, f0, amp, dist, B, T, S, K, w, sr, norm, None)


def _bwd(a=P, f=P, f0=P, ga=P, gd=P, da=P, df=P, d0=P, B=2, T=3, S=5, K=8, w=0.1,
         sr=16000.0, norm=0):
  return (a, f, f0, ga, gd, da, df, d0, B, T, S, K, w, sr, norm, None)


_F, _B = 'sinusoidal_to_harmonic', 'sinusoidal_to_harmonic_backward'
_ABI_CASES = [
    ('f-null-a', _F, _fwd(a=None), E_INVALID, b'sinusoidal_to_harmonic: null pointer'),
    ('f-null-f', _F, _fwd(f=None), E_INVALID, b'sinusoidal_to_harmonic: null pointer'),
    ('f-null-f0', _F, _fwd(f0=None), E_INVALID, b'sinusoidal_to_harmonic: null pointer'),
    ('f-null-amp', _F, _fwd(amp=None), E_INVALID, b'sinusoidal_to_harmonic: null pointer'),
    ('f-null-dist', _F, _fwd(dist=None), E_INVALID, b'sinusoidal_to_harmonic: null pointer'),
    ('f-null-f0-s0', _F, _fwd(f0=None, S=0), E_INVALID, b'sinusoidal_to_harmonic: null pointer'),
    ('f-B', _F, _fwd(B=-1), E_INVALID, b'sinusoidal_to_harmonic: bad shape B=-1 T=3 S=5 K=8'),
    ('f-T', _F, _fwd(T=-2), E_INVALID, b'sinusoidal_to_harmonic: bad shape B=2 T=-2 S=5 K=8'),
    ('f-S', _F, _fwd(S=-1), E_INVALID, b'sinusoidal_to_harmonic: bad shape B=2 T=3 S=-1 K=8'),
    ('f-K', _F, _fwd(K=-1), E_INVALID, b'sinusoidal_to_harmonic: bad shape B=2 T=3 S=5 K=-1'),
    ('f-width', _F, _fwd(w=0.0), E_INVALID, b'sinusoidal_to_harmonic: harmonic_width must be nonzero'),
    ('f-norm', _F, _fwd(norm=2), E_INVALID, b'sinusoidal_to_harmonic: normalize must be 0 or 1, got 2'),
    ('f-S-max', _F, _fwd(S=4097), E_UNSUPPORTED, b'sinusoidal_to_harmonic: S=4097 sinusoids exceed the 4096 supported'),
    ('f-grid', _F, _fwd(B=65536, T=32768), E_INVALID, b'sinusoidal_to_harmonic: B*T=2147483648 exceeds the 2^31 - 1 grid limit'),
    ('f-B0', _F, _fwd(B=0), 0, None),
    ('f-T0', _F, _fwd(T=0), 0, None),
    ('f-empty-null', _F, _fwd(None, None, None, None, None, B=0), 0, None),
    ('f-S-4096-empty', _F, _fwd(T=0, S=4096), 0, None),
    ('b-null-ga', _B, _bwd(ga=None), E_INVALID, b'sinusoidal_to_harmonic_backward: null pointer'),
    ('b-null-gd', _B, _bwd(gd=None), E_INVALID, b'sinusoidal_to_harmonic_backward: null pointer'),
    ('b-null-da', _B, _bwd(da=None), E_INVALID, b'sinusoidal_to_harmonic_backward: null pointer'),
    ('b-null-df', _B, _bwd(df=None), E_INVALID, b'sinusoidal_to_harmonic_backward: null pointer'),
    ('b-null-d0', _B, _bwd(d0=None), E_INVALID, b'sinusoidal_to_harmonic_backward: null pointer'),
    ('b-null-d0-k0', _B, _bwd(d0=None, K=0, S=0), E_INVALID, b'sinusoidal_to_harmonic_backward: null pointer'),
    ('b-S', _B, _bwd(S=-3), E_INVALID, b'sinusoidal_to_harmonic_backward: bad shape B=2 T=3 S=-3 K=8'),
    ('b-width', _B, _bwd(w=-0.0), E_INVALID, b'sinusoidal_to_harmonic_backward: harmonic_width must be nonzero'),
    ('b-norm', _B, _bwd(norm=-1), E_INVALID, b'sinusoidal_to_harmonic_backward: normalize must be 0 or 1, got -1'),
    ('b-S-max', _B, _bwd(S=8192), E_UNSUPPORTED, b'sinusoidal_to_harmonic_backward: S=8192 sinusoids exceed the 4096 supported'),
    ('b-grid', _B, _bwd(B=1 << 20, T=1 << 12), E_INVALID, b'sinusoidal_to_harmonic_backward: B*T=4294967296 exceeds the 2^31 - 1 grid limit'),
    ('b-B0', _B, _bwd(B=0), 0, None),
    ('b-empty-null', _B, _bwd(*([None] * 8), T=0), 0, None),
]


@pytest.mark.parametrize('fn,args,want,msg', [c[1:] for c in _ABI_CASES],
                         ids=[c[0] for c in _ABI_CASES])
def test_abi_check_table(fn, args, want, msg):
  """Every check of the two entry points: the status and the full message come back
  before any CUDA call, and nothing is launched."""
  lib = _lib.load()
  launches = lib.ddsp_b200_launch_count()
  assert getattr(lib, 'ddsp_b200_' + fn)(*args) == want
  assert lib.ddsp_b200_launch_count() == launches
  if msg is not None:
    assert lib.ddsp_b200_last_error() == msg


def test_no_workspace():
  """Neither entry point takes a workspace or has a query."""
  names = [n for n in _lib.SIGNATURES if 'sinusoidal_to_harmonic' in n]
  assert sorted(names) == ['ddsp_b200_sinusoidal_to_harmonic',
                           'ddsp_b200_sinusoidal_to_harmonic_backward']
  for n in names:
    assert _lib.SIGNATURES[n][1][-2] is not _lib._sz


# ---- the bounds ------------------------------------------------------------------------
def _bounds(a, f, f0, harmonic_width=0.1, n_harmonics=100, sample_rate=16000,
            normalize=False, g_amp=None, g_dist=None):
  """float64 forward values with their float32 error bounds (see the module docstring),
  and, given upstream gradients, the bounds of d a, d f and d f0.  Returns a dict."""
  a, f, f0 = (np.asarray(v, np.float64) for v in (a, f, f0))
  K, w_ = n_harmonics, float(np.float32(harmonic_width))
  rho = abs(w_ - harmonic_width) / abs(harmonic_width)    # the width as a float32
  S = a.shape[-1]
  k = np.arange(1, K + 1, dtype=np.float64)[None, None, :, None]       # [1,1,K,1]
  f0_ = f0[..., None]                                                   # [B,T,1,1]
  den = np.where(f0_ == 0.0, DEN0, f0_)
  hf = f0_ * k
  q = (f[:, :, None, :] - hf) / den                                     # [B,T,K,S]
  dq = U * (k * np.abs(f0_) / np.abs(den) + 3.0 * np.abs(q))
  r = np.abs(q) / abs(w_)
  w = np.exp(-r * r)
  eps = 2.0 * r * dq / abs(w_) + (3.0 * U + 2.0 * rho) * r * r + 2.0 * U
  dw = w * eps + 3e-45
  a4 = a[:, :, None, :]
  sw = w.sum(-1)
  swa = (w * a4).sum(-1)
  dsw = dw.sum(-1) + S * U * sw + S * TINY
  dswa = (dw * np.abs(a4)).sum(-1) + S * U * (w * np.abs(a4)).sum(-1) + S * TINY
  sel = (sw > 1.0) if normalize else np.zeros(sw.shape, bool)
  sw_sel = np.where(sel, sw, 1.0)
  hp = swa / sw_sel
  dhp = np.where(sel, dswa / sw_sel + np.abs(hp) * dsw / sw_sel + U * np.abs(hp), dswa)
  masked = hf[..., 0] >= sample_rate / 2.0
  ha = np.where(masked, 0.0, hp)
  dha = np.where(masked, 0.0, dhp)
  D = ha.sum(-1, keepdims=True)
  dD = dha.sum(-1, keepdims=True) + (K + 128) * U * np.abs(ha).sum(-1, keepdims=True)
  Ds = np.where(D == 0.0, DEN0, D)
  dist = ha / Ds
  ddist = dha / np.abs(Ds) + np.abs(ha) * dD / Ds**2 + U * np.abs(dist) + TINY
  out = dict(amp=D, d_amp=dD, dist=dist, d_dist=ddist)
  if g_amp is None:
    return out
  ga, gd = np.asarray(g_amp, np.float64), np.asarray(g_dist, np.float64)
  nz = D != 0.0
  rel_D = np.where(nz, dD / np.where(nz, np.abs(D), 1.0), 0.0)
  # dHA_k = g_A + (g_k - Gd) / Ds, Gd = sum_j g_j HA_j / Ds (0 where D = 0)
  Gd_mag = np.where(nz, (np.abs(gd) * np.abs(ha)).sum(-1, keepdims=True) / np.abs(Ds), 0.0)
  dGd = np.where(nz, ((np.abs(gd) * dha).sum(-1, keepdims=True) / np.abs(Ds)
                      + (K + 128 + 1) * U * Gd_mag + rel_D * Gd_mag
                      + (K + 128) * TINY * (1.0 + np.abs(gd).sum(-1, keepdims=True))), 0.0)
  num_mag = np.abs(gd) + Gd_mag
  dha_mag = np.abs(ga) + num_mag / np.abs(Ds)                           # [B,T,K]
  d_dha = (dGd + U * num_mag) / np.abs(Ds) + num_mag / np.abs(Ds) * (rel_D + U) + U * dha_mag
  al_mag = np.where(masked, 0.0, dha_mag / sw_sel)
  d_al = np.where(masked, 0.0, np.where(sel, d_dha / sw_sel + al_mag * (dsw / sw_sel + U),
                                        d_dha))
  be = np.where(sel, hp, 0.0)
  d_be = np.where(sel, dhp, 0.0)
  al4, dal4, be4, dbe4 = (x[..., None] for x in (al_mag, d_al, be, d_be))
  amb = np.abs(a4 - be4)
  # d a_s = sum_k alpha w
  da_err = (dal4 * w + al4 * dw).sum(-2) + K * U * (al4 * w).sum(-2)
  # T_ks = alpha (a - beta) w q and its bound
  t_mag = al4 * amb * w * np.abs(q)
  t_err = (dal4 * amb * w * np.abs(q) + al4 * amb * (dw * np.abs(q) + w * dq)
           + al4 * w * np.abs(q) * (dbe4 + U * amb) + 4 * U * t_mag
           + TINY * (np.abs(q) + 1.0))       # products that land among the denormals
  k2 = 2.0 / (w_ * w_)
  scale_err = 4 * U + 2 * rho          # k2 / den in float32, from the float32 width
  den3 = np.abs(den[..., 0])                                            # [B,T,1]
  df_err = (k2 / den3 * (t_err.sum(-2) + (K + 1) * U * t_mag.sum(-2)
                         + scale_err * t_mag.sum(-2)) + TINY * (1.0 + 1.0 / den3))
  kq = np.abs(k + np.where(f0_ != 0.0, q, 0.0))
  n_f0 = math.ceil(S / 128) * K + 128
  f0_mag = (t_mag * kq).sum((-2, -1))[..., None]
  df0_err = (k2 / den3 * ((t_err * kq + t_mag * (dq + U * kq)).sum((-2, -1))[..., None]
                          + (n_f0 + 1) * (U * f0_mag + TINY) + scale_err * f0_mag)
             + TINY * (1.0 + 1.0 / den3))
  out.update(da=da_err + K * TINY, df=df_err, df0=df0_err)
  return out


def _check(what, got, want, tol):
  got = got.detach().cpu().numpy().astype(np.float64) if torch.is_tensor(got) else got
  want = want.detach().cpu().numpy() if torch.is_tensor(want) else np.asarray(want)
  assert got.shape == want.shape, (what, got.shape, want.shape)
  err = np.abs(got - want)
  bad = ~(err <= tol)
  assert not bad.any(), (what, int(bad.sum()), got[bad][:4], want[bad][:4], tol[bad][:4])


def _cuda(*xs, grad=False):
  return [torch.as_tensor(np.asarray(x, np.float32), device=DEV).requires_grad_(grad)
          for x in xs]


# ---- GPU ---------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('i', range(len(mg.CASES)), ids=[c[0] for c in mg.CASES])
def test_forward_fixture_cases(i):
  name = mg.CASES[i][0]
  want = _fixture()
  x = mg.inputs(i)
  kw = _case_kw(i)
  amp, dist = core.sinusoidal_to_harmonic(*x, **kw)
  assert amp.dtype == torch.float32 and amp.device.type == 'cuda'
  b = _bounds(*x, **kw)
  _check(name + ' amp', amp, want[name + '_amp_wide'], b['d_amp'])
  _check(name + ' dist', dist, want[name + '_dist_wide'], b['d_dist'])


# (name, B, T, S, K, width, sample_rate, normalize): the fixture's regimes plus K = 257
# (two harmonic chunks of the backward) and S = 4096 (the staging limit)
GRAD_CASES = [c[:1] + (None,) * 3 + c[4:] for c in mg.CASES] + [
    ('k257', 2, 3, 100, 257, 0.1, 44100, False),
    ('k257_norm', 2, 3, 100, 257, 0.03, 16000, True),
    ('s4096', 1, 3, 4096, 100, 0.1, 16000, False),
    ('s4096_norm', 1, 3, 4096, 257, 1.0, 44100, True),
]


def _grad_inputs(j):
  name, b, t, s, k, width, sr, norm = GRAD_CASES[j]
  if b is None:
    i = [c[0] for c in mg.CASES].index(name)
    return mg.inputs(i), _case_kw(i)
  return mg.inputs(100 + j, b, t, s), dict(harmonic_width=width, n_harmonics=k,
                                           sample_rate=sr, normalize=norm)


@pytest.mark.gpu
@pytest.mark.parametrize('j', range(len(GRAD_CASES)), ids=[c[0] for c in GRAD_CASES])
def test_gradients_against_float64(j):
  """d sin_amps, d sin_freqs and d f0 against float64 autograd of the restatement, for
  random upstream gradients of both outputs.  The inputs hold f0 = 0, harmonics above
  Nyquist, sinusoids on harmonics, 0 Hz sinusoids and an all-zero amplitude frame, whose
  d harm_dist reaches the harmonics times 1e7."""
  x, kw = _grad_inputs(j)
  xs = _cuda(*x, grad=True)
  amp, dist = core.sinusoidal_to_harmonic(*xs, **kw)
  rng = np.random.default_rng(j)
  ga = rng.normal(size=amp.shape).astype(np.float32)
  gd = rng.normal(size=dist.shape).astype(np.float32)
  torch.autograd.backward([amp, dist], _cuda(ga, gd))
  x64 = [torch.from_numpy(v.astype(np.float64)).requires_grad_(True) for v in x]
  a64, d64 = ref.sinusoidal_to_harmonic(*x64, **kw)
  torch.autograd.backward([a64, d64], [torch.from_numpy(ga).double(),
                                       torch.from_numpy(gd).double()])
  b = _bounds(*x, **kw, g_amp=ga, g_dist=gd)
  _check('amp', amp, a64, b['d_amp'])
  _check('dist', dist, d64, b['d_dist'])
  for n, got, want, tol in zip(('d sin_amps', 'd sin_freqs', 'd f0'), xs, x64,
                               (b['da'], b['df'], b['df0'])):
    _check(n, got.grad, want.grad, tol)
  assert xs[2].grad[0, 0, 0].item() == 0.0 or x[2][0, 0, 0] != 0.0   # f0 = 0 frame


@pytest.mark.gpu
@pytest.mark.parametrize('sr', [16000, 44100])
def test_round_trip_through_harmonic_to_sinusoidal(sr):
  """Known answer, no restatement: sinusoids placed on the harmonics by
  harmonic_to_sinusoidal come back as the amplitude and the distribution renormalised
  over the harmonics below Nyquist.  A neighbour's weight is exp(-100) ~ 4e-44 (a
  float32 denormal), far below the results' resolution; the sums of K terms give the
  bound."""
  rng = np.random.default_rng(sr)
  b, t, k = 3, 50, 100
  a = rng.uniform(0.1, 2.0, (b, t, 1)).astype(np.float32)
  d = rng.uniform(0.0, 1.0, (b, t, k)).astype(np.float32)
  f0 = np.exp(rng.uniform(np.log(60.0), np.log(sr / 4.0), (b, t, 1))).astype(np.float32)
  ag, dg, f0g = _cuda(a, d, f0)
  amps, freqs = core.harmonic_to_sinusoidal(ag, dg, f0g, sample_rate=sr)
  amp, dist = core.sinusoidal_to_harmonic(amps, freqs, f0g, n_harmonics=k, sample_rate=sr)
  below = (f0.astype(np.float64) * np.arange(1, k + 1) < sr / 2.0)
  dn = np.where(below, d, 0.0)
  dn = dn / dn.sum(-1, keepdims=True)
  tol = (2 * k + 8) * U
  _check('harm_amp', amp, a.astype(np.float64), tol * a)
  _check('harm_dist', dist, dn, tol * dn + 1e-30)


def _poisoned_zero_grads(b, t, s, k):
  torch.full((1 << 16,), math.nan, device=DEV)      # freed NaN memory first
  x = mg.inputs(0, b, t, s) if b * t else [np.zeros((b, t, n), np.float32) for n in (s, s, 1)]
  xs = _cuda(*x, grad=True)
  amp, dist = core.sinusoidal_to_harmonic(*xs, n_harmonics=k)
  assert tuple(amp.shape) == (b, t, 1) and tuple(dist.shape) == (b, t, k)
  (amp.sum() + dist.sum()).backward()
  return amp, dist, xs


@pytest.mark.gpu
@pytest.mark.parametrize('b,t,s,k', [(0, 3, 4, 5), (2, 0, 4, 5), (2, 3, 0, 5), (2, 3, 4, 0),
                                     (2, 3, 0, 0)])
def test_zero_sizes(b, t, s, k):
  """The reference's shapes; S = 0 writes zero outputs and every gradient buffer is
  written, zeros where nothing contributes (d f0 at S = 0, everything at K = 0)."""
  amp, dist, xs = _poisoned_zero_grads(b, t, s, k)
  if s == 0 or k == 0:
    assert torch.equal(amp, torch.zeros_like(amp)) and torch.equal(dist, torch.zeros_like(dist))
  for x in xs:
    assert x.grad is not None and x.grad.shape == x.shape
    if s == 0 or k == 0:
      assert torch.equal(x.grad, torch.zeros_like(x.grad)), x.grad


_BIG = (32, 1000, 100, 100)


def _big_inputs(seed):
  b, t, s, _ = _BIG
  return _cuda(*mg.inputs(seed, b, t, s), grad=True)


def _step(xs, normalize, g=None):
  for x in xs:
    x.grad = None
  amp, dist = core.sinusoidal_to_harmonic(*xs, n_harmonics=_BIG[3], normalize=normalize)
  (amp.sum() + (dist * (g if g is not None else 1.0)).sum()).backward()
  return [amp.detach().clone(), dist.detach().clone()] + [x.grad.clone() for x in xs]


@pytest.mark.gpu
@pytest.mark.parametrize('normalize', [False, True])
def test_backward_is_bit_reproducible(normalize):
  xs = _big_inputs(7)
  g = torch.randn((_BIG[0], _BIG[1], _BIG[3]), device=DEV,
                  generator=torch.Generator(DEV).manual_seed(3))
  first, second = _step(xs, normalize, g), _step(xs, normalize, g)
  for a, b in zip(first, second):
    assert torch.equal(a, b)


@pytest.mark.gpu
def test_cuda_graph_capture_equals_eager():
  xs = _cuda(*mg.inputs(8, 4, 50, 60), grad=True)
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    for _ in range(2):
      eager = _step(xs, True)
  torch.cuda.current_stream().wait_stream(s)
  graph = torch.cuda.CUDAGraph()
  for x in xs:
    x.grad = None
  with torch.cuda.graph(graph):
    amp, dist = core.sinusoidal_to_harmonic(*xs, n_harmonics=_BIG[3], normalize=True)
    (amp.sum() + dist.sum()).backward()
  graph.replay()
  torch.cuda.synchronize()
  assert torch.equal(amp, eager[0]) and torch.equal(dist, eager[1])
  for x, g in zip(xs, eager[2:]):
    assert torch.equal(x.grad, g)


@pytest.mark.gpu
def test_memory_has_no_pairwise_tensors():
  """B = 32, T = 1000, S = K = 100 under grad: one [B, T, K, S] tensor would be
  1.28 GB; the outputs and gradients are 12.9 MB + 25.6 MB."""
  xs = _big_inputs(9)
  torch.cuda.synchronize()
  base = torch.cuda.memory_allocated()
  torch.cuda.reset_peak_memory_stats()
  amp, dist = core.sinusoidal_to_harmonic(*xs, n_harmonics=_BIG[3])
  (amp.sum() + dist.sum()).backward()
  torch.cuda.synchronize()
  rise = torch.cuda.max_memory_allocated() - base
  assert rise < 64 * 2**20, rise / 2**20
  assert all(torch.isfinite(x.grad).all() for x in xs)


@pytest.mark.gpu
def test_harmonic_consistency_chain():
  """sinusoids -> sinusoidal_to_harmonic -> HarmonicConsistencyLoss -> backward.  The
  loss is torch on both sides; the d harm_amp and d harm_dist it sends back are fed to
  the float64 restatement's backward, and the sinusoids' and f0's gradients compared
  within the bounds of those upstream gradients."""
  x = mg.inputs(11, 4, 30, 40)
  xs = _cuda(*x, grad=True)
  amp, dist = core.sinusoidal_to_harmonic(*xs, n_harmonics=60)
  amp.retain_grad()
  dist.retain_grad()
  rng = np.random.default_rng(12)
  amp_t = rng.uniform(0.0, 3.0, amp.shape).astype(np.float32)
  amp_t[0, :3] = 0.0                                   # below amp_threshold
  dist_t = rng.uniform(0.0, 1.0, dist.shape).astype(np.float32)
  f0_t = (x[2] * np.float32(1.01)).astype(np.float32)
  hc = losses.HarmonicConsistencyLoss(amp_weight=0.5, dist_weight=2.0, f0_weight=1.5)
  terms = hc(amp, amp_t, dist, dist_t, xs[2], f0_t)
  sum(terms.values()).backward()
  x64 = [torch.from_numpy(v.astype(np.float64)).requires_grad_(True) for v in x]
  a64, d64 = ref.sinusoidal_to_harmonic(*x64, n_harmonics=60)
  want = cref.harmonic_consistency(a64, amp_t, d64, dist_t, x64[2], f0_t, amp_weight=0.5,
                                   dist_weight=2.0, f0_weight=1.5)
  for key, v in terms.items():
    assert abs(v.item() - want[key].item()) <= 1e-4 * max(1.0, abs(want[key].item())), key
  ga, gd = amp.grad.cpu().numpy(), dist.grad.cpu().numpy()
  x64 = [torch.from_numpy(v.astype(np.float64)).requires_grad_(True) for v in x]
  a64, d64 = ref.sinusoidal_to_harmonic(*x64, n_harmonics=60)
  torch.autograd.backward([a64, d64], [torch.from_numpy(ga).double(),
                                       torch.from_numpy(gd).double()])
  b = _bounds(*x, n_harmonics=60, g_amp=ga, g_dist=gd)
  _check('d sin_amps', xs[0].grad, x64[0].grad, b['da'])
  _check('d sin_freqs', xs[1].grad, x64[1].grad, b['df'])
  # f0 also reaches the loss directly through freq_loss, in torch: take that part out
  f0_leaf = xs[2].detach().clone().requires_grad_(True)
  sum(hc(amp.detach(), amp_t, dist.detach(), dist_t, f0_leaf, f0_t).values()).backward()
  direct = f0_leaf.grad.cpu().numpy().astype(np.float64)
  total = xs[2].grad.cpu().numpy().astype(np.float64)
  _check('d f0', total - direct, x64[2].grad, b['df0'] + 2 * U * (np.abs(direct) + np.abs(total)))


@pytest.mark.gpu
@pytest.mark.parametrize('b,t,s,k,norm', [(2, 3, 5, 8, False), (3, 4, 100, 257, True),
                                          (2, 3, 0, 5, False), (2, 3, 4, 0, True),
                                          (1, 2, 4096, 3, False)])
def test_under_every_poison(b, t, s, k, norm):
  """Forward and backward under the guarded allocator of test_gpu_memory_bounds.py:
  fences intact and bit-identical results whatever the fresh memory holds."""
  from tests.test_gpu_memory_bounds import POISONS, guarded
  x = mg.inputs(13, b, t, s)
  g = np.random.default_rng(14).normal(size=(b, t, k)).astype(np.float32)
  runs = []
  for p in POISONS:
    with guarded(p):
      xs = _cuda(*x, grad=True)
      amp, dist = core.sinusoidal_to_harmonic(*xs, n_harmonics=k, normalize=norm)
      torch.autograd.backward([amp, dist], [torch.ones_like(amp), *_cuda(g)])
      runs.append([amp.detach().clone(), dist.detach().clone()] +
                  [v.grad.clone() for v in xs])
  for run in runs[1:]:
    for got, want in zip(run, runs[0]):
      assert torch.equal(got.view(torch.int32), want.view(torch.int32))
  assert all(torch.isfinite(v).all() for v in runs[0])
