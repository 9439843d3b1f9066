"""losses.wasserstein_distance, losses.WassersteinConsistencyLoss (csrc/wasserstein.cuh)
and losses.LossGroup: argument checks, the C entry points, the float64 restatement and
LossGroup's plumbing on the CPU; the kernels against the restatement, ties, NaN
propagation, the loss end to end, reproducibility, CUDA graphs, streams, devices,
poisoned and fenced memory on the GPU.  Reference: tests/wasserstein_ref.py, pinned to
the unmodified reference by tests/golden/wasserstein.npz.

Tolerances, for the kernel against float64 on the same float32 inputs.

* D.  Every D_j is one value of a float32 scan of the signed weights in sorted order: a
  run of at most L = 16 serial additions per thread, 5 warp-shuffle levels, at most 15
  serial additions of warp totals and the final prefix add, so at most 38 additions.
  Every partial sum along the way is a sum of contiguous signed weights, the difference
  of two prefixes, so at most 2 Pmax in size (Pmax the row's largest |prefix|, in
  float64).  So |D_err| <= e_D = 38 * 2^-24 * 2 Pmax (first order); 40 is used.
* c = |D|^p moves by e_D at p = 1, by p (|D| + e_D)^(p-1) e_D at p > 1 and by at most
  e_D^p at p < 1 (|D|^p is subadditive); powf adds 4 ulp of c.  delta is one rounding.
* S = sum delta c: sum_i delta_i (dc_i + 2^-20 c_i) plus the summation's own 38
  roundings of at most S; the distance S^(1/p) is checked within the float64 image of
  [S - e_S, S + e_S] plus 4 ulp for powf.
* Gradients.  The value gradient G (c_{j-1} - c_j) and the weight gradients (suffix sums
  of g = G delta p |D|^(p-1) sgn D) inherit these relative errors; each is compared
  normwise (|got - want|_2 <= 1e-4 |want|_2 + atol) and elementwise within
  5e-3 |want| + 1e-3 max |want| + atol, where atol covers a sign of D that the scan's
  error could flip: 2 |G delta_i| summed over the |D_i| <= e_D.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, core, losses
from tests import wasserstein_ref as ref
from tests.golden import make_wasserstein_golden as wg
from tests.test_launch import Recorder

P = 0x1000        # a device pointer the library never dereferences on the host
E_INVALID, E_UNSUPPORTED = _lib.E_INVALID, _lib.E_UNSUPPORTED
DEV = 'cuda'
K_SCAN = 40


# ---- CPU: the restatement and the fixture --------------------------------------------
def _rel_close(got, want, rtol=1e-9):
  got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
  assert got.shape == want.shape, (got.shape, want.shape)
  assert np.all(np.abs(got - want) <= rtol * (1.0 + np.abs(want))), (got, want)


def test_restatement_matches_the_reference():
  """tests/wasserstein_ref.py against the unmodified reference run wide on the shim, at
  1e-9 relative, over every case of the fixture."""
  want = np.load(wg.PATH)
  for i, (name, batch, *_, p, _) in enumerate(wg.DISTANCE_CASES):
    got = ref.wasserstein_distance(*wg.distance_inputs(i), p=p).numpy()
    assert got.shape == batch
    _rel_close(got, want[name])
  for i, (name, *_, w, m) in enumerate(wg.LOSS_CASES):
    _rel_close(ref.wasserstein_consistency(*wg.loss_inputs(i), weight=w, midi=m).numpy(),
               want[name])


def test_fixture_regenerates():
  """Where the reference is checked out, the fixture is what it computes."""
  from oracle import ref_on_shim
  try:
    ref_on_shim.load()
  except Exception as e:  # pylint: disable=broad-except
    pytest.skip('reference sources not available: %s' % e)
  from tests.golden.make_golden import compare
  compare('wasserstein', wg.wasserstein(), np.load(wg.PATH))


# ---- CPU: the C entry points ---------------------------------------------------------
def _wf(u=P, v=P, wu=P, wv=P, out=P, R=6, Nu=10, Nv=7, p=1.0):
  return (u, v, wu, wv, out, R, Nu, Nv, p, None)


def _wb(u=P, v=P, wu=P, wv=P, g=P, du=P, dv=P, dwu=P, dwv=P, R=6, Nu=10, Nv=7, p=1.0):
  return (u, v, wu, wv, g, du, dv, dwu, dwv, R, Nu, Nv, p, None)


_WF, _WB = 'wasserstein_forward', 'wasserstein_backward'
_ABI_CASES = [
    ('wf-null-u', _WF, _wf(u=None), E_INVALID, b'wasserstein_forward: null pointer'),
    ('wf-null-v', _WF, _wf(v=None), E_INVALID, b'wasserstein_forward: null pointer'),
    ('wf-null-wu', _WF, _wf(wu=None), E_INVALID, b'wasserstein_forward: null pointer'),
    ('wf-null-wv', _WF, _wf(wv=None), E_INVALID, b'wasserstein_forward: null pointer'),
    ('wf-null-out', _WF, _wf(out=None), E_INVALID, b'wasserstein_forward: null pointer'),
    ('wf-R', _WF, _wf(R=-1), E_INVALID, b'wasserstein_forward: bad shape R=-1 Nu=10 Nv=7'),
    ('wf-Nu', _WF, _wf(Nu=-2), E_INVALID, b'wasserstein_forward: bad shape R=6 Nu=-2 Nv=7'),
    ('wf-Nv', _WF, _wf(Nv=-1), E_INVALID, b'wasserstein_forward: bad shape R=6 Nu=10 Nv=-1'),
    ('wf-p0', _WF, _wf(p=0.0), E_INVALID, b'wasserstein_forward: p must be positive and finite, got 0'),
    ('wf-p-neg', _WF, _wf(p=-1.0), E_INVALID, b'wasserstein_forward: p must be positive and finite, got -1'),
    ('wf-p-nan', _WF, _wf(p=math.nan), E_INVALID, b'wasserstein_forward: p must be positive and finite, got nan'),
    ('wf-p-inf', _WF, _wf(p=math.inf), E_INVALID, b'wasserstein_forward: p must be positive and finite, got inf'),
    ('wf-Nu-max', _WF, _wf(Nu=4097), E_UNSUPPORTED, b'wasserstein_forward: Nu=4097 or Nv=7 elements exceed the 4096 supported per side'),
    ('wf-Nv-max', _WF, _wf(Nv=5000), E_UNSUPPORTED, b'wasserstein_forward: Nu=10 or Nv=5000 elements exceed the 4096 supported per side'),
    ('wf-grid', _WF, _wf(R=1 << 31), E_INVALID, b'wasserstein_forward: R=2147483648 exceeds the 2^31 - 1 grid limit'),
    ('wf-R0', _WF, _wf(R=0), 0, None),
    ('wf-Nu0', _WF, _wf(Nu=0), 0, None),
    ('wf-Nv0', _WF, _wf(Nv=0), 0, None),
    ('wf-4096', _WF, _wf(R=0, Nu=4096, Nv=4096), 0, None),
    ('wf-empty-null', _WF, _wf(u=None, v=None, wu=None, wv=None, out=None, R=0), 0, None),
    ('wb-null-g', _WB, _wb(g=None), E_INVALID, b'wasserstein_backward: null pointer'),
    ('wb-null-du', _WB, _wb(du=None), E_INVALID, b'wasserstein_backward: null pointer'),
    ('wb-null-dv', _WB, _wb(dv=None), E_INVALID, b'wasserstein_backward: null pointer'),
    ('wb-null-dwu', _WB, _wb(dwu=None), E_INVALID, b'wasserstein_backward: null pointer'),
    ('wb-null-dwv', _WB, _wb(dwv=None), E_INVALID, b'wasserstein_backward: null pointer'),
    ('wb-R', _WB, _wb(R=-3), E_INVALID, b'wasserstein_backward: bad shape R=-3 Nu=10 Nv=7'),
    ('wb-p', _WB, _wb(p=-0.5), E_INVALID, b'wasserstein_backward: p must be positive and finite, got -0.5'),
    ('wb-Nu-max', _WB, _wb(Nu=8192), E_UNSUPPORTED, b'wasserstein_backward: Nu=8192 or Nv=7 elements exceed the 4096 supported per side'),
    ('wb-grid', _WB, _wb(R=1 << 40), E_INVALID, b'wasserstein_backward: R=1099511627776 exceeds the 2^31 - 1 grid limit'),
    ('wb-R0', _WB, _wb(R=0), 0, None),
    ('wb-Nv0', _WB, _wb(Nv=0), 0, None),
    ('wb-empty-null', _WB, _wb(*([None] * 9), R=0), 0, None),
]


@pytest.mark.parametrize('fn,args,want,msg', [c[1:] for c in _ABI_CASES],
                         ids=[c[0] for c in _ABI_CASES])
def test_wasserstein_abi_check_table(fn, args, want, msg):
  """Every check of the two entry points: the status and the full message come back
  before any CUDA call, and nothing is launched."""
  lib = _lib.load()
  launches = lib.ddsp_b200_launch_count()
  assert getattr(lib, 'ddsp_b200_' + fn)(*args) == want
  assert lib.ddsp_b200_launch_count() == launches
  if msg is not None:
    assert lib.ddsp_b200_last_error() == msg


def test_entry_points_take_no_workspace():
  for name in ('ddsp_b200_wasserstein_forward', 'ddsp_b200_wasserstein_backward'):
    args = _lib.SIGNATURES[name][1]
    assert ctypes.c_size_t not in args, name
    assert args[5 if name.endswith('forward') else 9] is ctypes.c_int64, name
  assert not any(n.startswith('ddsp_b200_wasserstein') and n.endswith('_workspace')
                 for n in _lib.SIGNATURES)


@pytest.fixture
def recorder(monkeypatch):
  rec = Recorder()
  monkeypatch.setattr(_lib, 'load', lambda: rec)
  return rec


def test_errors_before_the_library_is_looked_up(recorder, monkeypatch):
  def fail(*a, **k):
    raise AssertionError('device work before the argument checks')
  monkeypatch.setattr(core, 'torch_float32', fail)
  z = np.zeros((2, 3, 4), np.float32)
  z5 = np.zeros((2, 3, 5), np.float32)
  wd = losses.wasserstein_distance
  cases = [
      (ValueError, 'weights are required', lambda: wd(z, z, None, z)),
      (ValueError, 'weights are required', lambda: wd(z, z, z, None)),
      (ValueError, r'u_values \(2, 3, 4\) and u_weights \(2, 3, 5\)', lambda: wd(z, z, z5, z)),
      (ValueError, r'v_values \(2, 3, 5\) and v_weights \(2, 3, 4\)', lambda: wd(z, z5, z, z)),
      (ValueError, 'must be one shape', lambda: wd(np.float32(1), z, np.float32(1), z)),
      (ValueError, r'u has batch shape \(2, 3\), v \(2, 4\)',
       lambda: wd(z, np.zeros((2, 4, 4)), z, np.zeros((2, 4, 4)))),
      (ValueError, 'n_u=0', lambda: wd(z[..., :0], z, z[..., :0], z)),
      (ValueError, 'n_v=0', lambda: wd(z, z[..., :0], z, z[..., :0])),
      (ValueError, 'p must be positive and finite, got 0.0', lambda: wd(z, z, z, z, p=0.0)),
      (ValueError, 'p must be positive and finite, got -2.0', lambda: wd(z, z, z, z, p=-2)),
      (ValueError, 'p must be positive and finite, got nan', lambda: wd(z, z, z, z, p=math.nan)),
      (ValueError, 'p must be positive and finite, got inf', lambda: wd(z, z, z, z, p=math.inf)),
      (NotImplementedError, 'n_u=4097',
       lambda: wd(np.zeros((1, 4097)), z[0, :1], np.zeros((1, 4097)), z[0, :1])),
      (NotImplementedError, 'n_v=5000',
       lambda: wd(z[0, :1], np.zeros((1, 5000)), z[0, :1], np.zeros((1, 5000)))),
      (ValueError, 'amps_a, freqs_a must be two',
       lambda: losses.WassersteinConsistencyLoss()(z, z5, z, z)),
      (ValueError, r'amps_b, freqs_b has \[batch, time\] \(2, 4\)',
       lambda: losses.WassersteinConsistencyLoss()(z, z, np.zeros((2, 4, 4)),
                                                   np.zeros((2, 4, 4)))),
      (ValueError, 'amps_b, freqs_b must be two',
       lambda: losses.WassersteinConsistencyLoss(weight=0.0)(z, z, z[0], z[0])),
  ]
  for exc, msg, call in cases:
    with pytest.raises(exc, match=msg):
      call()
  assert recorder.looked_up == []


def test_rows_over_the_grid_limit_raise_before_device_work(recorder, monkeypatch):
  class Shaped:
    def __init__(self, shape):
      self.shape = shape
  monkeypatch.setattr(core, 'torch_float32', None)
  big = Shaped((1 << 16, 1 << 15, 3))
  with pytest.raises(NotImplementedError, match='2147483648 rows exceed'):
    losses.wasserstein_distance(big, big, big, big)
  assert recorder.looked_up == []


def test_loss_without_weight_or_midi_is_plain_zero(recorder):
  x = np.ones((2, 3, 4), np.float32)
  for w, m in ((0.0, True), (-1.0, True), (1.0, False), (0.3, False)):
    got = losses.WassersteinConsistencyLoss(weight=w, midi=m)(x, x, x, x)
    assert got == 0.0 and isinstance(got, float)
  assert recorder.looked_up == []
  assert losses.WassersteinConsistencyLoss().name == 'wasserstein_consistency_loss'
  assert losses.WassersteinConsistencyLoss(name='w').name == 'w'


# ---- CPU: LossGroup ------------------------------------------------------------------
RECON_DAG = [
    ['synth_spectral_loss', ['audio', 'synth_audio']],
    ['f0_loss', ['f0_midi', 'f0_midi_pred', 'f0_loss_weights']],
    ['amps_loss', ['amps', 'amps_pred']],
    ['hd_loss', ['hd', 'hd_pred']],
    ['noise_loss', ['noise', 'noise_pred']],
]


def _recon_losses(spectral):
  """The keyword losses of gin/models/midiae/mixins/recon_lossgroup.gin."""
  return dict(
      amps_loss=losses.ParamLoss(weight=0.5, loss_type='L1', name='amplitude_reconstruction'),
      f0_loss=losses.ParamLoss(weight=50.0, loss_type='L2', name='f0_reconstruction'),
      hd_loss=losses.ParamLoss(weight=500.0, loss_type='L1',
                               name='harmonic_distribution_reconstruction'),
      noise_loss=losses.ParamLoss(weight=0.5, loss_type='L1', name='noise_reconstruction'),
      synth_spectral_loss=spectral)


def _recon_outputs(device, n_samples=4096):
  g = torch.Generator().manual_seed(3)
  r = lambda *s: torch.rand(*s, generator=g).to(device)
  return {'audio': r(2, n_samples), 'synth_audio': r(2, n_samples),
          'f0_midi': 60 * r(2, 10, 1), 'f0_midi_pred': 60 * r(2, 10, 1),
          'f0_loss_weights': (r(2, 10, 1) > 0.3).float(),
          'amps': r(2, 10, 1), 'amps_pred': r(2, 10, 1), 'hd': r(2, 10, 20),
          'hd_pred': r(2, 10, 20), 'noise': r(2, 10, 65), 'noise_pred': r(2, 10, 65)}


class _L1(losses.Loss):
  def call(self, a, b):
    return torch.mean(torch.abs(a - b))


def test_loss_group_runs_the_recon_dag_on_cpu(monkeypatch):
  """The MIDI autoencoder's reconstruction LossGroup with its four ParamLosses and a CPU
  stand-in for the spectral loss.  The package moves every operand to CUDA; the
  coercion is kept on the CPU here so that the DAG plumbing runs without a device."""
  monkeypatch.setattr(core, 'torch_float32',
                      lambda x, device=None: torch.as_tensor(x, dtype=torch.float32))
  kw = _recon_losses(_L1(name='spectral_loss_synth'))
  group = losses.LossGroup(RECON_DAG, name='recon_lossgroup', **kw)
  assert group.name == 'recon_lossgroup'
  assert group.loss_names == list(kw)
  assert [getattr(group, k) for k in kw] == list(kw.values()) == group.losses
  out = _recon_outputs('cpu')
  got = group(out)
  assert list(got) == [kw[k].name for k in group.loss_names]
  assert set(got) == {'f0_reconstruction', 'amplitude_reconstruction',
                      'harmonic_distribution_reconstruction', 'noise_reconstruction',
                      'spectral_loss_synth'}
  want = {
      'f0_reconstruction': kw['f0_loss'](out['f0_midi'], out['f0_midi_pred'],
                                         out['f0_loss_weights']),
      'amplitude_reconstruction': kw['amps_loss'](out['amps'], out['amps_pred']),
      'harmonic_distribution_reconstruction': kw['hd_loss'](out['hd'], out['hd_pred']),
      'noise_reconstruction': kw['noise_loss'](out['noise'], out['noise_pred']),
      'spectral_loss_synth': kw['synth_spectral_loss'](out['audio'], out['synth_audio'])}
  for k, v in want.items():
    assert torch.equal(got[k], v), k
  w = out['f0_loss_weights']
  assert torch.allclose(got['f0_reconstruction'],
                        50.0 * torch.mean((out['f0_midi'] - out['f0_midi_pred'])**2 * w))
  assert group.get_losses_dict(out).keys() == got.keys()
  assert losses.LossGroup(RECON_DAG, **kw).name == 'loss_group'


def test_loss_group_takes_instances_in_the_dag_and_checks_keyword_losses(monkeypatch):
  monkeypatch.setattr(core, 'torch_float32',
                      lambda x, device=None: torch.as_tensor(x, dtype=torch.float32))
  direct = losses.ParamLoss(name='direct')
  out = _recon_outputs('cpu')
  group = losses.LossGroup([[direct, ['amps', 'amps_pred']]])
  assert group.loss_names == ['direct']
  assert list(group(out)) == ['direct']
  unused = losses.LossGroup([['amps_loss', ['amps', 'amps_pred']]],
                            amps_loss=losses.ParamLoss(name='a'),
                            noise_loss=losses.ParamLoss(name='n'))
  with pytest.raises(KeyError):
    unused(out)


# ---- GPU: helpers --------------------------------------------------------------------
def _cuda(*xs, grad=False):
  return [torch.as_tensor(np.asarray(x, np.float32), device=DEV).requires_grad_(grad)
          for x in xs]


def _terms(u, v, wu, wv):
  """Per row, in float64 on the float32 inputs: the sorted gaps delta [R, N-1], D at
  the N - 1 positions and the largest |prefix| of the signed weights in sorted order."""
  u, v, wu, wv = (ref.t64(x) for x in (u, v, wu, wv))
  s, order = torch.sort(torch.cat([u, v], -1), dim=-1, stable=True)
  sw = torch.gather(torch.cat([wu, -wv], -1), -1, order)
  pmax = torch.max(torch.abs(torch.cumsum(sw, -1)), -1).values
  d = ref._cdf(u, wu, s[..., :-1]) - ref._cdf(v, wv, s[..., :-1])
  return (s[..., 1:] - s[..., :-1]).numpy(), d.numpy(), pmax.numpy()


def _bounds(u, v, wu, wv, p):
  """(forward tolerance [R], e_D [R]) as the module docstring derives them."""
  delta, d, pmax = _terms(u, v, wu, wv)
  e_d = K_SCAN * 2.0**-24 * 2.0 * pmax[..., None]
  ad = np.abs(d)
  c = ad**p
  if p == 1.0:
    dc = e_d + 0 * ad
  elif p > 1.0:
    dc = p * (ad + e_d)**(p - 1.0) * e_d
  else:
    dc = e_d**p + 0 * ad
  s = np.sum(delta * c, -1)
  e_s = np.sum(delta * (dc + 2.0**-20 * c), -1) + K_SCAN * 2.0**-24 * s
  hi = (s + e_s)**(1.0 / p)
  lo = np.maximum(s - e_s, 0.0)**(1.0 / p)
  out = s**(1.0 / p)
  tol = np.maximum(hi - out, out - lo) + 2.0**-21 * out + 1e-30
  return tol, e_d, delta, d


def _check_forward(got, want, tol):
  got = got.detach().cpu().numpy().astype(np.float64)
  want = want.detach().numpy()
  assert got.shape == want.shape, (got.shape, want.shape)
  assert np.array_equal(np.isnan(got), np.isnan(want))
  ok = ~np.isnan(want)
  err = np.abs(got[ok] - want[ok])
  assert np.all(err <= np.broadcast_to(tol, want.shape)[ok]), (np.max(err - tol[ok]),)


def _check_grad(got, want, name, atol=0.0):
  got = got.detach().cpu().numpy().astype(np.float64)
  want = want.detach().numpy()
  assert np.array_equal(np.isnan(got), np.isnan(want)), name
  ok = np.isfinite(want)
  got, want = got[ok], want[ok]
  atol = np.broadcast_to(atol, ok.shape)[ok] if np.ndim(atol) else atol
  scale = np.max(np.abs(want)) if want.size else 0.0
  err = np.abs(got - want)
  assert np.all(err <= 5e-3 * np.abs(want) + 1e-3 * scale + atol + 1e-30), (
      name, np.max(err), scale)
  assert np.linalg.norm(err) <= 1e-4 * np.linalg.norm(want) + np.linalg.norm(
      np.broadcast_to(atol, err.shape)) + 1e-30, (name, np.linalg.norm(err))


def _run_both(x, p, gr):
  """The kernel and the restatement on the same float32 inputs x = (u, v, wu, wv),
  forward and, for the upstream gradient gr, the four gradients."""
  xs = _cuda(*x, grad=True)
  got = losses.wasserstein_distance(*xs, p=p)
  x64 = [torch.from_numpy(np.asarray(a, np.float64)).requires_grad_(True) for a in x]
  want = ref.wasserstein_distance(*x64, p=p)
  got.backward(torch.as_tensor(gr, dtype=torch.float32, device=DEV))
  want.backward(torch.from_numpy(np.asarray(gr, np.float64)))
  return got, want, xs, x64


def _weight_atol(p, gr, e_d, delta, d):
  """2 |G delta_i| over the positions whose sign of D the scan error could flip, as a
  bound on every suffix sum of the row."""
  s = np.sum(delta * np.abs(d)**p, -1)
  G = np.abs(gr) * (1.0 / p) * np.where(s > 0, s, 1.0)**(1.0 / p - 1.0)
  flip = np.abs(d) <= e_d
  return np.sum(np.where(flip, 2.0 * G[..., None] * delta, 0.0), -1)


def _inputs(rows, nu, nv, seed, spread=3.0):
  rng = np.random.default_rng(seed)
  return (rng.uniform(-spread, spread, (rows, nu)).astype(np.float32),
          rng.uniform(-spread, spread, (rows, nv)).astype(np.float32),
          rng.uniform(0.0, 1.0, (rows, nu)).astype(np.float32),
          rng.uniform(0.0, 1.0, (rows, nv)).astype(np.float32))


_KERNEL_CASES = (
    [(f'n{n}', 4, n, n, 1.0) for n in (1, 2, 31, 33, 100, 127, 129, 1000, 4096)] +
    [('1-vs-4096', 3, 1, 4096, 1.0), ('33-vs-127', 5, 33, 127, 1.0),
     ('1000-vs-129', 3, 1000, 129, 1.0), ('icml', 32 * 125, 100, 100, 1.0),
     ('p2-100', 6, 100, 100, 2.0), ('p2-31-vs-1000', 3, 31, 1000, 2.0),
     ('p2-4096', 2, 4096, 4096, 2.0), ('p_half-100', 6, 100, 100, 0.5),
     ('p_half-129-vs-2', 4, 129, 2, 0.5), ('p_half-4096-vs-1000', 2, 4096, 1000, 0.5)])


# ---- GPU: the kernels against the restatement ----------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('rows,nu,nv,p', [c[1:] for c in _KERNEL_CASES],
                         ids=[c[0] for c in _KERNEL_CASES])
def test_kernel_against_float64(rows, nu, nv, p):
  x = _inputs(rows, nu, nv, nu * 31 + nv + int(4 * p))
  gr = np.random.default_rng(5).normal(size=(rows,))
  got, want, xs, x64 = _run_both(x, p, gr)
  tol, e_d, delta, d = _bounds(*x, p)
  _check_forward(got, want, tol)
  watol = _weight_atol(p, gr, e_d, delta, d)[:, None]
  for name, a, e, atol in (('du', xs[0], x64[0], 0.0), ('dv', xs[1], x64[1], 0.0),
                           ('dwu', xs[2], x64[2], watol), ('dwv', xs[3], x64[3], watol)):
    _check_grad(a.grad, e.grad, name, atol)


@pytest.mark.gpu
@pytest.mark.parametrize('i', range(len(wg.DISTANCE_CASES)),
                         ids=[c[0] for c in wg.DISTANCE_CASES])
def test_fixture_cases(i):
  """Every fixture case, batch shapes 1-D to 4-D, against the unmodified reference's
  values and the restatement's gradients."""
  name, batch, _, _, p, _ = wg.DISTANCE_CASES[i]
  x = wg.distance_inputs(i)
  got = losses.wasserstein_distance(*x, p=p)
  assert tuple(got.shape) == batch
  want = torch.from_numpy(np.load(wg.PATH)[name])
  flat = [a.reshape(-1, a.shape[-1]) for a in x]
  tol, *_ = _bounds(*flat, p)
  _check_forward(got.reshape(-1), want.reshape(-1), tol)


@pytest.mark.gpu
@pytest.mark.parametrize('p', [1.0, 2.0, 0.5])
def test_ties_take_the_stable_concat_order(p):
  """Values on a grid of 1/4 (ties within u, within v and across them, -0 against +0):
  the value gradients land on the elements the stable concat order gives them, and the
  weight gradients read the suffix sum at the start of each tie group."""
  rng = np.random.default_rng(int(10 * p))
  rows, nu, nv = 8, 40, 25
  u = (rng.integers(-6, 7, (rows, nu)) / 4.0).astype(np.float32)
  v = (rng.integers(-6, 7, (rows, nv)) / 4.0).astype(np.float32)
  u[0, :3] = -0.0
  v[0, :3] = 0.0
  wu = rng.uniform(0.1, 1.0, (rows, nu)).astype(np.float32)
  wv = rng.uniform(0.1, 1.0, (rows, nv)).astype(np.float32)
  x = (u, v, wu, wv)
  gr = rng.normal(size=(rows,))
  got, want, xs, x64 = _run_both(x, p, gr)
  tol, e_d, delta, d = _bounds(*x, p)
  _check_forward(got, want, tol)
  watol = _weight_atol(p, gr, e_d, delta, d)[:, None]
  for name, a, e, atol in (('du', xs[0], x64[0], 0.0), ('dv', xs[1], x64[1], 0.0),
                           ('dwu', xs[2], x64[2], watol), ('dwv', xs[3], x64[3], watol)):
    _check_grad(a.grad, e.grad, name, atol)
  # within a tie group only the first and the last element can get a value gradient
  du = xs[0].grad.cpu().numpy()
  assert np.count_nonzero(du[0, :3]) <= 1


@pytest.mark.gpu
def test_nan_where_autograd_has_nan():
  """Weights in eighths, so that every running sum is exact and U = V holds exactly
  where the sides agree: D = 0 at p = 1/2 gives 0 * inf in the weight gradients, S = 0 at
  p = 2 an infinite G; an infinite value and a NaN weight propagate.  NaN at the
  restatement's positions, the finite values alike."""
  rng = np.random.default_rng(9)
  u = rng.uniform(-1, 1, (5, 5)).astype(np.float32)
  w = (rng.integers(1, 9, (5, 5)) / 8.0).astype(np.float32)
  v, wv = u.copy(), w.copy()
  v[1] += 0.5
  wv[2, 0] = 0.25                      # D = 0 on part of row 2 only
  v[3, 1] = np.inf
  wv[4, 2] = np.nan
  for p in (0.5, 2.0, 1.0):
    gr = rng.normal(size=(5,))
    got, want, xs, x64 = _run_both((u, v, w, wv), p, gr)
    g, e = got.detach().cpu().numpy(), want.detach().numpy()
    assert np.array_equal(np.isnan(g), np.isnan(e)), (p, g, e)
    for name, a, b in zip(('du', 'dv', 'dwu', 'dwv'), xs, x64):
      ga, gb = a.grad.cpu().numpy(), b.grad.numpy()
      assert np.array_equal(np.isnan(ga), np.isnan(gb)), (p, name, ga, gb)
      fin = np.isfinite(gb)
      np.testing.assert_allclose(ga[fin], gb[fin], rtol=1e-4, atol=1e-5, err_msg=name)
    if p == 1.0:
      assert np.all(np.isfinite(xs[0].grad.cpu().numpy()[:3]))


# ---- GPU: the loss ----------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('i', range(len(wg.LOSS_CASES)), ids=[c[0] for c in wg.LOSS_CASES])
def test_loss_fixture_cases(i):
  name, *_, w, m = wg.LOSS_CASES[i]
  x = wg.loss_inputs(i)
  got = losses.WassersteinConsistencyLoss(weight=w, midi=m)(*_cuda(*x))
  want = float(np.load(wg.PATH)[name])
  # hz_to_midi in float32 is off by up to 1.2e-4 MIDI (16 ulp at MIDI 128); each value
  # moves the distance by at most that times its side's weight total
  a_tot = np.sum(x[0], -1) + np.sum(x[2], -1)
  tol = w * np.mean(2.4e-4 * a_tot) + 2.0**-18 * abs(want) + 1e-6
  assert abs(float(got) - want) <= tol, (float(got), want, tol)


@pytest.mark.gpu
def test_loss_gradients_through_hz_to_midi():
  """WassersteinConsistencyLoss at B = 4, T = 25, 30 against 20 sinusoids.  Its value is
  checked against the restatement from hertz (within hz_to_midi's float32 error), and
  its gradients against float64 autograd from the same float32 MIDI values, chained
  through d midi / d f = 12 / (f ln 2) (0 at f <= 0): float32 MIDI values that differ
  from float64's by an ulp may swap two close sinusoids, which moves the value gradients
  of both by a whole weight."""
  rng = np.random.default_rng(12)
  b, t = 4, 25
  x = (rng.uniform(0.05, 1.0, (b, t, 30)), np.exp(rng.uniform(4.0, 8.5, (b, t, 30))),
       rng.uniform(0.05, 1.0, (b, t, 20)), np.exp(rng.uniform(4.0, 8.5, (b, t, 20))))
  x = [a.astype(np.float32) for a in x]
  x[1][0, 0, 0] = 0.0
  xs = _cuda(*x, grad=True)
  loss = losses.WassersteinConsistencyLoss(weight=0.7)
  got = loss(*xs)
  want_hz = ref.wasserstein_consistency(*x, weight=0.7).item()
  a_tot = np.sum(x[0], -1) + np.sum(x[2], -1)
  assert abs(got.item() - want_hz) <= 0.7 * np.mean(2.4e-4 * a_tot) + 1e-5 * want_hz
  got.backward()
  midi = [core.hz_to_midi(xs[k].detach()).double().cpu().requires_grad_(True) for k in (1, 3)]
  amps = [torch.from_numpy(x[k].astype(np.float64)).requires_grad_(True) for k in (0, 2)]
  want = torch.mean(0.7 * ref.wasserstein_distance(midi[0], midi[1], amps[0], amps[1]))
  assert abs(got.item() - want.item()) <= 1e-5 * want.item()
  want.backward()
  dfreq = [m.grad.numpy() * np.where(x[k] > 0, 12.0 / (np.maximum(x[k], 1e-30) * np.log(2.0)),
                                     0.0) for m, k in zip(midi, (1, 3))]
  for n, a, e in (('amps_a', xs[0], amps[0].grad.numpy()), ('freqs_a', xs[1], dfreq[0]),
                  ('amps_b', xs[2], amps[1].grad.numpy()), ('freqs_b', xs[3], dfreq[1])):
    gg = a.grad.cpu().numpy().astype(np.float64)
    scale = np.max(np.abs(e))
    assert np.all(np.abs(gg - e) <= 5e-3 * np.abs(e) + 1e-3 * scale), (
        n, np.max(np.abs(gg - e)), scale)
  assert xs[1].grad[0, 0, 0].item() == 0.0        # no gradient through the 0 Hz floor


# ---- GPU: reproducibility, graphs, streams, devices, memory ----------------------------
def _step(xs, p=1.0):
  for x in xs:
    x.grad = None
  out = losses.wasserstein_distance(*xs, p=p)
  out.sum().backward()
  return out.detach().clone(), [x.grad.clone() for x in xs]


@pytest.mark.gpu
@pytest.mark.parametrize('nu,nv', [(100, 100), (4096, 1000)])
def test_bit_reproducible(nu, nv):
  xs = _cuda(*_inputs(64, nu, nv, 4), grad=True)
  first, second = _step(xs), _step(xs)
  assert torch.equal(first[0], second[0])
  for a, b in zip(first[1], second[1]):
    assert torch.equal(a, b)


@pytest.mark.gpu
def test_cuda_graph_capture_equals_eager():
  xs = _cuda(*_inputs(500, 100, 80, 6), grad=True)
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    for _ in range(2):
      eager, eager_grads = _step(xs)
  torch.cuda.current_stream().wait_stream(s)
  graph = torch.cuda.CUDAGraph()
  for x in xs:
    x.grad = None
  with torch.cuda.graph(graph):
    static = losses.wasserstein_distance(*xs)
    static.sum().backward()
  graph.replay()
  torch.cuda.synchronize()
  assert torch.equal(static, eager)
  for x, g in zip(xs, eager_grads):
    assert torch.equal(x.grad, g)


@pytest.mark.gpu
def test_empty_batch():
  for shape in ((0, 5), (3, 0, 5)):
    xs = [torch.zeros(shape, device=DEV, requires_grad=True) for _ in range(4)]
    out = losses.wasserstein_distance(*xs)
    assert out.shape == shape[:-1]
    out.sum().backward()
    assert all(x.grad.shape == shape for x in xs)


@pytest.mark.gpu
def test_runs_on_the_current_stream(recorder):
  xs = _cuda(*_inputs(3, 4, 5, 1))
  s = torch.cuda.Stream()
  with torch.cuda.stream(s):
    losses.wasserstein_distance(*xs)
  (name, _, args), = recorder.calls
  assert name == 'ddsp_b200_wasserstein_forward'
  assert args[-1] == s.cuda_stream
  assert args[5:9] == (3, 4, 5, 1.0)


@pytest.mark.gpu
def test_side_stream_equals_default_stream():
  xs = _cuda(*_inputs(200, 50, 70, 2), grad=True)
  want = _step(xs)
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    got = _step(xs)
  torch.cuda.current_stream().wait_stream(s)
  torch.cuda.synchronize()
  assert torch.equal(got[0], want[0])
  for a, b in zip(got[1], want[1]):
    assert torch.equal(a, b)


@pytest.mark.gpu
def test_runs_on_the_operands_device():
  if torch.cuda.device_count() < 2:
    pytest.skip('needs a second GPU')
  x = _inputs(20, 30, 40, 8)
  want = _step(_cuda(*x, grad=True))
  with torch.cuda.device(0):
    xs = [torch.as_tensor(a, device='cuda:1').requires_grad_(True) for a in x]
    got = _step(xs)
  assert got[0].device == torch.device('cuda:1')
  assert torch.equal(got[0].cpu(), want[0].cpu())
  for a, b in zip(got[1], want[1]):
    assert torch.equal(a.cpu(), b.cpu())


@pytest.mark.gpu
@pytest.mark.parametrize('nu,nv', [(1, 1), (33, 129), (100, 100), (4096, 3)])
def test_poisoned_outputs_and_fenced_operands(nu, nv):
  """Every output and gradient buffer poisoned (0x00, 0xFF, 0x7F) between canary fences,
  and every input and the upstream gradient between 64 KiB fences of NaN and of 7.0:
  the same bits every time, and every fence intact."""
  from tests.test_gpu_memory_bounds import POISONS, _fenced, _fences_intact, guarded
  x = _inputs(7, nu, nv, 13)
  gr = torch.as_tensor(np.random.default_rng(3).normal(size=(7,)), dtype=torch.float32,
                       device=DEV)

  def run(ins, g):
    ins = [a.detach().requires_grad_(True) for a in ins]
    out = losses.wasserstein_distance(*ins)
    out.backward(g)
    return [out.detach().clone()] + [a.grad.clone() for a in ins]

  want = run(_cuda(*x), gr)
  for poison in POISONS:
    with guarded(poison):
      got = run(_cuda(*x), gr)
    for a, b in zip(got, want):
      assert torch.equal(a.view(torch.int32), b.view(torch.int32)), poison
  for fill in (math.nan, 7.0):
    for off in (0, 1):
      regions, ins = [], []
      for a in _cuda(*x):
        fa, r = _fenced(a, fill, off)
        ins.append(fa)
        regions.append(r)
      fg, r = _fenced(gr, fill, off)
      regions.append(r)
      got = run(ins, fg)
      for a, b in zip(got, want):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (fill, off)
      torch.cuda.synchronize()
      for r in regions:
        _fences_intact(r, (fill, off))


@pytest.mark.gpu
def test_memory_holds_no_row_intermediates():
  """B = 32, T = 125, 1024 against 1024: forward and backward allocate the [R] distances
  and the four gradients, nothing of [R, N]'s size beyond them."""
  xs = _cuda(*_inputs(32 * 125, 1024, 1024, 14), grad=True)
  torch.cuda.synchronize()
  base = torch.cuda.memory_allocated()
  torch.cuda.reset_peak_memory_stats()
  out = losses.wasserstein_distance(*xs)
  out.sum().backward()
  torch.cuda.synchronize()
  rise = torch.cuda.max_memory_allocated() - base
  grads = sum(x.numel() * 4 for x in xs)
  assert rise <= grads + 2 * 2**20, (rise, grads)


# ---- GPU: LossGroup ---------------------------------------------------------------------
@pytest.mark.gpu
def test_loss_group_with_spectral_loss_on_cuda():
  """The recon LossGroup with the real SpectralLoss (L1, mag and logmag weight 1) on CUDA
  tensors: the values of the direct calls, and gradients reaching the audio."""
  spectral = losses.SpectralLoss(loss_type='L1', mag_weight=1.0, logmag_weight=1.0,
                                 name='spectral_loss_synth')
  kw = _recon_losses(spectral)
  group = losses.LossGroup(RECON_DAG, **kw)
  out = _recon_outputs(DEV, 16000)
  out['synth_audio'].requires_grad_(True)
  got = group(out)
  assert set(got) == {'spectral_loss_synth', 'f0_reconstruction', 'amplitude_reconstruction',
                      'harmonic_distribution_reconstruction', 'noise_reconstruction'}
  direct = spectral(out['audio'], out['synth_audio'])
  assert torch.equal(got['spectral_loss_synth'], direct)
  assert torch.equal(got['f0_reconstruction'],
                     kw['f0_loss'](out['f0_midi'], out['f0_midi_pred'], out['f0_loss_weights']))
  total = sum(got.values())
  total.backward()
  g = out['synth_audio'].grad
  assert g is not None and bool(torch.isfinite(g).all()) and float(g.abs().max()) > 0
