"""losses.HmmTranscriber and core.hmm_log_prob / core.hmm_posterior_mode (csrc/hmm.cuh):
the float64 restatement against the unmodified reference's fixture and against
brute-force enumeration, the C ABI's checks, the Python errors and B = 0 (CPU); the
kernels against float64, Viterbi decodes, the loss chain and the library's conventions
(GPU).

Tolerances.  log_prob is within 1e-5 relative of float64: every step's log normaliser
M_t + log S_t is formed in float32 from terms of relative error a few u = 2^-24 of
|l_t| + |log q_t|, and summed in double, so the total is off by a few u of
sum_t (|l_t| + |log q_t|) - 1e-6 relative where the per-step terms share a sign, as
they do for these inputs (|log_prob| / T is 0.4 .. 2e5 here).  The gradients are
posterior-weighted sums of K terms each step, with float32 marginals of relative error
~1e-6 after the normalised forward and backward scans; 2e-4 of the peak and 1e-4
relative L2 leave a factor of 100 over that.  Viterbi decodes must equal the float64
decode exactly wherever the optimum is not within float32 rounding of a rival.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, core, losses
from oracle import ref_on_shim
from tests import hmm_ref as ref
from tests.golden import make_hmm_golden as mg
from tests.util import HostQueriesOnly

DEV = 'cuda'


def _fixture():
  return np.load(mg.PATH)


def _params(kw, device='cpu'):
  return [p.to(device) for p in ref.transcriber_params(**kw)]


def _pa(pitch, amps):
  return np.concatenate([pitch, amps], -1).astype(np.float32)


def _rel(got, want):
  got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
  return float(np.max(np.abs(got - want) / np.maximum(np.abs(want), 1e-30)))


# ---- CPU: the restatement ---------------------------------------------------------
def test_restatement_matches_the_reference():
  """tests/hmm_ref.py with its own HmmTranscriber parameters against the reference run
  wide on the shim."""
  want = _fixture()
  for i, (name, _, _) in enumerate(mg.CASES):
    kw = mg.case_kwargs(i)
    pitch, amps = mg.inputs(i)
    x = torch.from_numpy(_pa(pitch, amps)).double()
    lp = ref.log_prob(x, *_params(kw)).numpy()
    t = kw['n_timesteps']
    assert _rel(lp, want[name + '_log_prob']) <= 1e-12, name
    assert _rel(kw['weight'] * -lp / t, want[name + '_nll_per_example']) <= 1e-12, name
    assert _rel(np.mean(kw['weight'] * -lp / t), want[name + '_nll']) <= 1e-12, name
    path = ref.posterior_mode(x, *_params(kw))
    assert np.array_equal(path[..., None], want[name + '_predict_midi']), name


@pytest.mark.skipif(not ref_on_shim.available(), reason='reference sources absent')
def test_fixture_regenerates_from_reference():
  """In a fresh process: the generator restates tfp before the reference is imported."""
  subprocess.run([sys.executable, os.path.abspath(mg.__file__), '--check'], check=True)


@pytest.mark.parametrize('k', [2, 3])
@pytest.mark.parametrize('t', [1, 2, 5, 7])
@pytest.mark.parametrize('avg_length', [1.0, 1.7, 30.0])
def test_restatement_against_brute_force(k, t, avg_length):
  """The dense forward algorithm and Viterbi against every one of the K^T paths."""
  rng = np.random.default_rng(k * 100 + t * 10 + int(avg_length))
  kw = dict(avg_length=avg_length, n_pitches=k, midi_std=0.7)
  x = torch.from_numpy(np.stack([rng.uniform(-0.5, k - 0.5, (3, t)),
                                 rng.uniform(-0.2, 1.8, (3, t))], -1))
  params = _params(kw)
  lp, best, gap = ref.brute_force(x, *params)
  assert np.allclose(ref.log_prob(x, *params).numpy(), lp, rtol=1e-12, atol=1e-12)
  path = ref.posterior_mode(x, *params)
  for i in range(3):
    if gap[i] > 1e-9:
      assert np.array_equal(path[i], best[i]), (i, path[i], best[i])


def test_value_errors_before_device_work_or_launches(monkeypatch):
  """Every error is raised from static shapes and arguments, before any tensor is moved
  or anything but the library's host queries (the Viterbi size rule) is called."""
  def touched(*a, **k):
    raise AssertionError('device work before the argument checks')
  monkeypatch.setattr(core, 'torch_float32', touched)
  rec = HostQueriesOnly(_lib.load())
  monkeypatch.setattr(core._lib, 'load', lambda: rec)
  for kw in (dict(n_pitches=1), dict(n_pitches=0), dict(n_timesteps=0),
             dict(avg_length=0.999), dict(avg_length=-3.0), dict(n_pitches=2.5)):
    with pytest.raises(ValueError):
      losses.HmmTranscriber(**kw)
  hmm = losses.HmmTranscriber(n_timesteps=10, n_pitches=16)
  ok = np.zeros((2, 10, 1), np.float32)
  for pitch, amps in ((np.zeros((2, 9, 1)), ok), (ok, np.zeros((2, 10, 2))),
                      (np.zeros((2, 10)), ok), (ok, np.zeros((3, 10, 1))),
                      (torch.zeros((2, 11, 1), requires_grad=True), ok)):
    for call in (hmm, hmm.nll, hmm.predict_midi):
      with pytest.raises(ValueError):
        call(pitch, amps)
  for pa in (np.zeros((2, 10, 1)), np.zeros((2, 9, 2))):
    for call in (hmm.log_prob, hmm.posterior_mode):
      with pytest.raises(ValueError):
        call(pa)
  with pytest.raises(NotImplementedError, match='1025 pitches'):
    losses.HmmTranscriber(n_timesteps=10, n_pitches=1025).nll(ok, ok)
  with pytest.raises(NotImplementedError, match='10241 steps of 128 states'):
    big = np.zeros((1, 10241, 1), np.float32)
    losses.HmmTranscriber(n_timesteps=10241).predict_midi(big, big)
  # core: shapes, states and transitions
  x = np.zeros((2, 5, 2), np.float32)
  ls = np.ones((8, 2), np.float32)
  for fn in (core.hmm_log_prob, core.hmm_posterior_mode):
    for args in ((x[..., :1], ls, ls, 0.9, 0.01), (np.zeros((2, 0, 2)), ls, ls, 0.9, 0.01),
                 (x, ls[:, :1], ls, 0.9, 0.01), (x, ls, ls[:4], 0.9, 0.01),
                 (x, ls[:1], ls[:1], 0.9, 0.01), (x, ls, ls, -0.1, 0.01),
                 (x, ls, ls, 0.0, 0.0), (x, ls, ls, np.inf, 0.01), (x, ls, ls, 0.5, np.nan)):
      with pytest.raises(ValueError):
        fn(*args)
    big = np.ones((1025, 2), np.float32)
    with pytest.raises(NotImplementedError, match='1025 states'):
      fn(x, big, big, 0.9, 1e-4)
  with pytest.raises(NotImplementedError, match='loc and scale are constants'):
    core.hmm_log_prob(x, torch.ones((8, 2), requires_grad=True), ls, 0.9, 0.01)


def test_transcriber_attributes():
  hmm = losses.HmmTranscriber()
  assert (hmm.avg_length, hmm.midi_std, hmm.n_timesteps, hmm.n_pitches, hmm.weight,
          hmm.name) == (200, 0.5, 1000, 128, 1.0, 'HiddenMarkovModel')
  assert losses.HmmTranscriber(name='hmm_prior', weight=5.0).name == 'hmm_prior'
  log_init, log_trans, loc, scale = _params({})
  assert np.array_equal(hmm.loc, loc.numpy().astype(np.float32))
  assert np.array_equal(hmm.scale, scale.numpy().astype(np.float32))
  t = np.exp(log_trans.numpy())
  assert abs(hmm.hold - t[0, 0]) < 1e-15 and abs(hmm.other - t[0, 1]) < 1e-15


def test_size_rules():
  assert core.hmm_viterbi_takes(1000, 1024) and core.hmm_viterbi_takes(10000, 128)
  assert core.hmm_viterbi_takes(1551, 1024) and not core.hmm_viterbi_takes(1552, 1024)
  assert core.hmm_viterbi_takes(10240, 128) and not core.hmm_viterbi_takes(10241, 128)
  assert core.hmm_segment(1000, 128) == 32 and core.hmm_segment(1, 2) == 1
  assert core.hmm_segment(10000, 1024) == 48 and core.hmm_segment(1024, 128) == 32


P = 0x1000        # a device pointer the library never dereferences on the host
E_INVALID, E_UNSUPPORTED = _lib.E_INVALID, _lib.E_UNSUPPORTED


def _fwd(x=P, loc=P, scale=P, out=P, B=2, T=10, K=8, hold=0.9, other=0.01):
  return (x, loc, scale, out, B, T, K, hold, other, None)


def _bwd(x=P, loc=P, scale=P, g=P, dx=P, ck=P, seg=4, B=2, T=10, K=8, hold=0.9, other=0.01):
  return (x, loc, scale, g, dx, ck, seg, B, T, K, hold, other, None)


_F, _B, _V = 'hmm_log_prob', 'hmm_log_prob_backward', 'hmm_viterbi'
_ABI_CASES = [
    ('f-null-x', _F, _fwd(x=None), E_INVALID, b'hmm_log_prob: null pointer'),
    ('f-null-loc', _F, _fwd(loc=None), E_INVALID, b'hmm_log_prob: null pointer'),
    ('f-null-scale', _F, _fwd(scale=None), E_INVALID, b'hmm_log_prob: null pointer'),
    ('f-null-out', _F, _fwd(out=None), E_INVALID, b'hmm_log_prob: null pointer'),
    ('f-B', _F, _fwd(B=-1), E_INVALID, b'hmm_log_prob: bad shape B=-1 T=10 K=8'),
    ('f-T', _F, _fwd(T=0), E_INVALID, b'hmm_log_prob: bad shape B=2 T=0 K=8'),
    ('f-K', _F, _fwd(K=1), E_INVALID, b'hmm_log_prob: bad shape B=2 T=10 K=1'),
    ('f-K-max', _F, _fwd(K=1025), E_UNSUPPORTED, b'hmm_log_prob: K=1025 states exceed the 1024 supported'),
    ('f-hold', _F, _fwd(hold=-0.5), E_INVALID, b'hmm_log_prob: hold=-0.5 and other=0.01 must be finite, non-negative and not both 0'),
    ('f-other', _F, _fwd(other=float('inf')), E_INVALID, b'hmm_log_prob: hold=0.9 and other=inf must be finite, non-negative and not both 0'),
    ('f-nan', _F, _fwd(hold=float('nan')), E_INVALID, b'hmm_log_prob: hold=nan and other=0.01 must be finite, non-negative and not both 0'),
    ('f-zero', _F, _fwd(hold=0.0, other=0.0), E_INVALID, b'hmm_log_prob: hold=0 and other=0 must be finite, non-negative and not both 0'),
    ('f-B0', _F, _fwd(None, None, None, None, B=0), 0, None),
    ('f-hold0', _F, _fwd(B=0, hold=0.0), 0, None),
    ('b-null-g', _B, _bwd(g=None), E_INVALID, b'hmm_log_prob_backward: null pointer'),
    ('b-null-dx', _B, _bwd(dx=None), E_INVALID, b'hmm_log_prob_backward: null pointer'),
    ('b-null-ck', _B, _bwd(ck=None), E_INVALID, b'hmm_log_prob_backward: null pointer'),
    ('b-T', _B, _bwd(T=-1), E_INVALID, b'hmm_log_prob_backward: bad shape B=2 T=-1 K=8'),
    ('b-K-max', _B, _bwd(K=2048), E_UNSUPPORTED, b'hmm_log_prob_backward: K=2048 states exceed the 1024 supported'),
    ('b-seg0', _B, _bwd(seg=0), E_INVALID, b'hmm_log_prob_backward: seg=0 must be at least 1 with seg*K at most 49152'),
    ('b-seg-max', _B, _bwd(seg=49, K=1024), E_INVALID, b'hmm_log_prob_backward: seg=49 must be at least 1 with seg*K at most 49152'),
    ('b-seg-ok-B0', _B, _bwd(seg=48, K=1024, B=0), 0, None),
    ('b-B0', _B, _bwd(*([None] * 6), B=0), 0, None),
    ('v-null-path', _V, _fwd(out=None), E_INVALID, b'hmm_viterbi: null pointer'),
    ('v-K', _V, _fwd(K=0), E_INVALID, b'hmm_viterbi: bad shape B=2 T=10 K=0'),
    ('v-other', _V, _fwd(other=-1e-3), E_INVALID, b'hmm_viterbi: hold=0.9 and other=-0.001 must be finite, non-negative and not both 0'),
    ('v-T-max', _V, _fwd(T=10241, K=128), E_UNSUPPORTED, b'hmm_viterbi: T=10241 steps of K=128 states need 204820 B of back pointers, more than the 204800 supported'),
    ('v-T-max-1024', _V, _fwd(T=1552, K=1024), E_UNSUPPORTED, b'hmm_viterbi: T=1552 steps of K=1024 states need 204864 B of back pointers, more than the 204800 supported'),
    ('v-T-max-B0', _V, _fwd(T=10241, K=128, B=0), E_UNSUPPORTED, b'hmm_viterbi: T=10241 steps of K=128 states need 204820 B of back pointers, more than the 204800 supported'),
    ('v-B0', _V, _fwd(None, None, None, None, B=0, T=10240, K=128), 0, None),
]


@pytest.mark.parametrize('fn,args,want,msg', [c[1:] for c in _ABI_CASES],
                         ids=[c[0] for c in _ABI_CASES])
def test_abi_check_table(fn, args, want, msg):
  """Every check of the three entry points: the status and the full message come back
  before any CUDA call, and nothing is launched (B = 0 included)."""
  lib = _lib.load()
  launches = lib.ddsp_b200_launch_count()
  assert getattr(lib, 'ddsp_b200_' + fn)(*args) == want
  assert lib.ddsp_b200_launch_count() == launches
  if msg is not None:
    assert lib.ddsp_b200_last_error() == msg


def test_no_workspace_and_one_size_query():
  names = sorted(n for n in _lib.SIGNATURES if 'hmm' in n)
  assert names == ['ddsp_b200_hmm_log_prob', 'ddsp_b200_hmm_log_prob_backward',
                   'ddsp_b200_hmm_viterbi', 'ddsp_b200_hmm_viterbi_takes']
  for n in names:
    assert _lib.SIGNATURES[n][1][-2] is not _lib._sz


# ---- GPU ------------------------------------------------------------------------------
def _cuda(x, grad=False):
  return torch.as_tensor(np.asarray(x, np.float32), device=DEV).requires_grad_(grad)


def _hmm_args(kw):
  hmm = losses.HmmTranscriber(**kw)
  return _cuda(hmm.loc), _cuda(hmm.scale), hmm.hold, hmm.other


def _ref_log_prob(x, kw, grad=False):
  """float64 dense log_prob on the GPU, and with grad the float64 leaf."""
  x64 = torch.as_tensor(np.asarray(x), dtype=torch.float64, device=DEV)
  x64.requires_grad_(grad)
  return ref.log_prob(x64, *_params(kw, DEV)), x64


def _notes(seed, b, t, k=128, **kw):
  pitch, amps = mg.notes(np.random.default_rng(seed), b, t, k, **kw)
  return _pa(pitch, amps)


def _extreme(seed, b, t, k=128):
  """Pitch pinned at 0 and K - 1 and amplitudes far outside the loc / scale range."""
  rng = np.random.default_rng(seed)
  pitch = rng.choice([0.0, k - 1.0], (b, t, 1))
  amps = rng.choice([-40.0, 0.0, 60.0], (b, t, 1)) + rng.normal(size=(b, t, 1))
  return _pa(pitch, amps)


LOG_PROB_CASES = [('K2', 2, 1000, 2), ('K33', 33, 1000, 2), ('K128', 128, 1000, 2),
                  ('K1024', 1024, 1000, 2), ('T1', 128, 1, 3), ('T31', 128, 31, 3),
                  ('T10000', 128, 10000, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize('i', range(len(mg.CASES)), ids=[c[0] for c in mg.CASES])
def test_fixture_cases(i):
  """log_prob, nll (both forms) and predict_midi against the reference's fixture."""
  name = mg.CASES[i][0]
  want = _fixture()
  kw = mg.case_kwargs(i)
  pitch, amps = mg.inputs(i)
  hmm = losses.HmmTranscriber(**mg.CASES[i][2])
  p, a = _cuda(pitch), _cuda(amps)
  assert _rel(hmm.log_prob(torch.cat([p, a], -1)).cpu(), want[name + '_log_prob']) <= 1e-5
  assert _rel(hmm.nll(p, a).cpu(), want[name + '_nll']) <= 1e-5
  assert _rel(hmm(p, a).cpu(), want[name + '_nll']) <= 1e-5
  assert _rel(hmm.nll(p, a, per_example_loss=True).cpu(),
              want[name + '_nll_per_example']) <= 1e-5
  midi = hmm.predict_midi(p, a)
  assert midi.dtype == torch.float32 and tuple(midi.shape) == pitch.shape
  assert np.array_equal(midi.cpu().numpy(), want[name + '_predict_midi']), name
  assert kw['n_timesteps'] == pitch.shape[1]


@pytest.mark.gpu
@pytest.mark.parametrize('name,k,t,b', LOG_PROB_CASES, ids=[c[0] for c in LOG_PROB_CASES])
@pytest.mark.parametrize('inputs', ['notes', 'extreme'])
def test_log_prob_against_float64(name, k, t, b, inputs):
  seed = 10 * [c[0] for c in LOG_PROB_CASES].index(name) + (inputs == 'extreme')
  x = (_notes if inputs == 'notes' else _extreme)(seed, b, t, k)
  kw = dict(n_pitches=k)
  got = core.hmm_log_prob(_cuda(x), *_hmm_args(kw))
  want, _ = _ref_log_prob(x, kw)
  assert got.shape == (b,) and got.dtype == torch.float32
  assert _rel(got.cpu(), want.cpu()) <= 1e-5, (got, want)


def _grad_check(x, kw, g=None):
  """d observations of the kernel against float64 autograd of the dense restatement."""
  b = x.shape[0]
  g = np.random.default_rng(5).normal(size=b) if g is None else g
  xs = _cuda(x, grad=True)
  core.hmm_log_prob(xs, *_hmm_args(kw)).backward(_cuda(g))
  want, x64 = _ref_log_prob(x, kw, grad=True)
  want.backward(torch.as_tensor(g, dtype=torch.float64, device=DEV))
  got, w = xs.grad.double().cpu().numpy(), x64.grad.cpu().numpy()
  for d in range(2):       # pitch and amplitude separately, each against its own peak
    gd, wd = got[..., d], w[..., d]
    peak = np.abs(wd).max()
    assert np.abs(gd - wd).max() <= 2e-4 * peak, (d, np.abs(gd - wd).max() / peak)
    assert np.linalg.norm(gd - wd) <= 1e-4 * np.linalg.norm(wd), d
  return xs.grad


GRAD_CASES = [(name, mg.case_kwargs(i), i) for i, (name, _, _) in enumerate(mg.CASES)] + [
    ('K33_T1000', dict(n_pitches=33), 1000), ('K1024_T60', dict(n_pitches=1024), 60),
    ('extreme', dict(), 300), ('avg1_K128', dict(avg_length=1), 300)]


@pytest.mark.gpu
@pytest.mark.parametrize('j', range(len(GRAD_CASES)), ids=[c[0] for c in GRAD_CASES])
def test_gradients_against_float64(j):
  name, kw, arg = GRAD_CASES[j]
  if j < len(mg.CASES):
    x = _pa(*mg.inputs(arg))
  elif name == 'extreme':
    x = _extreme(31, 2, arg)
  else:
    x = _notes(30 + j, 2, arg, kw.get('n_pitches', 128))
  _grad_check(x, kw)


@pytest.mark.gpu
@pytest.mark.parametrize('k,t', [(128, 10000), (1024, 2500), (2, 4000)])
def test_gradient_inner_product_against_finite_differences(k, t):
  """<d log_prob / d x, v> against the central difference of the float64 log_prob
  along v, at sizes (long T; K = 1024, where the segment is capped at 48 steps) whose
  dense float64 autograd would not fit."""
  x = _notes(40 + k, 1, t, k)
  kw = dict(n_pitches=k)
  xs = _cuda(x, grad=True)
  core.hmm_log_prob(xs, *_hmm_args(kw)).sum().backward()
  v = np.random.default_rng(41).normal(size=x.shape)
  h = 1e-3
  plus, _ = _ref_log_prob(x + h * v, kw)
  minus, _ = _ref_log_prob(x - h * v, kw)
  fd = float((plus - minus).sum()) / (2 * h)
  grad = xs.grad.double().cpu().numpy()
  got = float(np.sum(grad * v))
  assert abs(got - fd) <= 1e-4 * float(np.sum(np.abs(grad * v))), (got, fd)


def _decode(x, kw):
  return core.hmm_posterior_mode(_cuda(x), *_hmm_args(kw)).cpu().numpy()


@pytest.mark.gpu
def test_viterbi_on_noisy_notes_at_the_reference_shape():
  x = _notes(50, 16, 1000)
  got = _decode(x, {})
  want = ref.posterior_mode(torch.from_numpy(x).double(), *_params({}))
  assert got.dtype == np.int64 and got.shape == (16, 1000)
  assert np.array_equal(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize('k,t,avg', [(128, 1000, 200), (33, 500, 3), (1024, 1000, 200),
                                     (128, 10000, 50), (16, 300, 1), (64, 400, 1e6)])
def test_viterbi_path_is_optimal(k, t, avg):
  """Random observations (noisy and ambiguous): where the decode differs from the
  float64 one, its float64 log-joint is within 1e-3 nats of the optimum."""
  rng = np.random.default_rng(k + t)
  x = _notes(60 + k, 4, t, k)
  x[..., 0] += rng.uniform(-0.5, 0.5, x.shape[:2]).astype(np.float32)
  kw = dict(n_pitches=k, avg_length=avg)
  got = _decode(x, kw)
  params = _params(kw)
  x64 = torch.from_numpy(x).double()
  want = ref.posterior_mode(x64, *params)
  lj_got = ref.log_joint(got, x64, *params)
  lj_want = ref.log_joint(want, x64, *params)
  assert np.all(lj_got >= lj_want - 1e-3), lj_want - lj_got
  assert np.all((got >= 0) & (got < k))


@pytest.mark.gpu
@pytest.mark.parametrize('k', [128, 1024])
def test_halfway_decodes_to_the_lower_pitch(k):
  """An observation exactly between pitches p and p + 1 for the whole run: both states
  tie at every step, and the lower one wins."""
  t = 200
  x = np.zeros((3, t, 2), np.float32)
  x[:, :, 0] = np.array([60.5, 1.5, k - 1.5], np.float32)[:, None]
  x[:, :, 1] = 1.5
  got = _decode(x, dict(n_pitches=k))
  assert np.array_equal(got, np.broadcast_to(np.array([60, 1, k - 2])[:, None], (3, t)))


@pytest.mark.gpu
def test_predict_midi_shape_and_dtype():
  hmm = losses.HmmTranscriber(n_timesteps=50)
  x = _notes(70, 3, 50)
  p, a = _cuda(x[..., :1]), _cuda(x[..., 1:])
  base = hmm.predict_midi(p, a)
  for dtype in (torch.float32, torch.float16, torch.int32, torch.int64, torch.float64):
    got = hmm.predict_midi(p, a, dtype=dtype)
    assert got.dtype == dtype and tuple(got.shape) == (3, 50, 1)
    assert torch.equal(got.to(torch.float32), base)
  flat = hmm.predict_midi(p, a, channel_dim=False)
  assert tuple(flat.shape) == (3, 50) and torch.equal(flat, base[..., 0])
  assert torch.equal(hmm.posterior_mode(torch.cat([p, a], -1)), base[..., 0].long())


@pytest.mark.gpu
def test_viterbi_size_rule_is_the_entry_points():
  """`core.hmm_viterbi_takes` against `ddsp_b200_hmm_viterbi` itself."""
  for t, k in ((1551, 1024), (1552, 1024), (10240, 128), (10241, 128), (10240, 97),
               (8533, 160), (8534, 160), (1, 1024)):
    x = torch.zeros((1, t, 2), device=DEV)
    ls = torch.ones((k, 2), device=DEV)
    path = torch.empty((1, t), dtype=torch.int64, device=DEV)
    try:
      core._launch('ddsp_b200_hmm_viterbi', x, ls, ls, path, 1, t, k, 0.9, 0.001)
      took = True
    except NotImplementedError:
      took = False
    assert took == core.hmm_viterbi_takes(t, k), (t, k)


@pytest.mark.gpu
def test_zero_batch():
  hmm = losses.HmmTranscriber(n_timesteps=20)
  z = torch.zeros((0, 20, 1), device=DEV, requires_grad=True)
  loss = hmm.nll(z, z, per_example_loss=True)
  assert tuple(loss.shape) == (0,)
  loss.sum().backward()
  assert tuple(z.grad.shape) == (0, 20, 1)
  assert tuple(hmm.predict_midi(z, z).shape) == (0, 20, 1)


@pytest.mark.gpu
def test_straight_through():
  x = torch.linspace(-3.0, 3.0, 17, device=DEV, requires_grad=True)
  q = torch.round(x.detach())
  y = losses.HmmTranscriber.straight_through(x, q)
  assert torch.equal(y, q)
  g = torch.arange(17.0, device=DEV)
  y.backward(g)
  assert torch.equal(x.grad, g)


@pytest.mark.gpu
def test_chain_from_f0_through_hz_to_midi():
  """nll as a loss on core.hz_to_midi(f0), backward to f0 in Hz: the gradient is the
  float64 HMM's d pitch, at the pitch hz_to_midi produced, times d midi / d f0 =
  12 / (f0 ln 2)."""
  t = 400
  x = _notes(80, 3, t)
  f0 = (440.0 * 2.0 ** ((x[..., :1].astype(np.float64) - 69.0) / 12.0)).astype(np.float32)
  f0_t = _cuda(f0, grad=True)
  hmm = losses.HmmTranscriber(n_timesteps=t, weight=5.0)
  pitch = core.hz_to_midi(f0_t)
  loss = hmm(pitch, _cuda(x[..., 1:]))
  loss.backward()
  pitch32 = pitch.detach().double().cpu().numpy()
  x64 = torch.from_numpy(np.concatenate([pitch32, x[..., 1:]], -1)).to(DEV).requires_grad_()
  want = 5.0 * torch.mean(-ref.log_prob(x64, *_params({}, DEV)) / t)
  want.backward()
  assert _rel(loss.item(), want.item()) <= 1e-5
  w = x64.grad[..., :1].cpu().numpy() * 12.0 / (f0.astype(np.float64) * np.log(2.0))
  got = f0_t.grad.double().cpu().numpy()
  assert np.abs(got - w).max() <= 2e-4 * np.abs(w).max()


# ---- conventions ------------------------------------------------------------------------
def _step(x, kw):
  loc, scale, hold, other = _hmm_args(kw)
  x.grad = None
  lp = core.hmm_log_prob(x, loc, scale, hold, other)
  lp.backward(torch.linspace(-1.0, 2.0, x.shape[0], device=DEV))
  return lp.detach().clone(), x.grad.clone()


@pytest.mark.gpu
def test_gradients_are_bit_reproducible():
  x = _cuda(_notes(90, 256, 1000), grad=True)
  (a0, g0), (a1, g1) = _step(x, {}), _step(x, {})
  assert torch.equal(a0, a1) and torch.equal(g0, g1)


@pytest.mark.gpu
def test_cuda_graph_capture_equals_eager():
  x = _cuda(_notes(91, 8, 300), grad=True)
  hmm = losses.HmmTranscriber(n_timesteps=300)
  p, a = x[..., :1].detach().clone().requires_grad_(), x[..., 1:].detach().clone()
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    for _ in range(2):
      p.grad = None
      eager = hmm.nll(p, a)
      eager.backward()
      eager_midi = hmm.predict_midi(p, a)
  torch.cuda.current_stream().wait_stream(s)
  eager_grad = p.grad.clone()
  graph = torch.cuda.CUDAGraph()
  p.grad = None
  with torch.cuda.graph(graph):
    loss = hmm.nll(p, a)
    loss.backward()
    midi = hmm.predict_midi(p, a)
  graph.replay()
  torch.cuda.synchronize()
  assert torch.equal(loss, eager) and torch.equal(p.grad, eager_grad)
  assert torch.equal(midi, eager_midi)


@pytest.mark.gpu
def test_side_stream():
  """Launched on the caller's current stream: results on a busy side stream equal the
  default stream's."""
  x = _cuda(_notes(92, 16, 500))
  kw = dict(n_pitches=128)
  want = core.hmm_log_prob(x, *_hmm_args(kw))
  want_path = core.hmm_posterior_mode(x, *_hmm_args(kw))
  args = _hmm_args(kw)
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    torch.cuda._sleep(10_000_000)
    xs = x.clone().requires_grad_()
    got = core.hmm_log_prob(xs, *args)
    got.sum().backward()
    path = core.hmm_posterior_mode(xs, *args)
  torch.cuda.synchronize()
  assert torch.equal(got, want) and torch.equal(path, want_path)
  _, g = _step(x.clone().requires_grad_(), kw)
  xs.grad = None
  with torch.cuda.stream(s):
    torch.cuda._sleep(10_000_000)
    core.hmm_log_prob(xs, *args).backward(torch.linspace(-1.0, 2.0, 16, device=DEV))
  torch.cuda.synchronize()
  assert torch.equal(xs.grad, g)


@pytest.mark.gpu
@pytest.mark.parametrize('form', ['float16', 'bfloat16', 'float64', 'strided', 'offset'])
def test_input_forms_give_the_canonical_bits(form):
  """Other dtypes, strided and offset pitch / amps: the bits of the float32 contiguous
  call on the same values (after the cast), gradients cast back, inputs unchanged."""
  from tests.test_gpu_input_conventions import at_offset, strided
  t = 200
  x = _notes(93, 4, t)
  hmm = losses.HmmTranscriber(n_timesteps=t)

  def make(v):
    v = torch.as_tensor(v, device=DEV)
    if form in ('float16', 'bfloat16', 'float64'):
      return v.to(getattr(torch, form))
    return strided(v) if form == 'strided' else at_offset(v, 3)
  p, a = make(x[..., :1]), make(x[..., 1:])
  p.requires_grad_()
  before = (p.detach().clone(), a.clone())
  loss = hmm.nll(p, a, per_example_loss=True)
  loss.sum().backward()
  midi = hmm.predict_midi(p, a)
  assert torch.equal(p.detach(), before[0]) and torch.equal(a, before[1])
  pc = p.detach().float().contiguous().requires_grad_()
  ac = a.float().contiguous()
  want = hmm.nll(pc, ac, per_example_loss=True)
  want.sum().backward()
  assert torch.equal(loss, want)
  assert p.grad.dtype == p.dtype and torch.equal(p.grad, pc.grad.to(p.dtype))
  assert torch.equal(midi, hmm.predict_midi(pc, ac))


@pytest.mark.gpu
@pytest.mark.parametrize('k,t', [(128, 1000), (33, 97), (1024, 100), (2, 3), (128, 1)])
def test_under_every_poison(k, t):
  """Forward, backward (checkpoints included) and Viterbi under the guarded allocator of
  test_gpu_memory_bounds.py: fences intact and bit-identical results whatever the fresh
  memory holds."""
  from tests.test_gpu_memory_bounds import POISONS, guarded
  x = _notes(94 + k, 3, t, k)
  kw = dict(n_pitches=k)
  runs = []
  for p in POISONS:
    with guarded(p):
      xs = _cuda(x, grad=True)
      lp, g = _step(xs, kw)
      path = core.hmm_posterior_mode(xs, *_hmm_args(kw))
      runs.append([lp, g, path])
  for run in runs[1:]:
    for got, want in zip(run, runs[0]):
      assert torch.equal(got, want)
  assert torch.isfinite(runs[0][0]).all() and torch.isfinite(runs[0][1]).all()


@pytest.mark.gpu
def test_peak_memory():
  """B = 256, T = 1000, K = 128, forward and backward: the checkpoints are 4 MB, the
  gradient 2 MB; a stored [B, T, K] alpha would be 131 MB."""
  x = _cuda(_notes(95, 256, 1000), grad=True)
  args = _hmm_args({})
  torch.cuda.synchronize()
  base = torch.cuda.memory_allocated()
  torch.cuda.reset_peak_memory_stats()
  core.hmm_log_prob(x, *args).sum().backward()
  torch.cuda.synchronize()
  rise = torch.cuda.max_memory_allocated() - base
  assert rise < 16 * 2**20, rise / 2**20
  assert torch.isfinite(x.grad).all()
