"""core.harmonic_oscillator_bank (core.py:966-1025) and streaming_harmonic_synthesis on
top of it (core.py:1114-1164): forward against the float64 oracle, gradients against a
differentiable float64 restatement (tests/harmonic_bank_ref.py), routing, and the input
conventions of the other ops.  The float64 references are pinned on CPU to the
unmodified reference run on the shim (tests/golden/harmonic_oscillator_bank.npz)."""
import math
import os

import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, core
from oracle import ddsp_oracle as oracle
from tests import harmonic_bank_ref as ref
from tests.golden import make_harmonic_oscillator_bank_golden as hg
from tests.test_gpu_input_conventions import assert_same_bits, at_offset
from tests.test_gpu_memory_bounds import POISONS, _fenced, _fences_intact, guarded
from tests.util import HostQueriesOnly, rel_err

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'harmonic_oscillator_bank.npz')
TOL = 1e-4


# ---- CPU: the references against the reference ------------------------------------
def test_restatement_matches_the_reference():
  g = np.load(GOLDEN)
  for i, ((_, _, _, mode), (f, a, p)) in enumerate(zip(hg.BANK_CASES, hg.bank_inputs())):
    audio, final = ref.harmonic_oscillator_bank(f, a, p, 16000, mode)
    np.testing.assert_allclose(audio.numpy(), g['bank_audio_wide_%d' % i], atol=1e-9)
    np.testing.assert_allclose(final.numpy(), g['bank_phase_wide_%d' % i], atol=1e-9)
    o_audio, o_final = oracle.harmonic_oscillator_bank(f, a, p, 16000, mode)
    np.testing.assert_allclose(o_audio, g['bank_audio_wide_%d' % i], atol=1e-9)
    np.testing.assert_allclose(o_final, g['bank_phase_wide_%d' % i], atol=1e-9)


def test_streaming_oracle_matches_the_reference():
  g = np.load(GOLDEN)
  for i, ((_, n, _, method, _), (f0, amp, hd, p)) in enumerate(
      zip(hg.STREAM_CASES, hg.stream_inputs())):
    audio, final = oracle.streaming_harmonic_synthesis(f0, amp, hd, p, n, 16000, method)
    np.testing.assert_allclose(audio, g['stream_audio_wide_%d' % i], atol=1e-9)
    np.testing.assert_allclose(final, g['stream_phase_wide_%d' % i], atol=1e-9)


# ---- CPU: routing --------------------------------------------------------------------
@pytest.fixture
def no_device(monkeypatch):
  monkeypatch.setattr(_lib, 'load', lambda real=_lib.load(): HostQueriesOnly(real))
  monkeypatch.setattr(torch.Tensor, 'to', lambda *a, **k: pytest.fail('tensor moved'))


@pytest.mark.parametrize('shapes', [
    ((2, 10), (2, 10, 3), None),            # frequency not 3-D
    ((2, 10, 2), (2, 10, 3), None),         # two frequency channels
    ((2, 10, 1), (2, 11, 3), None),         # N differs
    ((2, 0, 1), (2, 0, 3), None),           # N = 0
    ((2, 10, 1), (2, 10, 0), None),         # K = 0
    ((2, 10, 1), (2, 10, 3), (2, 1)),       # initial phase not [B, 1, 1]
    ((2, 10, 1), (2, 10, 3), (3, 1, 1)),    # initial phase of another batch
])
def test_bank_shapes_raise_before_device_work(shapes, no_device):
  sf, sa, sp = shapes
  with pytest.raises(ValueError):
    core.harmonic_oscillator_bank(torch.zeros(sf), torch.zeros(sa),
                                  None if sp is None else torch.zeros(sp))


def test_streaming_shapes_raise_before_device_work(no_device):
  with pytest.raises(ValueError):
    core.streaming_harmonic_synthesis(torch.zeros(2, 4, 1), torch.zeros(2, 4, 1),
                                      torch.zeros(2, 5, 3), n_samples=64)


def test_under_grad_a_shape_without_backward_raises(no_device):
  """A batch past the backward's grid limit has no backward: the composition reaches
  _no_grad_path instead of returning detached audio."""
  b = 65536
  f0 = torch.full((b, 1, 1), 100.0, requires_grad=True)
  with pytest.raises(RuntimeError, match='requires grad'):
    core.streaming_harmonic_synthesis(f0, torch.ones(b, 1, 1), n_samples=2,
                                      amp_resample_method='nearest')
  with pytest.raises(RuntimeError, match='requires grad'):
    core.harmonic_oscillator_bank(torch.zeros(b, 1, 1), torch.ones(b, 1, 2),
                                  torch.zeros(b, 1, 1, requires_grad=True))


def test_backward_takes():
  lib = _lib.load()
  assert lib.ddsp_b200_harmonic_oscillator_bank_backward_takes(65535, 1, 1) == 1
  assert lib.ddsp_b200_harmonic_oscillator_bank_backward_takes(65536, 1, 1) == 0
  assert lib.ddsp_b200_harmonic_oscillator_bank_backward_takes(1, 0, 1) == 0


# ---- GPU -----------------------------------------------------------------------------
def _inputs(b, n, k, seed=0, init=True):
  rng = np.random.default_rng(seed)
  f = rng.uniform(40.0, 1200.0, (b, n, 1)).astype(np.float32)
  a = rng.uniform(-1.0, 1.0, (b, n, k)).astype(np.float32)
  p = rng.uniform(-7.0, 7.0, (b, 1, 1)).astype(np.float32) if init else None
  return f, a, p


def _cuda(x):
  return None if x is None else torch.as_tensor(x, device='cuda')


def _check_bank(f, a, p, mode):
  audio, final = core.harmonic_oscillator_bank(_cuda(f), _cuda(a), _cuda(p), 16000, mode)
  want_audio, want_final = oracle.harmonic_oscillator_bank(f, a, p, 16000, mode)
  assert audio.shape == want_audio.shape and final.shape == (f.shape[0], 1, 1)
  assert rel_err(audio.cpu().numpy(), want_audio)[0] <= TOL
  got = final.double().cpu().numpy()
  if mode:   # compared mod 2 pi
    d = np.remainder(got - want_final + np.pi, 2 * np.pi) - np.pi
    assert np.abs(d).max() <= TOL
  else:   # the exact unwrapped sum, rounded once to float32: one lost turn would show
    ulp = np.spacing(np.abs(want_final).astype(np.float32)).astype(np.float64)
    assert np.all(np.abs(got - want_final) <= ulp)
  return audio, final


@pytest.mark.gpu
@pytest.mark.parametrize('n,k', [(1, 1), (1, 100), (63, 7), (63, 64), (64000, 1),
                                 (64000, 64), (64000, 100), (1000000, 1), (1000000, 7)])
@pytest.mark.parametrize('init', [False, True])
@pytest.mark.parametrize('mode', [True, False])
def test_bank_matches_float64(n, k, init, mode):
  f, a, p = _inputs(2 if n * k < 10**7 else 1, n, k, seed=n + k, init=init)
  _check_bank(f, a, p, mode)


@pytest.mark.gpu
def test_audio_does_not_depend_on_the_mode():
  f, a, p = _inputs(3, 5000, 9)
  x = core.harmonic_oscillator_bank(_cuda(f), _cuda(a), _cuda(p), 16000, True)[0]
  y = core.harmonic_oscillator_bank(_cuda(f), _cuda(a), _cuda(p), 16000, False)[0]
  assert torch.equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize('mode', [True, False])
def test_chained_calls_match_one_call(mode):
  """Eight calls, each fed the previous final_phase, against one call.  The wrapped phase
  (use_angular_cumsum=True, the streaming mode) stays in [0, 2 pi) + initial_phase, so
  the chained audio matches; the unwrapped one grows to ~1e4 rad here, and the float32
  phase carried between calls is then only good to ~1e-3 rad, as in the reference, so
  that mode checks the carried phase alone, to float32 rounding."""
  f, a, p = _inputs(2, 8 * 3000, 16, seed=5)
  whole, final = core.harmonic_oscillator_bank(_cuda(f), _cuda(a), _cuda(p), 16000, mode)
  phase, parts = _cuda(p), []
  for i in range(8):
    s = slice(3000 * i, 3000 * (i + 1))
    out, phase = core.harmonic_oscillator_bank(_cuda(f[:, s]), _cuda(a[:, s]), phase, 16000,
                                               mode)
    parts.append(out)
  chained = torch.cat(parts, 1)
  d = (phase - final).double().cpu().numpy()
  if mode:
    assert rel_err(chained.cpu().numpy(), whole.cpu().numpy())[0] <= TOL
    d = np.remainder(d + np.pi, 2 * np.pi) - np.pi
    assert np.abs(d).max() <= TOL
  else:
    assert np.abs(d).max() <= 8 * 2**-23 * float(final.abs().max())


@pytest.mark.gpu
def test_empty_batch():
  audio, final = core.harmonic_oscillator_bank(torch.zeros(0, 5, 1, device='cuda'),
                                               torch.zeros(0, 5, 3, device='cuda'))
  assert audio.shape == (0, 5) and final.shape == (0, 1, 1)


def _grads(f, a, p, g, g_phi, mode=True, f_scale=1.0):
  """Kernel and float64 gradients of <g, audio> + <g_phi, final_phase>."""
  out = []
  for dtype, fn in ((torch.float32, core.harmonic_oscillator_bank),
                    (torch.float64, ref.harmonic_oscillator_bank)):
    ft = torch.tensor(f, dtype=dtype, device='cuda', requires_grad=True)
    at = torch.tensor(a, dtype=dtype, device='cuda', requires_grad=True)
    pt = torch.tensor(p, dtype=dtype, device='cuda', requires_grad=True)
    audio, final = fn(ft, at, pt, 16000, mode)
    loss = 0.0
    if g is not None:
      loss = loss + (audio * torch.as_tensor(g, dtype=dtype, device='cuda')).sum()
    if g_phi is not None:
      loss = loss + (final * torch.as_tensor(g_phi, dtype=dtype, device='cuda')).sum()
    loss.backward()
    out.append([np.zeros(t.shape) if t.grad is None else t.grad.double().cpu().numpy()
                for t in (ft, at, pt)])
  return out


def _assert_grads(got, want):
  for x, y, name in zip(got, want, ('d f', 'd a', 'd init')):
    assert rel_err(x, y)[0] <= TOL, name


@pytest.mark.gpu
@pytest.mark.parametrize('n,k', [(1, 1), (63, 7), (5000, 64), (64000, 3)])
def test_gradients_match_float64(n, k):
  f, a, p = _inputs(2, n, k, seed=11)
  rng = np.random.default_rng(3)
  got, want = _grads(f, a, p, rng.standard_normal((2, n)), rng.standard_normal((2, 1, 1)))
  _assert_grads(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize('mode', [True, False])
def test_final_phase_gradient_alone(mode):
  f, a, p = _inputs(2, 700, 5, seed=12)
  got, want = _grads(f, a, p, None, np.array([[[1.5]], [[-0.5]]]), mode)
  _assert_grads(got, want)
  assert np.all(got[1] == 0.0)


@pytest.mark.gpu
def test_backward_reruns_bitwise():
  f, a, p = _inputs(3, 20000, 33, seed=13)
  g = torch.randn(3, 20000, device='cuda')
  runs = []
  for _ in range(2):
    ts = [_cuda(x).requires_grad_() for x in (f, a, p)]
    audio, final = core.harmonic_oscillator_bank(*ts)
    ((audio * g).sum() + final.sum()).backward()
    runs.append([t.grad for t in ts])
  for x, y in zip(*runs):
    assert torch.equal(x, y)


@pytest.mark.gpu
def test_amplitude_gradient_does_not_depend_on_the_others():
  f, a, p = _inputs(2, 3000, 20, seed=14)
  g = torch.randn(2, 3000, device='cuda')
  at = _cuda(a).requires_grad_()
  (core.harmonic_oscillator_bank(_cuda(f), at, _cuda(p))[0] * g).sum().backward()
  ts = [_cuda(x).requires_grad_() for x in (f, a, p)]
  (core.harmonic_oscillator_bank(*ts)[0] * g).sum().backward()
  assert torch.equal(at.grad, ts[1].grad)


# ---- streaming_harmonic_synthesis ------------------------------------------------------
def _stream_inputs(b, f, k, seed):
  rng = np.random.default_rng(seed)
  return (rng.uniform(100.0, 2500.0, (b, f, 1)).astype(np.float32),
          rng.uniform(0.1, 1.0, (b, f, 1)).astype(np.float32),
          rng.uniform(0.0, 1.0, (b, f, k)).astype(np.float32),
          rng.uniform(0.0, 6.0, (b, 1, 1)).astype(np.float32))


@pytest.mark.gpu
@pytest.mark.parametrize('method', ['linear', 'window', 'nearest', 'cubic'])
@pytest.mark.parametrize('n', [4000, 4037])
def test_streaming_forward_matches_float64(method, n):
  if method == 'window' and n % 20:
    pytest.skip('window upsampling needs an integer hop (the reference raises)')
  f0, amp, hd, p = _stream_inputs(2, 20, 12, seed=n)
  audio, final = core.streaming_harmonic_synthesis(_cuda(f0), _cuda(amp), _cuda(hd), _cuda(p),
                                                   n_samples=n, amp_resample_method=method)
  want_audio, want_final = _oracle_streaming(f0, amp, hd, p, n, method)
  assert rel_err(audio.cpu().numpy(), want_audio)[0] <= TOL
  d = np.remainder(final.double().cpu().numpy() - want_final + np.pi, 2 * np.pi) - np.pi
  assert np.abs(d).max() <= TOL


def _oracle_streaming(f0, amp, hd, p, n, method):
  """core.py:1140-1164 in float64.  The composition's resample kernel reproduces
  TensorFlow's float32 index arithmetic (so 'nearest' picks the same frames); the fused
  kernel that no-grad calls at an integer hop keep interpolates at exact positions."""
  fused = method in ('linear', 'window') and n % f0.shape[1] == 0
  hd = oracle.normalize_harmonics(hd, f0, 16000)
  fe = oracle.resample(f0, n, tf_index_math=not fused)
  ae = oracle.resample(amp * hd, n, method=method, tf_index_math=not fused)
  return oracle.harmonic_oscillator_bank(fe, ae, p, 16000)


def _torch_streaming(f0, amp, hd, p, n, method):
  """core.py:1140-1164 in float64 torch: the reference's composition, each resample an
  explicit linear map (the oracle's resample of one-hot frames, with TensorFlow's index
  arithmetic)."""
  b, f, _ = f0.shape
  eye = np.eye(f)[None, :, :]                                   # [1, F, F]
  def rs(x, m):
    basis = oracle.resample(eye, n, method=m, tf_index_math=True)  # [1, N, F]
    return torch.einsum('nf,bfc->bnc', torch.as_tensor(basis[0], device=x.device), x)
  k = hd.shape[-1]
  harm = f0 * torch.arange(1, k + 1, dtype=f0.dtype, device=f0.device)
  hd = torch.where(harm >= 8000.0, torch.zeros_like(hd), hd)
  hd = hd / torch.where(hd.sum(-1, keepdim=True) == 0, torch.full_like(hd[..., :1], 1e-7),
                        hd.sum(-1, keepdim=True))
  return ref.harmonic_oscillator_bank(rs(f0, 'linear'), rs(amp * hd, method), p, 16000)


@pytest.mark.gpu
@pytest.mark.parametrize('method', ['linear', 'window', 'nearest', 'cubic'])
@pytest.mark.parametrize('n', [2000, 2013])
def test_streaming_gradients_match_float64(method, n):
  if method == 'window' and n % 10:
    pytest.skip('window upsampling needs an integer hop (the reference raises)')
  f0, amp, hd, p = _stream_inputs(2, 10, 6, seed=n + 1)
  rng = np.random.default_rng(n)
  g, g_phi = rng.standard_normal((2, n)), rng.standard_normal((2, 1, 1))
  res = []
  for dtype in (torch.float32, torch.float64):
    ts = [torch.tensor(x, dtype=dtype, device='cuda', requires_grad=True)
          for x in (f0, amp, hd, p)]
    if dtype == torch.float32:
      audio, final = core.streaming_harmonic_synthesis(*ts, n_samples=n,
                                                       amp_resample_method=method)
    else:
      audio, final = _torch_streaming(*ts, n, method)
    ((audio * torch.as_tensor(g, dtype=dtype, device='cuda')).sum() +
     (final * torch.as_tensor(g_phi, dtype=dtype, device='cuda')).sum()).backward()
    res.append([t.grad.double().cpu().numpy() for t in ts])
  for x, y, name in zip(*res, ('d f0', 'd amplitudes', 'd distribution', 'd phase')):
    assert rel_err(x, y)[0] <= TOL, name


@pytest.mark.gpu
def test_streaming_integer_hop_without_grad_keeps_the_fused_kernel(monkeypatch):
  f0, amp, hd, p = _stream_inputs(2, 20, 12, seed=21)
  calls = []
  real = core._launch
  monkeypatch.setattr(core, '_launch', lambda name, *a: (calls.append(name), real(name, *a)))
  core.streaming_harmonic_synthesis(_cuda(f0), _cuda(amp), _cuda(hd), _cuda(p), n_samples=4000)
  assert 'ddsp_b200_streaming_harmonic_forward' in calls
  assert 'ddsp_b200_harmonic_oscillator_bank' not in calls


# ---- input conventions ---------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_half_inputs_give_the_canonical_bits_and_gradients_in_their_dtype(dtype):
  f, a, p = _inputs(2, 3000, 10, seed=31)
  fh, ah, ph = [torch.as_tensor(x, device='cuda').to(dtype) for x in (f, a, p)]
  want = core.harmonic_oscillator_bank(fh.float(), ah.float(), ph.float())
  got = core.harmonic_oscillator_bank(fh, ah, ph)
  for x, y in zip(got, want):
    assert torch.equal(x, y)
  ts = [t.clone().requires_grad_() for t in (fh, ah, ph)]
  audio, final = core.harmonic_oscillator_bank(*ts)
  (audio.sum() + final.sum()).backward()
  assert all(t.grad.dtype == dtype for t in ts)


@pytest.mark.gpu
def test_strided_and_offset_inputs_give_the_canonical_bits():
  f, a, p = _inputs(2, 3000, 10, seed=32)
  want = core.harmonic_oscillator_bank(_cuda(f), _cuda(a), _cuda(p))
  big = torch.zeros(2, 3000, 23, device='cuda')
  big[..., 3:13] = _cuda(a)
  fs = torch.zeros(2, 3000, 2, device='cuda')
  fs[..., 1:] = _cuda(f)
  got = core.harmonic_oscillator_bank(fs[..., 1:], big[..., 3:13], _cuda(p))
  for x, y in zip(got, want):
    assert torch.equal(x, y)


# ---- poisoned and fenced memory (the patterns of test_gpu_memory_bounds.py) --------------
# (B, N, K, what requires grad, use_angular_cumsum): partial 1024-sample chunks, partial
# backward segments, spans of several chunks (N = 140000), partial lanes over k, and the
# backward with every output and with d a only.
MEMORY_CASES = [(2, 3037, 33, 'all', True), (2, 3037, 33, 'a', True),
                (1, 140000, 3, 'all', False), (3, 1, 1, 'all', True), (2, 700, 64, 'f', False)]


def _memory_inputs(case):
  b, n, k, _, _ = case
  f, a, p = _inputs(b, n, k, seed=n + k)
  rng = np.random.default_rng(k)
  t = {'f': _cuda(f), 'a': _cuda(a), 'p': _cuda(p)}
  gs = [_cuda(rng.standard_normal((b, n)).astype(np.float32)),
        _cuda(rng.standard_normal((b, 1, 1)).astype(np.float32))]
  return t, gs


def _memory_run(case, t, gs):
  """Outputs and the gradients of <g, audio> + <g_phi, final_phase> to what requires grad;
  the inputs must come back unchanged."""
  want = {'all': 'fap', 'a': 'a', 'f': 'f'}[case[3]]
  before = {k: v.clone() for k, v in t.items()}
  leaves = {k: v.detach().requires_grad_(k in want) for k, v in t.items()}
  audio, final = core.harmonic_oscillator_bank(leaves['f'], leaves['a'], leaves['p'], 16000,
                                               case[4])
  torch.autograd.backward([audio, final], gs)
  for k, v in t.items():
    assert torch.equal(v, before[k]), ('input changed', k)
  return [audio.detach(), final.detach()], {k: leaves[k].grad for k in want}


@pytest.mark.gpu
@pytest.mark.parametrize('case', MEMORY_CASES, ids=[str(c) for c in MEMORY_CASES])
def test_poisoned_allocations_give_the_canonical_bits(case):
  """Every allocation of core and autograd is poisoned with 0x00, 0xFF (NaN) and 0x7F and
  fenced with canaries: outputs and gradients are bit-identical to a plain run, and no
  fence is written."""
  t, gs = _memory_inputs(case)
  want_outs, want_grads = _memory_run(case, t, gs)
  for p in POISONS:
    with guarded(p):
      outs, grads = _memory_run(case, t, gs)
    assert_same_bits(outs, want_outs, (case, p))
    for k in want_grads:
      assert_same_bits(grads[k], want_grads[k], (case, p, k))


@pytest.mark.gpu
@pytest.mark.parametrize('case', MEMORY_CASES, ids=[str(c) for c in MEMORY_CASES])
def test_fenced_operands_give_the_canonical_bits(case):
  """Every input and upstream gradient between 64 KiB fences of NaN, and of 7.0, at
  storage offsets of 0 and 1 element: the bits of fresh operands at that offset, with the
  fences unchanged."""
  t, gs = _memory_inputs(case)
  for off in (0, 1):
    want_outs, want_grads = _memory_run(case, {k: at_offset(v, off) for k, v in t.items()},
                                        [at_offset(g, off) for g in gs])
    for fill in (math.nan, 7.0):
      regions, ins, fgs = [], {}, []
      for k, v in t.items():
        ins[k], r = _fenced(v, fill, off)
        regions.append(r)
      for g in gs:
        fg, r = _fenced(g, fill, off)
        fgs.append(fg)
        regions.append(r)
      outs, grads = _memory_run(case, ins, fgs)
      assert_same_bits(outs, want_outs, (case, fill, off))
      for k in want_grads:
        assert_same_bits(grads[k], want_grads[k], (case, fill, off, k))
      torch.cuda.synchronize()
      for r in regions:
        _fences_intact(r, (case, fill, off))


@pytest.mark.gpu
def test_forward_takes_more_than_65535_items():
  """The forward puts the batch on grid.x; the backward's cluster grid takes at most
  65535 items, and under grad a larger batch is refused before any launch."""
  f, a, p = _inputs(70000, 3, 2, seed=40)
  audio, final = core.harmonic_oscillator_bank(_cuda(f), _cuda(a), _cuda(p), 16000, True)
  want_audio, want_final = oracle.harmonic_oscillator_bank(f, a, p, 16000, True)
  assert rel_err(audio.cpu().numpy(), want_audio)[0] <= TOL
  d = np.remainder(final.double().cpu().numpy() - want_final + np.pi, 2 * np.pi) - np.pi
  assert np.abs(d).max() <= TOL
  with pytest.raises(RuntimeError, match='requires grad'):
    core.harmonic_oscillator_bank(_cuda(f), _cuda(a).requires_grad_(), _cuda(p))


@pytest.mark.gpu
def test_cuda_graph_replay_equals_eager():
  f, a, p = [_cuda(x) for x in _inputs(2, 4000, 12, seed=34)]
  eager = core.harmonic_oscillator_bank(f, a, p)
  s = torch.cuda.Stream()
  with torch.cuda.stream(s):
    core.harmonic_oscillator_bank(f, a, p)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
      out = core.harmonic_oscillator_bank(f, a, p)
  graph.replay()
  torch.cuda.synchronize()
  for x, y in zip(out, eager):
    assert torch.equal(x, y)
