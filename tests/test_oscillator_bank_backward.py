"""The backward of core.oscillator_bank and core.angular_cumsum (csrc/oscbank.cuh,
`oscbank_backward`): the C ABI's checks and the routing errors (CPU); the gradients
against float64 autograd of tests/grad_ref.py, exact zeros, inner-product identities
against the forward kernels, a chain through resample and SpectralLoss,
reproducibility, CUDA-graph capture, poisoned and fenced memory, input forms, streams
and devices (GPU).

Tolerance: max-abs error <= 2e-4 of each gradient's peak and rel-L2 <= 1e-4 against
float64 (DESIGN.md §3.8, §3.14).  The float64 reference uses the kernel's float32
Nyquist decision (grad_ref decides the mask on the float32 frequencies).
"""
import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, core, losses
from tests import grad_ref, routing_ref

DEV = 'cuda'
SEGMENTS = 128          # time segments of one cluster: 8 CTAs x 16 warps


# ---- CPU ---------------------------------------------------------------------
P = 0x1000        # a device pointer the library never dereferences on the host
E_INVALID = _lib.E_INVALID
SR = 16000.0


def _ob(f=P, a=P, g=P, df=P, da=P, B=2, N=640, K=4, sr=SR, ss=1):
  return (f, a, g, df, da, B, N, K, sr, ss, None)


def _ac(g=P, d=P, B=2, N=640, C=4):
  return (g, d, B, N, C, None)


_F, _C = 'oscillator_bank_backward', 'angular_cumsum_backward'
_ABI_CASES = [
    ('ob-null-f', _F, _ob(f=None), E_INVALID, b'oscillator_bank_backward: null pointer'),
    ('ob-null-a', _F, _ob(a=None), E_INVALID, b'oscillator_bank_backward: null pointer'),
    ('ob-null-g', _F, _ob(g=None), E_INVALID, b'oscillator_bank_backward: null pointer'),
    ('ob-B', _F, _ob(B=-1), E_INVALID, b'oscillator_bank_backward: bad shape B=-1 N=640 K=4'),
    ('ob-N', _F, _ob(N=-2), E_INVALID, b'oscillator_bank_backward: bad shape B=2 N=-2 K=4'),
    ('ob-K', _F, _ob(K=-3), E_INVALID, b'oscillator_bank_backward: bad shape B=2 N=640 K=-3'),
    ('ob-sr0', _F, _ob(sr=0.0), E_INVALID,
     b'oscillator_bank_backward: sample_rate must be positive'),
    ('ob-sr-neg', _F, _ob(sr=-16000.0), E_INVALID,
     b'oscillator_bank_backward: sample_rate must be positive'),
    ('ob-flag', _F, _ob(ss=2), E_INVALID,
     b'oscillator_bank_backward: sum_sinusoids must be 0 or 1, got 2'),
    ('ob-flag-neg', _F, _ob(ss=-1), E_INVALID,
     b'oscillator_bank_backward: sum_sinusoids must be 0 or 1, got -1'),
    ('ob-grid', _F, _ob(B=65536), E_INVALID,
     b'oscillator_bank_backward: B=65536 exceeds the 65535 grid limit'),
    ('ob-B0', _F, _ob(B=0), 0, None),
    ('ob-N0', _F, _ob(N=0), 0, None),
    ('ob-K0', _F, _ob(K=0), 0, None),
    ('ob-empty-null', _F, _ob(None, None, None, None, None, N=0), 0, None),
    ('ob-no-gradients', _F, _ob(df=None, da=None), 0, None),
    ('ac-null-g', _C, _ac(g=None), E_INVALID, b'angular_cumsum_backward: null pointer'),
    ('ac-null-d', _C, _ac(d=None), E_INVALID, b'angular_cumsum_backward: null pointer'),
    ('ac-B', _C, _ac(B=-1), E_INVALID, b'angular_cumsum_backward: bad shape B=-1 N=640 C=4'),
    ('ac-N', _C, _ac(N=-1), E_INVALID, b'angular_cumsum_backward: bad shape B=2 N=-1 C=4'),
    ('ac-C', _C, _ac(C=-5), E_INVALID, b'angular_cumsum_backward: bad shape B=2 N=640 C=-5'),
    ('ac-grid', _C, _ac(B=70000), E_INVALID,
     b'angular_cumsum_backward: B=70000 exceeds the 65535 grid limit'),
    ('ac-B0', _C, _ac(B=0), 0, None),
    ('ac-N0', _C, _ac(N=0), 0, None),
    ('ac-C0', _C, _ac(C=0), 0, None),
    ('ac-empty-null', _C, _ac(None, None, C=0), 0, None),
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
  """Neither backward entry point takes a workspace or has a query."""
  for n in ('ddsp_b200_oscillator_bank_backward', 'ddsp_b200_angular_cumsum_backward'):
    args = _lib.SIGNATURES[n][1]
    assert _lib._sz not in args, n
    assert n + '_workspace' not in _lib.SIGNATURES


def test_tf_sequential_refuses_grad(monkeypatch):
  """The float32 debug modes have no backward: under grad they raise
  NotImplementedError before anything is launched."""
  monkeypatch.setattr(core, 'torch_float32', lambda x, device=None: x.float())
  monkeypatch.setattr(core, '_launch', lambda *a: pytest.fail('launched'))
  f = torch.zeros((1, 8, 2), requires_grad=True)
  with pytest.raises(NotImplementedError, match='forward-only'):
    core.oscillator_bank(f, torch.ones((1, 8, 2)), phase_mode='tf_sequential')
  with pytest.raises(NotImplementedError, match='forward-only'):
    core.angular_cumsum(f, tf_sequential=True)


# ---- GPU helpers -------------------------------------------------------------
def _gate(what, got, want):
  got, want = got.detach().double(), want.detach().double().to(got.device)
  assert got.shape == want.shape, (what, got.shape, want.shape)
  err = (got - want).abs().max().item() if got.numel() else 0.0
  peak = want.abs().max().item() if want.numel() else 0.0
  assert err <= 2e-4 * peak, (what, err, peak)
  norm = want.norm().item()
  if norm > 0:
    assert (got - want).norm().item() <= 1e-4 * norm, (what, (got - want).norm().item(), norm)


def _inputs(B, N, K, sr, seed):
  """Frequencies in [-0.3, 0.55] sr (negative ones and masked ones above Nyquist);
  every 7th sample of oscillator 0 exactly at sr / 2 and of oscillator 1 one float32
  ulp below it."""
  gen = torch.Generator(device=DEV).manual_seed(seed)
  f = (torch.rand(B, N, K, device=DEV, generator=gen) * 0.85 - 0.3) * sr
  a = torch.rand(B, N, K, device=DEV, generator=gen) + 0.1
  nyq = np.float32(sr / 2.0)
  f[:, ::7, 0] = float(nyq)
  if K > 1:
    f[:, ::7, 1] = float(np.nextafter(nyq, np.float32(0)))
  return f, a


def _upstream(B, N, K, sum_sinusoids, seed):
  gen = torch.Generator(device=DEV).manual_seed(seed + 1)
  return torch.randn((B, N) if sum_sinusoids else (B, N, K), device=DEV, generator=gen)


def _grads(f, a, g, sr, sum_sinusoids, want=(True, True), clone=True):
  """(out, d f, d a) of one forward and backward; clone=False makes f and a
  themselves the leaves, so the kernels read their memory."""
  fl = (f.clone() if clone else f).requires_grad_(want[0])
  al = (a.clone() if clone else a).requires_grad_(want[1])
  out = core.oscillator_bank(fl, al, sample_rate=sr, sum_sinusoids=sum_sinusoids)
  out.backward(g)
  return out.detach(), fl.grad, al.grad


def _ref_grads(f, a, g, sr, sum_sinusoids):
  f64 = f.double().requires_grad_(True)
  a64 = a.double().requires_grad_(True)
  grad_ref.oscillator_bank(f64, a64, sr, sum_sinusoids).backward(g.double())
  return f64.grad, a64.grad


# the shapes of test_gpu_generic_edges.py::test_oscillator_bank_over_oscillator_blocks_and_chunks,
# and N one below, at and one past the number of time segments
SHAPES = [
    (1, 1, 1, 16000),
    (64, 127, 127, 16000),
    (5, 128, 128, 44100),
    (3, 129, 129, 16000),
    (2, 12345, 300, 48000),
    (1, 64000, 1000, 16000),
    (7, 12345, 1, 44100),
    (2, SEGMENTS - 1, 33, 16000),
    (2, SEGMENTS, 33, 44100),
    (2, SEGMENTS + 1, 33, 48000),
]


@pytest.mark.gpu
@pytest.mark.parametrize('sum_sinusoids', [True, False])
@pytest.mark.parametrize('B,N,K,sr', SHAPES)
def test_gradients_against_float64(B, N, K, sr, sum_sinusoids):
  f, a = _inputs(B, N, K, sr, seed=N + K)
  g = _upstream(B, N, K, sum_sinusoids, seed=N + K)
  _, df, da = _grads(f, a, g, sr, sum_sinusoids)
  want_df, want_da = _ref_grads(f, a, g, sr, sum_sinusoids)
  _gate('d f', df, want_df)
  _gate('d a', da, want_da)


@pytest.mark.gpu
@pytest.mark.parametrize('sum_sinusoids', [True, False])
@pytest.mark.parametrize('N', [SEGMENTS - 1, SEGMENTS + 1, 5000])
def test_every_request_combination(N, sum_sinusoids):
  """d a is bit-identical with and without d f, d f with and without d a, and a
  gradient that is not asked for is not returned."""
  B, K, sr = 3, 45, 16000
  f, a = _inputs(B, N, K, sr, seed=N)
  g = _upstream(B, N, K, sum_sinusoids, seed=N)
  out, df, da = _grads(f, a, g, sr, sum_sinusoids)
  out_a, df_none, da_only = _grads(f, a, g, sr, sum_sinusoids, want=(False, True))
  out_f, df_only, da_none = _grads(f, a, g, sr, sum_sinusoids, want=(True, False))
  assert df_none is None and da_none is None
  assert torch.equal(out, out_a) and torch.equal(out, out_f)
  assert torch.equal(da.view(torch.int32), da_only.view(torch.int32))
  assert torch.equal(df.view(torch.int32), df_only.view(torch.int32))
  want_df, want_da = _ref_grads(f, a, g, sr, sum_sinusoids)
  _gate('d f only', df_only, want_df)
  _gate('d a only', da_only, want_da)


@pytest.mark.gpu
@pytest.mark.parametrize('sum_sinusoids', [True, False])
def test_exact_zeros_at_and_above_nyquist(sum_sinusoids):
  """d a is exactly 0 wherever f >= sr / 2; an oscillator at or above Nyquist at every
  sample has d f and d a exactly 0."""
  B, N, K, sr = 2, 3000, 40, 16000
  f, a = _inputs(B, N, K, sr, seed=3)
  f[:, :, 5] = sr / 2.0
  f[:, :, 6] = 0.7 * sr
  g = _upstream(B, N, K, sum_sinusoids, seed=3)
  _, df, da = _grads(f, a, g, sr, sum_sinusoids)
  assert not da[f >= sr / 2.0].any()
  assert not df[:, :, 5:7].any() and not da[:, :, 5:7].any()
  assert da[f < sr / 2.0].abs().max() > 0.1


@pytest.mark.gpu
@pytest.mark.parametrize('sum_sinusoids', [True, False])
def test_inner_product_identity_for_amplitudes(sum_sinusoids):
  """oscillator_bank is linear in the amplitudes: <d a, v> = <g, oscillator_bank(f, v)>
  against the forward kernel, for three random directions v."""
  B, N, K, sr = 2, 20000, 60, 44100
  f, a = _inputs(B, N, K, sr, seed=5)
  g = _upstream(B, N, K, sum_sinusoids, seed=5)
  _, _, da = _grads(f, a, g, sr, sum_sinusoids)
  gen = torch.Generator(device=DEV).manual_seed(6)
  for _ in range(3):
    v = torch.randn(B, N, K, device=DEV, generator=gen)
    lhs = (da.double() * v.double()).sum().item()
    y = core.oscillator_bank(f, v, sample_rate=sr, sum_sinusoids=sum_sinusoids)
    rhs = (g.double() * y.double()).sum().item()
    scale = (da.double() * v.double()).abs().sum().item()
    assert abs(lhs - rhs) <= 1e-5 * scale, (lhs, rhs, scale)


def _cumsum_grad(x, g):
  xl = x.clone().requires_grad_(True)
  out = core.angular_cumsum(xl)
  out.backward(g)
  return out.detach(), xl.grad


@pytest.mark.gpu
@pytest.mark.parametrize('shape', [(4, 1000), (3, 129, 5), (2, 300, 3, 4), (2, SEGMENTS - 1, 7),
                                   (2, SEGMENTS, 7), (2, SEGMENTS + 1, 7), (1, 64000, 1000),
                                   (5, 1, 33)])
def test_angular_cumsum_gradient_against_float64(shape):
  gen = torch.Generator(device=DEV).manual_seed(len(shape) + shape[1])
  x = (torch.rand(shape, device=DEV, generator=gen) - 0.3) * 2.0
  g = torch.randn(shape, device=DEV, generator=gen)
  _, d = _cumsum_grad(x, g)
  x64 = x.double().requires_grad_(True)
  grad_ref.angular_cumsum(x64).backward(g.double())
  assert d.shape == x.shape
  _gate('d omega', d, x64.grad)


@pytest.mark.gpu
def test_inner_product_identity_for_angular_cumsum():
  """<d omega, v> = <g, running sum of v> for three random directions v."""
  B, N, C = 3, 30000, 20
  gen = torch.Generator(device=DEV).manual_seed(9)
  x = torch.rand(B, N, C, device=DEV, generator=gen)
  g = torch.randn(B, N, C, device=DEV, generator=gen)
  _, d = _cumsum_grad(x, g)
  for _ in range(3):
    v = torch.randn(B, N, C, device=DEV, generator=gen).double()
    lhs = (d.double() * v).sum().item()
    rhs = (g.double() * torch.cumsum(v, 1)).sum().item()
    scale = (g.double().abs() * torch.cumsum(v.abs(), 1)).sum().item()
    assert abs(lhs - rhs) <= 1e-6 * scale, (lhs, rhs, scale)


@pytest.mark.gpu
def test_tutorial_chain_through_resample_and_spectral_loss():
  """Frame-rate frequencies and amplitudes -> core.resample to N -> core.oscillator_bank
  -> SpectralLoss -> backward.  The loss matches the same chain in float64, and the
  gradients reaching the frame-rate inputs match float64 autograd of resample +
  oscillator_bank driven by the audio gradient SpectralLoss sent back, evaluated at the
  float32 envelopes core.resample produced (d envelopes / d frame-rate inputs stays
  float64 resample).  d f sums g a cos(phi) over the rest of the signal, which cancels,
  so the float32 rounding of the spectral loss's gradient and of the envelopes would
  otherwise dominate the comparison."""
  B, F, K, N, sr = 2, 50, 8, 16000, 16000
  gen = torch.Generator(device=DEV).manual_seed(11)
  f = (torch.rand(B, F, K, device=DEV, generator=gen) * 3000 + 100)
  a = torch.rand(B, F, K, device=DEV, generator=gen) * 0.2
  target = torch.randn(B, N, device=DEV, generator=gen) * 0.3
  fl, al = f.clone().requires_grad_(True), a.clone().requires_grad_(True)
  fe, ae = core.resample(fl, N), core.resample(al, N)
  audio = core.oscillator_bank(fe, ae, sample_rate=sr)
  audio.retain_grad()
  loss = losses.SpectralLoss()(target, audio)
  loss.backward()
  f64, a64 = f.double().requires_grad_(True), a.double().requires_grad_(True)
  fe64, ae64 = routing_ref.resample(f64, N), routing_ref.resample(a64, N)
  audio64 = grad_ref.oscillator_bank(fe64 + (fe.detach().double() - fe64).detach(),
                                     ae64 + (ae.detach().double() - ae64).detach(), sr)
  loss64 = grad_ref.spectral_loss(target.double(), audio64.detach())
  assert abs(loss.item() - loss64.item()) <= 1e-5 * abs(loss64.item())
  audio64.backward(audio.grad.double())
  _gate('d frame-rate frequencies', fl.grad, f64.grad)
  _gate('d frame-rate amplitudes', al.grad, a64.grad)


def _step(f, a, g, sum_sinusoids):
  out, df, da = _grads(f, a, g, 16000, sum_sinusoids)
  return [out, df, da]


@pytest.mark.gpu
@pytest.mark.parametrize('sum_sinusoids', [True, False])
def test_bit_reproducible_at_full_size(sum_sinusoids):
  B, N, K = 32, 64000, 100
  gen = torch.Generator(device=DEV).manual_seed(13)
  f = torch.rand(B, N, K, device=DEV, generator=gen) * 7900 + 20
  a = torch.rand(B, N, K, device=DEV, generator=gen) * 0.05
  g = _upstream(B, N, K, sum_sinusoids, seed=13)
  first = _step(f, a, g, sum_sinusoids)
  second = _step(f, a, g, sum_sinusoids)
  for x, y in zip(first, second):
    assert torch.equal(x.view(torch.int32), y.view(torch.int32))
  if not sum_sinusoids:
    x = torch.rand(B, N, K, device=DEV, generator=gen)
    first, second = _cumsum_grad(x, g), _cumsum_grad(x, g)
    for x, y in zip(first, second):
      assert torch.equal(x.view(torch.int32), y.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize('sum_sinusoids', [True, False])
def test_cuda_graph_capture_equals_eager(sum_sinusoids):
  B, N, K, sr = 3, 2000, 70, 16000
  f, a = _inputs(B, N, K, sr, seed=17)
  g = _upstream(B, N, K, sum_sinusoids, seed=17)
  fl, al = f.clone().requires_grad_(True), a.clone().requires_grad_(True)
  xl = (f / sr).clone().requires_grad_(True)
  gx = torch.randn(B, N, K, device=DEV)

  def run():
    for t in (fl, al, xl):
      t.grad = None
    core.oscillator_bank(fl, al, sample_rate=sr, sum_sinusoids=sum_sinusoids).backward(g)
    core.angular_cumsum(xl).backward(gx)

  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    for _ in range(2):
      run()
  torch.cuda.current_stream().wait_stream(s)
  eager = [fl.grad.clone(), al.grad.clone(), xl.grad.clone()]
  graph = torch.cuda.CUDAGraph()
  for t in (fl, al, xl):
    t.grad = None
  with torch.cuda.graph(graph):
    core.oscillator_bank(fl, al, sample_rate=sr, sum_sinusoids=sum_sinusoids).backward(g)
    core.angular_cumsum(xl).backward(gx)
  graph.replay()
  torch.cuda.synchronize()
  for got, want in zip((fl.grad, al.grad, xl.grad), eager):
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize('B,N,K,sum_sinusoids', [(2, 1, 129, True), (2, 129, 129, False),
                                                 (3, 1000, 33, True), (1, 5, 1, False)])
def test_under_every_poison(B, N, K, sum_sinusoids):
  """Forward and backward under the guarded allocator of test_gpu_memory_bounds.py:
  fences intact and bit-identical results whatever the fresh memory holds."""
  from tests.test_gpu_memory_bounds import POISONS, guarded
  f, a = _inputs(B, N, K, 16000, seed=19)
  g = _upstream(B, N, K, sum_sinusoids, seed=19)
  gx = torch.randn(B, N, K, device=DEV)
  runs = []
  for p in POISONS:
    with guarded(p):
      fl, al = f.clone().requires_grad_(True), a.clone().requires_grad_(True)
      out = core.oscillator_bank(fl, al, sample_rate=16000, sum_sinusoids=sum_sinusoids)
      out.backward(g)
      xl = (f / 16000).clone().requires_grad_(True)
      ph = core.angular_cumsum(xl)
      ph.backward(gx)
      runs.append([out.detach().clone(), fl.grad.clone(), al.grad.clone(),
                   ph.detach().clone(), xl.grad.clone()])
  for run in runs[1:]:
    for got, want in zip(run, runs[0]):
      assert torch.equal(got.view(torch.int32), want.view(torch.int32))
  assert all(torch.isfinite(v).all() for v in runs[0])


@pytest.mark.gpu
@pytest.mark.parametrize('fill', [float('nan'), 7.0])
@pytest.mark.parametrize('off', [0, 1])
def test_fenced_operands_give_the_canonical_bits(fill, off):
  """Inputs and upstream gradients placed between fences of NaN or 7.0, at offsets of
  0 and 1 float, give the bits of fresh operands, and the fences stay intact."""
  from tests.test_gpu_memory_bounds import _fenced, _fences_intact
  B, N, K = 2, 300, 40
  f, a = _inputs(B, N, K, 16000, seed=23)
  g = _upstream(B, N, K, False, seed=23)
  want = _grads(f, a, g, 16000, False)
  ff, rf = _fenced(f, fill, off)
  af, ra = _fenced(a, fill, off)
  gf, rg = _fenced(g, fill, off)
  got = _grads(ff, af, gf, 16000, False, clone=False)
  for x, y in zip(got, want):
    assert torch.equal(x.view(torch.int32), y.view(torch.int32))
  for region, what in ((rf, 'f'), (ra, 'a'), (rg, 'g')):
    _fences_intact(region, what)


@pytest.mark.gpu
def test_strided_and_offset_inputs_and_side_stream():
  """Transposed, offset and expanded inputs and upstream gradients, and a side stream,
  give the canonical bits; the gradients reach the strided leaves in their shapes."""
  from tests.test_gpu_input_conventions import assert_same_bits
  B, N, K, sr = 2, 700, 24, 16000
  f, a = _inputs(B, N, K, sr, seed=29)
  g = _upstream(B, N, K, False, seed=29)
  want = _grads(f, a, g, sr, False)
  # transposed storage: leaves [B, K, N] seen as [B, N, K]
  ft = f.transpose(1, 2).contiguous().requires_grad_(True)
  at = a.transpose(1, 2).contiguous().requires_grad_(True)
  out = core.oscillator_bank(ft.transpose(1, 2), at.transpose(1, 2), sample_rate=sr,
                             sum_sinusoids=False)
  out.backward(g.transpose(1, 2).contiguous().transpose(1, 2))
  assert_same_bits(out, want[0], 'out (strided)')
  assert_same_bits(ft.grad.transpose(1, 2), want[1], 'd f (strided)')
  assert_same_bits(at.grad.transpose(1, 2), want[2], 'd a (strided)')
  # offset: a view one element into a larger buffer
  buf = torch.empty(f.numel() + 1, device=DEV)
  buf[1:] = f.reshape(-1)
  fo = buf[1:].view(B, N, K)
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    got = _grads(fo, a.clone(), g, sr, False, clone=False)
  torch.cuda.current_stream().wait_stream(s)
  torch.cuda.synchronize()
  for x, y, what in zip(got, want, ('out', 'd f', 'd a')):
    assert_same_bits(x, y, what + ' (offset, side stream)')
  # an expanded upstream gradient: out.sum() sends ones with stride 0
  gs = torch.ones(B, N, device=DEV)
  ref = _grads(f, a, gs, sr, True)
  fl, al = f.clone().requires_grad_(True), a.clone().requires_grad_(True)
  core.oscillator_bank(fl, al, sample_rate=sr).sum().backward()
  assert_same_bits(fl.grad, ref[1], 'd f (expanded g)')
  assert_same_bits(al.grad, ref[2], 'd a (expanded g)')


@pytest.mark.gpu
def test_operands_on_a_non_current_device():
  if torch.cuda.device_count() < 2:
    pytest.skip('needs two CUDA devices')
  B, N, K, sr = 2, 500, 10, 16000
  f, a = _inputs(B, N, K, sr, seed=31)
  g = _upstream(B, N, K, True, seed=31)
  want = _grads(f, a, g, sr, True)
  dev = torch.device('cuda', torch.cuda.device_count() - 1)
  got = _grads(f.to(dev), a.to(dev), g.to(dev), sr, True)
  assert torch.cuda.current_device() == 0
  for x, y in zip(got, want):
    assert x.device == dev
    assert torch.equal(x.cpu(), y.cpu())


@pytest.mark.gpu
@pytest.mark.parametrize('b,n,k', [(0, 5, 3), (2, 0, 3), (2, 5, 0), (0, 0, 0)])
def test_zero_sizes_launch_nothing(b, n, k):
  """The backward entry points on empty CUDA tensors: no error and no launch."""
  lib = _lib.load()
  z = torch.empty((b, n, k), device=DEV)
  gz = torch.empty((b, n), device=DEV)
  launches = lib.ddsp_b200_launch_count()
  for ss, g in ((1, gz), (0, z)):
    core._launch('ddsp_b200_oscillator_bank_backward', z, z, g, torch.empty_like(z),
                 torch.empty_like(z), b, n, k, 16000.0, ss)
  core._launch('ddsp_b200_angular_cumsum_backward', z, torch.empty_like(z), b, n, k)
  assert lib.ddsp_b200_launch_count() == launches
