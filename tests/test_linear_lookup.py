"""core.linear_lookup (core.py:1168-1214): forward and gradients against a float64
restatement on the float32 grid (tests/harmonic_bank_ref.py), routing, and the input
conventions of the other ops.  The restatement is pinned on CPU to the unmodified
reference run on the shim (tests/golden/linear_lookup.npz)."""
import math
import os

import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, core
from tests import harmonic_bank_ref as ref
from tests.golden import make_linear_lookup_golden as lg
from tests.test_gpu_input_conventions import assert_same_bits, at_offset
from tests.test_gpu_memory_bounds import POISONS, _fenced, _fences_intact, guarded
from tests.util import HostQueriesOnly

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'linear_lookup.npz')
TOL = 1e-4
LAYOUTS = ('item', 'item3', 'sample')


def test_restatement_matches_the_reference():
  g = np.load(GOLDEN)
  for i, (_, _, _, phase, tab) in enumerate(lg.lookup_inputs()):
    np.testing.assert_allclose(ref.linear_lookup(phase, tab).numpy(),
                               g['lookup_wide_%02d' % i], atol=1e-6, rtol=1e-6)


@pytest.fixture
def no_device(monkeypatch):
  monkeypatch.setattr(_lib, 'load', lambda real=_lib.load(): HostQueriesOnly(real))
  monkeypatch.setattr(torch.Tensor, 'to', lambda *a, **k: pytest.fail('tensor moved'))


@pytest.mark.parametrize('shapes', [
    ((2,), (2, 8)),                 # phase 1-D
    ((2, 5, 2), (2, 8)),            # two phase channels
    ((2, 0), (2, 8)),               # N = 0
    ((2, 5), (3, 8)),               # batch differs
    ((1, 5), (2, 8)),               # no batch broadcasting
    ((2, 5), (2, 3, 8)),            # tables neither per item nor per sample
    ((2, 5), (2, 0)),               # W = 0
    ((2, 5), (2, 5, 8, 1)),         # 4-D tables
])
def test_shapes_raise_before_device_work(shapes, no_device):
  with pytest.raises(ValueError):
    core.linear_lookup(torch.zeros(shapes[0]), torch.zeros(shapes[1]))


def _case(layout, b, n, w, kind, seed):
  rng = np.random.default_rng(seed)
  phase = lg.lookup_phase(kind, b, n, w, rng)
  shape = {'item': (b, w), 'item3': (b, 1, w), 'sample': (b, n, w)}[layout]
  return phase, rng.standard_normal(shape).astype(np.float32)


def _cuda(x):
  return torch.as_tensor(x, device='cuda')


@pytest.mark.gpu
@pytest.mark.parametrize('layout', LAYOUTS)
@pytest.mark.parametrize('w', [1, 2, 64, 2048])
@pytest.mark.parametrize('kind', ['inside', 'grid', 'edges', 'far', 'rank3'])
def test_forward_matches_float64(layout, w, kind):
  n = 300 if layout == 'sample' and w == 2048 else 5000
  phase, tab = _case(layout, 2, n, w, kind, seed=w)
  got = core.linear_lookup(_cuda(phase), _cuda(tab))
  want = ref.linear_lookup(phase, tab).numpy()
  assert got.shape == (2, n)
  assert np.abs(got.cpu().numpy() - want).max() <= TOL * max(1.0, np.abs(want).max())


def _grads(phase, tab):
  rng = np.random.default_rng(7)
  g = rng.standard_normal(phase.shape[:2])
  out = []
  for dtype, fn in ((torch.float32, core.linear_lookup), (torch.float64, ref.linear_lookup)):
    p = torch.tensor(phase, dtype=dtype, device='cuda', requires_grad=True)
    t = torch.tensor(tab, dtype=dtype, device='cuda', requires_grad=True)
    (fn(p, t) * torch.as_tensor(g, dtype=dtype, device='cuda')).sum().backward()
    out.append((p.grad.double().cpu().numpy(), t.grad.double().cpu().numpy()))
  return out


@pytest.mark.gpu
@pytest.mark.parametrize('layout', LAYOUTS)
@pytest.mark.parametrize('w', [1, 2, 64, 2048])
@pytest.mark.parametrize('kind', ['inside', 'grid', 'edges', 'far'])
def test_gradients_match_float64(layout, w, kind):
  n = 200 if layout == 'sample' and w == 2048 else 9000
  phase, tab = _case(layout, 2, n, w, kind, seed=w + 1)
  (dp, dt), (wp, wt) = _grads(phase, tab)
  assert np.abs(dp - wp).max() <= TOL * max(1.0, np.abs(wp).max())
  assert np.abs(dt - wt).max() <= TOL * max(1.0, np.abs(wt).max())
  if kind == 'grid':
    assert np.all(dp == 0.0)


@pytest.mark.gpu
@pytest.mark.parametrize('layout', LAYOUTS)
def test_backward_reruns_bitwise(layout):
  n = 20000 if layout != 'sample' else 2000
  phase, tab = _case(layout, 3, n, 512, 'inside', seed=5)
  phase = np.sort(phase, axis=1)        # many samples per column: the shared-target path
  runs = []
  for _ in range(2):
    p, t = _cuda(phase).requires_grad_(), _cuda(tab).requires_grad_()
    (core.linear_lookup(p, t) * torch.linspace(-1, 1, n, device='cuda')).sum().backward()
    runs.append((p.grad, t.grad))
  assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_half_inputs_give_the_canonical_bits_and_gradients_in_their_dtype(dtype):
  phase, tab = _case('item', 2, 3000, 64, 'inside', seed=9)
  ph, th = _cuda(phase).to(dtype), _cuda(tab).to(dtype)
  assert torch.equal(core.linear_lookup(ph, th), core.linear_lookup(ph.float(), th.float()))
  p, t = ph.clone().requires_grad_(), th.clone().requires_grad_()
  core.linear_lookup(p, t).sum().backward()
  assert p.grad.dtype == dtype and t.grad.dtype == dtype


@pytest.mark.gpu
def test_strided_and_offset_inputs_give_the_canonical_bits():
  phase, tab = _case('sample', 2, 500, 40, 'inside', seed=10)
  want = core.linear_lookup(_cuda(phase), _cuda(tab))
  big = torch.zeros(2, 500, 50, device='cuda')
  big[..., 7:47] = _cuda(tab)
  ps = torch.zeros(2, 1000, device='cuda')
  ps[:, 1::2] = _cuda(phase)
  assert torch.equal(core.linear_lookup(ps[:, 1::2], big[..., 7:47]), want)


# ---- poisoned and fenced memory (the patterns of test_gpu_memory_bounds.py) --------------
# (layout, B, N, W, what requires grad): every table shape, an N that leaves a partial
# 256-sample block and eight uneven time segments, per-item tables of two column tiles
# (the second partial), columns that are not a multiple of 32, and each gradient alone.
MEMORY_CASES = [('item', 2, 5001, 5000, 'both'), ('item', 3, 5001, 37, 'both'),
                ('item3', 2, 777, 64, 'both'), ('sample', 2, 501, 37, 'both'),
                ('item', 2, 901, 33, 'phase'), ('sample', 2, 301, 40, 'tables')]


def _memory_inputs(case):
  layout, b, n, w, _ = case
  phase, tab = _case(layout, b, n, w, 'edges', seed=n + w)
  g = np.random.default_rng(w).standard_normal((b, n)).astype(np.float32)
  return {'phase': _cuda(phase), 'tab': _cuda(tab)}, [_cuda(g)]


def _memory_run(case, t, gs):
  want = {'both': ('phase', 'tab'), 'phase': ('phase',), 'tables': ('tab',)}[case[4]]
  before = {k: v.clone() for k, v in t.items()}
  leaves = {k: v.detach().requires_grad_(k in want) for k, v in t.items()}
  out = core.linear_lookup(leaves['phase'], leaves['tab'])
  out.backward(gs[0])
  for k, v in t.items():
    assert torch.equal(v, before[k]), ('input changed', k)
  return [out.detach()], {k: leaves[k].grad for k in want}


@pytest.mark.gpu
@pytest.mark.parametrize('case', MEMORY_CASES, ids=[str(c) for c in MEMORY_CASES])
def test_poisoned_allocations_give_the_canonical_bits(case):
  """Every allocation of core and autograd is poisoned with 0x00, 0xFF (NaN) and 0x7F and
  fenced with canaries: output and gradients are bit-identical to a plain run, and no
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
  """Phase, tables and the upstream gradient between 64 KiB fences of NaN, and of 7.0, at
  storage offsets of 0 and 1 element: the bits of fresh operands at that offset, with the
  fences unchanged."""
  t, gs = _memory_inputs(case)
  for off in (0, 1):
    want_outs, want_grads = _memory_run(case, {k: at_offset(v, off) for k, v in t.items()},
                                        [at_offset(g, off) for g in gs])
    for fill in (math.nan, 7.0):
      regions, ins = [], {}
      for k, v in t.items():
        ins[k], r = _fenced(v, fill, off)
        regions.append(r)
      fg, r = _fenced(gs[0], fill, off)
      regions.append(r)
      outs, grads = _memory_run(case, ins, [fg])
      assert_same_bits(outs, want_outs, (case, fill, off))
      for k in want_grads:
        assert_same_bits(grads[k], want_grads[k], (case, fill, off, k))
      torch.cuda.synchronize()
      for r in regions:
        _fences_intact(r, (case, fill, off))


@pytest.mark.gpu
@pytest.mark.parametrize('layout', LAYOUTS)
def test_more_than_65535_items(layout):
  """No kernel puts the batch on a 65535-limited grid axis."""
  phase, tab = _case(layout, 70000, 3, 5, 'inside', seed=13)
  (dp, dt), (wp, wt) = _grads(phase, tab)
  got = core.linear_lookup(_cuda(phase), _cuda(tab)).cpu().numpy()
  want = ref.linear_lookup(phase, tab).numpy()
  assert np.abs(got - want).max() <= TOL * max(1.0, np.abs(want).max())
  assert np.abs(dp - wp).max() <= TOL * max(1.0, np.abs(wp).max())
  assert np.abs(dt - wt).max() <= TOL * max(1.0, np.abs(wt).max())


@pytest.mark.gpu
def test_cuda_graph_replay_equals_eager():
  phase, tab = [_cuda(x) for x in _case('item', 2, 4000, 256, 'inside', seed=12)]
  eager = core.linear_lookup(phase, tab)
  s = torch.cuda.Stream()
  with torch.cuda.stream(s):
    core.linear_lookup(phase, tab)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
      out = core.linear_lookup(phase, tab)
  graph.replay()
  torch.cuda.synchronize()
  assert torch.equal(out, eager)


@pytest.mark.gpu
def test_empty_batch():
  assert core.linear_lookup(torch.zeros(0, 5, device='cuda'),
                            torch.zeros(0, 8, device='cuda')).shape == (0, 5)
