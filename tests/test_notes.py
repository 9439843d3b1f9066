"""nn.get_note_mask, get_note_mask_from_onset, get_note_moments, pool_over_notes and the
torch helpers of ddsp_b200/nn.py (csrc/notes.cuh).  On the CPU: the float64 restatement
against the reference's fixture, the C entry points' checks, and the argument errors
raised before any device work.  On the GPU: the masks bit for bit against the
restatement, the moments and the pooled values against float64, d x against float64
autograd with its NaN positions, the MIDI-autoencoder pattern end to end,
reproducibility, CUDA graphs, streams, devices, poisoned and fenced memory, and peak
memory.  Reference: tests/notes_ref.py, pinned to the unmodified reference by
tests/golden/notes.npz.

Tolerances.  Every sum is float32 in a fixed order: a thread adds its chunk of 32 terms
serially and then adds the chunk to its total, so a sum of T terms carries at most
32 + T / 32 roundings, each at most 2^-24 of the sum of the terms' magnitudes.  The
forward is held to K = 8 (32 + T / 32 + 4) roundings of the float64 sum of magnitudes
of each output (for the std, of the squared deviations, halved through the square
root), and the gradients normwise to 1e-4 and elementwise to 1e-3 of the largest
element.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, autograd, core, nn
from tests import notes_ref as ref
from tests.golden import make_notes_golden as ng
from tests.test_launch import Recorder

P = 0x1000        # a device pointer the library never dereferences on the host
E_INVALID, E_WORKSPACE = _lib.E_INVALID, _lib.E_WORKSPACE
DEV = 'cuda'
U = 2.0**-24


# ---- CPU: the restatement and the fixture --------------------------------------------
def _rel_close(got, want, rtol=1e-9):
  got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
  assert got.shape == want.shape, (got.shape, want.shape)
  np.testing.assert_allclose(got, want, rtol=rtol, atol=rtol)


def _restated():
  """The restatement's value of every fixture entry, by name."""
  out = {}
  for i, (name, _, r) in enumerate(ng.MASK_CASES):
    for on in (True, False):
      out[f'{name}_on{int(on)}'] = ref.get_note_mask(ng.mask_input(i), r, on)
  for i, (name, _, _, r) in enumerate(ng.ONSET_CASES):
    for on in (True, False):
      out[f'{name}_on{int(on)}'] = ref.get_note_mask_from_onset(*ng.onset_inputs(i), r, on)
  for i, (name, _, _) in enumerate(ng.MOMENT_CASES):
    x, m = ng.moment_inputs(i)
    out[f'{name}_mean'], out[f'{name}_std'] = ref.get_note_moments(x, m)
    out[f'{name}_mean_only'] = ref.get_note_moments(x, m, False)
    if x.ndim == 3:
      out[f'{name}_pool_mean'], out[f'{name}_pool_std'] = ref.pool_over_notes(x, m)
    lengths = ref.get_note_lengths(m)
    out[f'{name}_lengths'] = lengths
    mean = out[f'{name}_mean']
    out[f'{name}_short'] = ref.get_short_note_loss_mask(
        m, lengths, mean if mean.dim() == 2 else mean[..., 0], min_length=4)
  return out


def test_restatement_matches_the_reference():
  """tests/notes_ref.py against the unmodified reference run wide on the shim: the masks
  exactly, everything else at 1e-9.  The cases hold the last-frame rule, T = 1, 2 and 3,
  more transitions than max_regions, note_on_only both ways, a 3-D q_pitch with three
  channels, onsets of 1.7, -1 and 2, NaN and infinite pitches, 2-D and 3-D x, soft
  masks, and empty and constant notes."""
  want = np.load(ng.PATH)
  got = _restated()
  assert set(got) == set(want.files)
  for k, v in got.items():
    if k.endswith(('_on0', '_on1')):
      assert np.array_equal(v.numpy(), want[k]), k
    else:
      _rel_close(v.numpy(), want[k])


def test_fixture_pins_the_edge_rules():
  """The fixture's statements in the issue's words: the last frame joins region 3 of
  [0,0,60,60,60,62,62,0,0,64], one frame gives two rows, onsets truncate."""
  want = np.load(ng.PATH)
  regions = want['last_frame_on0'][0].argmax(-1)
  assert regions.tolist() == [0, 0, 1, 1, 1, 2, 2, 3, 3, 3]
  assert want['last_frame_on1'][0, :, 3].tolist() == [0] * 7 + [1] * 3
  assert want['t1_on1'].shape == (3, 2, 3)
  assert want['t1_on1'][:, :, 0].tolist() == [[1, 1], [0, 0], [0, 0]]
  assert want['onset_trunc_on0'][0].argmax(-1).tolist() == [0, 1, 0, 2, 2, 2, 3, 3, 3, 3]
  assert not want['nonfinite_on1'][:2].any()   # a non-finite frame elsewhere: all off


def test_fixture_regenerates():
  """Where the reference is checked out, the fixture is what it computes."""
  from oracle import ref_on_shim
  try:
    ref_on_shim.load()
  except Exception as e:  # pylint: disable=broad-except
    pytest.skip('reference sources not available: %s' % e)
  from tests.golden.make_golden import compare
  compare('notes', ng.notes(), np.load(ng.PATH))


def test_straight_through_int_quantization():
  x = torch.tensor([-2.5, -1.5, -0.5, 0.5, 1.5, 2.5, 0.4, 2.6], requires_grad=True)
  y = nn.straight_through_int_quantization(x)
  assert y.tolist() == [-2.0, -2.0, -0.0, 0.0, 2.0, 2.0, 0.0, 3.0]
  y.sum().backward()
  assert x.grad.tolist() == [1.0] * 8


# ---- CPU: the C entry points ---------------------------------------------------------
def _mask(q=P, on=None, out=P, ws=P, nbytes=1 << 20, B=2, T=10, R=4, note_on=1):
  return (q, on, out, ws, nbytes, B, T, R, note_on, None)


def _mom(x=P, m=P, mean=P, std=P, pm=None, ps=None, B=2, T=10, N=4, D=3):
  return (x, m, mean, std, pm, ps, B, T, N, D, None)


def _bwd(x=P, m=P, mean=P, std=P, gm=P, gs=None, gpm=None, gps=None, dx=P, ws=P,
         nbytes=1 << 20, B=2, T=10, N=4, D=3):
  return (x, m, mean, std, gm, gs, gpm, gps, dx, ws, nbytes, B, T, N, D, None)


_M, _F, _B = 'note_mask', 'note_moments', 'note_moments_backward'
_ABI_CASES = [
    ('mask-B', _M, _mask(B=-1), E_INVALID, b'note_mask: bad shape B=-1 T=10 R=4'),
    ('mask-T0', _M, _mask(T=0), E_INVALID, b'note_mask: bad shape B=2 T=0 R=4'),
    ('mask-R', _M, _mask(R=-1), E_INVALID, b'note_mask: bad shape B=2 T=10 R=-1'),
    ('mask-flag', _M, _mask(note_on=2), E_INVALID,
     b'note_mask: note_on_only must be 0 or 1, got 2'),
    ('mask-null-q', _M, _mask(q=None), E_INVALID, b'note_mask: null pointer'),
    ('mask-null-out', _M, _mask(out=None), E_INVALID, b'note_mask: null pointer'),
    ('mask-ws', _M, _mask(nbytes=7), E_WORKSPACE,
     b'note_mask: workspace of 7 B is smaller than the 8 B needed'),
    ('mask-ws-null', _M, _mask(ws=None), E_WORKSPACE,
     b'note_mask: workspace of 1048576 B is smaller than the 8 B needed'),
    ('mask-B0', _M, _mask(q=None, out=None, ws=None, nbytes=0, B=0), 0, None),
    ('mask-R0', _M, _mask(q=None, out=None, ws=None, nbytes=0, R=0), 0, None),
    ('mom-shape', _F, _mom(N=-1), E_INVALID, b'note_moments: bad shape B=2 T=10 N=-1 D=3'),
    ('mom-T0', _F, _mom(T=0), E_INVALID, b'note_moments: bad shape B=2 T=0 N=4 D=3'),
    ('mom-null-x', _F, _mom(x=None), E_INVALID, b'note_moments: null pointer'),
    ('mom-null-mean', _F, _mom(mean=None), E_INVALID, b'note_moments: null pointer'),
    ('mom-pool-std', _F, _mom(std=None, pm=P, ps=P), E_INVALID,
     b'note_moments: pooled_std needs std and pooled_mean'),
    ('mom-grid', _F, _mom(B=1 << 20, N=1 << 20, D=1 << 10), E_INVALID,
     b'note_moments: 549755813888 tiles exceed the 2^31 - 1 grid limit'),
    ('mom-B0', _F, _mom(x=None, m=None, mean=None, std=None, B=0), 0, None),
    ('bwd-shape', _B, _bwd(D=-2), E_INVALID,
     b'note_moments_backward: bad shape B=2 T=10 N=4 D=-2'),
    ('bwd-null-dx', _B, _bwd(dx=None), E_INVALID, b'note_moments_backward: null pointer'),
    ('bwd-std', _B, _bwd(std=None, gs=P), E_INVALID,
     b'note_moments_backward: a std gradient needs std'),
    ('bwd-ws', _B, _bwd(nbytes=100), E_WORKSPACE,
     b'note_moments_backward: workspace of 100 B is smaller than the 448 B needed'),
    ('bwd-B0', _B, _bwd(*([None] * 10), nbytes=0, B=0), 0, None),
]


@pytest.mark.parametrize('fn,args,want,msg', [c[1:] for c in _ABI_CASES],
                         ids=[c[0] for c in _ABI_CASES])
def test_notes_abi_check_table(fn, args, want, msg):
  """Every check of the three entry points: the status and the full message come back
  before any CUDA call, and nothing is launched."""
  lib = _lib.load()
  launches = lib.ddsp_b200_launch_count()
  assert getattr(lib, 'ddsp_b200_' + fn)(*args) == want
  assert lib.ddsp_b200_launch_count() == launches
  if msg is not None:
    assert lib.ddsp_b200_last_error() == msg


def test_entry_points_take_stated_scratch_not_queries():
  """The two scratch buffers' sizes are stated in the header; there is no size query."""
  assert not any(n.startswith('ddsp_b200_note') and n.endswith('_workspace')
                 for n in _lib.SIGNATURES)
  for name in ('ddsp_b200_note_mask', 'ddsp_b200_note_moments_backward'):
    args = _lib.SIGNATURES[name][1]
    assert args[args.index(ctypes.c_size_t) - 1] is ctypes.c_void_p, name


@pytest.fixture
def recorder(monkeypatch):
  rec = Recorder()
  monkeypatch.setattr(_lib, 'load', lambda: rec)
  return rec


def test_errors_before_the_library_is_looked_up(recorder, monkeypatch):
  def fail(*a, **k):
    raise AssertionError('device work before the argument checks')
  monkeypatch.setattr(core, 'torch_float32', fail)
  q = np.zeros((2, 5), np.float32)
  x = np.zeros((2, 5, 3), np.float32)
  m = np.zeros((2, 5, 4), np.float32)
  cases = [
      (ValueError, r'expected \[batch, time\]', lambda: nn.get_note_mask(q[0])),
      (ValueError, 'at least one frame', lambda: nn.get_note_mask(q[:, :0])),
      (ValueError, 'max_regions must be a non-negative integer',
       lambda: nn.get_note_mask(q, max_regions=-1)),
      (ValueError, 'max_regions must be a non-negative integer',
       lambda: nn.get_note_mask(q, max_regions=2.5)),
      (ValueError, r'onset \(2, 4\) and q_pitch \(2, 5\)',
       lambda: nn.get_note_mask_from_onset(q, q[:, :4])),
      (ValueError, r'x must be \[batch, time\]', lambda: nn.get_note_moments(q[0], m)),
      (ValueError, r'note_mask must be \[batch, time, notes\]',
       lambda: nn.pool_over_notes(x, q)),
      (ValueError, r'x \(2, 5, 3\) and note_mask \(2, 1, 4\) must share',
       lambda: nn.get_note_moments(x, m[:, :1])),
      (ValueError, r'x \(1, 5, 3\) and note_mask \(2, 5, 4\) must share',
       lambda: nn.pool_over_notes(x[:1], m)),
      (ValueError, 'at least one frame', lambda: nn.get_note_moments(x[:, :0], m[:, :0])),
  ]
  for exc, msg, call in cases:
    with pytest.raises(exc, match=msg):
      call()
  assert recorder.looked_up == []


def test_mask_that_requires_grad_raises(recorder):
  x = torch.zeros((2, 5, 3))
  m = torch.zeros((2, 5, 4), requires_grad=True)
  for fn in (nn.get_note_moments, nn.pool_over_notes):
    with pytest.raises(RuntimeError, match='an input requires grad'):
      fn(x, m)
  assert recorder.looked_up == []


def test_torch_helpers_on_cpu():
  x, m = ng.moment_inputs(0)
  lengths = nn.get_note_lengths(torch.as_tensor(m))
  assert torch.equal(lengths.double(), ref.get_note_lengths(m))
  pitches = torch.as_tensor(x[:, :6, 0] - 3.0)
  got = nn.get_short_note_loss_mask(torch.as_tensor(m), lengths, pitches, min_length=4)
  assert torch.equal(got.double(), ref.get_short_note_loss_mask(m, lengths, pitches, 4))


# ---- GPU: masks -------------------------------------------------------------------------
def _pitches(b, t, seed, runs=6.0):
  """Integer pitches in runs of mean length `runs`, a third of them 0 or below."""
  rng = np.random.default_rng(seed)
  q = np.zeros((b, t), np.float32)
  for i in range(b):
    k = 0
    while k < t:
      n = 1 + int(rng.exponential(runs))
      q[i, k:k + n] = rng.integers(-20, 40)
      k += n
  return q


def _onsets(b, t, seed):
  rng = np.random.default_rng(seed)
  return rng.choice(np.array([0.0, 0.0, 0.0, 1.0, 1.7, 2.0, -1.0], np.float32), (b, t))


def _cuda_ref(fn, *args, **kw):
  """A restatement function on CUDA float64 tensors (the [B, T, R] products are large)."""
  args = [torch.as_tensor(a, device=DEV).double() for a in args]
  return fn(*args, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize('t', [1, 2, 3, 31, 32, 33, 1000, 4097])
@pytest.mark.parametrize('r', [1, 3, 100, 1000])
def test_masks_bit_exact(t, r):
  for b in (0, 1, 5, 64):
    if b * t * r > 64 * 1000 * 1000:
      b = 5   # B = 64 at T = 4097, R = 1000 is covered at R = 100
    q = _pitches(b, t, 10 * t + r + b)
    on = _onsets(b, t, 7 * t + r + b)
    for note_on in (True, False):
      got = nn.get_note_mask(torch.as_tensor(q, device=DEV), r, note_on)
      want = _cuda_ref(ref.get_note_mask, q, max_regions=r, note_on_only=note_on)
      assert got.dtype == torch.float32 and not got.requires_grad
      assert torch.equal(got.double(), want), (b, t, r, note_on)
      got = nn.get_note_mask_from_onset(torch.as_tensor(q, device=DEV),
                                        torch.as_tensor(on, device=DEV), r, note_on)
      want = _cuda_ref(ref.get_note_mask_from_onset, q, on, max_regions=r,
                       note_on_only=note_on)
      assert torch.equal(got.double(), want), (b, t, r, note_on, 'onset')


@pytest.mark.gpu
def test_mask_fixture_cases():
  """The kernel on every mask case of the fixture: NaN and infinite pitches, the last
  frame's sign, three channels, onset truncation."""
  want = np.load(ng.PATH)
  for i, (name, _, r) in enumerate(ng.MASK_CASES):
    for on in (True, False):
      got = nn.get_note_mask(torch.as_tensor(ng.mask_input(i), device=DEV), r, on)
      assert np.array_equal(got.cpu().numpy(), want[f'{name}_on{int(on)}']), (name, on)
  for i, (name, _, _, r) in enumerate(ng.ONSET_CASES):
    q, onset = ng.onset_inputs(i)
    for on in (True, False):
      got = nn.get_note_mask_from_onset(torch.as_tensor(q, device=DEV),
                                        torch.as_tensor(onset, device=DEV), r, on)
      assert np.array_equal(got.cpu().numpy(), want[f'{name}_on{int(on)}']), (name, on)


@pytest.mark.gpu
def test_mask_region_sum_sign():
  """A region of four frames of 1 and a last frame that (nearly) cancels them: on for a
  positive sum, off for an exact zero and for a negative one."""
  q = np.array([[0, 1, 1, 1, 1, -3.9999998], [0, 1, 1, 1, 1, -4.0], [0, 1, 1, 1, 1, -4.0000005]],
               np.float32)
  got = nn.get_note_mask(torch.as_tensor(q, device=DEV), 4)
  assert got[:, 1:, 1].sum(-1).tolist() == [5.0, 0.0, 0.0]
  assert torch.equal(got.double(), _cuda_ref(ref.get_note_mask, q, max_regions=4))


# ---- GPU: moments and pool ----------------------------------------------------------------
def _moment_inputs(b, t, n, d, kind, seed):
  rng = np.random.default_rng(seed)
  x = (rng.normal(size=(b, t, d)) + 3.0).astype(np.float32)
  if kind == 'soft':
    m = rng.uniform(0.0, 1.0, (b, t, n)).astype(np.float32)
  else:
    idx = np.sort(rng.integers(0, n, (b, t)), axis=1)
    m = (idx[..., None] == np.arange(n)).astype(np.float32)
  return x, m


def _sum_bound(t):
  return 8 * (32 + t / 32 + 4) * U


def _check_moments(got, x, m, pool):
  """got (mean, std) or pooled (mean, std) against float64, each element within the
  summation bound of its own terms' magnitudes."""
  x64, m64 = (torch.as_tensor(a, device=DEV).double() for a in (x, m))
  t = x.shape[1]
  k = _sum_bound(t)
  ls = m64.sum(1)
  ls = torch.where(ls == 0, torch.full_like(ls, 1e-7), ls)[..., None]
  mean, std = ref.get_note_moments(x64, m64)
  mag_mean = torch.einsum('btn,btd->bnd', m64.abs(), x64.abs()) / ls.abs()
  dev2 = (x64[:, :, None, :] - mean[:, None]) if m.shape[2] * t * x.shape[2] <= 2**26 else None
  if dev2 is not None:
    mag_var = torch.einsum('btnd,btn->bnd', (dev2.abs() + mag_mean[:, None] * k)**2,
                           m64**2) / ls.abs()
  else:
    mag_var = (mag_mean**2 + x64.abs().amax(1, keepdim=True)**2) * 4 * m64.sum(1)[..., None]
  tol_mean = k * mag_mean + 1e-30
  tol_std = (k * mag_var / (2 * std.clamp_min(1e-30)) + k * std).nan_to_num(posinf=math.inf)
  tol_std = torch.where(std == 0, (k * mag_var).sqrt(), tol_std)
  if pool:
    want = ref.pool_over_notes(x64, m64)
    tols = (torch.einsum('btn,bnd->btd', m64.abs(), mean.abs() + tol_mean) * k +
            torch.einsum('btn,bnd->btd', m64.abs(), tol_mean),
            torch.einsum('btn,bnd->btd', m64.abs(), std + tol_std) * k +
            torch.einsum('btn,bnd->btd', m64.abs(), tol_std))
  else:
    want, tols = (mean, std), (tol_mean, tol_std)
  for g, w, tol, what in zip(got, want, tols, ('mean', 'std')):
    err = (g.double() - w).abs()
    assert bool((err <= tol).all()), (what, float((err / tol).max()))


@pytest.mark.gpu
@pytest.mark.parametrize('d', [1, 3, 32, 128, 129])
@pytest.mark.parametrize('n', [1, 100, 257, 4096])
@pytest.mark.parametrize('kind', ['binary', 'soft'])
def test_moments_and_pool_against_float64(d, n, kind):
  t = 48 if n == 4096 else 200
  x, m = _moment_inputs(2, t, n, d, kind, n + d)
  xc, mc = torch.as_tensor(x, device=DEV), torch.as_tensor(m, device=DEV)
  _check_moments(nn.get_note_moments(xc, mc), x, m, pool=False)
  _check_moments(nn.pool_over_notes(xc, mc), x, m, pool=True)
  assert torch.equal(nn.get_note_moments(xc, mc, return_std=False),
                     nn.get_note_moments(xc, mc)[0])
  assert torch.equal(nn.pool_over_notes(xc, mc, return_std=False),
                     nn.pool_over_notes(xc, mc)[0])
  if d == 1:
    mean2, std2 = nn.get_note_moments(xc[:, :, 0], mc)
    mean3, std3 = nn.get_note_moments(xc, mc)
    assert mean2.shape == (2, n) and torch.equal(mean2, mean3[..., 0])
    assert torch.equal(std2, std3[..., 0])


@pytest.mark.gpu
def test_moment_fixture_cases():
  want = np.load(ng.PATH)
  for i, (name, _, _) in enumerate(ng.MOMENT_CASES):
    x, m = ng.moment_inputs(i)
    xc, mc = torch.as_tensor(x, device=DEV), torch.as_tensor(m, device=DEV)
    mean, std = nn.get_note_moments(xc, mc)
    np.testing.assert_allclose(mean.cpu().numpy(), want[f'{name}_mean'], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(std.cpu().numpy(), want[f'{name}_std'], rtol=1e-5, atol=1e-5)
    if x.ndim == 3:
      pm, ps = nn.pool_over_notes(xc, mc)
      np.testing.assert_allclose(pm.cpu().numpy(), want[f'{name}_pool_mean'], rtol=1e-5,
                                 atol=1e-5)
      np.testing.assert_allclose(ps.cpu().numpy(), want[f'{name}_pool_std'], rtol=1e-5,
                                 atol=1e-5)


# ---- GPU: gradients ------------------------------------------------------------------------
def _grads(fn, x, m, w_mean, w_std, return_std=True):
  """d x of sum(w_mean * mean) (+ sum(w_std * std)) through `fn`, on the kernels and in
  float64 autograd of the restatement."""
  xc = torch.as_tensor(x, device=DEV).requires_grad_(True)
  mc = torch.as_tensor(m, device=DEV)
  out = fn(nn, xc, mc, return_std)
  loss = (out[0] if return_std else out) * torch.as_tensor(w_mean, device=DEV)
  loss = loss.sum()
  if w_std is not None:
    loss = loss + (out[1] * torch.as_tensor(w_std, device=DEV)).sum()
  loss.backward()
  x64 = torch.as_tensor(x, device=DEV).double().requires_grad_(True)
  out = fn(ref, x64, torch.as_tensor(m, device=DEV).double(), True)
  loss = (out[0] * torch.as_tensor(w_mean, device=DEV).double()).sum()
  if w_std is not None:
    loss = loss + (out[1] * torch.as_tensor(w_std, device=DEV).double()).sum()
  loss.backward()
  return xc.grad.double(), x64.grad


_MOMENTS = lambda mod, x, m, s: mod.get_note_moments(x, m, s)
_POOL = lambda mod, x, m, s: mod.pool_over_notes(x, m, s)


def _check_grad(got, want):
  assert torch.equal(torch.isnan(got), torch.isnan(want))
  ok = ~torch.isnan(want)
  g, w = got[ok], want[ok]
  if w.numel():
    assert float((g - w).norm()) <= 1e-4 * float(w.norm()) + 1e-30, float((g - w).norm())
    assert bool(((g - w).abs() <= 1e-3 * w.abs().max() + 1e-3 * w.abs()).all())


def _weights(shape, seed):
  return np.random.default_rng(seed).normal(size=shape).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize('fn', [_MOMENTS, _POOL], ids=['moments', 'pool'])
@pytest.mark.parametrize('kind', ['binary', 'soft'])
@pytest.mark.parametrize('n,d', [(1, 1), (100, 128), (257, 129), (4096, 3)])
def test_grad_through_the_mean(fn, kind, n, d):
  """Binary masks with empty notes and soft masks: the mean's gradient is finite and
  matches, with the std returned and unused, and with return_std=False."""
  t = 64 if n == 4096 else 150
  x, m = _moment_inputs(2, t, n, d, kind, 5 * n + d)
  shape = (2, n, d) if fn is _MOMENTS else (2, t, d)
  w = _weights(shape, 1)
  for return_std in (True, False):
    got, want = _grads(fn, x, m, w, None, return_std)
    assert bool(torch.isfinite(got).all())
    _check_grad(got, want)


def _full_regions(b, t, n, seed):
  """A binary mask whose n notes each hold at least two frames."""
  rng = np.random.default_rng(seed)
  m = np.zeros((b, t, n), np.float32)
  for i in range(b):
    cuts = np.sort(rng.choice(np.arange(1, t // 2), n - 1, replace=False)) * 2
    idx = np.searchsorted(cuts, np.arange(t), side='right')
    m[i, np.arange(t), idx] = 1.0
  return m


@pytest.mark.gpu
@pytest.mark.parametrize('fn', [_MOMENTS, _POOL], ids=['moments', 'pool'])
@pytest.mark.parametrize('n,d,kind', [(1, 1, 'full'), (10, 128, 'full'), (100, 33, 'full'),
                                      (40, 129, 'soft'), (257, 5, 'soft')])
def test_grad_through_the_std(fn, n, d, kind):
  """Masks without empty or constant notes: the std's gradient is finite and matches."""
  t = 300
  rng = np.random.default_rng(n + d)
  x = (rng.normal(size=(2, t, d)) + 3.0).astype(np.float32)
  m = _full_regions(2, t, n, n) if kind == 'full' else rng.uniform(0.0, 1.0, (2, t, n)).astype(np.float32)
  shape = (2, n, d) if fn is _MOMENTS else (2, t, d)
  got, want = _grads(fn, x, m, _weights(shape, 2), _weights(shape, 3))
  assert bool(torch.isfinite(want).all())
  _check_grad(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize('fn', [_MOMENTS, _POOL], ids=['moments', 'pool'])
def test_grad_nan_where_autograd_has_nan(fn):
  """Empty notes (max_regions beyond the notes) and integer-valued constant notes: NaN in
  exactly the (b, d) columns where float64 autograd puts it, and the same values
  elsewhere; the std's weights are zero on some notes (0 * inf is NaN as well)."""
  t, d = 60, 4
  q = _pitches(3, t, 21, runs=8.0)
  q[0] = np.arange(t) // 10 + 1      # no empty note below region 6 in item 0
  m = _cuda_ref(ref.get_note_mask, q, max_regions=8, note_on_only=False).float().cpu().numpy()
  rng = np.random.default_rng(4)
  x = np.round(rng.normal(size=(3, t, d)) * 4).astype(np.float32)
  x[1, :, 1] = 5.0                   # constant over every note of item 1, dim 1
  shape = (3, 8, d) if fn is _MOMENTS else (3, t, d)
  w_std = _weights(shape, 6)
  w_std[..., 2] = 0.0
  got, want = _grads(fn, x, m, _weights(shape, 5), w_std)
  assert bool(torch.isnan(want).any())
  _check_grad(got, want)


@pytest.mark.gpu
def test_midi_autoencoder_pattern():
  """z_note_encode and add_slowness_loss: a quantized pitch that requires grad gives a
  mask that does not; pool_over_notes of the latents backpropagates a loss on the mean
  to the latents with finite gradients, equal to float64 autograd; the slowness-loss
  mask equals the restatement's."""
  b, t, d = 4, 250, 16
  rng = np.random.default_rng(9)
  raw = torch.as_tensor(_pitches(b, t, 31) + rng.normal(size=(b, t)).astype(np.float32) * 0.3,
                        device=DEV).requires_grad_(True)
  q = nn.straight_through_int_quantization(raw)
  z = torch.as_tensor(rng.normal(size=(b, t, d)).astype(np.float32),
                      device=DEV).requires_grad_(True)
  mask = nn.get_note_mask(q)
  assert not mask.requires_grad and mask.shape == (b, t, 100)
  z_pooled = nn.pool_over_notes(z, mask)[0]
  w = torch.as_tensor(_weights((b, t, d), 8), device=DEV)
  (z_pooled * w).sum().backward()
  assert bool(torch.isfinite(z.grad).all())
  z64 = z.detach().double().requires_grad_(True)
  want_mask = ref.get_note_mask(q.detach().double())
  assert torch.equal(mask.double(), want_mask)
  (ref.pool_over_notes(z64, want_mask)[0] * w.double()).sum().backward()
  _check_grad(z.grad.double(), z64.grad)
  # add_slowness_loss
  mask_all = nn.get_note_mask(q, note_on_only=False)
  lengths = nn.get_note_lengths(mask_all)
  pitches = nn.get_note_moments(q, mask_all, return_std=False)
  assert pitches.requires_grad
  short = nn.get_short_note_loss_mask(mask_all, lengths, pitches)
  q64 = q.detach().double()
  m64 = ref.get_note_mask(q64, note_on_only=False)
  want = ref.get_short_note_loss_mask(m64, ref.get_note_lengths(m64),
                                      ref.get_note_moments(q64, m64, return_std=False))
  assert torch.equal(short.double(), want)


# ---- GPU: reproducibility, graphs, streams, devices, memory ----------------------------
def _step(x, m):
  x.grad = None
  pm, ps = nn.pool_over_notes(x, m)
  mean, std = nn.get_note_moments(x, m)
  ((pm * 0.5).sum() + (ps * 0.25).sum() + mean.sum() + std.sum()).backward()
  return [o.detach().clone() for o in (pm, ps, mean, std)] + [x.grad.clone()]


def _train_inputs(b=8, t=300, n=100, d=64, seed=3):
  rng = np.random.default_rng(seed)
  x = torch.as_tensor(rng.normal(size=(b, t, d)).astype(np.float32), device=DEV)
  m = torch.as_tensor(rng.uniform(0.0, 1.0, (b, t, n)).astype(np.float32), device=DEV)
  return x.requires_grad_(True), m


@pytest.mark.gpu
def test_bit_reproducible():
  x, m = _train_inputs()
  q = torch.as_tensor(_pitches(16, 1000, 2), device=DEV)
  first = _step(x, m) + [nn.get_note_mask(q)]
  second = _step(x, m) + [nn.get_note_mask(q)]
  for a, b in zip(first, second):
    assert torch.equal(a, b)


@pytest.mark.gpu
def test_cuda_graph_capture_equals_eager():
  x, m = _train_inputs(seed=5)
  q = torch.as_tensor(_pitches(8, 300, 3), device=DEV)
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    for _ in range(2):
      eager = _step(x, m) + [nn.get_note_mask(q)]
  torch.cuda.current_stream().wait_stream(s)
  graph = torch.cuda.CUDAGraph()
  x.grad = None
  with torch.cuda.graph(graph):
    pm, ps = nn.pool_over_notes(x, m)
    mean, std = nn.get_note_moments(x, m)
    ((pm * 0.5).sum() + (ps * 0.25).sum() + mean.sum() + std.sum()).backward()
    mask = nn.get_note_mask(q)
  graph.replay()
  torch.cuda.synchronize()
  for a, b in zip([pm, ps, mean, std, x.grad, mask], eager):
    assert torch.equal(a, b)


@pytest.mark.gpu
def test_side_stream_equals_default_stream():
  x, m = _train_inputs(seed=6)
  want = _step(x, m)
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    got = _step(x, m)
  torch.cuda.current_stream().wait_stream(s)
  torch.cuda.synchronize()
  for a, b in zip(got, want):
    assert torch.equal(a, b)


@pytest.mark.gpu
def test_runs_on_the_current_stream(recorder):
  q = torch.zeros((3, 7), device=DEV)
  x = torch.zeros((3, 7, 2), device=DEV)
  m = torch.zeros((3, 7, 5), device=DEV)
  s = torch.cuda.Stream()
  with torch.cuda.stream(s):
    nn.get_note_mask(q, 5)
    nn.pool_over_notes(x, m)
  launches = [(name, args) for name, _, args in recorder.calls]
  assert [name for name, _ in launches] == ['ddsp_b200_note_mask', 'ddsp_b200_note_moments']
  for _, args in launches:
    assert args[-1] == s.cuda_stream
  assert launches[0][1][5:9] == (3, 7, 5, 1)
  assert launches[1][1][6:10] == (3, 7, 5, 2)


@pytest.mark.gpu
def test_runs_on_the_operands_device():
  if torch.cuda.device_count() < 2:
    pytest.skip('needs a second GPU')
  x, m = _train_inputs(b=2, t=50, n=10, d=8, seed=7)
  want = _step(x, m)
  with torch.cuda.device(0):
    x1 = x.detach().to('cuda:1').requires_grad_(True)
    got = _step(x1, m.to('cuda:1'))
    mask = nn.get_note_mask(torch.zeros((2, 9), device='cuda:1'))
  assert mask.device == torch.device('cuda:1')
  for a, b in zip(got, want):
    assert a.device == torch.device('cuda:1')
    assert torch.equal(a.cpu(), b.cpu())


@pytest.mark.gpu
def test_empty_batch():
  x = torch.zeros((0, 5, 3), device=DEV, requires_grad=True)
  m = torch.zeros((0, 5, 4), device=DEV)
  pm, ps = nn.pool_over_notes(x, m)
  mean, std = nn.get_note_moments(x, m)
  assert pm.shape == (0, 5, 3) and mean.shape == (0, 4, 3)
  (pm.sum() + ps.sum() + mean.sum() + std.sum()).backward()
  assert x.grad.shape == (0, 5, 3)
  assert nn.get_note_mask(torch.zeros((0, 5), device=DEV)).shape == (0, 5, 100)
  assert nn.get_note_mask(torch.zeros((0, 1), device=DEV)).shape == (0, 2, 100)
  assert nn.get_note_mask(torch.ones((2, 5), device=DEV), 0).shape == (2, 5, 0)
  # no notes: zero pooled values and a zero gradient
  x = torch.randn((2, 5, 3), device=DEV, requires_grad=True)
  pm, ps = nn.pool_over_notes(x, torch.zeros((2, 5, 0), device=DEV))
  assert not pm.any() and not ps.any()
  (pm.sum() + ps.sum()).backward()
  assert x.grad.shape == (2, 5, 3) and not x.grad.any()


@pytest.mark.gpu
@pytest.mark.parametrize('t,n,d', [(1, 1, 1), (33, 5, 65), (200, 100, 128)])
def test_poisoned_outputs_and_fenced_operands(t, n, d):
  """Every output, workspace and gradient buffer poisoned (0x00, 0xFF, 0x7F) between
  canary fences, and every input and upstream gradient between 64 KiB fences of NaN and
  of 7.0: the same bits every time, and every fence intact."""
  from tests.test_gpu_memory_bounds import POISONS, _fenced, _fences_intact, guarded
  rng = np.random.default_rng(t + n + d)
  x0 = torch.as_tensor(rng.normal(size=(3, t, d)).astype(np.float32), device=DEV)
  m0 = torch.as_tensor(rng.uniform(0.0, 1.0, (3, t, n)).astype(np.float32), device=DEV)
  q0 = torch.as_tensor(_pitches(3, t, 5), device=DEV)
  on0 = torch.as_tensor(_onsets(3, t, 5), device=DEV)
  g0 = [torch.as_tensor(rng.normal(size=s).astype(np.float32), device=DEV)
        for s in ((3, t, d), (3, t, d), (3, n, d), (3, n, d))]

  def run(x, m, q, on, g):
    x = x.detach().requires_grad_(True)
    outs = list(nn.pool_over_notes(x, m)) + list(nn.get_note_moments(x, m))
    torch.autograd.backward(outs, g)
    return [o.detach().clone() for o in outs] + [x.grad.clone(), nn.get_note_mask(q, n),
                                                 nn.get_note_mask_from_onset(q, on, n)]

  want = run(x0, m0, q0, on0, g0)
  for poison in POISONS:
    with guarded(poison):
      got = run(x0, m0, q0, on0, g0)
    for a, b in zip(got, want):
      assert torch.equal(a.view(torch.int32), b.view(torch.int32)), poison
  for fill in (math.nan, 7.0):
    for off in (0, 1):
      regions, ins = [], []
      for a in [x0, m0, q0, on0] + g0:
        fa, r = _fenced(a, fill, off)
        ins.append(fa)
        regions.append(r)
      got = run(*ins[:4], ins[4:])
      for a, b in zip(got, want):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (fill, off)
      torch.cuda.synchronize()
      for r in regions:
        _fences_intact(r, (fill, off))


@pytest.mark.gpu
def test_memory_holds_no_note_by_frame_products():
  """B = 32, T = 1000, R = 100, D = 128: get_note_mask, pool_over_notes and its backward
  allocate the mask, the two pooled outputs, autograd's two upstream gradients, the
  gradient, the per-note moments and the backward's scratch: nothing near the
  reference's [B, T, N, D] products (1.6 GB each)."""
  b, t, r, d = 32, 1000, 100, 128
  q = torch.as_tensor(_pitches(b, t, 12, runs=15.0), device=DEV)
  z = torch.randn((b, t, d), device=DEV, requires_grad=True)
  torch.cuda.synchronize()
  base = torch.cuda.memory_allocated()
  torch.cuda.reset_peak_memory_stats()
  mask = nn.get_note_mask(q, r)
  pm, ps = nn.pool_over_notes(z, mask)
  (pm.sum() + ps.sum()).backward()
  torch.cuda.synchronize()
  rise = torch.cuda.max_memory_allocated() - base
  mask_bytes, x_bytes, note_bytes = b * t * r * 4, b * t * d * 4, b * r * d * 4
  assert rise <= mask_bytes + 6 * x_bytes + 6 * note_bytes + 4 * 2**20, rise
