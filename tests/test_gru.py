"""The GRU recurrence (csrc/gru.cuh) and the Keras-semantics layers around it
(ddsp_b200.nn: Dense, LayerNormalization, Fc, FcStack, Gru, Rnn, split_to_dict).

CPU: the float64 restatement (tests/gru_ref.py) against torch.nn.GRU, the layers'
shapes, parameter names and initialisers, every refusal raised before device work, and
the C ABI's refusals in a process without a CUDA device.
GPU: forward and every gradient against float64 at every H where the kernel's tiling
changes (see gru.cuh), bitwise reproducibility, batch independence, launches per call
and the takes-query."""
import copy
import ctypes
import io
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, autograd, core, nn
from tests import gru_ref
from tests.util import rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu


# ---- CPU ---------------------------------------------------------------------------
def test_reference_matches_torch_gru_in_float64():
  n_in, units = 5, 8
  kernel, rk, bias = gru_ref.random_weights(n_in, units, seed=1)
  x = torch.randn((3, 7, n_in), dtype=torch.float64, generator=torch.Generator().manual_seed(2))
  want = torch.nn.GRU(n_in, units, batch_first=True).double()
  want.load_state_dict(gru_ref.torch_gru_weights(kernel, rk, bias))
  got = gru_ref.gru(x, kernel, rk, bias)
  np.testing.assert_allclose(got.numpy(), want(x)[0].detach().numpy(), rtol=0, atol=1e-12)


def test_split_to_dict():
  x = torch.arange(24.0).reshape(2, 3, 4)
  d = nn.split_to_dict(x, (('a', 1), ('b', 3)))
  assert list(d) == ['a', 'b']
  assert torch.equal(d['a'], x[..., :1]) and torch.equal(d['b'], x[..., 1:])
  with pytest.raises(ValueError, match='add up'):
    nn.split_to_dict(x, (('a', 1), ('b', 2)))


def test_fc_stack_shapes_names_and_initialisers():
  torch.manual_seed(0)
  stack = nn.FcStack(256, 3)
  x = torch.randn(2, 5, 40)
  y = stack(x)
  assert y.shape == (2, 5, 256)
  names = [n for n, _ in stack.named_parameters()]
  assert names == [f'{i}.{k}' for i in range(3) for k in
                   ('0.kernel', '0.bias', '1.gamma', '1.beta')]
  k0 = stack[0][0].kernel
  assert k0.shape == (40, 256)
  lim = (6.0 / (40 + 256))**0.5
  assert k0.abs().max() <= lim and abs(k0.std().item() - lim / 3**0.5) < 0.05 * lim
  assert torch.all(stack[0][0].bias == 0) and torch.all(stack[0][1].gamma == 1)
  assert torch.all(stack[0][1].beta == 0)
  # Dense -> LayerNormalization (epsilon 1e-3) -> leaky ReLU 0.2
  d = x @ k0
  m, v = d.mean(-1, keepdim=True), d.var(-1, unbiased=False, keepdim=True)
  want = torch.nn.functional.leaky_relu((d - m) / torch.sqrt(v + 1e-3), 0.2)
  torch.testing.assert_close(stack[0](x), want, rtol=1e-5, atol=1e-5)
  with pytest.raises(ValueError, match='width 40'):
    stack(torch.randn(2, 5, 41))


def test_gru_parameters_and_initialisers():
  torch.manual_seed(0)
  g = nn.Gru(64)
  g.build(20, 'cpu')
  assert [n for n, _ in g.named_parameters()] == ['kernel', 'recurrent_kernel', 'bias']
  assert g.kernel.shape == (20, 192) and g.recurrent_kernel.shape == (64, 192)
  assert g.bias.shape == (2, 192) and torch.all(g.bias == 0)
  assert g.kernel.abs().max() <= (6.0 / (20 + 192))**0.5
  u = g.recurrent_kernel.detach().double()
  torch.testing.assert_close(u @ u.t(), torch.eye(64, dtype=torch.float64), rtol=0, atol=1e-5)


@pytest.mark.parametrize('units', [0, 16, 33, 100, 544, 1024])
def test_unsupported_units_refused_at_construction(units):
  with pytest.raises(NotImplementedError, match='multiples of 32 from 32 to 512'):
    nn.Rnn(units, 'gru')


def test_rnn_refusals():
  with pytest.raises(NotImplementedError, match="rnn_type='gru'"):
    nn.Rnn(64, 'lstm')
  with pytest.raises(NotImplementedError, match="rnn_type='gru'"):
    nn.Rnn(64, 'gru', bidir=True)
  with pytest.raises(KeyError):
    nn.Rnn(64, 'vanilla')
  with pytest.raises(ValueError, match='CUDA'):
    nn.Rnn(64, 'gru')(torch.zeros(1, 2, 3))
  with pytest.raises(ValueError, match=r'\[batch, time, features\]'):
    nn.Rnn(64, 'gru')(torch.zeros(2, 3))


def _stub_handle(units, ptr):
  """A GruHandle object that stands for a created one without a device: its pointer is
  never passed to the library (the test clears it before the object is freed)."""
  h = object.__new__(autograd.GruHandle)
  h.units, h.device, h.ptr, h.loaded = units, torch.device('cuda', 0), ptr, None
  return h


def test_handles_are_never_copied():
  """A copied or pickled layer holds no handle of the original's (two objects would
  free one handle, and the survivor would launch into freed memory); the handle itself
  refuses to be copied."""
  rnn = nn.Rnn(64, 'gru')
  rnn.rnn.build(20, 'cpu')
  stub = _stub_handle(64, 0xdead)
  rnn.rnn._handles[stub.device] = stub
  try:
    buf = io.BytesIO()
    torch.save(rnn, buf)
    buf.seek(0)
    copies = [copy.deepcopy(rnn), copy.copy(rnn.rnn), torch.load(buf, weights_only=False)]
    for c in copies:
      g = c if isinstance(c, nn.Gru) else c.rnn
      assert g._handles == {}
      assert torch.equal(g.recurrent_kernel, rnn.rnn.recurrent_kernel)
    assert rnn.rnn._handles[stub.device] is stub and stub.ptr == 0xdead
    for fn in (copy.copy, copy.deepcopy, lambda h: torch.save(h, io.BytesIO())):
      with pytest.raises(TypeError, match='cannot be copied or pickled'):
        fn(stub)
  finally:
    stub.ptr = None


@pytest.mark.parametrize('units', range(0, 545, 16))
def test_takes_query(units):
  lib = _lib.load()
  assert lib.ddsp_b200_gru_takes(units) == int(32 <= units <= 512 and units % 32 == 0)


def _abi_refusals():
  """Status, message and launches of each refused call, run where no device is seen."""
  lib = _lib.load()
  h = ctypes.c_void_p()
  calls = {
      'create_null_out': lambda: lib.ddsp_b200_gru_create(None, 64),
      'create_units': lambda: lib.ddsp_b200_gru_create(ctypes.byref(h), 48),
      'create_no_device': lambda: lib.ddsp_b200_gru_create(ctypes.byref(h), 64),
      'load_null_handle': lambda: lib.ddsp_b200_gru_load(None, 16, 16, None),
      'forward_null_handle': lambda: lib.ddsp_b200_gru_forward(None, 16, 1 << 20, 2, 3, None),
      'backward_null_handle': lambda: lib.ddsp_b200_gru_backward(
          None, 16, 1 << 20, 2 << 20, 3 << 20, 4 << 20, 2, 3, None),
  }
  rows = {}
  for name, call in calls.items():
    before = lib.ddsp_b200_launch_count()
    rc = call()
    rows[name] = [rc, lib.ddsp_b200_last_error().decode(), lib.ddsp_b200_launch_count() - before]
  rows['destroy_null'] = [lib.ddsp_b200_gru_destroy(None), '', 0]
  rows['clusters_null'] = [lib.ddsp_b200_gru_clusters(None, 4, 0), '', 0]
  rows['handle'] = [h.value, '', 0]
  return rows


def test_abi_refusals_without_a_device():
  proc = subprocess.run(
      [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [
          '-c', 'import json; from tests.test_gru import _abi_refusals; '
                'print(json.dumps(_abi_refusals()))'],
      cwd=ROOT, env=dict(os.environ, CUDA_VISIBLE_DEVICES=''), capture_output=True,
      text=True)
  assert proc.returncode == 0, proc.stderr
  rows = json.loads(proc.stdout.strip().splitlines()[-1])
  want = {
      'create_null_out': (_lib.E_INVALID, 'gru_create: null out'),
      'create_units': (_lib.E_UNSUPPORTED, 'units=48; the GRU takes multiples of 32'),
      'create_no_device': (_lib.E_CUDA, 'gru_create: cudaGetDevice'),
      'load_null_handle': (_lib.E_INVALID, 'gru_load: null handle'),
      'forward_null_handle': (_lib.E_INVALID, 'gru_forward: null handle'),
      'backward_null_handle': (_lib.E_INVALID, 'gru_backward: null handle'),
  }
  for name, (rc, msg) in want.items():
    assert rows[name][0] == rc, (name, rows[name])
    assert msg in rows[name][1], (name, rows[name])
    assert rows[name][2] == 0, name
  assert rows['destroy_null'][0] == 0 and rows['clusters_null'][0] == 0
  assert rows['handle'][0] is None


# ---- GPU ---------------------------------------------------------------------------
N_IN = 24
# (H, B, T): every H where gru.cuh's tiling changes (Q = 16 / 8 / 4, registers from
# H = 384), B = 1, 2, 5, 33 and 64 (several items per cluster: 33 -> 3, 64 -> 4 in the
# forward, and more clusters than fit at once in the H = 512 backward), T = 1, 2, 201, 1000.
CASES = [(32, 1, 1), (32, 33, 201), (32, 64, 1000), (64, 2, 2), (64, 5, 1000),
         (128, 33, 1), (256, 1, 1000), (256, 5, 201), (288, 2, 201), (320, 1, 2),
         (352, 33, 2), (384, 5, 201), (416, 1, 1), (448, 2, 201), (480, 1, 2),
         (512, 1, 1000), (512, 2, 201), (512, 5, 2), (512, 33, 201), (512, 64, 201)]


def _setup(units, b, t, seed, dev='cuda'):
  kernel, rk, bias = gru_ref.random_weights(N_IN, units, seed)
  g = torch.Generator().manual_seed(seed + 1)
  x = torch.randn((b, t, N_IN), dtype=torch.float64, generator=g)
  up = torch.randn((b, t, units), dtype=torch.float64, generator=g)
  return [v.to(dev) for v in (x, kernel, rk, bias, up)]


def _run(handle, x, kernel, rk, bias, up):
  """The GRU in float32 through GruFn: (output, d x, d kernel, d recurrent_kernel, d bias)."""
  ins = [v.to(torch.float32).contiguous().requires_grad_(True) for v in (x, kernel, rk, bias)]
  out = autograd.GruFn.apply(*ins, handle, True)
  out.backward(up.to(torch.float32))
  return [out.detach()] + [v.grad for v in ins]


def _float64(x, kernel, rk, bias, up):
  ins = [v.clone().requires_grad_(True) for v in (x, kernel, rk, bias)]
  out = gru_ref.gru(*ins)
  out.backward(up)
  return [out.detach()] + [v.grad for v in ins]


@gpu
@pytest.mark.parametrize('units,b,t', CASES, ids=[f'H{h}-B{b}-T{t}' for h, b, t in CASES])
def test_forward_and_gradients_against_float64(units, b, t):
  args = _setup(units, b, t, seed=units + b + t)
  handle = autograd.GruHandle(units, 'cuda')
  got = _run(handle, *args)
  want = _float64(*args)
  names = ['out', 'd_x', 'd_kernel', 'd_recurrent_kernel', 'd_bias_input', 'd_bias_recurrent']
  got = got[:4] + [got[4][0], got[4][1]]
  want = want[:4] + [want[4][0], want[4][1]]
  for name, g, w in zip(names, got, want):
    emax, el2 = rel_err(g.cpu().numpy(), w.cpu().numpy())
    tol = (1e-4, 1e-4) if name == 'out' else (2e-3, 1e-3)
    assert emax < tol[0] and el2 < tol[1], (name, emax, el2)


def _kernel_outputs(handle, xw, rk, bias, up):
  """The two launches' own results, (states, d_pre, d_rec), through the C ABI from the
  input projection xw [B, T, 3H]: the torch GEMMs around them choose their kernels by
  shape, so only these are compared across batch sizes.  d_rec starts as NaN: the
  backward writes all of it, zeros in each item's last row."""
  b, t, _ = xw.shape
  h = handle.units
  gates = torch.zeros((b, t, 4 * h), device='cuda')
  gates[..., :3 * h] = xw
  states = torch.zeros((b, t + 1, h), device='cuda')
  handle.load(rk.float().contiguous(), bias[1].float().contiguous())
  core._launch('ddsp_b200_gru_forward', handle.ptr, gates, states, b, t)
  d_pre = torch.zeros((b, t, 3 * h), device='cuda')
  d_rec = torch.full((b, t + 1, 3 * h), float('nan'), device='cuda')
  core._launch('ddsp_b200_gru_backward', handle.ptr, gates, states, up.float().contiguous(),
               d_pre, d_rec, b, t)
  return states, d_pre, d_rec


@gpu
def test_bitwise_reproducible_and_batch_independent():
  units, b, t = 512, 33, 64
  args = _setup(units, b, t, seed=5)
  handle = autograd.GruHandle(units, 'cuda')
  first, second = _run(handle, *args), _run(handle, *args)
  for f, s in zip(first, second):
    assert torch.equal(f, s)
  x, kernel, rk, bias, up = args
  xw = (x @ kernel + bias[0]).float()
  whole = _kernel_outputs(handle, xw, rk, bias, up)
  assert torch.equal(whole[2][:, t], torch.zeros_like(whole[2][:, t]))
  assert not torch.isnan(whole[2]).any()
  for i in (0, 17, 32):   # each item alone: its own slice of one
    alone = _kernel_outputs(handle, xw[i:i + 1], rk, bias, up[i:i + 1])
    for a, w in zip(alone, whole):
      assert torch.equal(a[0], w[i])


def _counter():
  lib = _lib.load()
  return lib.ddsp_b200_launch_count


@gpu
@pytest.mark.parametrize('units', [64, 512])
def test_launches_per_call(units):
  """One pack and one recurrence launch per forward, one launch per backward; none
  under no_grad beyond the forward's two.  The backward runs on autograd's device
  thread, where the thread-local counter is read by hooks."""
  count = _counter()
  x, kernel, rk, bias, up = _setup(units, 3, 10, seed=1)
  layer = nn.Gru(units).cuda()
  xf = x.float().requires_grad_(True)
  layer(xf)   # builds
  with torch.no_grad():
    layer.kernel.copy_(kernel)
    layer.recurrent_kernel.copy_(rk)
    layer.bias.copy_(bias)
  before = count()
  out = layer(xf)
  assert count() - before == 2
  seen = {}
  out.register_hook(lambda g: seen.__setitem__('before', count()))
  xf.register_hook(lambda g: seen.__setitem__('after', count()))
  out.backward(up.float())
  assert seen['after'] - seen['before'] == 1
  before = count()
  with torch.no_grad():
    out2 = layer(xf)
  assert count() - before == 2 and out2.grad_fn is None
  assert torch.equal(out2, out.detach())


@gpu
@pytest.mark.parametrize('units', [32, 64, 96, 256, 288, 352, 384, 480, 512])
def test_takes_query_agrees_with_the_entry_points(units):
  lib = _lib.load()
  assert lib.ddsp_b200_gru_takes(units) == 1
  handle = autograd.GruHandle(units, 'cuda')
  for backward in (0, 1):
    assert lib.ddsp_b200_gru_clusters(handle.ptr, 1, backward) >= 1
  x, kernel, rk, bias, up = _setup(units, 2, 3, seed=3)
  out = _run(handle, x, kernel, rk, bias, up)[0]
  assert torch.isfinite(out).all()
  h = ctypes.c_void_p()
  for bad in (units + 16, units - 1):
    assert lib.ddsp_b200_gru_create(ctypes.byref(h), bad) == _lib.E_UNSUPPORTED


@gpu
def test_gpu_abi_refusals():
  lib = _lib.load()
  h = ctypes.c_void_p()
  assert lib.ddsp_b200_gru_create(ctypes.byref(h), 64) == 0
  try:
    gates = torch.zeros(2 * 3 * 256 + 2 * 4 * 64, device='cuda')
    stream = torch.cuda.current_stream().cuda_stream
    before = lib.ddsp_b200_launch_count()
    rc = lib.ddsp_b200_gru_forward(h, gates.data_ptr(), gates.data_ptr() + 4 * 1536, 2, 3,
                                   stream)
    assert rc == _lib.E_INVALID and b'call ddsp_b200_gru_load first' in lib.ddsp_b200_last_error()
    u = torch.zeros(64 * 192 + 192, device='cuda')
    assert lib.ddsp_b200_gru_load(h, u.data_ptr(), u.data_ptr() + 4 * 64 * 192, stream) == 0
    rc = lib.ddsp_b200_gru_forward(h, gates.data_ptr(), gates.data_ptr() + 4 * 1000, 2, 3,
                                   stream)
    assert rc == _lib.E_INVALID
    assert b'gates must not overlap states' in lib.ddsp_b200_last_error()
    assert lib.ddsp_b200_gru_forward(h, None, None, 0, 3, stream) == 0
    for b, t in ((-1, 3), (2, -1)):
      assert lib.ddsp_b200_gru_forward(h, gates.data_ptr(), gates.data_ptr() + 4 * 1536, b, t,
                                       stream) == _lib.E_INVALID
      assert b'gru_forward: bad shape' in lib.ddsp_b200_last_error()
      assert lib.ddsp_b200_gru_backward(h, *[gates.data_ptr() + 4 * 512 * i for i in range(5)],
                                        b, t, stream) == _lib.E_INVALID
      assert b'gru_backward: bad shape' in lib.ddsp_b200_last_error()
    assert lib.ddsp_b200_launch_count() - before == 1   # the load
  finally:
    lib.ddsp_b200_gru_destroy(h)


@gpu
def test_a_copied_layer_has_its_own_handle():
  layer = nn.Gru(64).cuda()
  x = torch.randn(2, 50, 12, device='cuda')
  want = layer(x)
  twin = copy.deepcopy(layer)
  assert twin._handles == {}
  got = twin(x)
  assert twin._handles[x.device].ptr != layer._handles[x.device].ptr
  del layer
  assert torch.equal(twin(x), got) and torch.equal(got, want)
