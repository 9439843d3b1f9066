"""nn.DilatedConvStack and its residual site on the fused kernel of csrc/norm.cuh
(nn.norm_residual), the conditional norms, and the MIDI autoencoders' encoders and
decoders.  On the CPU: 'same' padding with dilation, the layers' names, shapes and
initialisers, the refusals, and the C ABI's refusals in a process without a device.  On
the GPU: the kernel's forward and every gradient against float64 for every norm type and
parameter mode, its determinism and coverage, and the stack, decoders and encoders
against the float64 restatement (tests/midi_autoencoder_ref.py)."""
import json
import os
import subprocess
import sys

import pytest
import torch

from ddsp_b200 import _lib, core, decoders, encoders, nn
from tests import midi_autoencoder_ref as ref
from tests.util import rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu


@pytest.fixture(autouse=True)
def no_tf32():
  """FP32 convolutions and matmuls for this module's comparisons with float64; the
  defaults come back after each test."""
  saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
  torch.backends.cudnn.allow_tf32 = False
  torch.backends.cuda.matmul.allow_tf32 = False
  yield
  torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


# ---- CPU ---------------------------------------------------------------------------
@pytest.mark.parametrize('t,k,d', [(64, 3, 256), (1000, 3, 1), (1000, 3, 16), (5, 3, 4),
                                   (7, 2, 3), (1, 3, 2)])
def test_dilated_same_padding(t, k, d):
  """TensorFlow pads a 'same' dilated convolution by its dilated extent (k - 1) d + 1,
  also when that is longer than the input (d = 256 at T = 64)."""
  x = torch.randn(2, t, 1, 3, dtype=torch.float64)
  conv = nn.Conv2D(4, (k, 1), dilation_rate=(d, 1))
  conv(x.float())
  conv.double()
  y = conv(x)
  assert y.shape == (2, t, 1, 4)
  want = ref.conv_time(x[:, :, 0], conv.kernel, conv.bias, d)
  torch.testing.assert_close(y[:, :, 0], want)
  assert nn.same_padding(t, (k - 1) * d + 1, 1) == ((k - 1) * d // 2,
                                                    (k - 1) * d - (k - 1) * d // 2)


def test_conv2d_dilation_default_and_refusals():
  x = torch.randn(1, 9, 1, 2)
  a, b = nn.Conv2D(5, (3, 1)), nn.Conv2D(5, (3, 1), dilation_rate=1)
  torch.manual_seed(0)
  ya = a(x)
  torch.manual_seed(0)
  assert torch.equal(ya, b(x)) and a.dilation_rate == (1, 1)
  with pytest.raises(ValueError):
    nn.Conv2D(5, (3, 1), strides=(2, 1), dilation_rate=(2, 1))
  with pytest.raises(NotImplementedError):
    nn.Conv2D(5, 3, kernel_initializer='he_normal')
  ortho = nn.Conv2D(8, (3, 1), kernel_initializer='orthogonal')
  ortho(torch.zeros(1, 4, 1, 4))
  m = ortho.kernel.reshape(12, 8)
  torch.testing.assert_close(m.T @ m, torch.eye(8), atol=1e-5, rtol=0)


def test_stack_structure_names_and_dilations():
  s = nn.DilatedConvStack(ch=128, layers_per_stack=5, stacks=4, norm_type='layer')
  assert [l.dilation_rate[0] for l in s.layers] == [1, 2, 4, 8, 16] * 4
  assert all(l.kernel_size == (3, 1) and l.filters == 128 for l in s.layers)
  assert all(isinstance(n, nn.Normalize) and n.norm_type == 'layer' for n in s.norms)
  neg = nn.DilatedConvStack(ch=8, layers_per_stack=4, stacks=1, dilation=-3)
  assert [l.dilation_rate[0] for l in neg.layers] == [27, 9, 3, 1]
  c = nn.DilatedConvStack(ch=16, layers_per_stack=2, stacks=1, conditional=True,
                          shift_only=True, ortho_init=True)
  assert all(isinstance(n, nn.ConditionalNorm) and n.norm_type is None for n in c.norms)
  assert c.conv_in.kernel_initializer == 'orthogonal'
  # built by hand on the CPU: every lazy layer takes its input width
  c.conv_in(torch.zeros(1, 3, 1, 2))
  for layer, norm in zip(c.layers, c.norms):
    layer(torch.zeros(1, 3, 1, 16))
    norm.conditional_scale_and_shift.film(16, torch.zeros(1, 3, 5))
  names = [n for n, _ in c.named_parameters()]
  assert names == (['conv_in.kernel', 'conv_in.bias', 'layers.0.kernel', 'layers.0.bias',
                    'layers.1.kernel', 'layers.1.bias'] +
                   [f'norms.{i}.conditional_scale_and_shift.dense.{p}' for i in (0, 1)
                    for p in ('kernel', 'bias')])
  assert c.norms[0].conditional_scale_and_shift.dense.kernel.shape == (5, 16)


@pytest.mark.parametrize('kwargs', [dict(resample_type='upsample', resample_stride=2),
                                    dict(resample_type='downsample', resample_stride=2),
                                    dict(resample_stride=2), dict(spectral_norm=True)])
def test_stack_refusals(kwargs):
  with pytest.raises(NotImplementedError):
    nn.DilatedConvStack(ch=8, **kwargs)


def test_stack_unknown_norm_and_cpu():
  with pytest.raises(KeyError):
    nn.DilatedConvStack(ch=8, norm_type='batch')
  for ch in (6, 2052):
    with pytest.raises(NotImplementedError, match='ch='):
      nn.DilatedConvStack(ch=ch)
  with pytest.raises(ValueError, match='ch=48'):
    nn.DilatedConvStack(ch=48, norm_type='group')
  nn.DilatedConvStack(ch=2048, norm_type='instance')
  with pytest.raises(ValueError, match='CUDA'):
    nn.DilatedConvStack(ch=8, layers_per_stack=1, stacks=1)(torch.zeros(1, 4, 2))
  with pytest.raises(ValueError, match='CUDA'):
    nn.norm_residual(torch.zeros(1, 4, 8), torch.zeros(1, 4, 8), 'layer', torch.ones(8),
                     torch.zeros(8))


def test_conditional_norms_on_the_cpu():
  torch.manual_seed(1)
  x, z = torch.randn(2, 5, 1, 8), torch.randn(2, 5, 1, 3)
  cn = nn.ConditionalNorm('instance')
  out = cn([x, z])
  film = cn.conditional_scale_and_shift.dense(z)
  torch.testing.assert_close(out, nn.normalize_op(x, 'instance') * film[..., :8] +
                             film[..., 8:])
  so = nn.ConditionalScaleAndShift(shift_only=True)
  torch.testing.assert_close(so([x, z]), x + so.dense(z))
  assert so.dense.units == 8 and cn.conditional_scale_and_shift.dense.units == 16
  with pytest.raises(ValueError):
    so([torch.zeros(2, 5, 1, 4), z])


def test_embedding_and_fc_stack_out():
  torch.manual_seed(2)
  emb = nn.get_embedding(vocab_size=13, n_dims=6)
  assert emb(torch.tensor([3, 4])).shape == (2, 6)
  assert emb(torch.tensor([[3.0], [12.0]])).shape == (2, 1, 6)
  assert emb.embeddings.shape == (13, 6) and emb.embeddings.abs().max() <= 0.05
  torch.testing.assert_close(emb(torch.tensor([5]))[0], emb.embeddings[5])
  fc = nn.FcStackOut(ch=16, layers=3, n_out=7)
  assert fc(torch.zeros(2, 4, 5)).shape == (2, 4, 7) and len(fc.stack) == 3


def test_one_hot_encoder_skip_expand():
  keep = encoders.OneHotEncoder(vocab_size=13, n_dims=4)
  assert keep.input_keys == ['instrument', 'f0_scaled']
  assert keep({'instrument': torch.tensor([1]),
               'f0_scaled': torch.zeros(1, 10, 1)})['z'].shape == (1, 4)
  assert keep({'instrument': torch.tensor([[1]]),
               'f0_scaled': torch.zeros(1, 10, 1)})['z'].shape == (1, 1, 4)


@gpu
def test_one_hot_encoder_expands_over_time():
  enc = encoders.OneHotEncoder(one_hot_key='instrument_id', vocab_size=13, n_dims=4,
                               skip_expand=False)
  for ids in (torch.tensor([2, 7]), torch.tensor([[2], [7]])):
    z = enc({'instrument_id': ids.cuda(), 'f0_scaled': torch.zeros(2, 10, 1).cuda()})['z']
    assert z.shape == (2, 10, 4)
    torch.testing.assert_close(z[1], enc.embedding.embeddings[7].expand(10, 4))


def test_encoder_and_decoder_refusals():
  with pytest.raises(NotImplementedError, match='audio'):
    encoders.ExpressionEncoder(input_keys=('f0_scaled', 'audio'))
  with pytest.raises(ValueError, match='conditioning keys'):
    decoders.DilatedConvDecoder(conditioning_keys=None, precondition_stack=nn.FcStack())
  with pytest.raises(NotImplementedError):
    decoders.DilatedConvDecoder(resample_stride=2)
  d = decoders.DilatedConvDecoder(conditioning_keys=('z',))
  assert d.input_keys == ['ld_scaled', 'f0_scaled', 'z'] and d.conditional
  assert decoders.DilatedConvDecoder().input_keys == ['ld_scaled', 'f0_scaled', 'z']
  assert decoders.MidiToHarmonicDecoder(net=None).output_keys[-1] == 'f0_hz'


@pytest.mark.parametrize('c,g', [(c, g) for c in (0, 2, 4, 6, 8, 128, 2048, 2052)
                                 for g in (-1, 0, 1, 3, 4, 32, c)])
def test_takes_query(c, g):
  want = 4 <= c <= 2048 and c % 4 == 0 and (g == 0 or (g >= 1 and c % g == 0))
  assert _lib.load().ddsp_b200_norm_residual_takes(c, g) == int(want)


def _abi_refusals():
  lib = _lib.load()
  M = 1 << 20
  f = lib.ddsp_b200_norm_residual_forward
  bw = lib.ddsp_b200_norm_residual_backward
  calls = {
      'forward_channels': lambda: f(16, M, 32, 48, 0, 2 * M, 3 * M, 4 * M, 5 * M, 2, 3, 6, 1,
                                    1e-5, None),
      'forward_groups': lambda: f(16, M, 32, 48, 0, 2 * M, 3 * M, 4 * M, 5 * M, 2, 3, 8, 3,
                                  1e-5, None),
      'forward_ld': lambda: f(16, M, 32, 48, 6, 2 * M, 3 * M, 4 * M, 5 * M, 2, 3, 8, 1, 1e-5,
                              None),
      'forward_align': lambda: f(20, M, 32, 48, 0, 2 * M, 3 * M, 4 * M, 5 * M, 2, 3, 8, 1,
                                 1e-5, None),
      'forward_null': lambda: f(16, M, None, 48, 0, 2 * M, None, 4 * M, 5 * M, 2, 3, 8, 1,
                                1e-5, None),
      'forward_overlap': lambda: f(M, 16, 32, 48, 0, M, None, None, None, 2, 3, 8, 0, 1e-5,
                                   None),
      'forward_outputs': lambda: f(16, M, 32, 48, 0, 2 * M, 2 * M, 4 * M, 5 * M, 2, 3, 8, 1,
                                   1e-5, None),
      'backward_workspace': lambda: bw(16, 32, 0, M, 48, 64, 2 * M, None, 3 * M, 4 * M,
                                       5 * M, 6 * M, 7 * M, 4 * 2 * 8 * 2 * 8 - 4, 2, 3, 8, 1,
                                       None),
      'backward_overlap': lambda: bw(16, 32, 0, M, 48, 64, 2 * M, None, 2 * M, 4 * M, 5 * M,
                                     6 * M, 7 * M, 1 << 16, 2, 3, 8, 1, None),
      'backward_columns': lambda: bw(16, M, 16, M, 48, 64, 2 * M, None, 3 * M, 4 * M,
                                     5 * M, 5 * M + 16, None, 0, 2, 3, 8, 1, None),
      'backward_channels': lambda: bw(16, 32, 0, M, 48, 64, 2 * M, None, 3 * M, 4 * M,
                                      5 * M, 6 * M, 7 * M, 1 << 16, 2, 3, 4096, 1, None),
      'forward_empty': lambda: f(None, None, None, None, 0, None, None, None, None, 0, 3, 8,
                                 1, 1e-5, None),
      'backward_empty': lambda: bw(None, None, 0, None, None, None, None, None, None, None,
                                   None, None, None, 0, 2, 0, 8, 1, None),
  }
  rows = {}
  for name, call in calls.items():
    before = lib.ddsp_b200_launch_count()
    rc = call()
    rows[name] = [rc, lib.ddsp_b200_last_error().decode(), lib.ddsp_b200_launch_count() - before]
  return rows


def test_abi_refusals_without_a_device():
  proc = subprocess.run(
      [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [
          '-c', 'import json; from tests.test_dilated_conv import _abi_refusals; '
                'print(json.dumps(_abi_refusals()))'],
      cwd=ROOT, env=dict(os.environ, CUDA_VISIBLE_DEVICES=''), capture_output=True,
      text=True)
  assert proc.returncode == 0, proc.stderr
  rows = json.loads(proc.stdout.strip().splitlines()[-1])
  want = {
      'forward_channels': (_lib.E_UNSUPPORTED, 'C=6 channels in G=1 groups'),
      'forward_groups': (_lib.E_UNSUPPORTED, 'C=8 channels in G=3 groups'),
      'forward_ld': (_lib.E_INVALID, 'row stride ld=6'),
      'forward_align': (_lib.E_INVALID, 'must be 16-byte aligned'),
      'forward_null': (_lib.E_INVALID, 'norm_residual_forward: null pointer'),
      'forward_overlap': (_lib.E_INVALID, 'x_next must not overlap y'),
      'forward_outputs': (_lib.E_INVALID, 'x_next, r, mean and rstd must not overlap'),
      'backward_workspace': (_lib.E_INVALID, 'the workspace has'),
      'backward_overlap': (_lib.E_INVALID, 'dy must not overlap gx'),
      'backward_columns': (_lib.E_INVALID, 'disjoint column blocks'),
      'backward_channels': (_lib.E_UNSUPPORTED, 'C=4096'),
      'forward_empty': (0, ''),
      'backward_empty': (0, ''),
  }
  for name, (rc, msg) in want.items():
    assert rows[name][0] == rc, (name, rows[name])
    assert msg in rows[name][1], (name, rows[name])
    assert rows[name][2] == 0, (name, rows[name])


# ---- GPU: the kernel against float64 -----------------------------------------------
def _site_inputs(b, t, c, mode, offset=0.0, seed=0, ld_width=None):
  g = torch.Generator().manual_seed(seed)
  y = torch.randn(b, t, c, generator=g, dtype=torch.float64) * 3.0 + offset
  x = torch.randn(b, t, c, generator=g, dtype=torch.float64)
  if mode == 'channel':
    p = (1.0 + 0.3 * torch.randn(c, generator=g, dtype=torch.float64),
         0.3 * torch.randn(c, generator=g, dtype=torch.float64))
  else:
    width = c if mode == 'shift' else 2 * c
    p = (torch.randn(b, t, width, generator=g, dtype=torch.float64),)
  return y, x, p


def _run_site(y, x, p, norm_type, mode, relu, dev='cuda', ups=None):
  """(outputs, grads) of the fused site (float32) and of the float64 restatement, for
  the same upstream gradients `ups` (random by default)."""
  b, t, c = y.shape
  g = torch.Generator().manual_seed(99)
  if ups is None:
    ups = [torch.randn(b, t, c, generator=g, dtype=torch.float64) for _ in range(2)]
  leaves64 = [v.clone().requires_grad_(True) for v in (y, x) + p]
  leaves32 = [v.float().to(dev).requires_grad_(True) for v in (y, x) + p]
  if mode == 'channel':
    s, h = leaves64[2], leaves64[3]
    out32 = nn.norm_residual(leaves32[0], leaves32[1], norm_type, leaves32[2], leaves32[3],
                             relu=relu)
  else:
    s, h = ref.film_split(leaves64[2], c, mode == 'shift')
    out32 = nn.norm_residual(leaves32[0], leaves32[1], norm_type, film=leaves32[2],
                             shift_only=mode == 'shift', relu=relu)
  out64 = ref.site(leaves64[0], leaves64[1], norm_type, s, h)
  out64 = out64 if relu else out64[:1]
  out32 = out32 if relu else (out32,)
  loss64 = sum((o * u).sum() for o, u in zip(out64, ups))
  loss32 = sum((o * u.float().to(dev)).sum() for o, u in zip(out32, ups))
  g64 = torch.autograd.grad(loss64, leaves64)
  g32 = torch.autograd.grad(loss32, leaves32)
  return ([o.detach().cpu() for o in out32], [o.detach() for o in out64],
          [v.cpu() for v in g32], list(g64))


def _check(got, want, tol, what, tol_l2=None):
  for i, (a, w) in enumerate(zip(got, want)):
    emax, el2 = rel_err(a.double().numpy(), w.numpy())
    assert emax < tol and el2 < (tol_l2 or tol), (what, i, emax, el2)


SITES = ([(n, m, r, (2, 37, 128)) for n in (None, 'layer', 'group', 'instance')
          for m in ('channel', 'row', 'shift') for r in (True, False)] +
         [('layer', 'channel', True, (3, 1, 4)), ('layer', 'row', True, (2, 1, 12)),
          ('instance', 'row', True, (2, 2, 12)),
          ('layer', 'row', False, (1, 1000, 2048)), ('group', 'channel', True, (2, 300, 2048)),
          ('instance', 'shift', True, (2, 5, 4)), (None, 'row', True, (2, 9, 4)),
          ('layer', 'channel', True, (32, 1000, 128))])


@gpu
@pytest.mark.parametrize('norm_type,mode,relu,shape', SITES)
def test_site_against_float64(norm_type, mode, relu, shape):
  y, x, p = _site_inputs(*shape, mode, seed=SITES.index((norm_type, mode, relu, shape)))
  out32, out64, g32, g64 = _run_site(y, x, p, norm_type, mode, relu)
  _check(out32, out64, 2e-5, 'outputs')
  _check(g32, g64, 5e-4, 'gradients', 2e-4)


@gpu
@pytest.mark.parametrize('norm_type,mode', [('layer', 'channel'), ('instance', 'row'),
                                            ('group', 'shift')])
def test_site_large_mean(norm_type, mode):
  """Inputs of mean 1e3: the Welford statistics keep the normalized values exact to
  float32's resolution of the input."""
  y, x, p = _site_inputs(2, 500, 64, mode, offset=1e3, seed=5)
  out32, out64, g32, g64 = _run_site(y, x, p, norm_type, mode, True)
  _check(out32, out64, 2e-4, 'outputs')
  # y itself carries float32's 6e-8 relative rounding of 1e3, 2e-5 of its spread
  _check(g32, g64, 5e-2, 'gradients', 1e-3)


@gpu
def test_site_relu_ties_and_no_upstream_relu():
  """Where x_next is exactly 0 the ReLU passes no gradient; without a ReLU output the
  gradient of x is the upstream gradient itself."""
  b, t, c = 2, 16, 8
  y = torch.randn(b, t, c, device='cuda')
  x = torch.zeros(b, t, c, device='cuda', requires_grad=True)
  scale = torch.zeros(c, device='cuda', requires_grad=True)
  shift = torch.zeros(c, device='cuda', requires_grad=True)
  x_next, r = nn.norm_residual(y, x, 'layer', scale, shift)
  assert not x_next.any()
  (gx,) = torch.autograd.grad(r.sum(), [x])
  assert not gx.any()
  out = nn.norm_residual(y, x, None, scale, shift, relu=False)
  u = torch.randn_like(y)
  (gx,) = torch.autograd.grad((out * u).sum(), [x])
  assert torch.equal(gx, u)


@gpu
@pytest.mark.parametrize('norm_type,mode', [('layer', 'channel'), ('layer', 'row'),
                                            (None, 'channel'), ('instance', 'shift')])
def test_site_determinism_and_batch_independence(norm_type, mode):
  y, x, p = _site_inputs(5, 203, 128, mode, seed=3)
  ups = [torch.randn(5, 203, 128, dtype=torch.float64) for _ in range(2)]
  runs = []
  for _ in range(2):
    out32, _, g32, _ = _run_site(y, x, p, norm_type, mode, True, ups=ups)
    runs.append((out32, g32))
  assert all(torch.equal(a, b) for a, b in zip(runs[0][0] + runs[0][1], runs[1][0] + runs[1][1]))
  one = _run_site(y[1:2], x[1:2], tuple(v[1:2] if v.dim() == 3 else v for v in p),
                  norm_type, mode, True, ups=[u[1:2] for u in ups])
  assert torch.equal(one[0][0], runs[0][0][0][1:2])
  assert torch.equal(one[2][0], runs[0][1][0][1:2])
  assert torch.equal(one[2][1], runs[0][1][1][1:2])


@gpu
@pytest.mark.parametrize('groups,ld', [(1, 0), (0, 0), (1, 256), (32, 128)])
def test_site_writes_every_output(groups, ld):
  """Outputs poisoned with NaN are fully written (per row, the gradient columns in the
  Dense output's layout), with one launch forward and one (per row) or two (per
  channel) backward."""
  b, t, c = 3, 77, 128
  dev = 'cuda'
  y, x = torch.randn(b, t, c, device=dev), torch.randn(b, t, c, device=dev)
  nan = lambda *s: torch.full(s, float('nan'), device=dev)
  if ld:
    film = torch.randn(b, t, ld, device=dev)
    s = film.data_ptr() if ld == 2 * c else None
    h = film.data_ptr() + (4 * c if ld == 2 * c else 0)
  else:
    s, h = torch.randn(c, device=dev), torch.randn(c, device=dev)
  x_next, r = nan(b, t, c), nan(b, t, c)
  mean, rstd = (nan(b, groups), nan(b, groups)) if groups else (None, None)
  count = _lib.load().ddsp_b200_launch_count
  before = count()
  core._launch('ddsp_b200_norm_residual_forward', y, x, s, h, ld, x_next, r, mean, rstd, b,
               t, c, groups, 1e-5)
  assert count() - before == 1
  outs = [x_next, r] + ([mean, rstd] if groups else [])
  assert all(torch.isfinite(o).all() for o in outs)
  dy, dx, gx, gr = nan(b, t, c), nan(b, t, c), torch.randn_like(y), torch.randn_like(y)
  if ld:
    dfilm = nan(b, t, ld)
    ds = dfilm.data_ptr() if s is not None else None
    dh = dfilm.data_ptr() + (4 * c if s is not None else 0)
    core._launch('ddsp_b200_norm_residual_backward', y, s, ld, x_next, mean, rstd, gx, gr,
                 dy, dx, ds, dh, None, 0, b, t, c, groups)
    assert count() - before == 2   # one launch per row
    grads = [dy, dx, dfilm]
  else:
    ds, dh = nan(c), nan(c)
    ws = torch.empty(4 * 2 * 8 * b * c, dtype=torch.uint8, device=dev)
    core._launch('ddsp_b200_norm_residual_backward', y, s, 0, x_next, mean, rstd, gx, gr,
                 dy, dx, ds, dh, ws, ws.numel(), b, t, c, groups)
    assert count() - before == 3   # the site, then the fixed-order parameter sums
    grads = [dy, dx, ds, dh]
  assert all(torch.isfinite(o).all() for o in grads)


# ---- GPU: layers against float64 -------------------------------------------------
def _grads_against_float64(module, call32, call64, tol_out=1e-4, tol_grad=1e-3):
  out32 = call32()
  out64, leaves = call64()
  up = torch.randn(out64.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(7))
  (out32 * up.float().cuda()).sum().backward()
  (out64 * up).sum().backward()
  emax, el2 = rel_err(out32.detach().cpu().double().numpy(), out64.detach().numpy())
  assert emax < tol_out and el2 < tol_out, (emax, el2)
  names = [n for n, _ in module.named_parameters()]
  assert names and set(names) == set(leaves)
  scale = max(float(v.grad.abs().max()) for v in leaves.values())
  for name, p in module.named_parameters():
    want = leaves[name].grad
    if float(want.abs().max()) < 1e-9 * scale:
      # a gradient that is 0 exactly (a convolution bias before instance norm)
      assert float(p.grad.abs().max()) < 1e-5 * scale, name
      continue
    emax, el2 = rel_err(p.grad.cpu().double().numpy(), want.numpy())
    assert el2 < tol_grad, (name, emax, el2)


@gpu
@pytest.mark.parametrize('kwargs,zshape', [
    (dict(ch=128, layers_per_stack=5, stacks=2, norm_type='layer'), None),
    (dict(ch=32, layers_per_stack=3, stacks=2, norm_type=None, dilation=-2,
          ortho_init=True), None),
    (dict(ch=64, layers_per_stack=4, stacks=1, norm_type='instance', kernel_size=2), None),
    (dict(ch=128, layers_per_stack=5, stacks=1, norm_type='layer', conditional=True),
     (3, 200, 24)),
    (dict(ch=64, layers_per_stack=3, stacks=1, norm_type='group', conditional=True,
          shift_only=True), (3, 1, 16)),
    (dict(ch=32, layers_per_stack=2, stacks=1, norm_type='layer', conditional=True),
     (3, 16)),
])
def test_stack_against_float64(kwargs, zshape):
  torch.manual_seed(11)
  stack = nn.DilatedConvStack(**kwargs)
  x = torch.randn(3, 200, 2, dtype=torch.float64)
  z = None if zshape is None else torch.randn(*zshape, dtype=torch.float64)
  arg32 = (x.float().cuda() if z is None else [x.float().cuda(), z.float().cuda()])
  stack(arg32)   # builds
  _grads_against_float64(stack, lambda: stack(arg32), lambda: ref.stack(stack, x, z))


@gpu
def test_stack_short_input_and_large_dilation():
  torch.manual_seed(12)
  stack = nn.DilatedConvStack(ch=16, layers_per_stack=9, stacks=1, norm_type='layer')
  x = torch.randn(2, 64, 3, dtype=torch.float64)
  stack(x.float().cuda())
  assert stack.layers[-1].dilation_rate == (256, 1)
  _grads_against_float64(stack, lambda: stack(x.float().cuda()), lambda: ref.stack(stack, x))


def _normalize_layer(norm, x, leaves, prefix):
  c = x.shape[-1]
  return (ref.normalize(x, 'layer') * leaves[prefix + 'scale'].reshape(c) +
          leaves[prefix + 'shift'].reshape(c))


def _dense(x, leaves, prefix):
  return torch.matmul(x, leaves[prefix + 'kernel']) + leaves[prefix + 'bias']


@gpu
@pytest.mark.parametrize('conditional', [False, True])
def test_dilated_conv_decoder_against_float64(conditional):
  torch.manual_seed(13)
  dec = decoders.DilatedConvDecoder(
      ch=64, layers_per_stack=3, stacks=2, input_keys=('ld_scaled', 'f0_scaled'),
      conditioning_keys=('z',) if conditional else None,
      precondition_stack=nn.Dense(12) if conditional else None,
      output_splits=(('amplitudes', 1), ('harmonic_distribution', 7)))
  f = {k: torch.randn(2, 100, 1, dtype=torch.float64) for k in ('ld_scaled', 'f0_scaled')}
  f['z'] = torch.randn(2, 100, 5, dtype=torch.float64)
  f32 = {k: v.float().cuda() for k, v in f.items()}
  cat = lambda d: torch.cat([d[k] for k in dec.output_keys], -1)
  cat(dec(f32))

  def call64():
    x = torch.cat([f['ld_scaled'], f['f0_scaled']], -1)
    leaves = {}
    z = None
    if conditional:
      pre = {n: p.detach().double().cpu().requires_grad_(True)
             for n, p in dec.precondition_stack.named_parameters()}
      leaves.update({'precondition_stack.' + n: v for n, v in pre.items()})
      z = _dense(f['z'], pre, '')
    out, sl = ref.stack(dec.dilated_conv_stack, x, z)
    leaves.update({'dilated_conv_stack.' + n: v for n, v in sl.items()})
    for n, p in dec.dense_out.named_parameters():
      leaves['dense_out.' + n] = p.detach().double().cpu().requires_grad_(True)
    return _dense(out, leaves, 'dense_out.'), leaves

  _grads_against_float64(dec, lambda: cat(dec(f32)), call64)


@gpu
def test_midi_to_harmonic_decoder_against_float64():
  torch.manual_seed(14)
  net = nn.DilatedConvStack(ch=32, layers_per_stack=3, stacks=1, norm_type='layer',
                            conditional=True)
  dec = decoders.MidiToHarmonicDecoder(net=net, output_splits=(('f0_midi', 1),
                                                               ('amplitudes', 1),
                                                               ('harmonic_distribution', 5)))
  q = torch.round(40 + 20 * torch.rand(2, 80, 1, dtype=torch.float64))
  z = torch.randn(2, 80, 6, dtype=torch.float64)
  out = dec(q.float().cuda(), None, z.float().cuda())
  assert set(out) == {'f0_midi', 'amplitudes', 'harmonic_distribution', 'f0_hz'}
  torch.testing.assert_close(out['f0_hz'], core.midi_to_hz(out['f0_midi'],
                                                           midi_zero_silence=True))

  def call32():
    o = dec(q.float().cuda(), None, z.float().cuda())
    return torch.cat([o['f0_midi'], o['amplitudes'], o['harmonic_distribution']], -1)

  def call64():
    h, leaves = ref.stack(net, q, z)
    leaves = {'net.' + n: v for n, v in leaves.items()}
    for sub in ('norm', 'dense_out'):
      for n, p in getattr(dec, sub).named_parameters():
        leaves[f'{sub}.{n}'] = p.detach().double().cpu().requires_grad_(True)
    o = _dense(_normalize_layer(None, h, leaves, 'norm.'), leaves, 'dense_out.')
    return torch.cat([o[..., :1] + q, o[..., 1:]], -1), leaves

  _grads_against_float64(dec, call32, call64)


@gpu
@pytest.mark.parametrize('which', ['harmonic_to_midi', 'expression_pooled', 'expression'])
def test_encoders_against_float64(which):
  torch.manual_seed(15)
  net = nn.DilatedConvStack(ch=32, layers_per_stack=3, stacks=1, norm_type='layer')
  ins = [torch.randn(2, 90, w, dtype=torch.float64) for w in (1, 1, 6, 5)]
  if which == 'harmonic_to_midi':
    enc = encoders.HarmonicToMidiEncoder(net=net)
    call32 = lambda: torch.cat(list(enc(*[v.float().cuda() for v in ins]).values()), -1)
  else:
    enc = encoders.ExpressionEncoder(net=net, z_dims=8,
                                     input_keys=('f0_scaled', 'amps_scaled', 'hd_scaled',
                                                 'noise_scaled'),
                                     pool_time=which == 'expression_pooled')
    feats = dict(zip(('f0_scaled', 'amps_scaled', 'hd_scaled', 'noise_scaled'),
                     [v.float().cuda() for v in ins]))
    call32 = lambda: enc(feats)['z']
  call32()

  def call64():
    h, leaves = ref.stack(net, torch.cat(ins, -1))
    leaves = {'net.' + n: v for n, v in leaves.items()}
    for sub in ('norm', 'dense_out'):
      for n, p in getattr(enc, sub).named_parameters():
        leaves[f'{sub}.{n}'] = p.detach().double().cpu().requires_grad_(True)
    o = _dense(_normalize_layer(None, h, leaves, 'norm.'), leaves, 'dense_out.')
    if which == 'harmonic_to_midi':
      return torch.cat([o[..., :1] + ins[0], o[..., 1:]], -1), leaves
    if which == 'expression_pooled':
      o = o.mean(dim=1, keepdim=True).expand(-1, 90, -1)
    return o, leaves

  _grads_against_float64(enc, call32, call64)
