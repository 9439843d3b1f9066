"""Every CUDA op on poisoned and fenced memory.

A kernel can leave part of its output unwritten, read memory it never wrote, or
read or write just outside its buffers, and still pass a test by luck: a fresh
allocation often reads as zero, and neighbouring tensors share one `cudaMalloc`
segment, so an access past the end lands in someone else's memory without a fault.
This file takes that luck away.

  * A guarded allocator stands in for `torch.empty` / `torch.empty_like` inside the
    library modules that allocate (GUARDED_MODULES).  Every CUDA allocation of n
    bytes becomes the middle of `fence + n + fence` bytes: the fences hold the
    canary byte 0xA5 and the payload a poison byte, 0x00 (what a fresh segment
    often holds), 0xFF (NaN in float32) or 0x7F (3.39e38, finite, for paths that
    would hide a NaN).  The payload is 512-byte aligned, as the real allocator's
    blocks are, so every kernel takes its usual route.  On exit every fence must
    still hold the canary.  CPU allocations (the host decoder's pinned output) and
    non-contiguous `empty_like`s are poisoned without fences.
  * Every row of the input-conventions table, and a table of edge shapes that leave a
    partial tile or vector on every tiled axis, runs under all three poisons: outputs
    and gradients must be bit-identical across poisons, finite wherever the float64
    reference is, and match that reference.
  * Every input and upstream gradient is placed between 64 KiB fences of NaN, and
    separately of 7.0: the results must be the bits of fresh contiguous operands.
  * Every entry point that takes a workspace is handed exactly the bytes it asked for,
    at 0, 16, 128 and 240 bytes past a 256-byte boundary, between canary fences: its
    alignment slack is used up to the last byte and the outputs must not change.
"""
import ast
import contextlib
import ctypes
import glob
import math
import os
import sys
import tempfile
import types

import numpy as np
import pytest
import torch

from ddsp_b200 import (_lib, autograd, core, host, losses, sharding, spectral_ops)
from oracle import ddsp_oracle as oracle
from tests import (consistency_ref, grad_ref, loudness_ref, mel_ref, mod_delay_ref,
                   routing_ref, sinc_ref, sinusoidal_ref, wavetable_ref)
from tests.test_gpu_input_conventions import (ROWS, SR, Row, _flat, _np,
                                              _phasor, _t, assert_same_bits, at_offset,
                                              assert_unchanged, run_grad, snapshot, u,
                                              upstream, with_leaves)

# The library modules that allocate uninitialised memory (test_allocations_go_through_
# the_guard checks that no other module does).
GUARDED_MODULES = (core, autograd, spectral_ops, host, sharding)
FENCE = 64 * 1024
CANARY = 0xA5
POISONS = (0x00, 0xFF, 0x7F)
POISON_IDS = ['0x00', '0xFF', '0x7F']


# ---- the guarded allocator --------------------------------------------------------
def _fill_bytes(t, byte):
  """Every byte of t's storage set to `byte`, whatever its dtype."""
  if t.untyped_storage().nbytes():
    raw = torch.empty(0, dtype=torch.uint8, device=t.device)
    raw.set_(t.untyped_storage())
    raw.fill_(byte)


class Guard:
  """The allocations made while one `guarded` block is active, and their fences."""

  def __init__(self, poison, fence_devices=('cuda',), allocates=True):
    assert FENCE % 512 == 0
    self.poison, self.allocates = poison, allocates
    self.fence_devices = fence_devices
    self.fenced = []      # (buffer, payload bytes, shape, dtype, call site)
    self.unfenced = []    # (shape, dtype, device, call site)

  @staticmethod
  def _site():
    """file:line of the allocating call (the innermost frame outside this file)."""
    f = sys._getframe(1)
    while f is not None and f.f_code.co_filename == __file__:
      f = f.f_back
    return '?' if f is None else '%s:%d' % (os.path.basename(f.f_code.co_filename),
                                           f.f_lineno)

  def wrap(self, t):
    """t, or a fenced stand-in for it with the same shape, dtype and device."""
    if (t.device.type not in self.fence_devices or t.layout != torch.strided or
        not t.is_contiguous()):
      _fill_bytes(t, self.poison)
      self.unfenced.append((tuple(t.shape), t.dtype, t.device, self._site()))
      return t
    n = t.numel() * t.element_size()
    buf = torch.empty((2 * FENCE + n,), dtype=torch.uint8, device=t.device)
    buf[:FENCE].fill_(CANARY)
    buf[FENCE + n:].fill_(CANARY)
    buf[FENCE:FENCE + n].fill_(self.poison)
    v = buf[FENCE:FENCE + n].view(t.dtype).view(t.shape)
    if t.requires_grad:
      v.requires_grad_(True)
    self.fenced.append((buf, n, tuple(t.shape), t.dtype, self._site()))
    return v

  def check(self):
    """Every fence still holds the canary, and something went through the guard."""
    assert self.fenced or self.unfenced or not self.allocates, (
        'no allocation went through the guard')
    if torch.cuda.is_available():
      torch.cuda.synchronize()
    for buf, n, shape, dtype, site in self.fenced:
      intact = bool(torch.all(buf[:FENCE] == CANARY)) and bool(
          torch.all(buf[FENCE + n:] == CANARY))
      assert intact, ('fence overwritten', shape, dtype, site)


class _TorchProxy:
  """`torch` as the guarded modules see it: everything passes through but `empty`
  and `empty_like`, whose results go through the guard."""

  def __init__(self, guard):
    self._guard = guard

  def __getattr__(self, name):
    return getattr(torch, name)

  def empty(self, *args, **kwargs):
    return self._guard.wrap(torch.empty(*args, **kwargs))

  def empty_like(self, *args, **kwargs):
    return self._guard.wrap(torch.empty_like(*args, **kwargs))


@contextlib.contextmanager
def guarded(poison, modules=GUARDED_MODULES, fence_devices=('cuda',), allocates=True):
  """Inside the block, `modules` allocate through a Guard (yielded); on a normal exit
  the fences are checked (and, unless `allocates` is False, that something was
  allocated)."""
  guard = Guard(poison, fence_devices, allocates)
  proxy = _TorchProxy(guard)
  saved = [(m, m.torch) for m in modules]
  for m in modules:
    m.torch = proxy
  try:
    yield guard
  finally:
    for m, t in saved:
      m.torch = t
  guard.check()


# ---- comparisons -------------------------------------------------------------------
def _bits(t):
  t = t.detach()
  if t.is_complex():
    t = torch.view_as_real(t)
  return t.contiguous().reshape(-1).view(torch.uint8)


def assert_close(what, got, want, tol, cmp=None):
  """got within max-relative `tol` of the float64 `want` (after `cmp`), finite
  wherever want is."""
  got, want = _flat(got), _flat(want)
  assert len(got) == len(want), (what, len(got), len(want))
  cmps = cmp if isinstance(cmp, tuple) else (cmp,) * len(want)
  for i, (g, w, c) in enumerate(zip(got, want, cmps)):
    g, w = _np(g), _np(w)
    if c is not None:
      g, w = c(g), c(w)
    g = np.asarray(g, np.complex128)
    w = np.asarray(w, np.complex128)
    assert g.shape == w.shape, (what, i, g.shape, w.shape)
    fin = np.isfinite(w)
    assert np.all(np.isfinite(g[fin])), (what, i, 'not finite where the reference is')
    if not fin.any():
      continue
    peak = max(np.abs(w[fin]).max(), 1e-30)
    err = np.abs(g[fin] - w[fin]).max() / peak
    assert err <= tol, (what, i, err)


def assert_poison_independent(runs, what):
  """runs: one (outputs, grads) per poison; every one must have the first one's bits."""
  outs0, grads0 = runs[0]
  for p, (outs, grads) in zip(POISON_IDS[1:], runs[1:]):
    assert_same_bits(outs, outs0, (what, 'output', p))
    for k in grads0:
      assert_same_bits(grads[k], grads0[k], (what, 'grad', k, p))


def _run(row, t, gs=None):
  """The row's outputs (and gradients for the grad rows) on inputs t; the inputs
  must come back unchanged."""
  ins = with_leaves(row, t) if row.grads else dict(t)
  before = snapshot(ins)
  if row.grads:
    outs, grads = run_grad(row, ins, gs)
    outs = [o.detach() for o in _flat(outs)]
  else:
    with torch.no_grad():
      outs, grads = _flat(row(ins)), {}
  assert_unchanged(before, ins, row.name)
  return outs, grads


# rows whose call is torch on the caller's tensors, or a view of them
NO_ALLOCATION = ('compute_logmag', 'Crop')


def _poisoned_runs(row, t):
  runs = []
  for p in POISONS:
    with guarded(p, allocates=row.name not in NO_ALLOCATION):
      runs.append(_run(row, t))
  assert_poison_independent(runs, row.name)
  return runs


# ---- CPU: the guard itself ---------------------------------------------------------
_standin = types.ModuleType('standin')
_standin.torch = torch


def _standin_op(x, bug=None):
  """2 x, into an output `empty_like` allocates, done right or with one bug."""
  out = _standin.torch.empty_like(x)
  if bug == 'unwritten':
    out[:-1] = 2.0 * x[:-1]
  elif bug == 'overrun':
    out.copy_(2.0 * x)
    torch.as_strided(out, (out.numel() + 1,), (1,))[-1] = 1.0
  elif bug == 'reads_poison':
    out.copy_(torch.maximum(out, 2.0 * x))   # assumes a fresh buffer holds -inf or 0
  else:
    out.copy_(2.0 * x)
  return out


def _standin_runs(bug):
  x = torch.linspace(-1.0, 1.0, 37)
  runs = []
  for p in POISONS:
    with guarded(p, modules=(_standin,), fence_devices=('cpu',)):
      runs.append(([_standin_op(x, bug).clone()], {}))
  assert_poison_independent(runs, bug)
  assert_close(bug, runs[0][0], [2.0 * x.double()], 0.0)


def test_guard_passes_a_correct_op():
  _standin_runs(None)


@pytest.mark.parametrize('bug', ['unwritten', 'reads_poison'])
def test_guard_catches_a_result_that_depends_on_the_poison(bug):
  with pytest.raises(AssertionError):
    _standin_runs(bug)


def test_guard_catches_a_write_one_element_past_the_payload():
  with pytest.raises(AssertionError, match='fence overwritten'):
    _standin_runs('overrun')


def test_guard_poisons_every_dtype_and_fences_only_where_asked():
  for p in POISONS:
    with guarded(p, modules=(_standin,), fence_devices=('cpu',)) as g:
      for dt in (torch.float32, torch.complex64, torch.uint8, torch.float64):
        t = _standin.torch.empty((5, 3), dtype=dt)
        assert t.dtype == dt and t.shape == (5, 3) and t.is_contiguous()
        assert torch.all(_bits(t) == p), (dt, p)
      like = _standin.torch.empty_like(torch.zeros(4, 6, dtype=torch.complex64))
      assert torch.all(_bits(like) == p)
      assert len(g.fenced) == 5 and not g.unfenced
    # CPU tensors are poisoned but not fenced by default; so are non-contiguous ones
    with guarded(p, modules=(_standin,)) as g:
      t = _standin.torch.empty((7,), dtype=torch.float32)
      s = _standin.torch.empty_like(torch.zeros(4, 6).t())
      assert torch.all(_bits(t) == p) and not s.is_contiguous()
      raw = torch.empty(0, dtype=torch.uint8).set_(s.untyped_storage())
      assert torch.all(raw == p)
      assert len(g.unfenced) == 2 and not g.fenced


def test_guard_insists_on_an_allocation():
  with pytest.raises(AssertionError, match='no allocation'):
    with guarded(0xFF, modules=(_standin,)):
      pass


def test_guard_restores_the_modules():
  with guarded(0x7F, modules=(_standin,), fence_devices=('cpu',)):
    assert _standin.torch is not torch
    _standin.torch.empty(1)
  assert _standin.torch is torch
  for m in GUARDED_MODULES:
    assert m.torch is torch


# ---- CPU: every uninitialised allocation goes through the guard -----------------------
_PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    'ddsp_b200')
_UNGUARDED = {'new_empty', 'new_empty_strided', 'empty_strided', 'Tensor', 'FloatTensor',
              'DoubleTensor', 'HalfTensor', 'IntTensor', 'LongTensor', 'ByteTensor',
              'empty_permuted'}


def _scan(path):
  """(uses of torch.empty / torch.empty_like, [violations]) of one source file."""
  tree = ast.parse(open(path, encoding='utf-8').read(), path)
  uses, bad = 0, []
  for node in ast.walk(tree):
    where = '%s:%d' % (os.path.basename(path), getattr(node, 'lineno', 0))
    if isinstance(node, ast.ImportFrom) and node.module and node.module.split('.')[0] == 'torch':
      for a in node.names:
        if a.name in ('empty', 'empty_like', '*') or a.name in _UNGUARDED:
          bad.append((where, 'from torch import ' + a.name))
    if isinstance(node, ast.Import):
      for a in node.names:
        if a.name == 'torch' and a.asname not in (None, 'torch'):
          bad.append((where, 'import torch as ' + a.asname))
    if not isinstance(node, ast.Call) or not isinstance(node.func, ast.Attribute):
      continue
    attr, base = node.func.attr, node.func.value
    if attr in _UNGUARDED:
      bad.append((where, attr))
    elif attr in ('empty', 'empty_like'):
      if isinstance(base, ast.Name) and base.id == 'torch':
        uses += 1
      elif not (isinstance(base, ast.Name) and base.id in ('np', 'numpy')):
        bad.append((where, ast.unparse(node.func)))
  return uses, bad


def test_allocations_go_through_the_guard():
  """Every uninitialised allocation in the package is `torch.empty` /
  `torch.empty_like` on the module's own `torch` name, in a module the guard covers."""
  guarded_names = {m.__name__.split('.')[-1] for m in GUARDED_MODULES}
  allocating, bad = set(), []
  for path in sorted(glob.glob(os.path.join(_PKG, '*.py'))):
    uses, b = _scan(path)
    bad += b
    if uses:
      allocating.add(os.path.splitext(os.path.basename(path))[0])
  assert not bad, bad
  assert allocating <= guarded_names, allocating - guarded_names
  assert allocating == guarded_names, ('a guarded module allocates nothing',
                                       guarded_names - allocating)


def test_scan_flags_the_ways_around_the_guard():
  src = ('import torch\nfrom torch import empty\nx = torch.Tensor(3)\n'
         'y = x.new_empty(3)\nz = torch.empty_strided((3,), (1,))\n'
         'w = torch.cuda.empty(3)\nv = torch.empty(3)\n')
  with tempfile.TemporaryDirectory() as d:
    path = os.path.join(d, 'probe.py')
    with open(path, 'w', encoding='utf-8') as f:
      f.write(src)
    uses, bad = _scan(path)
  assert uses == 1
  assert sorted(b[1] for b in bad) == sorted(
      ['from torch import empty', 'Tensor', 'new_empty', 'empty_strided',
       'torch.cuda.empty'])


# ---- the edge-shape table ----------------------------------------------------------
class Edge(Row):
  """A Row with, for the grad rows, `gref`: the float64 torch restatement of the call
  on the inputs in builder order, whose autograd gradients (for `gcheck`, default all
  of `grads`) the kernel's must match at max-relative `gtol`; and `zero(n_samples)`: the
  slice of the audio gradient that no frame covers, which must be exactly 0."""

  def __init__(self, name, build, call, ref=None, tol=1e-4, grads=(), gref=None,
               gtol=5e-4, gcheck=None, zero=None, cmp=None):
    if ref is None:
      ref = lambda *a: [_np(o) for o in _flat(gref(*[_t(x) for x in a]))]
    super().__init__(name, build, call, ref, tol=tol, grads=grads, cmp=cmp)
    self.gref, self.gtol, self.zero = gref, gtol, zero
    self.gcheck = grads if gcheck is None else gcheck


B3 = 3


def _harm_build(b, f, k):
  def build(rng):
    f0 = u(rng, 100.0, 230.0, b, 1, 1) * (1.0 + 0.02 * u(rng, -1, 1, b, f, 1))
    return {'amps': u(rng, 0.1, 1.0, b, f, 1), 'hd': u(rng, 0.0, 1.0, b, f, k),
            'f0': f0}
  return build


def _harmonic(name, b, f, k, hop, method='window', phase_mode='recurrence'):
  n = f * hop
  return Edge(name, _harm_build(b, f, k),
              lambda amps, hd, f0: core.harmonic_synthesis(
                  f0, amps, harmonic_distribution=hd, n_samples=n, sample_rate=SR,
                  amp_resample_method=method, phase_mode=phase_mode),
              lambda amps, hd, f0: oracle.harmonic_synthesis(
                  f0, amps, harmonic_distribution=hd, n_samples=n, sample_rate=SR,
                  amp_resample_method=method))


def _harmonic_fn(name, b, f, k, hop, method='window'):
  n = f * hop
  return Edge(name, _harm_build(b, f, k),
              lambda amps, hd, f0: autograd.HarmonicSynthesisFn.apply(
                  f0, amps, hd, n, SR, method),
              grads=('amps', 'hd', 'f0'), gcheck=('amps', 'hd'),
              gref=lambda amps, hd, f0: grad_ref.harmonic(f0, amps, hd, n, SR, method))


def _decoder_build(b, f, k, nb, n):
  def build(rng):
    f0 = u(rng, 100.0, 230.0, b, 1, 1) * (1.0 + 0.02 * u(rng, -1, 1, b, f, 1))
    return {'amps': rng.standard_normal((b, f, 1)), 'hd': rng.standard_normal((b, f, k)),
            'f0': f0, 'mags': rng.standard_normal((b, f, nb)), 'noise': u(rng, -1, 1, b, n)}
  return build


def _decoder_ref(n):
  return lambda amps, hd, f0, mags, noise: oracle.decoder(
      amps, hd, f0, mags, noise, n_samples=n)['add']['signal']


def _noise_build(f, nb, n):
  return lambda rng: {'mags': u(rng, 0.0, 1.0, 2, f, nb), 'noise': u(rng, -1, 1, 2, n)}


def _noise(name, f, nb, n):
  return Edge(name, _noise_build(f, nb, n),
              lambda mags, noise: core.filtered_noise(mags, n, window_size=0, noise=noise),
              lambda mags, noise: oracle.noise_get_signal(mags, noise, window_size=0))


def _noise_fn(name, f, nb, n):
  return Edge(name, _noise_build(f, nb, n),
              lambda mags, noise: autograd.FilteredNoiseFn.apply(mags, n, 0, noise, 0, 0),
              grads=('mags',),
              gref=lambda mags, noise: grad_ref.frequency_filter(noise, mags, 0))


def _fir(name, n, f, s, ib=2, padding='same', delay=-1):
  return Edge(name, lambda rng: {'audio': u(rng, -1, 1, 2, n),
                                 'ir': u(rng, -1, 1, ib, f, s) / math.sqrt(s)},
              lambda audio, ir: core.fft_convolve(audio, ir, padding=padding,
                                                  delay_compensation=delay),
              grads=('audio', 'ir'), tol=1e-5,
              gref=lambda audio, ir: grad_ref.fft_convolve(audio, ir, padding, delay))


def _long_ir(name, n, s):
  return Edge(name, lambda rng: {'audio': u(rng, -1, 1, 2, n),
                                 'ir': u(rng, -1, 1, 2, s) / math.sqrt(s)},
              lambda audio, ir: core.fft_convolve(audio, ir),
              grads=('audio', 'ir'), tol=1e-5,
              gref=lambda audio, ir: grad_ref.fft_convolve(audio, ir[:, None, :]))


def _sinc(name, n, f, ws, padding='same', cb=2):
  s = sinc_ref.n_taps(ws)
  return Edge(name, lambda rng: {'audio': u(rng, -1, 1, 2, n),
                                 'c': u(rng, 0.05, 0.45, cb, f, 1)},
              lambda audio, c: core.sinc_filter(audio, c, window_size=ws, padding=padding),
              lambda audio, c: sinc_ref.sinc_filter(audio, c, ws, padding=padding),
              tol=1e-5, grads=('audio', 'c'),
              gref=lambda audio, c: sinc_ref.torch_sinc_filter(audio, c, s, padding))


def _per_sample(x):
  return x[..., 0] if x.dim() == 3 else x


def _mod_delay(name, n, length, per_sample=True):
  shape = (2, n, 1) if per_sample else (2, 1)
  return Edge(name, lambda rng: {'audio': u(rng, -1, 1, 2, n), 'g': u(rng, 0, 1, *shape),
                                 'p': u(rng, 0.05, 0.95, *shape)},
              lambda audio, g, p: core.mod_delay(audio, g, p, length, add_dry=True),
              grads=('audio', 'g', 'p'), tol=1e-5,
              gref=lambda audio, g, p: mod_delay_ref.torch_mod_delay(
                  audio, _per_sample(g), _per_sample(p), length, add_dry=True))


def _sinusoidal(name, f, k, hop, method='window'):
  n = f * hop
  return Edge(name, lambda rng: {'f': u(rng, 100, 7000, 2, f, k), 'a': u(rng, 0, 1, 2, f, k)},
              lambda f_, a: core.sinusoidal_synthesis(f_, a, n_samples=n,
                                                      amp_resample_method=method),
              grads=('f', 'a'), gcheck=('a',),
              gref=lambda f_, a: sinusoidal_ref.torch_sinusoidal(f_, a, n, SR, method))


def _oscbank(name, n, k):
  return Edge(name, lambda rng: {'f': u(rng, 100, 9000, 2, n, k), 'a': u(rng, 0, 1, 2, n, k)},
              lambda f, a: core.oscillator_bank(f, a, SR),
              lambda f, a: oracle.oscillator_bank(f, a, SR))


def _cumsum(name, n, k):
  return Edge(name, lambda rng: {'x': u(rng, 0.0, 0.5, 2, n, k)}, core.angular_cumsum,
              oracle.angular_cumsum, tol=2e-5, cmp=_phasor)


def _resample(name, f, n, method):
  return Edge(name, lambda rng: {'x': u(rng, -1, 1, 2, f, 3)},
              lambda x: core.resample(x, n, method=method),
              grads=('x',), tol=1e-5,
              gref=lambda x: routing_ref.resample(x, n, method))


def _covered(n, frame, hop):
  """Samples [0, covered) lie in some frame of an unpadded framing."""
  frames = 1 + (n - frame) // hop if n >= frame else 0
  return (frames - 1) * hop + frame if frames else 0


def _audio_build(n):
  return lambda rng: {'audio': u(rng, -1, 1, 2, n)}


def _no_frames(*shape):
  """The reference of a framing without frames: nothing (the float64 FFT takes no
  empty batch); the gradient's check is that it is exactly 0 everywhere."""
  return lambda audio: np.zeros((2, 0) + shape)


def _stft(name, n):
  return Edge(name, _audio_build(n), lambda audio: spectral_ops.stft_cuda(audio, 256),
              tol=1e-5, grads=('audio',),
              gref=lambda audio: mel_ref.stft(audio, 256),
              cmp=lambda x: np.stack([np.real(_np(x)), np.imag(_np(x))]))


def _loudness(name, n, padding='center'):
  zero = (lambda m: slice(_covered(m, 512, 64), None)) if padding == 'valid' else None
  empty = padding == 'valid' and n < 512
  return Edge(name, _audio_build(n),
              lambda audio: spectral_ops.compute_loudness(audio, padding=padding),
              _no_frames() if empty else None, grads=('audio',), zero=zero,
              gref=None if empty else (
                  lambda audio: loudness_ref.compute_loudness(audio, padding=padding)))


def _power(name, n, padding='center'):
  empty = padding == 'valid' and n < 512
  return Edge(name, _audio_build(n),
              lambda audio: [spectral_ops.compute_power(audio, padding=padding),
                             spectral_ops.compute_rms_energy(audio, padding=padding)],
              (lambda audio: [np.zeros((2, 0))] * 2) if empty else lambda audio: [
                  _np(loudness_ref.compute_power(_t(audio), padding=padding)),
                  np.sqrt(np.mean(_np(loudness_ref.frames(_t(audio), 512, 64, padding))**2,
                                  -1))])


def _mel(name, which, n, pad_end=True):
  fn = {'mel': (spectral_ops.compute_mel, mel_ref.compute_mel),
        'logmel': (spectral_ops.compute_logmel, mel_ref.compute_logmel),
        'mfcc': (spectral_ops.compute_mfcc, mel_ref.compute_mfcc)}[which]
  zero = None if pad_end else (lambda m: slice(_covered(m, 256, 64), None))
  empty = not pad_end and n < 256
  return Edge(name, _audio_build(n),
              lambda audio: fn[0](audio, fft_size=256, pad_end=pad_end),
              _no_frames(13 if which == 'mfcc' else 64) if empty else None,
              grads=('audio',), zero=zero,
              gref=None if empty else (
                  lambda audio: fn[1](audio, fft_size=256, pad_end=pad_end)))


def _kde_build(q, j, bt=(2, 3)):
  return lambda rng: {'a': u(rng, 0.01, 1, *bt, q), 'f': u(rng, 100, 2000, *bt, q),
                      'at': u(rng, 0.01, 1, *bt, j), 'ft': u(rng, 100, 2000, *bt, j)}


def _kde(name, q, j):
  return Edge(name, _kde_build(q, j),
              lambda a, f, at, ft: losses.KDEConsistencyLoss().nll(a, f, at, ft, 0.1),
              lambda a, f, at, ft: _np(consistency_ref.kde_nll(a, f, at, ft, 0.1)),
              tol=1e-3, grads=('a', 'f', 'at', 'ft'))


def _twm(name, c, p):
  return Edge(name, lambda rng: {'f0c': u(rng, 80, 400, 2, 3, c),
                                 'freqs': u(rng, 100, 2000, 2, 3, p),
                                 'amps': u(rng, 0.01, 1, 2, 3, p)},
              lambda f0c, freqs, amps: losses.TWMLoss().get_loss_tensors(f0c, freqs, amps),
              lambda f0c, freqs, amps: [_np(x) for x in consistency_ref.twm_loss_tensors(
                  f0c, freqs, amps)],
              tol=1e-3, grads=('f0c', 'freqs', 'amps'))


EDGES = [
    # harmonic v4: 33 frames leave a partial frame tile, K = 33 a partial 4-wide
    # harmonic vector (f0 below 240 Hz keeps all 33 below Nyquist, where the float64
    # reference could decide a boundary sample differently)
    _harmonic('harmonic_v4_window', B3, 33, 33, 192),
    _harmonic('harmonic_v4_linear', B3, 33, 33, 192, 'linear'),
    # generic kernel: hop 80 is not a multiple of 64 (partial frame tile at 33)
    _harmonic('harmonic_generic_hop80', B3, 33, 33, 80),
    _harmonic('harmonic_generic_k1', B3, 33, 1, 80),                 # one harmonic
    _harmonic('harmonic_generic_direct', B3, 33, 33, 192, 'linear', 'direct'),
    _harmonic('harmonic_v4_f1', B3, 1, 33, 192),                     # a single frame
    _harmonic_fn('HarmonicSynthesisFn_v4_window', B3, 33, 33, 192),
    _harmonic_fn('HarmonicSynthesisFn_v4_linear', B3, 33, 33, 192, 'linear'),
    _harmonic_fn('HarmonicSynthesisFn_k1', B3, 33, 1, 64),
    _harmonic_fn('HarmonicSynthesisFn_f1', B3, 1, 33, 192),
    Edge('decoder_train_f33_hop192', _decoder_build(B3, 33, 33, 9, 33 * 192),
         lambda amps, hd, f0, mags, noise: autograd.decoder_train(
             amps, hd, f0, mags, n_samples=33 * 192, noise=noise),
         _decoder_ref(33 * 192), grads=('amps', 'hd', 'f0', 'mags')),
    Edge('decoder_train_f1', _decoder_build(B3, 1, 33, 9, 192),
         lambda amps, hd, f0, mags, noise: autograd.decoder_train(
             amps, hd, f0, mags, n_samples=192, noise=noise),
         _decoder_ref(192), grads=('amps', 'hd', 'f0', 'mags')),
    # decoder_forward off the ring route (hop 192, 9 bands)
    Edge('decoder_forward_off_ring', _decoder_build(B3, 33, 33, 9, 33 * 192),
         lambda amps, hd, f0, mags, noise: core.decoder_forward(
             amps, hd, f0, mags, 33 * 192, noise=noise), _decoder_ref(33 * 192)),
    # filtered noise: 80-sample frames with a ragged last frame, N % 4 = 1, 2, 3 (fused)
    *[_noise(f'filtered_noise_fused_n{n}', 20, 9, n) for n in (1597, 1598, 1599)],
    # 81-sample frames (not a multiple of 16): generic route, ragged, N % 4 = 1, 2, 3
    *[_noise(f'filtered_noise_generic_n{n}', 20, 9, n) for n in (1601, 1602, 1603)],
    # ring route: 33 frames of 64 (its frame tile is partial); the ring takes no
    # ragged frame (N = 64 F)
    _noise('filtered_noise_ring_f33', 33, 65, 33 * 64),
    _noise_fn('FilteredNoiseFn_fused_n1599', 20, 9, 1599),
    _noise_fn('FilteredNoiseFn_generic_n1601', 20, 9, 1601),
    _noise_fn('FilteredNoiseFn_ring_f33', 33, 65, 33 * 64),
    # FIR: one tap; 2047 taps (the longest direct-form IR) over 7 ragged frames of 101;
    # one sample; 'valid'; a delay past the IR's length
    _fir('fir_s1', 700, 7, 1, delay=0),
    _fir('fir_s2047_ragged', 703, 7, 2047),
    _fir('fir_n1', 1, 1, 17),
    _fir('fir_valid_shared_ir', 703, 7, 17, ib=1, padding='valid'),
    _fir('fir_delay_past_s', 703, 7, 17, delay=20),
    # long convolution: one sample, odd lengths, IR longer than the crop (d IR past it)
    _long_ir('long_ir_n1_s2048', 1, 2048),
    _long_ir('long_ir_n1025_s2048', 1025, 2048),
    _long_ir('long_ir_n1025_s3073', 1025, 3073),
    # sinc filter: fewer samples than taps; 2047 taps over 7 ragged frames with a cutoff
    # per frame; 'valid'
    _sinc('sinc_n_lt_s', 100, 1, 256),
    _sinc('sinc_w2047_ragged', 703, 7, 2047),
    _sinc('sinc_valid', 703, 7, 63, padding='valid'),
    _sinc('sinc_shared_cutoff', 703, 7, 63, cb=1),                  # one cutoff row
    # frequency filter with one set of magnitudes for the batch, 7 ragged frames
    Edge('frequency_filter_shared_mags',
         lambda rng: {'audio': u(rng, -1, 1, 2, 703), 'm': u(rng, 0, 1, 1, 7, 9)},
         lambda audio, m: core.frequency_filter(audio, m, window_size=11),
         grads=('audio', 'm'), tol=1e-5,
         gref=lambda audio, m: grad_ref.frequency_filter(audio, m, 11)),
    # mod delay: one sample; a one-sample line; a line longer than the audio; [B, 1]
    # gain and phase
    _mod_delay('mod_delay_n1', 1, 100),
    _mod_delay('mod_delay_l1', 300, 1),
    _mod_delay('mod_delay_l_gt_n', 50, 100),
    _mod_delay('mod_delay_b1_gain_phase', 300, 100, per_sample=False),
    # wavetable: 257 frames (past the 256-frame phase tile), 5140 samples (past 4096:
    # d wavetables split into segments)
    Edge('wavetable_f257_n5140',
         lambda rng: {'f0': u(rng, 100, 600, 2, 1, 1) * (1 + 0.02 * u(rng, -1, 1, 2, 257, 1)),
                      'a': u(rng, 0, 1, 2, 257, 1), 'w': u(rng, -1, 1, 2, 257, 64)},
         lambda f0, a, w: core.wavetable_synthesis(f0, a, w, n_samples=257 * 20),
         lambda f0, a, w: wavetable_ref.wavetable_synthesis(f0, a, w, 257 * 20, SR),
         grads=('f0', 'a', 'w'), gcheck=('a', 'w'),
         gref=lambda f0, a, w: wavetable_ref.torch_wavetable_synthesis(
             f0[..., 0], a[..., 0], w, 257 * 20, SR)),
    # sinusoidal: hop 1; one sinusoid; K = 33 at hop 63; K = 420 (the tile shrinks)
    _sinusoidal('sinusoidal_hop1', 64, 4, 1, 'linear'),
    _sinusoidal('sinusoidal_k1', 20, 1, 80),
    _sinusoidal('sinusoidal_k33_hop63', 21, 33, 63),
    _sinusoidal('sinusoidal_k420', 20, 420, 64),
    # oscillator bank and angular cumsum: one sample; 129 samples of 129 sinusoids
    _oscbank('oscillator_bank_n1', 1, 129),
    _oscbank('oscillator_bank_n129', 129, 129),
    _cumsum('angular_cumsum_n1', 1, 129),
    _cumsum('angular_cumsum_n129', 129, 129),
    # resample from a single frame, to one sample and to five
    *[_resample(f'resample_{m}_f1_n{n}', 1, n, m)
      for m in ('linear', 'nearest', 'cubic') for n in (1, 5)],
    # mix of one sample; impulse responses of 1, 2047 and 2048 taps
    Edge('mix_n1', lambda rng: {'s1': u(rng, -1, 1, 2, 1, 1), 's2': u(rng, -1, 1, 2, 1, 1),
                                'm': u(rng, 0.05, 0.95, 2, 1, 1)},
         core.mix, grads=('s1', 's2', 'm'), tol=1e-6, gref=routing_ref.mix),
    *[Edge(f'exp_decay_ir_l{n}', lambda rng, n=n: {'g': u(rng, 0.1, 1, 2, 1),
                                                   'd': u(rng, 0, 2, 2, 1),
                                                   'nz': u(rng, -1, 1, 1, n)},
           lambda g, d, nz, n=n: core.exp_decay_ir(g, d, n, noise=nz),
           grads=('g', 'd'), tol=1e-5,
           gref=lambda g, d, nz, n=n: routing_ref.exp_decay_ir(g, d, n, nz))
      for n in (1, 2047, 2048)],
    # add: lengths that leave 1, 3 and 1 elements past a 4-wide vector
    *[Edge(f'add_n{n}', lambda rng, n=n: {'a': u(rng, -1, 1, 2, n), 'b': u(rng, -1, 1, 2, n)},
           core.add, grads=('a', 'b'), tol=1e-7, gref=lambda a, b: a + b)
      for n in (1, 3, 5)],
    # spectral features: one sample; fewer samples than the FFT; N not a multiple of
    # the hop; N just past 4096 (the backward's per-CTA ownership); unpadded framings
    # with no frame at all and with a tail no frame covers (gradient exactly 0 there)
    *[_stft(f'stft_cuda_n{n}', n) for n in (1, 100, 1601, 4097)],
    *[_loudness(f'loudness_n{n}', n) for n in (1, 100, 1601, 4097)],
    _loudness('loudness_valid_no_frames', 100, 'valid'),
    _loudness('loudness_valid_tail', 1601, 'valid'),
    *[_power(f'power_rms_n{n}', n) for n in (1, 100, 1601, 4097)],
    _power('power_rms_valid_no_frames', 100, 'valid'),
    _power('power_rms_valid_tail', 1601, 'valid'),
    *[_mel(f'{w}_n{n}', w, n) for w in ('mel', 'logmel', 'mfcc') for n in (1, 100, 1601, 4097)],
    *[_mel(f'{w}_no_pad_end_no_frames', w, 100, False) for w in ('mel', 'logmel', 'mfcc')],
    *[_mel(f'{w}_no_pad_end_tail', w, 1601, False) for w in ('mel', 'logmel', 'mfcc')],
    # mixture NLL: one query; 513 queries (past the query chunk); 4096 components;
    # comb NLL over 4096 points
    _kde('kde_nll_q1', 1, 6),
    _kde('kde_nll_q513', 513, 6),
    _kde('kde_nll_j4096', 6, 4096),
    _twm('twm_p4096', 4, 4096),
    # no queries but components: the mixture's gradients are exactly 0
    Edge('kde_nll_q0', _kde_build(0, 5),
         lambda a, f, at, ft: losses.KDEConsistencyLoss().nll(a, f, at, ft, 0.1),
         lambda a, f, at, ft: _np(consistency_ref.kde_nll(a, f, at, ft, 0.1)),
         grads=('at', 'ft'), zero=lambda m: slice(None)),
]
EDGE_IDS = [e.name for e in EDGES]


def test_edge_table_is_well_formed():
  assert len(set(EDGE_IDS)) == len(EDGES)
  for e in EDGES:
    if e.name.startswith(('filtered_noise_', 'FilteredNoiseFn_')):
      shapes = {k: v.shape for k, v in e.build(np.random.default_rng(0)).items()}
      _, f, nb = shapes['mags']
      want = e.name.split('_')[2 if e.name.startswith('filtered') else 1]
      assert grad_ref.noise_route(f, nb, shapes['noise'][1], 0) == want, e.name
    if e.name.startswith(('harmonic_v4', 'HarmonicSynthesisFn_v4')):
      shapes = {k: v.shape for k, v in e.build(np.random.default_rng(0)).items()}
      b, f, k = shapes['hd']
      assert grad_ref.harmonic_v4_tile_width(b, f, k, 192, 132) is not None, e.name
    assert set(e.gcheck) <= set(e.grads)


@pytest.mark.parametrize('row', EDGES, ids=EDGE_IDS)
def test_edge_references_run_on_the_host(row):
  d = {k: np.asarray(v, np.float64) for k, v in row.build(np.random.default_rng(0)).items()}
  for w in _flat(row.ref(*d.values())):
    assert isinstance(np.asarray(_np(w)), np.ndarray)


def _gref_grads(row, t, gs):
  x = {k: v.detach().double().cpu().requires_grad_(k in row.grads) for k, v in t.items()}
  outs = _flat(row.gref(*x.values()))
  torch.autograd.backward(outs, [g.detach().cpu().to(o.dtype) for g, o in zip(gs, outs)])
  return {k: torch.zeros_like(x[k]) if x[k].grad is None else x[k].grad
          for k in row.grads}


# ---- GPU ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('row', ROWS, ids=[r.name for r in ROWS])
def test_rows_under_every_poison(row):
  """Outputs and gradients of every input-conventions row: the unguarded call's bits
  under every poison, inside intact fences."""
  t = row.inputs()
  want = _run(row, t)
  runs = _poisoned_runs(row, t)
  assert_poison_independent([want] + runs[:1], row.name)
  want_ref = row.ref(*[v.double().cpu().numpy() for v in t.values()])
  assert_close(row.name, runs[0][0], want_ref, row.tol, row.cmp)
  for k, g in runs[0][1].items():
    assert torch.all(torch.isfinite(g)), (row.name, k)


@pytest.mark.gpu
@pytest.mark.parametrize('row', EDGES, ids=EDGE_IDS)
def test_edge_shapes_under_every_poison(row):
  t = row.inputs()
  runs = _poisoned_runs(row, t)
  outs, grads = runs[0]
  want = row.ref(*[v.double().cpu().numpy() for v in t.values()])
  assert_close(row.name, outs, want, row.tol, row.cmp)
  if not row.grads:
    return
  for k, g in grads.items():
    assert g is not None and g.shape == t[k].shape, (row.name, k)
    assert torch.all(torch.isfinite(g)), (row.name, k)
  if row.gref is not None:
    gw = _gref_grads(row, t, upstream(outs))
    for k in row.gcheck:
      assert_close((row.name, 'd ' + k), grads[k], gw[k], row.gtol)
  if row.zero is not None:
    for k in row.grads:
      tail = grads[k][..., row.zero(t[k].shape[-1])]
      assert torch.all(_bits(tail) == 0), (row.name, k, 'not exactly 0 where nothing '
                                           'depends on the input')


@pytest.mark.gpu
@pytest.mark.parametrize('poison', POISONS, ids=POISON_IDS)
def test_host_decoder_under_every_poison(poison):
  """HostDecoder, 7 items in 3 chunks, into a poisoned pinned output: the device
  ProcessorGroup's bits."""
  import ddsp_b200
  from tests.util import synth_inputs
  b, f, k, nb, n = 7, 125, 100, 65, 8000
  keys = ['amps', 'harmonic_distribution', 'f0_hz', 'noise_magnitudes']

  def group():
    return ddsp_b200.ProcessorGroup(dag=[
        (ddsp_b200.Harmonic(n_samples=n), ['amps', 'harmonic_distribution', 'f0_hz']),
        (ddsp_b200.FilteredNoise(n_samples=n, window_size=0, seed=9),
         ['noise_magnitudes']),
        (ddsp_b200.Add(), ['filtered_noise/signal', 'harmonic/signal'])])
  inp = synth_inputs(b, f, k, nb, n, seed=12)
  feats = {key: inp[key] for key in keys}
  want = group()({key: torch.from_numpy(v).cuda() for key, v in feats.items()})
  with guarded(poison) as g:
    dec = ddsp_b200.HostDecoder(group(), max_batch=b, n_frames=f, n_harmonics=k,
                                n_bands=nb, n_chunks=3)
    got = dec({key: host.pin(v) for key, v in feats.items()})
    dec.close()
  assert any(d.type == 'cpu' for _, _, d, _ in g.unfenced), 'output not poisoned'
  assert got.is_pinned() and torch.equal(_bits(got), _bits(want.cpu()))


@pytest.mark.gpu
@pytest.mark.parametrize('hop,method', [(1, 'linear'), (33, 'window'), (80, 'linear'),
                                        (192, 'window')])
def test_harmonic_d_f0_is_bit_reproducible_at_any_hop(hop, method):
  """`ddsp_b200_harmonic_backward_f0` sums each frame's terms in a fixed order: at a
  hop of 1, 33 or 80 a warp's 32 samples straddle frames, at 192 they do not.  d f0
  matches float64 autograd and repeated calls give the same bits."""
  b, f, k = 3, 33, 20
  n = f * hop
  rng = np.random.default_rng(hop)
  d = _harm_build(b, f, k)(rng)
  f0, amps, hd = (torch.as_tensor(d[key], dtype=torch.float32, device='cuda')
                  for key in ('f0', 'amps', 'hd'))
  g = torch.as_tensor(rng.standard_normal((b, n)), dtype=torch.float32, device='cuda')
  runs = [autograd._harmonic_d_f0(f0, amps, hd, g, n, SR, method) for _ in range(3)]
  for r in runs[1:]:
    assert_same_bits(r, runs[0], (hop, 'd f0'))
  f0d = f0.double().cpu().requires_grad_(True)
  grad_ref.harmonic(f0d, amps.double().cpu(), hd.double().cpu(), n, SR, method).backward(
      g.double().cpu())
  assert_close((hop, 'd f0'), runs[0], f0d.grad, 5e-4)


# ---- fenced operands ---------------------------------------------------------------
def _fenced(x, fill, off):
  """x's values in a view `off` elements past a FENCE-byte run of `fill`, followed by
  another; returns (view, buffer, the fence bytes as they were)."""
  pad = FENCE // x.element_size()
  buf = torch.full((2 * pad + off + x.numel(),), fill, dtype=x.dtype, device=x.device)
  v = buf[pad + off:pad + off + x.numel()].view(x.shape)
  v.copy_(x)
  fences = torch.cat([_bits(buf[:pad + off]), _bits(buf[pad + off + x.numel():])]).clone()
  return v, (buf, pad + off, x.numel(), fences)


def _fences_intact(region, what):
  buf, start, n, fences = region
  now = torch.cat([_bits(buf[:start]), _bits(buf[start + n:])])
  assert torch.equal(now, fences), (what, 'fence modified')


@pytest.mark.gpu
@pytest.mark.parametrize('row', ROWS + EDGES, ids=[r.name for r in ROWS + EDGES])
def test_fenced_operands_give_the_canonical_bits(row):
  """Every input and the upstream gradient between 64 KiB fences of NaN, and of 7.0,
  at storage offsets of 0 and 1 element: the bits of fresh contiguous operands at the
  same offset (torch's own reductions may round differently at another alignment),
  with fences and inputs unchanged."""
  t = row.inputs()
  want_outs, _ = _run(row, t)
  gs = upstream(want_outs) if row.grads else None
  for off in (0, 1):
    fresh = {k: at_offset(v, off) for k, v in t.items()}
    want_outs, want_grads = _run(row, fresh, None if gs is None else [
        at_offset(g, off) for g in gs])
    for fill in (math.nan, 7.0):
      what = (row.name, fill, off)
      regions = []
      ins = {}
      for k, v in t.items():
        ins[k], r = _fenced(v, fill, off)
        regions.append(r)
      fgs = None
      if gs is not None:
        fgs = []
        for g in gs:
          fg, r = _fenced(g, fill, off)
          fgs.append(fg)
          regions.append(r)
      outs, grads = _run(row, ins, fgs)
      assert_same_bits(outs, want_outs, what)
      for k in row.grads:
        assert_same_bits(grads[k].contiguous(), want_grads[k], what + (k,))
      torch.cuda.synchronize()
      for r in regions:
        _fences_intact(r, what)


# ---- workspaces at the C ABI -------------------------------------------------------
WS_OFFSETS = (0, 16, 128, 240)
# every entry point whose last three parameters are (workspace, workspace_bytes, stream)
WORKSPACE_CALLS = {
    'ddsp_b200_filtered_noise_forward', 'ddsp_b200_harmonic_backward_f0',
    'ddsp_b200_fir_time_varying_backward', 'ddsp_b200_frequency_filter_backward',
    'ddsp_b200_sinc_filter_backward', 'ddsp_b200_oscillator_bank',
    'ddsp_b200_fft_convolve_lti', 'ddsp_b200_angular_cumsum',
    'ddsp_b200_sinusoidal_forward', 'ddsp_b200_sinusoidal_backward',
    'ddsp_b200_wavetable_forward', 'ddsp_b200_wavetable_backward'}


def test_workspace_entry_points_are_the_ones_tested():
  """The ten *_workspace queries and harmonic_backward_f0 (12 B F bytes, stated in the
  header) cover every entry point that takes a workspace."""
  takes = {name for name, (_, args) in _lib.SIGNATURES.items()
           if len(args) >= 3 and args[-3] is ctypes.c_void_p and
           args[-2] is ctypes.c_size_t and not name.endswith('_workspace')}
  assert takes == WORKSPACE_CALLS
  queries = {n for n in _lib.SIGNATURES if n.endswith('_workspace')}
  assert len(queries) == 10


class _Relocator:
  """Stands in for the loaded library: every workspace-taking entry point gets, in
  place of the caller's workspace, a fresh one of exactly the bytes the caller passes,
  `off` bytes past a 256-byte boundary between canary fences, its payload poisoned."""

  def __init__(self, real, off):
    self.real, self.off = real, off
    self.calls = []

  def __getattr__(self, name):
    fn = getattr(self.real, name)
    if name not in WORKSPACE_CALLS:
      return fn

    def call(*args):
      args = list(args)
      nbytes = int(args[-2])
      if nbytes == 0 or not args[-3]:
        return fn(*args)
      buf = torch.full((2 * FENCE + 256 + nbytes,), CANARY, dtype=torch.uint8,
                       device='cuda')
      assert buf.data_ptr() % 256 == 0
      start = FENCE + self.off
      buf[start:start + nbytes].fill_(0xFF)
      args[-3] = buf.data_ptr() + start
      self.calls.append((name, buf, start, nbytes))
      return fn(*args)
    return call


# row name -> the workspace entry points it reaches
WS_ROWS = {
    'filtered_noise_generic': {'ddsp_b200_filtered_noise_forward'},
    'filtered_noise_generic_n1601': {'ddsp_b200_filtered_noise_forward'},
    'HarmonicSynthesisFn_v4_window': {'ddsp_b200_harmonic_backward_f0'},
    'HarmonicSynthesisFn_k1': {'ddsp_b200_harmonic_backward_f0'},
    # the FIR, frequency-filter and sinc-filter backwards ask for a workspace when
    # one operand is shared by the batch
    'fir_valid_shared_ir': {'ddsp_b200_fir_time_varying_backward'},
    'frequency_filter_shared_mags': {'ddsp_b200_frequency_filter_backward'},
    'sinc_shared_cutoff': {'ddsp_b200_sinc_filter_backward'},
    'oscillator_bank': {'ddsp_b200_oscillator_bank'},
    'oscillator_bank_n129': {'ddsp_b200_oscillator_bank'},
    'angular_cumsum': {'ddsp_b200_angular_cumsum'},
    'angular_cumsum_n129': {'ddsp_b200_angular_cumsum'},
    'fft_convolve_lti': {'ddsp_b200_fft_convolve_lti'},
    'long_ir_n1025_s3073': {'ddsp_b200_fft_convolve_lti'},
    'sinusoidal_synthesis': {'ddsp_b200_sinusoidal_forward',
                             'ddsp_b200_sinusoidal_backward'},
    'sinusoidal_k420': {'ddsp_b200_sinusoidal_forward', 'ddsp_b200_sinusoidal_backward'},
    'wavetable_synthesis': {'ddsp_b200_wavetable_forward', 'ddsp_b200_wavetable_backward'},
    'wavetable_f257_n5140': {'ddsp_b200_wavetable_forward',
                             'ddsp_b200_wavetable_backward'},
}
_BY_NAME = {r.name: r for r in ROWS + EDGES}


def test_workspace_rows_cover_every_workspace_entry_point():
  assert set(WS_ROWS) <= set(_BY_NAME)
  assert set().union(*WS_ROWS.values()) == WORKSPACE_CALLS


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(WS_ROWS))
def test_workspace_at_every_alignment(name, monkeypatch):
  row = _BY_NAME[name]
  t = row.inputs()
  want = _run(row, t)
  gs = upstream(want[0]) if row.grads else None
  real = _lib.load()
  seen = set()
  for off in WS_OFFSETS:
    rel = _Relocator(real, off)
    monkeypatch.setattr(_lib, 'load', lambda rel=rel: rel)
    got = _run(row, t, gs)
    monkeypatch.setattr(_lib, 'load', lambda: real)
    torch.cuda.synchronize()
    assert_poison_independent([want, got], (name, off))
    for fn, buf, start, n in rel.calls:
      assert (buf.data_ptr() + start) % 256 == off, (fn, off)
      assert torch.all(buf[:start] == CANARY) and torch.all(buf[start + n:] == CANARY), (
          name, fn, off, 'workspace fence overwritten')
      seen.add(fn)
  assert seen >= WS_ROWS[name], (name, WS_ROWS[name] - seen)
