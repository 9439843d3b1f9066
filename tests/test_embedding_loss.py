"""losses.EmbeddingLoss, PretrainedCREPEEmbeddingLoss and PretrainedCREPE, and the CUDA
framing they train through (csrc/crepe.cuh: crepe_frames with
DDSP_B200_CREPE_LOSS_FRAMES, and ddsp_b200_crepe_frames_backward), against the float64
restatement tests/embedding_ref.py, which tests/golden/embedding_loss.npz pins to the
unmodified reference."""
import copy
import ctypes
import os

import numpy as np
import pytest
import torch

import ddsp_b200
from ddsp_b200 import _lib, autograd, losses
from tests import embedding_ref as ref
from tests.golden import make_embedding_loss_golden as golden

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'embedding_loss.npz'))
gpu = pytest.mark.gpu
FLAG = _lib.CREPE_LOSS_FRAMES
# The backward against torch.autograd of the float64 restatement on the same float32
# audio: the kernel's sums are in double, so only the final rounding to float32 and the
# float32 frames the forward reads differ.
BWD_RTOL, BWD_ATOL = 1e-5, 1e-6


# ---- the restatement against the reference --------------------------------------------
@pytest.mark.parametrize('i', range(len(golden.FRAME_CASES)), ids=[c[0] for c in golden.FRAME_CASES])
def test_frames_restatement(i):
  name, hop, center, _ = golden.FRAME_CASES[i]
  frames = ref.frame_audio(golden.frame_input(i), hop, center).numpy()
  np.testing.assert_allclose(frames[:, golden.kept_rows(frames.shape[1])],
                             GOLDEN['frames_' + name], rtol=1e-9, atol=1e-9)


def test_call_and_losses_restatement():
  np.testing.assert_allclose(ref.call(golden.call_input()), GOLDEN['call'], rtol=1e-9,
                             atol=1e-12)
  target, audio = golden.loss_inputs()
  for loss_type in golden.LOSS_TYPES:
    np.testing.assert_allclose(ref.embedding_loss(target, audio, golden.LOSS_WEIGHT, loss_type),
                               GOLDEN['loss_' + loss_type], rtol=1e-9)
  assert ref.embedding_loss(target, audio, 0.0, 'L1') == GOLDEN['loss_weight0'] == 0.0


def test_layer_weights(monkeypatch):
  assert tuple(losses.CREPE_LAYER_SCALE) == golden.LAYERS
  monkeypatch.setattr(losses, 'PretrainedCREPE', lambda **kwargs: None)
  got = [losses.PretrainedCREPEEmbeddingLoss(weight=golden.LAYER_WEIGHT,
                                             activation_layer=l).weight
         for l in golden.LAYERS]
  np.testing.assert_allclose(got, GOLDEN['layer_weights'], rtol=1e-15)


@pytest.mark.parametrize('hop,center', [(1, True), (160, True), (512, False), (1024, True),
                                        (2048, True), (2048, False)])
def test_closed_form_gradient_is_autograd(hop, center):
  """The closed form the kernel evaluates is torch.autograd of the restatement, NaN
  where a frame has variance 0 included."""
  rng = np.random.default_rng(hop)
  x = rng.normal(size=(2, 5000))
  x[1, 1000:3200] = 0.25
  xt = torch.tensor(x, requires_grad=True)
  frames = ref.frame_audio(xt, hop, center)
  g = torch.as_tensor(rng.normal(size=frames.shape))
  frames.backward(g)
  want = xt.grad.numpy()
  got = ref.frame_audio_grad(x, g.numpy(), hop, center)
  np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
  assert np.isnan(want[1]).any() and not np.isnan(want[0]).any()
  ok = ~np.isnan(want)
  np.testing.assert_allclose(got[ok], want[ok], rtol=1e-9, atol=1e-9)


# ---- argument errors (no device work) ---------------------------------------------------
def _net():
  return torch.nn.Sequential(torch.nn.Linear(1024, 8))


def test_errors():
  with pytest.raises(KeyError):     # before the network is looked at
    losses.PretrainedCREPEEmbeddingLoss(model_capacity=3, activation_layer='conv7-BN')
  with pytest.raises(ValueError, match='activation layer conv5-maxpool not found'):
    losses.PretrainedCREPE(_net())
  with pytest.raises(ValueError, match='activation layer classifier not found'):
    losses.PretrainedCREPEEmbeddingLoss(model_capacity=_net())
  for size in ('tiny', 'small', 'medium', 'large', 'full'):
    with pytest.raises(NotImplementedError, match='crepe package'):
      losses.PretrainedCREPE(size)
    with pytest.raises(NotImplementedError, match='crepe package'):
      losses.PretrainedCREPEEmbeddingLoss(model_capacity=size)
  for bad in (3, lambda x: x, 'crepe.pt'):
    with pytest.raises(TypeError, match='torch.nn.Module'):
      losses.PretrainedCREPE(bad, activation_layer='0')
  with pytest.raises(TypeError, match='TorchScript'):
    losses.PretrainedCREPE(torch.jit.script(_net()), activation_layer='0')
  m = losses.PretrainedCREPE(_net(), activation_layer='0')
  assert (m.name, m.trainable, m.frame_length, m.layer_names) == (
      'pretrained_crepe', False, 1024, ['0'])
  with pytest.raises(ValueError, match='batch, length'):
    m.frame_audio(np.zeros(3000, np.float32))
  with pytest.raises(ValueError, match='hop_length'):
    m.frame_audio(np.zeros((1, 3000), np.float32), hop_length=0)


def test_weight_zero_does_not_call_the_model():
  def model(audio):
    raise AssertionError('called')
  for w in (0.0, -1.0):
    loss = losses.EmbeddingLoss(weight=w, pretrained_model=model)
    got = loss(np.zeros((1, 100)), np.zeros((1, 100)))
    assert type(got) is float and got == 0.0
  loss = losses.EmbeddingLoss(weight=0.0)
  assert (loss.name, loss.loss_type) == ('embedding_loss', 'L1')
  assert loss.get_losses_dict(None, None) == {'embedding_loss': 0.0}
  assert losses.PretrainedCREPEEmbeddingLoss.__init__.__defaults__ == (
      1.0, 'L1', 'tiny', 'classifier', 'pretrained_crepe_embedding_loss')


def test_abi_refusals():
  lib = _lib.load()
  fake = 1 << 20               # never dereferenced: the checks fail first
  C, V, S = _lib.PAD_CENTER, _lib.PAD_VALID, _lib.PAD_SAME
  before = lib.ddsp_b200_launch_count()
  fwd, bwd = lib.ddsp_b200_crepe_frames, lib.ddsp_b200_crepe_frames_backward
  # forward, flagged: any hop with CENTER, but frame counts, SAME and shapes are checked
  assert fwd(fake, fake, 1, 3000, 3, 2048, C | FLAG, None) == _lib.E_INVALID   # 2 frames
  assert b'n_frames=3, the padding gives 2' in lib.ddsp_b200_last_error()
  assert fwd(fake, fake, 1, 3000, 3, 1024, S | FLAG, None) == _lib.E_INVALID
  assert b'bad padding' in lib.ddsp_b200_last_error()
  assert fwd(fake, fake, 1, 3000, 3, 0, C | FLAG, None) == _lib.E_INVALID
  assert fwd(fake, fake, -1, 3000, 3, 1024, C | FLAG, None) == _lib.E_INVALID
  assert fwd(fake, None, 1, 3000, 3, 1024, C | FLAG, None) == _lib.E_INVALID
  assert fwd(fake, fake, 1, 3000, 3, 1024, C | FLAG, None) == _lib.E_INVALID   # overlap
  assert b'frames must not overlap audio' in lib.ddsp_b200_last_error()
  # without the flag the hop rule is spectral_ops.pad's, as before
  assert fwd(fake, fake, 1, 3000, 2, 2048, C, None) == _lib.E_INVALID
  assert b'must be greater than hop_size' in lib.ddsp_b200_last_error()
  # empty work returns after the checks
  assert fwd(None, None, 0, 3000, 3, 1024, C | FLAG, None) == _lib.OK
  assert fwd(fake, None, 2, 1000, 0, 160, V | FLAG, None) == _lib.OK
  assert fwd(None, None, 2, 0, 0, 160, V | FLAG, None) == _lib.OK
  # backward
  g, a, d = fake, fake + (1 << 24), fake + (1 << 26)
  assert bwd(a, g, d, 1, 3000, 4, 1024, C, None) == _lib.E_INVALID            # 3 frames
  assert bwd(a, g, d, 1, 3000, 3, 1024, S, None) == _lib.E_INVALID
  assert bwd(a, g, d, 1, 3000, 3, -5, C, None) == _lib.E_INVALID
  assert bwd(a, g, None, 1, 3000, 3, 1024, C, None) == _lib.E_INVALID
  assert b'null pointer' in lib.ddsp_b200_last_error()
  assert bwd(a, g, a + 400, 1, 3000, 3, 1024, C | FLAG, None) == _lib.E_INVALID
  assert b'grad_audio must not overlap audio' in lib.ddsp_b200_last_error()
  assert bwd(a, g, g + 4 * 3 * 1024 - 4, 1, 3000, 3, 1024, C, None) == _lib.E_INVALID
  assert b'grad_audio must not overlap grad_frames' in lib.ddsp_b200_last_error()
  assert bwd(None, None, None, 0, 3000, 3, 1024, C, None) == _lib.OK
  assert bwd(None, None, None, 3, 0, 1, 1024, C, None) == _lib.OK
  assert lib.ddsp_b200_launch_count() == before
  assert _lib.SIGNATURES['ddsp_b200_crepe_frames_backward'][1] == (
      [ctypes.c_void_p] * 3 + [ctypes.c_int] * 5 + [ctypes.c_void_p])


# ---- frames on the GPU -------------------------------------------------------------------
def _audio(rng, b, n, silent=True):
  x = rng.normal(size=(b, n)) * rng.uniform(0.01, 3.0, size=(b, 1))
  if silent and n >= 3000:
    x[:, 1000:2100] = 0.25       # frames of variance 0
  x[:, : n // 3] += 2.0          # frames with a large mean
  return x.astype(np.float32)


def _ref_rows(x, hop, center, rows):
  """The restatement's frames `rows` of the flattened [B * F, 1024], in float64, from
  the padded float32 audio, without building the others."""
  xp = np.pad(x.astype(np.float64), ((0, 0), (512, 512)) if center else ((0, 0), (0, 0)))
  f = ref.n_frames(x.shape[1], hop, center)
  b, k = np.divmod(rows, f)
  fr = xp[b[:, None], k[:, None] * hop + np.arange(1024)]
  mu = fr.mean(-1, keepdims=True)
  return (fr - mu) / (np.sqrt(((fr - mu) ** 2).mean(-1, keepdims=True)) + 1e-5)


def _frames(x, hop, center):
  return autograd.CrepeLossFramesFn.apply(x, hop, center)


@gpu
@pytest.mark.parametrize('center', [True, False])
@pytest.mark.parametrize('hop', golden.HOPS)
def test_frames(hop, center):
  rng = np.random.default_rng(hop + center)
  for b in (1, 3, 64):
    for n in golden.LENGTHS:
      f = ref.n_frames(n, hop, center)
      if f == 0 or (b > 1 and n == 64000 and hop < 512):
        continue
      x = _audio(rng, b, n)
      got = _frames(torch.as_tensor(x, device='cuda'), hop, center)
      assert got.shape == (b, f, 1024)
      got = got.reshape(-1, 1024)
      rows = np.arange(b * f)
      if len(rows) > 4096:
        rows = np.unique(np.r_[0, b * f - 1, rng.integers(0, b * f, 4094)])
      np.testing.assert_allclose(got[torch.as_tensor(rows, device='cuda')].cpu().numpy(),
                                 _ref_rows(x, hop, center, rows), rtol=0, atol=2e-5,
                                 err_msg=f'B={b} N={n}')


@gpu
def test_frames_match_the_reference():
  for i, (name, hop, center, _) in enumerate(golden.FRAME_CASES):
    x = torch.as_tensor(golden.frame_input(i), dtype=torch.float32, device='cuda')
    got = _frames(x, hop, center)
    np.testing.assert_allclose(got[:, golden.kept_rows(got.shape[1])].cpu().numpy(),
                               GOLDEN['frames_' + name], rtol=0, atol=2e-5, err_msg=name)


def _grads(x, g, hop, center):
  xt = torch.as_tensor(x, device='cuda').requires_grad_(True)
  _frames(xt, hop, center).backward(torch.as_tensor(g, device='cuda'))
  return xt.grad


def _want_grads(x, g, hop, center):
  xt = torch.tensor(x.astype(np.float64), requires_grad=True)
  ref.frame_audio(xt, hop, center).backward(torch.as_tensor(g, dtype=torch.float64))
  return xt.grad.numpy()


@gpu
@pytest.mark.parametrize('center', [True, False])
@pytest.mark.parametrize('hop', [1, 7, 160, 512, 1023, 1024, 1500, 2048])
def test_backward(hop, center):
  rng = np.random.default_rng(10 * hop + center)
  for b, n in ((1, 1000), (3, 3000), (2, 64000 if hop >= 160 else 9000)):
    f = ref.n_frames(n, hop, center)
    if f == 0:
      continue
    x = _audio(rng, b, n, silent=False)
    g = rng.normal(size=(b, f, 1024)).astype(np.float32)
    got = _grads(x, g, hop, center).cpu().numpy()
    want = _want_grads(x, g, hop, center)
    assert np.isfinite(want).all()
    np.testing.assert_allclose(got, want, rtol=BWD_RTOL,
                               atol=BWD_ATOL * np.abs(want).max(), err_msg=f'B={b} N={n}')


@gpu
@pytest.mark.parametrize('hop,center', [(160, True), (1024, True), (2048, False)])
def test_silent_frames_are_nan_where_they_read(hop, center):
  rng = np.random.default_rng(hop)
  x = _audio(rng, 3, 8000, silent=False)
  x[1, 3000:5200] = 0.5
  f = ref.n_frames(8000, hop, center)
  g = rng.normal(size=(3, f, 1024)).astype(np.float32)
  got = _grads(x, g, hop, center).cpu().numpy()
  want = _want_grads(x, g, hop, center)
  nan = np.isnan(want)
  assert nan[1].any() and not nan[0].any() and not nan[2].any()
  np.testing.assert_array_equal(np.isnan(got), nan)
  np.testing.assert_allclose(got[~nan], want[~nan], rtol=BWD_RTOL,
                             atol=BWD_ATOL * np.abs(want[~nan]).max())


@gpu
@pytest.mark.parametrize('hop,center', [(160, True), (1024, True), (2048, False)])
def test_uncovered_samples_get_zero(hop, center):
  """hop 2048 without centring leaves gaps between frames and a tail after the last."""
  rng = np.random.default_rng(1)
  x = _audio(rng, 2, 7000, silent=False)
  f = ref.n_frames(7000, hop, center)
  got = _grads(x, rng.normal(size=(2, f, 1024)).astype(np.float32), hop, center)
  covered = np.zeros(7000 + (1024 if center else 0), bool)
  for k in range(f):
    covered[k * hop:k * hop + 1024] = True
  covered = covered[512:512 + 7000] if center else covered[:7000]
  assert (got.cpu().numpy()[:, ~covered] == 0).all()
  assert (got.cpu().numpy()[:, covered] != 0).all()


@gpu
@pytest.mark.parametrize('hop', [160, 1024])
def test_reproducible_and_batch_independent(hop):
  rng = np.random.default_rng(hop)
  x = _audio(rng, 5, 16000, silent=False)
  f = ref.n_frames(16000, hop, True)
  g = rng.normal(size=(5, f, 1024)).astype(np.float32)
  first, second = _grads(x, g, hop, True), _grads(x, g, hop, True)
  assert torch.equal(first, second)
  for i in range(5):
    alone = _grads(x[i:i + 1], g[i:i + 1], hop, True)
    assert torch.equal(alone[0], first[i]), i
    frames = _frames(torch.as_tensor(x, device='cuda'), hop, True)
    assert torch.equal(_frames(torch.as_tensor(x[i:i + 1], device='cuda'), hop, True)[0],
                       frames[i])


@gpu
@pytest.mark.parametrize('poison', [0x00, 0xFF, 0x7F])
def test_poisoned_and_fenced_memory(poison):
  from tests.test_gpu_memory_bounds import guarded, _fenced, _fences_intact
  rng = np.random.default_rng(2)
  m = losses.PretrainedCREPE(_net().cuda(), activation_layer='0')
  for hop, center, n in ((160, True, 5001), (1024, True, 4000), (2048, False, 9000)):
    x = torch.as_tensor(_audio(rng, 2, n, silent=False), device='cuda')
    f = ref.n_frames(n, hop, center)
    g = torch.as_tensor(rng.normal(size=(2, f, 1024)), dtype=torch.float32, device='cuda')
    want_frames = _frames(x, hop, center)
    want_grad = _grads(x.cpu().numpy(), g.cpu().numpy(), hop, center)
    fx, rx = _fenced(x, float('nan'), 3)
    fg, rg = _fenced(g, float('nan'), 1)
    with guarded(poison):
      xt = fx.detach().requires_grad_(True)
      frames = m.frame_audio(xt, hop_length=hop, center=center)
      frames.backward(fg)
    _fences_intact(rx, 'audio')
    _fences_intact(rg, 'grad_frames')
    assert torch.equal(frames, want_frames)
    assert torch.equal(xt.grad, want_grad)


@gpu
def test_layouts_streams_and_devices():
  rng = np.random.default_rng(3)
  m = losses.PretrainedCREPE(_net().cuda(), activation_layer='0')
  x = torch.as_tensor(_audio(rng, 3, 5000, silent=False), device='cuda')
  want = _frames(x, 160, True)
  # non-contiguous, offset, CPU, NumPy and float64 audio
  strided = x.t().contiguous().t()
  assert not strided.is_contiguous()
  big = torch.cat([torch.zeros(1, 5000, device='cuda'), x])[1:]
  assert big.storage_offset() == 5000
  for a in (strided, big, x.cpu(), x.cpu().numpy(), x.double()):
    assert torch.equal(m.frame_audio(a, hop_length=160), want)
  g = torch.as_tensor(rng.normal(size=tuple(want.shape)), dtype=torch.float32, device='cuda')
  want_grad = _grads(x.cpu().numpy(), g.cpu().numpy(), 160, True)
  xs = strided.detach().requires_grad_(True)
  m.frame_audio(xs, hop_length=160).backward(g.transpose(0, 1).contiguous().transpose(0, 1))
  assert torch.equal(xs.grad, want_grad)
  # the current stream
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    xt = x.detach().requires_grad_(True)
    got = m.frame_audio(xt, hop_length=160)
    got.backward(g)
  s.synchronize()
  assert torch.equal(got, want) and torch.equal(xt.grad, want_grad)
  if torch.cuda.device_count() > 1:
    m1 = losses.PretrainedCREPE(_net().to('cuda:1'), activation_layer='0')
    got = m1.frame_audio(x.to('cuda:1'), hop_length=160)
    assert got.device == torch.device('cuda:1')
    assert torch.equal(got.cuda(0), want)


# ---- end to end --------------------------------------------------------------------------
class TinyCrepe(torch.nn.Module):
  """CREPE's layer structure at a small size: six conv blocks (conv, ReLU, BN, max-pool)
  named as Keras names them, and a sigmoid classifier on the time-major flattening."""

  def __init__(self, channels=8):
    super().__init__()
    c = channels
    for i in range(1, 7):
      if i == 1:
        conv = torch.nn.Conv2d(1, c, (64, 1), stride=(4, 1), padding=(30, 0))
      else:
        conv = torch.nn.Conv2d(c, c, (8, 1), padding='same')
      self.add_module(f'conv{i}', conv)
      self.add_module(f'conv{i}-BN', torch.nn.BatchNorm2d(c))
      self.add_module(f'conv{i}-maxpool', torch.nn.MaxPool2d((2, 1)))
    self.classifier = torch.nn.Sequential(torch.nn.Linear(4 * c, 360), torch.nn.Sigmoid())

  def forward(self, frames):
    y = frames[:, None, :, None]
    for i in range(1, 7):
      y = self._modules[f'conv{i}'](y).relu()
      y = self._modules[f'conv{i}-BN'](y)
      y = self._modules[f'conv{i}-maxpool'](y)
    return self.classifier(y.permute(0, 2, 3, 1).flatten(1))


def _tiny_crepe(seed=0):
  torch.manual_seed(seed)
  net = TinyCrepe()
  for mod in net.modules():
    if isinstance(mod, torch.nn.BatchNorm2d):
      mod.running_mean.uniform_(-0.1, 0.1)
      mod.running_var.uniform_(0.5, 2.0)
  return net.eval()


def _activation64(net, frames, layer):
  out = []
  net = copy.deepcopy(net).double().cpu()
  h = net.get_submodule(layer).register_forward_hook(lambda m, i, o: out.append(o))
  with torch.no_grad():
    net(frames.reshape(-1, 1024))
  h.remove()
  return out[0]


@gpu
@pytest.mark.parametrize('layer', golden.LAYERS)
def test_pretrained_crepe_embedding_loss_end_to_end(layer):
  net = _tiny_crepe().cuda()
  n = 8000
  rng = np.random.default_rng(5)
  f0 = torch.full((2, 20, 1), 220.0, device='cuda')
  f0[1] = 330.0
  amps = torch.full((2, 20, 1), -2.0, device='cuda', requires_grad=True)
  hd = torch.as_tensor(rng.normal(size=(2, 20, 16)), dtype=torch.float32, device='cuda')
  audio = ddsp_b200.Harmonic(n_samples=n)(amps, hd, f0)
  target = torch.as_tensor(_audio(rng, 2, n, silent=False) * 0.1, device='cuda')
  for loss_type in golden.LOSS_TYPES:
    loss_fn = losses.PretrainedCREPEEmbeddingLoss(weight=0.5, loss_type=loss_type,
                                                  model_capacity=net, activation_layer=layer)
    assert loss_fn.weight == 20.0 * losses.CREPE_LAYER_SCALE[layer] * 0.5
    loss = loss_fn(target, audio)
    # the same network in float64 on the restated frames
    emb = [_activation64(net, ref.frame_audio(a.detach().cpu().double(), 1024, True), layer)
           .reshape(2, ref.n_frames(n, 1024, True), -1) for a in (target, audio)]
    want = loss_fn.weight * losses.mean_difference(emb[0], emb[1], loss_type)
    # float32 network against float64; near cos = 1, 1 - cos cancels in float32
    np.testing.assert_allclose(loss.item(), want.item(), rtol=2e-4,
                               atol=1e-6 * loss_fn.weight, err_msg=loss_type)
    amps.grad = None
    loss.backward(retain_graph=True)
    assert amps.grad is not None and torch.isfinite(amps.grad).all()
    assert amps.grad.abs().max() > 0
    assert all(p.grad is None for p in net.parameters())
  assert all(p.requires_grad for p in net.parameters()) and not net.training
  # trainable: the network's parameters get gradients too
  model = losses.PretrainedCREPE(net, activation_layer=layer, trainable=True)
  loss = losses.EmbeddingLoss(pretrained_model=model)(target, audio.detach())
  loss.backward()
  grads = [p.grad for p in net.parameters()]
  assert any(g is not None and g.abs().max() > 0 for g in grads)


@gpu
def test_call_matches_the_reference_stub():
  """PretrainedCREPE.call with the fixture's stub network as a torch module: the
  [batch, n_frames, -1] reshape of the reference."""
  w = torch.as_tensor(ref.stub_weights(), dtype=torch.float32, device='cuda')

  class Stub(torch.nn.Module):
    def __init__(self):
      super().__init__()
      self.proj = torch.nn.Identity()

    def forward(self, frames):
      return self.proj(torch.tanh(frames @ w).reshape(-1, 4, 3))

  m = losses.PretrainedCREPE(Stub(), activation_layer='proj')
  got = m(torch.as_tensor(golden.call_input(), dtype=torch.float32, device='cuda'))
  assert got.shape == GOLDEN['call'].shape
  np.testing.assert_allclose(got.cpu().numpy(), GOLDEN['call'], rtol=0, atol=1e-4)
  loss = losses.EmbeddingLoss(weight=golden.LOSS_WEIGHT, pretrained_model=m)
  target, audio = golden.loss_inputs()
  np.testing.assert_allclose(loss(target, audio).item(), GOLDEN['loss_L1'], rtol=1e-4)
