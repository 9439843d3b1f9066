"""spectral_ops.pad and PretrainedCREPE (csrc/crepe.cuh: frames, Viterbi path, f0) and
the training preprocessors, against the float64 restatement tests/crepe_ref.py, which
tests/golden/crepe.npz pins to the unmodified reference."""
import os

import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, core, preprocessing, spectral_ops
from tests import crepe_ref as ref
from tests.golden import make_crepe_golden as golden

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'crepe.npz'))
gpu = pytest.mark.gpu


# ---- the restatement against the reference --------------------------------------------
@pytest.mark.parametrize('i', range(len(golden.PAD_CASES)))
def test_pad_matches_reference(i):
  name, _, frame, hop, padding, axis, mode = golden.PAD_CASES[i]
  x = golden.pad_input(i)
  want = GOLDEN['pad_' + name]
  got = spectral_ops.pad(torch.as_tensor(x), frame, hop, padding=padding, axis=axis,
                         mode=mode)
  assert got.dtype == torch.float32 and got.device.type == 'cpu'
  np.testing.assert_allclose(got.numpy(), want, rtol=1e-6, atol=1e-7)
  if mode == 'CONSTANT' and axis == 1 and len(x.shape) == 2:
    np.testing.assert_array_equal(ref.pad(x, frame, hop, padding), want)


@pytest.mark.parametrize('i', range(len(golden.FRAME_CASES)))
def test_frames_restatement(i):
  name, _, _, hop, padding = golden.FRAME_CASES[i]
  np.testing.assert_allclose(ref.frames(golden.frame_input(i), hop, padding),
                             GOLDEN['frames_' + name], rtol=1e-9, atol=1e-9)


def test_decode_restatement():
  acts, centers = golden.decode_input()
  for key, c in (('decode', None), ('decode_given', centers)):
    f0, conf = ref.activations_to_f0_and_confidence(acts, c)
    np.testing.assert_allclose(f0, GOLDEN[key + '_f0'], rtol=1e-6)
    np.testing.assert_array_equal(conf, GOLDEN[key + '_confidence'])


@pytest.mark.parametrize('i', range(len(golden.VITERBI_CASES)))
def test_viterbi_restatement(i):
  path, _ = ref.viterbi_decode(golden.viterbi_input(i))
  np.testing.assert_array_equal(path, GOLDEN['viterbi_' + golden.VITERBI_CASES[i][0]])


# ---- argument errors (no device work) ---------------------------------------------------
def test_pad_errors():
  x = torch.zeros(2, 100)
  with pytest.raises(ValueError, match='must be greater'):
    spectral_ops.pad(x, 64, 128, 'center')
  with pytest.raises(ValueError, match='padding'):
    spectral_ops.pad(x, 64, 16, 'full')
  assert spectral_ops.pad(x, 64, 128, 'valid') is not None   # 'valid' checks nothing
  with pytest.raises(ValueError):
    spectral_ops.pad(x, 512, 16, 'center', mode='reflect')


@pytest.mark.parametrize('size', ['full', 'large', 'small', 'tiny'])
def test_size_names_raise(size):
  with pytest.raises(NotImplementedError, match='crepe package'):
    spectral_ops.PretrainedCREPE(size)
  with pytest.raises(NotImplementedError):
    preprocessing.OnlineF0PowerPreprocessor(crepe_saved_model_path=size)


def test_model_argument():
  with pytest.raises(TypeError):
    spectral_ops.PretrainedCREPE(3)
  m = spectral_ops.PretrainedCREPE(lambda x: x, hop_size=256)
  assert (m.hop_size, m.frame_size, m.sample_rate) == (256, 1024, 16000)


def test_torchscript_path(tmp_path):
  net = torch.jit.script(torch.nn.Linear(1024, 360))
  path = str(tmp_path / 'crepe.pt')
  net.save(path)
  m = spectral_ops.PretrainedCREPE(path)
  x = torch.randn(3, 1024)
  torch.testing.assert_close(m.core_model(x), net(x))


def test_shape_errors():
  m = spectral_ops.PretrainedCREPE(lambda x: x)
  with pytest.raises(ValueError, match='activations'):
    m.activations_to_f0_and_confidence(np.zeros((4, 359)))
  with pytest.raises(ValueError, match='centers'):
    m.activations_to_f0_and_confidence(np.zeros((4, 360)), np.zeros(3, np.int64))
  for shape in ((4, 360), (2, 4, 361), (2, 0, 360)):
    with pytest.raises(ValueError, match='acts'):
      m.viterbi_decode(np.zeros(shape, np.float32))
  with pytest.raises(ValueError, match='frames'):
    m.normalize_frames(np.zeros((4, 1000), np.float32))
  with pytest.raises(ValueError, match='padding'):
    m.predict_f0_and_confidence(np.zeros((1, 2000), np.float32), padding='full')
  with pytest.raises(ValueError, match='audio'):
    m.predict_f0_and_confidence(np.zeros((1, 2, 2000), np.float32))


def test_batch_frames():
  m = spectral_ops.PretrainedCREPE(lambda x: x, hop_size=160)
  x = torch.randn(2, 3000)
  np.testing.assert_array_equal(m.batch_frames(x).numpy(),
                                ref.batch_frames(x.numpy(), 160).astype(np.float32))
  assert m.batch_frames(torch.zeros(3, 1024)).shape == (3, 1024)
  assert m.batch_frames(torch.zeros(3, 1000)).shape == (0, 1024)


def test_viterbi_abi_checks():
  lib = _lib.load()
  assert lib.ddsp_b200_crepe_viterbi_workspace_bytes(64, 1001) == 4 * 61 * 64 * 1000
  assert lib.ddsp_b200_crepe_viterbi_workspace_bytes(3, 1) == 0
  assert lib.ddsp_b200_crepe_viterbi_workspace_bytes(0, 10) == 0
  assert lib.ddsp_b200_crepe_viterbi(None, None, None, 0, 2, 0, None) == _lib.E_INVALID
  assert lib.ddsp_b200_crepe_viterbi(None, None, None, 0, 0, 5, None) == _lib.OK
  fake = 1 << 20     # never dereferenced: the checks fail first
  need = lib.ddsp_b200_crepe_viterbi_workspace_bytes(2, 5)
  assert lib.ddsp_b200_crepe_viterbi(fake, fake, fake, need - 1, 2, 5, None) == \
      _lib.E_WORKSPACE
  assert lib.ddsp_b200_crepe_frames(fake, fake, 1, 2000, 11, 2048, _lib.PAD_CENTER,
                                    None) == _lib.E_INVALID
  assert lib.ddsp_b200_crepe_frames(fake, fake, 1, 2000, 12, 160, _lib.PAD_CENTER,
                                    None) == _lib.E_INVALID   # 13 frames
  assert lib.ddsp_b200_crepe_decode(None, None, None, None, -1, None) == _lib.E_INVALID


def test_preprocessor_keys_and_errors():
  assert preprocessing.F0LoudnessPreprocessor.output_keys == (
      'f0_hz', 'loudness_db', 'f0_scaled', 'ld_scaled')
  assert preprocessing.F0PowerPreprocessor.output_keys == (
      'f0_hz', 'pw_db', 'f0_scaled', 'pw_scaled')
  assert preprocessing.OnlineF0PowerPreprocessor.output_keys == (
      'f0_hz', 'pw_db', 'f0_scaled', 'pw_scaled', 'f0_confidence')
  p = preprocessing.OnlineF0PowerPreprocessor(compute_f0=False, compute_power=False,
                                              crepe_saved_model_path=None)
  with pytest.raises(ValueError, match='compute_f0=True'):
    p({'audio': torch.zeros(1, 16000), 'f0_hz': torch.zeros(1, 251)})
  with pytest.raises(KeyError, match='audio'):
    p({'f0_hz': torch.zeros(1, 251)})
  with pytest.raises(KeyError, match='loudness_db'):
    preprocessing.F0LoudnessPreprocessor()({'f0_hz': torch.zeros(1, 10)})
  # without any computation the inputs pass through the scaling and the sanity check
  f0 = torch.full((2, 251), 440.0)     # 16000 samples, hop 64, 'center': 251 frames
  pw = torch.full((2, 251), -40.0)
  out = p({'audio': torch.zeros(2, 16000), 'f0_hz': f0, 'f0_confidence': f0, 'pw_db': pw})
  assert tuple(out) == p.output_keys
  assert out['f0_hz'].shape == (2, 251, 1)
  torch.testing.assert_close(out['pw_scaled'], torch.full((2, 251, 1), 0.5))
  torch.testing.assert_close(out['f0_scaled'], torch.full((2, 251, 1), 69.0 / 127.0))
  with pytest.raises(ValueError, match='does not have 251 timesteps'):
    p({'audio': torch.zeros(2, 16000), 'f0_hz': f0[:, :250], 'f0_confidence': f0,
       'pw_db': pw})


def test_scaling_helpers():
  assert preprocessing.at_least_3d(torch.tensor(1.0)).shape == (1, 1, 1)
  assert preprocessing.at_least_3d(torch.zeros(5)).shape == (1, 5, 1)
  assert preprocessing.at_least_3d(torch.zeros(2, 5)).shape == (2, 5, 1)
  db = torch.tensor([-80.0, -40.0, 0.0])
  torch.testing.assert_close(preprocessing.inv_scale_db(preprocessing.scale_db(db)), db)
  hz = torch.tensor([55.0, 440.0, 3000.0])
  torch.testing.assert_close(
      preprocessing.inv_scale_f0_hz(preprocessing.scale_f0_hz(hz)), hz, rtol=1e-5, atol=0)


# ---- frames on the GPU -------------------------------------------------------------------
def _frames(audio, hop, padding):
  frames, _ = spectral_ops._crepe_frames(audio, hop, padding)
  return frames


@gpu
@pytest.mark.parametrize('padding', ['center', 'same', 'valid'])
@pytest.mark.parametrize('hop', [16, 160, 333, 1024])
def test_frames(padding, hop):
  rng = np.random.default_rng(hop)
  for b, n in ((1, 1024), (3, 3000), (2, 1023 + hop)):
    x = rng.normal(size=(b, n)) * rng.uniform(0.01, 10.0, size=(b, 1))
    x[:, : n // 2] += 3.0     # frames with a large mean
    got = _frames(torch.as_tensor(x, dtype=torch.float32, device='cuda'), hop, padding)
    want = ref.frames(x.astype(np.float32), hop, padding)
    assert got.shape == want.shape
    np.testing.assert_allclose(got.cpu().numpy(), want, rtol=0, atol=2e-5)


@gpu
@pytest.mark.parametrize('b', [1, 7, 64, 256])
def test_frames_batch(b):
  x = np.random.default_rng(b).normal(size=(b, 2500)).astype(np.float32)
  got = _frames(torch.as_tensor(x, device='cuda'), 160, 'center')
  np.testing.assert_allclose(got.cpu().numpy(), ref.frames(x, 160, 'center'), atol=2e-5)


@gpu
def test_frames_exact_and_silent():
  m = spectral_ops.PretrainedCREPE(lambda x: x)
  x = np.zeros((4, 1024), np.float32)
  x[1] = 0.5                                    # constant: variance 0
  x[2] = np.random.default_rng(0).normal(size=1024)
  x[3, 100] = 1e-30                             # a tiny variance is still a variance
  got = _frames(torch.as_tensor(x, device='cuda'), 160, 'valid')
  assert got.shape == (4, 1024)
  want = ref.frames(x, 160, 'valid')
  np.testing.assert_allclose(got.cpu().numpy(), want, atol=2e-5)
  assert (got[:2] == 0).all()
  np.testing.assert_allclose(m.normalize_frames(x).cpu().numpy(), want, atol=2e-5)
  # 'valid' audio shorter than a frame has no frames
  assert _frames(torch.zeros(2, 1000, device='cuda'), 160, 'valid').shape == (0, 1024)


# ---- the Viterbi path on the GPU -----------------------------------------------------------
def _viterbi(acts):
  m = spectral_ops.PretrainedCREPE(lambda x: x)
  return m.viterbi_decode(torch.as_tensor(acts, dtype=torch.float32, device='cuda'))


@gpu
@pytest.mark.parametrize('b,t', [(1, 1), (3, 2), (2, 7), (4, 100), (2, 1001), (1, 2100)])
def test_viterbi_margin_cases(b, t):
  acts = golden.activations(np.random.default_rng(7 * t + b), b, t, noise=0.01)
  acts = acts.astype(np.float32)
  got = _viterbi(acts)
  assert got.dtype == torch.int64 and got.shape == (b, t)
  want, _ = ref.viterbi_decode(acts)
  np.testing.assert_array_equal(got.cpu().numpy(), want)


@gpu
def test_viterbi_planted_ties():
  t = 50
  acts = np.zeros((4, t, 360), np.float32)
  acts[0, :, 100] = acts[0, :, 200] = 0.8      # two equal, distant peaks
  acts[1, :, 0] = acts[1, :, 359] = 0.8        # the same at the edges
  acts[2, :, 100] = acts[2, :, 101] = 0.8      # two equal, adjacent peaks
  acts[3, :t // 2, 180] = 0.9                  # a jump to one of two equal peaks
  acts[3, t // 2:, 50] = acts[3, t // 2:, 300] = 0.9
  got = _viterbi(acts).cpu().numpy()
  want, _ = ref.viterbi_decode(acts)
  np.testing.assert_array_equal(got, want)
  assert (got[0] == 100).all() and (got[1] == 0).all() and (got[2] == 100).all()
  assert (got[3, t // 2:] == 50).all()


@gpu
def test_viterbi_near_ties_score():
  """Uniform noise leaves many near-ties, where the path is float-sensitive: the path
  found must score the oracle's best within rounding."""
  acts = np.random.default_rng(5).uniform(size=(3, 300, 360)).astype(np.float32)
  got = _viterbi(acts).cpu().numpy()
  want, best = ref.viterbi_decode(acts)
  score = ref.path_score(got, acts)
  np.testing.assert_allclose(score, best, rtol=0, atol=1e-3)
  assert (got == want).mean() > 0.5


# ---- f0 and confidence on the GPU -----------------------------------------------------------
@gpu
def test_decode():
  acts, centers = golden.decode_input()
  acts = acts.astype(np.float32)
  a = torch.as_tensor(acts, device='cuda')
  for c in (None, centers, centers.astype(np.int32), torch.as_tensor(centers)):
    f0, conf = spectral_ops.PretrainedCREPE.activations_to_f0_and_confidence(a, c)
    want_f0, want_conf = ref.activations_to_f0_and_confidence(
        acts, None if c is None else centers)
    assert f0.shape == (64,) and conf.shape == (64, 1)
    np.testing.assert_allclose(f0.cpu().numpy(), want_f0, rtol=2e-7)
    np.testing.assert_array_equal(conf.cpu().numpy(), want_conf)


@gpu
def test_decode_edges_and_zero_weights():
  acts = np.zeros((10, 360), np.float32)
  for r, c in enumerate([0, 1, 2, 3, 356, 357, 358, 359]):
    acts[r, c] = 1.0
    acts[r, (c + 2) % 360] = 0.25
  a = torch.as_tensor(acts, device='cuda')
  f0, conf = spectral_ops.PretrainedCREPE.activations_to_f0_and_confidence(a)
  want_f0, _ = ref.activations_to_f0_and_confidence(acts)
  got = f0.cpu().numpy()
  np.testing.assert_allclose(got[:8], want_f0[:8], rtol=2e-7)
  assert np.isnan(got[8:]).all() and np.isnan(want_f0[8:]).all()   # 0 / 0
  # many rows, more than one grid's worth of warps
  acts = np.random.default_rng(1).uniform(size=(50000, 360)).astype(np.float32)
  f0, conf = spectral_ops.PretrainedCREPE.activations_to_f0_and_confidence(
      torch.as_tensor(acts, device='cuda'))
  want_f0, want_conf = ref.activations_to_f0_and_confidence(acts)
  np.testing.assert_allclose(f0.cpu().numpy(), want_f0, rtol=2e-7)
  np.testing.assert_array_equal(conf.cpu().numpy(), want_conf)


# ---- end to end ---------------------------------------------------------------------------
def _network(seed=0):
  torch.manual_seed(seed)
  net = torch.nn.Sequential(torch.nn.Linear(1024, 64), torch.nn.Tanh(),
                            torch.nn.Linear(64, 360), torch.nn.Sigmoid())
  return net


def _network64(net, frames):
  x = torch.as_tensor(frames, dtype=torch.float64)
  w = [p.detach().cpu().double() for p in net.parameters()]
  h = torch.tanh(x @ w[0].T + w[1])
  return torch.sigmoid(h @ w[2].T + w[3]).numpy()


@gpu
@pytest.mark.parametrize('viterbi', [False, True])
@pytest.mark.parametrize('padding', ['center', 'same', 'valid'])
def test_predict_f0_and_confidence(viterbi, padding):
  net = _network().cuda()
  m = spectral_ops.PretrainedCREPE(net, hop_size=160)
  rng = np.random.default_rng(4)
  audio = (np.sin(2 * np.pi * 220.0 * np.arange(8000) / 16000.0)[None] *
           rng.uniform(0.1, 1.0, size=(3, 1)) + 0.1 * rng.normal(size=(3, 8000)))
  audio = audio.astype(np.float32)
  f0, conf = m.predict_f0_and_confidence(torch.as_tensor(audio, device='cuda'),
                                         viterbi=viterbi, padding=padding)
  n_frames = spectral_ops._framing(audio, 1024, 160, padding)[3]
  assert f0.shape == conf.shape == (3, n_frames)
  # the network in float64 on the float64 frames
  acts64 = _network64(net, ref.frames(audio, 160, padding))
  with torch.no_grad():
    acts32 = net(_frames(torch.as_tensor(audio, device='cuda'), 160, padding))
  np.testing.assert_allclose(acts32.cpu().numpy(), acts64, atol=1e-3)
  # decode of the GPU's activations in float64; a random network's activations are
  # full of near-ties, so the Viterbi centres are held to the best path's score
  a = acts32.cpu().numpy()
  centers = None
  if viterbi:
    centers = m.viterbi_decode(acts32.reshape(3, -1, 360)).cpu().numpy()
    _, best = ref.viterbi_decode(a.reshape(3, -1, 360))
    np.testing.assert_allclose(ref.path_score(centers, a.reshape(3, -1, 360)), best,
                               rtol=0, atol=1e-3)
    centers = centers.reshape(-1)
  want_f0, want_conf = ref.activations_to_f0_and_confidence(a, centers)
  np.testing.assert_allclose(f0.cpu().numpy().reshape(-1), want_f0, rtol=1e-6)
  np.testing.assert_array_equal(conf.cpu().numpy().reshape(-1), want_conf[:, 0])
  # 1-D audio is one item
  f0_1, conf_1 = m.predict_f0_and_confidence(torch.as_tensor(audio[0], device='cuda'),
                                             viterbi=viterbi, padding=padding)
  assert f0_1.shape == conf_1.shape == (1, n_frames)


# ---- preprocessors ---------------------------------------------------------------------
@gpu
def test_online_f0_power_preprocessor():
  net = _network(1).cuda()
  audio = torch.as_tensor(np.random.default_rng(2).normal(size=(2, 16000)) * 0.1,
                          dtype=torch.float32, device='cuda')
  for viterbi in (False, True):
    p = preprocessing.OnlineF0PowerPreprocessor(crepe_saved_model_path=net,
                                                viterbi=viterbi)
    out = p({'audio': audio})
    assert tuple(out) == p.output_keys
    for k in ('f0_hz', 'pw_db', 'f0_scaled', 'pw_scaled'):
      assert out[k].shape == (2, 251, 1), k
    assert out['f0_confidence'].shape == (2, 251)
    f0, conf = p.crepe_model.predict_f0_and_confidence(audio, viterbi=viterbi)
    torch.testing.assert_close(out['f0_hz'][..., 0], f0, rtol=0, atol=0)
    torch.testing.assert_close(out['f0_confidence'], conf, rtol=0, atol=0)
    pw = spectral_ops.compute_power(audio, 16000, 250, 1024)
    torch.testing.assert_close(out['pw_db'][..., 0], pw, rtol=0, atol=0)
  # a power frame that does not give CREPE's frame count fails the sanity check
  p = preprocessing.OnlineF0PowerPreprocessor(crepe_saved_model_path=net,
                                              frame_size=512, padding='valid')
  with pytest.raises(ValueError, match='timesteps'):
    p({'audio': audio})
  # audio_16k replaces audio
  p = preprocessing.OnlineF0PowerPreprocessor(crepe_saved_model_path=net)
  out = p({'audio': torch.zeros(2, 5, device='cuda'), 'audio_16k': audio})
  assert out['f0_hz'].shape == (2, 251, 1)


@gpu
def test_f0_loudness_and_power_preprocessors():
  rng = np.random.default_rng(3)
  audio = torch.as_tensor(rng.normal(size=(2, 16000)) * 0.1, dtype=torch.float32,
                          device='cuda')
  f0 = torch.as_tensor(rng.uniform(100, 500, size=(2, 250)), dtype=torch.float32,
                       device='cuda')
  p = preprocessing.F0LoudnessPreprocessor(time_steps=250)
  out = p({'audio': audio, 'f0_hz': f0, 'loudness_db': None})
  assert tuple(out) == p.output_keys
  ld = spectral_ops.compute_loudness(audio, 16000, 250)
  torch.testing.assert_close(out['loudness_db'], core.resample(ld[..., None], 250))
  torch.testing.assert_close(out['f0_scaled'], preprocessing.scale_f0_hz(out['f0_hz']))
  p = preprocessing.F0PowerPreprocessor(time_steps=250)
  out = p({'audio': audio, 'f0_hz': f0})
  assert tuple(out) == p.output_keys and out['pw_db'].shape == (2, 250, 1)
  pw = spectral_ops.compute_power(audio, 16000, 250, 64)
  torch.testing.assert_close(out['pw_db'], core.resample(pw[..., None], 250))
  out2 = p({'power_db': pw, 'f0_hz': f0})
  torch.testing.assert_close(out2['pw_db'], out['pw_db'])
  with pytest.raises(ValueError, match='"power_db" or "audio"'):
    p({'f0_hz': f0})


# ---- conventions: grad, devices, layouts, memory ------------------------------------------
@gpu
def test_refused_under_grad():
  m = spectral_ops.PretrainedCREPE(_network().cuda())
  audio = torch.zeros(1, 4000, device='cuda', requires_grad=True)
  acts = torch.rand(2, 5, 360, device='cuda', requires_grad=True)
  with pytest.raises(RuntimeError, match='requires grad'):
    m.predict_f0_and_confidence(audio)
  with pytest.raises(RuntimeError, match='requires grad'):
    m.viterbi_decode(acts)
  with pytest.raises(RuntimeError, match='requires grad'):
    m.activations_to_f0_and_confidence(acts[0])
  with pytest.raises(RuntimeError, match='requires grad'):
    m.normalize_frames(torch.zeros(2, 1024, device='cuda', requires_grad=True))
  with torch.no_grad():
    m.predict_f0_and_confidence(audio)
    m.viterbi_decode(acts)
  # the network's own parameters require grad; its output carries none
  f0, conf = m.predict_f0_and_confidence(audio.detach())
  assert not f0.requires_grad and not conf.requires_grad


@gpu
def test_layouts_and_devices():
  rng = np.random.default_rng(6)
  acts = golden.activations(rng, 2, 40).astype(np.float32)
  m = spectral_ops.PretrainedCREPE(lambda x: x)
  want = m.viterbi_decode(torch.as_tensor(acts, device='cuda'))
  # CPU and NumPy inputs run on the current device
  torch.testing.assert_close(m.viterbi_decode(acts), want, rtol=0, atol=0)
  torch.testing.assert_close(m.viterbi_decode(torch.as_tensor(acts)), want, rtol=0, atol=0)
  # a non-contiguous view, float64 and half precision inputs
  strided = torch.as_tensor(acts, device='cuda').transpose(0, 1).contiguous().transpose(0, 1)
  assert not strided.is_contiguous()
  torch.testing.assert_close(m.viterbi_decode(strided), want, rtol=0, atol=0)
  torch.testing.assert_close(m.viterbi_decode(torch.as_tensor(acts, dtype=torch.float64)),
                             want, rtol=0, atol=0)
  rows = torch.as_tensor(acts.reshape(-1, 360), device='cuda')
  f0, conf = m.activations_to_f0_and_confidence(rows)
  f0_t, conf_t = m.activations_to_f0_and_confidence(rows.t().contiguous().t())
  torch.testing.assert_close(f0_t, f0, rtol=0, atol=0)
  audio = torch.as_tensor(rng.normal(size=(2, 3000)), dtype=torch.float32)
  want_frames = _frames(audio.cuda(), 160, 'center')
  torch.testing.assert_close(_frames(audio, 160, 'center'), want_frames, rtol=0, atol=0)
  torch.testing.assert_close(_frames(audio.cuda()[:, None, :].expand(2, 2, 3000)[:, 0],
                                     160, 'center'), want_frames, rtol=0, atol=0)
  if torch.cuda.device_count() > 1:
    got = m.viterbi_decode(torch.as_tensor(acts, device='cuda:1'))
    assert got.device == torch.device('cuda:1')
    torch.testing.assert_close(got.cuda(0), want, rtol=0, atol=0)


@gpu
@pytest.mark.parametrize('poison', [0x00, 0xFF, 0x7F])
def test_poisoned_and_fenced_memory(poison):
  from tests.test_gpu_memory_bounds import guarded, _fenced, _fences_intact
  rng = np.random.default_rng(8)
  acts = torch.as_tensor(golden.activations(rng, 3, 130), dtype=torch.float32,
                         device='cuda')
  audio = torch.as_tensor(rng.normal(size=(2, 2999)), dtype=torch.float32, device='cuda')
  m = spectral_ops.PretrainedCREPE(lambda x: x)
  want = (m.viterbi_decode(acts), m.activations_to_f0_and_confidence(acts[0]),
          _frames(audio, 160, 'same'))
  fa, ra = _fenced(acts, float('nan'), 5)
  fx, rx = _fenced(audio, float('nan'), 3)
  with guarded(poison):
    got = (m.viterbi_decode(fa), m.activations_to_f0_and_confidence(fa[0]),
           _frames(fx, 160, 'same'))
  _fences_intact(ra, 'activations')
  _fences_intact(rx, 'audio')
  torch.testing.assert_close(got[0], want[0], rtol=0, atol=0)
  for g, w in zip(got[1], want[1]):
    torch.testing.assert_close(g, w, rtol=0, atol=0)
  torch.testing.assert_close(got[2], want[2], rtol=0, atol=0)


@gpu
def test_reproducible_and_streams():
  acts = torch.as_tensor(golden.activations(np.random.default_rng(9), 8, 500),
                         dtype=torch.float32, device='cuda')
  m = spectral_ops.PretrainedCREPE(lambda x: x)
  want = m.viterbi_decode(acts)
  s = torch.cuda.Stream()
  with torch.cuda.stream(s):
    got = m.viterbi_decode(acts)
  s.synchronize()
  torch.testing.assert_close(got, want, rtol=0, atol=0)
