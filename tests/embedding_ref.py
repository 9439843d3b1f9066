"""Float64 restatement of losses.PretrainedCREPE (losses.py:424-486) around its network,
and of EmbeddingLoss (losses.py:356-388): frame_audio, its gradient in closed form,
call's reshape and the embedding loss.  Pinned to the unmodified reference by
tests/golden/embedding_loss.npz (tests/golden/make_embedding_loss_golden.py).

`frame_audio` is torch float64 on the CPU, so that torch.autograd of it is the
reference gradient the CUDA backward is held to; it follows tf.nn.moments, whose
variance stops the gradient of the mean.  The stub networks are the ones the fixture
was made with.
"""
import numpy as np
import torch

FRAME = 1024
EPS = 1e-5
STUB_SHAPE = (4, 3)      # the stub network's activation per frame


def n_frames(n, hop, center):
  padded = n + (FRAME if center else 0)
  return 1 + (padded - FRAME) // hop if padded >= FRAME else 0


def frame_audio(audio, hop, center=True):
  """frames [B, F, 1024] of audio [B, N] (a float64 tensor, or anything numpy takes):
  512 zeros on both sides when `center`, tf.signal.frame with pad_end=False, then
  (x - mean) / (var**0.5 + 1e-5) per frame.  Differentiable in a tensor's values."""
  x = audio if torch.is_tensor(audio) else torch.as_tensor(np.asarray(audio, np.float64))
  x = x.to(torch.float64)
  if center:
    x = torch.nn.functional.pad(x, (FRAME // 2, FRAME // 2))
  f = n_frames(x.shape[-1], hop, False)
  if f == 0:
    return x.new_zeros((x.shape[0], 0, FRAME))
  frames = x.unfold(-1, FRAME, hop)[:, :f]
  mean = frames.mean(-1, keepdim=True)
  var = ((frames - mean.detach()) ** 2).mean(-1, keepdim=True)
  return (frames - mean) / (var ** 0.5 + EPS)


def frame_audio_grad(audio, grad_frames, hop, center=True):
  """d audio [B, N] for d frames [B, F, 1024], in closed form (numpy float64):
  dx_k = (g_k - gbar) / (s + eps) - c (x_k - mu) / ((s + eps)^2 1024 s) per frame,
  summed over the frames covering each sample."""
  x = np.asarray(audio, np.float64)
  g = np.asarray(grad_frames, np.float64)
  b, n = x.shape
  pad = FRAME // 2 if center else 0
  xp = np.pad(x, ((0, 0), (pad, pad)))
  out = np.zeros_like(xp)
  idx = np.arange(FRAME)
  with np.errstate(invalid='ignore', divide='ignore'):
    for f in range(g.shape[1]):
      fr = xp[:, f * hop + idx]
      mu = fr.mean(-1, keepdims=True)
      s = np.sqrt(((fr - mu) ** 2).mean(-1, keepdims=True))
      gf = g[:, f]
      c = (gf * (fr - mu)).sum(-1, keepdims=True)
      d = s + EPS
      out[:, f * hop + idx] += (gf - gf.mean(-1, keepdims=True)) / d - c * (fr - mu) / (
          d * d * FRAME * s)
  return out[:, pad:pad + n]


def stub_weights():
  """The stub network's projection [1024, 12]."""
  return np.random.default_rng(4100).normal(size=(FRAME, int(np.prod(STUB_SHAPE)))) / 32.0


def stub_activations(frames, unit=False):
  """The stub network: frames [M, 1024] -> tanh(frames W) as [M, 4, 3]; with `unit`, each
  frame's 12 values are scaled to unit length (the COSINE case, whose embedding is that
  frame's row of call's [B, n_frames, 12])."""
  fr = np.asarray(frames, np.float64)
  a = np.tanh(fr @ stub_weights())
  if unit:
    a = a / np.linalg.norm(a, axis=-1, keepdims=True)
  return a.reshape((fr.shape[0],) + STUB_SHAPE)


def unit_stub_activations(frames):
  return stub_activations(frames, unit=True)


def call(audio, activations=stub_activations):
  """PretrainedCREPE.call: frame_audio at hop 1024 with centring, the network on
  [-1, 1024], the result as [B, n_frames, -1]."""
  frames = frame_audio(audio, 1024, True).numpy()
  b, f = frames.shape[:2]
  return np.asarray(activations(frames.reshape(-1, FRAME))).reshape(b, f, -1)


def cosine_distance(labels, predictions, axis=-1):
  """tf.compat.v1.losses.cosine_distance with weights 1.0 (its default reduction,
  SUM_BY_NONZERO_WEIGHTS): mean(1 - sum(labels * predictions, axis)).  It assumes unit
  vectors, on which it is 1 - the cosine similarity."""
  return np.mean(1.0 - np.sum(np.asarray(labels) * np.asarray(predictions), axis=axis))


def embedding_loss(target_audio, audio, weight, loss_type):
  """EmbeddingLoss.call with a PretrainedCREPE on the stub network as pretrained_model
  (the unit-length stub for COSINE)."""
  if not weight > 0.0:
    return 0.0
  activations = unit_stub_activations if loss_type == 'COSINE' else stub_activations
  t, v = call(target_audio, activations), call(audio, activations)
  if loss_type == 'L1':
    return weight * np.mean(np.abs(t - v))
  if loss_type == 'L2':
    return weight * np.mean((t - v) ** 2)
  return weight * cosine_distance(t, v)
