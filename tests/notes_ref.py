"""Float64 torch restatement of the reference's note functions (training/nn.py:375-557),
step for step: the edges, the padded cumulative sum, the one-hot comparison against
range(max_regions), and the [batch, time, notes, dims] products of get_note_moments and
pool_over_notes.  Its gradients are torch autograd's.  Pinned to the unmodified reference
by tests/golden/notes.npz."""
import numpy as np
import torch


def t64(x):
  if torch.is_tensor(x):
    return x if x.dtype == torch.float64 else x.detach().cpu().double()
  return torch.as_tensor(np.asarray(x, np.float64))


def _safe_divide(a, b, eps=1e-7):
  return a / torch.where(b == 0.0, torch.full_like(b, eps), b)


def _one_hot(edge_idx, max_regions):
  return (edge_idx[..., None] == torch.arange(max_regions, device=edge_idx.device)).double()


def get_note_mask(q_pitch, max_regions=100, note_on_only=True):
  q = t64(q_pitch)
  if q.dim() == 3:
    q = q[:, :, 0]
  edges = torch.abs(q[:, 1:] - q[:, :-1]) > 0
  edges = edges[:, :-1]
  b = q.shape[0]
  edges = torch.cat([torch.ones((b, 1), dtype=torch.bool, device=q.device), edges,
                     torch.zeros((b, 1), dtype=torch.bool, device=q.device)], dim=1)
  mask = _one_hot(torch.cumsum(edges.long(), dim=1) - 1, max_regions)
  if note_on_only:
    pitches = get_note_moments(q, mask, return_std=False)
    mask = mask * (pitches > 0.0).double()[:, None, :]
  return mask


def get_note_mask_from_onset(q_pitch, onset, max_regions=100, note_on_only=True):
  q, on = t64(q_pitch), t64(onset)
  if q.dim() == 3:
    q = q[:, :, 0]
  if on.dim() == 3:
    on = on[:, :, 0]
  edges = torch.cat([torch.ones_like(on[:, :1]), on[:, 1:]], dim=1).to(torch.int32)
  mask = _one_hot(torch.cumsum(edges.long(), dim=1) - 1, max_regions)
  if note_on_only:
    mask = mask * (q > 0.0).double()[:, :, None]
  return mask


def get_note_moments(x, note_mask, return_std=True):
  x, m = t64(x), t64(note_mask)
  is_2d = x.dim() == 2
  if is_2d:
    x = x[:, :, None]
  md = m[..., None]
  lengths = torch.sum(md, dim=1)
  mean = _safe_divide(torch.sum(x[:, :, None, :] * md, dim=1), lengths)
  num = torch.sum(((x[:, :, None, :] - mean[:, None, :, :]) * md)**2.0, dim=1)
  std = _safe_divide(num, lengths)**0.5
  if is_2d:
    mean, std = mean[:, :, 0], std[:, :, 0]
  return (mean, std) if return_std else mean


def pool_over_notes(x, note_mask, return_std=True):
  m = t64(note_mask)
  mean, std = get_note_moments(x, m, return_std=True)
  pooled_mean = torch.sum(mean[:, None] * m[..., None], dim=2)
  if not return_std:
    return pooled_mean
  return pooled_mean, torch.sum(std[:, None] * m[..., None], dim=2)


def get_note_lengths(note_mask):
  return torch.sum(t64(note_mask), dim=1)


def get_short_note_loss_mask(note_mask, note_lengths, note_pitches, min_length=40):
  short = ((t64(note_lengths) < min_length) & (t64(note_pitches) > 0.0)).double()
  return torch.sum(t64(note_mask) * short[:, None, :], dim=-1)
