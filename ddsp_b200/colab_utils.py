"""The numeric helpers of `ddsp/colab/colab_utils.py` that the tone-transfer notebook
uses to adjust pitch: get_tuning_factor and auto_tune, with the reference's signatures.
They run on `ddsp_b200_tuning_factor` and `ddsp_b200_auto_tune`
(csrc/postprocessing.cuh, DESIGN.md section 3.29).  The notebook's play, record,
upload and plotting helpers are not part of this module.

Inputs are numpy arrays or torch tensors on any device.  get_tuning_factor returns a
numpy float64 scalar, as the reference does; auto_tune a CUDA tensor of the dtype numpy
promotion gives the reference's result.  Forward only: an input that requires grad
raises.
"""
import numpy as np
import torch

from ddsp_b200 import _lib
from ddsp_b200 import core

_SCALES = ['C', 'Db', 'D', 'Eb', 'E', 'F', 'Gb', 'G', 'Ab', 'A', 'Bb', 'B', 'C']


def _tensor(x, name, device=None):
  core._no_grad_path(name, x)
  t = x if torch.is_tensor(x) else torch.as_tensor(np.asarray(x))
  return t.detach().to(device or (t.device if t.is_cuda else core._device()))


def _masked(x, mask_on, name):
  """x[mask_on] flattened row-major, as float64 on x's device."""
  m = _tensor(mask_on, name, x.device)
  if tuple(m.shape) != tuple(x.shape):
    raise ValueError(f'{name}: mask_on {tuple(m.shape)} must have the shape of '
                     f'{tuple(x.shape)}')
  return x[m != 0].to(torch.float64).contiguous()


def _numpy_dtype(x):
  return np.dtype(str(x.dtype).replace('torch.', '')) if torch.is_tensor(x) else x.dtype


@core.on_operands_device
def get_tuning_factor(f0_midi, f0_confidence, mask_on):
  """colab_utils.get_tuning_factor: the offset of np.linspace(-0.5, 0.5, 101) (1-cent
  steps) that minimises the sum of the normalised mean weighted distance of the note
  frames' pitch to the offset chromatic grid and the normalised mean weighted count of
  grid-note changes between successive note frames.  The first factor when there are
  no note frames, or one."""
  f0 = _tensor(f0_midi, 'get_tuning_factor')
  conf = _tensor(f0_confidence, 'get_tuning_factor', f0.device)
  if tuple(conf.shape) != tuple(f0.shape):
    raise ValueError(f'get_tuning_factor: f0_confidence {tuple(conf.shape)} must have the '
                     f'shape of f0_midi {tuple(f0.shape)}')
  f0_on = _masked(f0, mask_on, 'get_tuning_factor')
  conf_on = _masked(conf, mask_on, 'get_tuning_factor')
  tuning_factors = np.linspace(-0.5, 0.5, 101)
  factors = torch.as_tensor(tuning_factors, device=f0.device)
  costs = torch.zeros((2, len(tuning_factors)), dtype=torch.float64, device=f0.device)
  index = torch.zeros((1,), dtype=torch.int32, device=f0.device)
  core._launch('ddsp_b200_tuning_factor', f0_on, conf_on, factors, costs, index,
               f0_on.numel(), len(tuning_factors))
  return tuning_factors[int(index.item())]


@core.on_operands_device
def auto_tune(f0_midi, tuning_factor, mask_on, amount=0.0, chromatic=False):
  """colab_utils.auto_tune: f0_midi - amount * midi_diff.  chromatic: midi_diff is
  (f0_midi - tuning_factor) % 1, less 1 above 0.5.  Otherwise the major scale whose
  notes lie nearest, on average, to the note frames' pitch is inferred (printed with the
  tuning offset in cents, as the reference prints it), and midi_diff is each frame's
  difference to its nearest note of that scale.  Scale mode takes [T] pitch and gives
  float64; chromatic mode any shape, float32 where numpy keeps float32."""
  f0 = _tensor(f0_midi, 'auto_tune')
  t = f0.numel()
  out = torch.zeros(tuple(f0.shape), dtype=torch.float64, device=f0.device)
  fd = f0.to(torch.float64).contiguous()
  if chromatic:
    dtype = np.result_type(_numpy_dtype(f0), tuning_factor, amount)
    f32 = dtype == np.float32
    core._launch('ddsp_b200_auto_tune', fd, None, None, None, out, t, 0,
                 float(tuning_factor), float(amount), 1, _lib.AUTO_TUNE_F32 if f32 else 0)
    return out.to(torch.float32) if f32 else out
  if f0.dim() != 1:
    raise ValueError(f'auto_tune: scale mode takes f0_midi [time], got {tuple(f0.shape)}')
  f0_on = _masked(f0, mask_on, 'auto_tune')
  scale_cost = torch.zeros((12,), dtype=torch.float64, device=f0.device)
  scale_index = torch.zeros((1,), dtype=torch.int32, device=f0.device)
  core._launch('ddsp_b200_auto_tune', fd, f0_on, scale_cost, scale_index, out, t,
               f0_on.numel(), float(tuning_factor), float(amount), 0, 0)
  scale = _SCALES[int(scale_index.item())]
  print('Autotuning... \nInferred key: {}  '
        '\nTuning offset: {} cents'.format(scale, int(tuning_factor * 100)))
  return out
