"""core._launch, the one path from Python to the library's launching entry points:
what reaches the C function for each kind of argument, the device and stream it runs
on, and the errors it raises before anything is launched."""
import pytest
import torch

from ddsp_b200 import _lib, core


class Recorder:
  """Stands in for the loaded library: records every name looked up on it, and every
  call with the current device and its arguments, and returns 0."""

  def __init__(self):
    self.looked_up, self.calls = [], []

  def __getattr__(self, name):
    self.looked_up.append(name)

    def call(*args):
      self.calls.append((name, torch.cuda.current_device(), args))
      return 0
    return call


@pytest.fixture
def recorder(monkeypatch):
  rec = Recorder()
  monkeypatch.setattr(_lib, 'load', lambda: rec)
  return rec


def test_cpu_tensor_raises_before_the_library_is_touched(recorder):
  with pytest.raises(ValueError, match=r'ddsp_b200_add: argument 0 is on cpu'):
    core._launch('ddsp_b200_add', torch.zeros(4), torch.zeros(4), torch.zeros(4), 4)
  assert recorder.looked_up == []


def test_non_contiguous_tensor_raises_before_the_library_is_touched(recorder):
  with pytest.raises(ValueError, match=r'ddsp_b200_add: argument 0 is not contiguous'):
    core._launch('ddsp_b200_add', torch.zeros(4, 4).t(), torch.zeros(16),
                 torch.zeros(16), 16)
  assert recorder.looked_up == []


@pytest.mark.gpu
def test_none_arrives_as_null_and_tensors_as_their_address(recorder):
  audio, phase, out = (torch.zeros((2, 64), device='cuda') for _ in range(3))
  core._launch('ddsp_b200_mod_delay_forward', audio, phase, None, out, 2, 64, 100, 1.0,
               0.0, 0)
  (name, _, args), = recorder.calls
  assert name == 'ddsp_b200_mod_delay_forward'
  assert args[:-1] == (audio.data_ptr(), phase.data_ptr(), 0, out.data_ptr(), 2, 64, 100,
                       1.0, 0.0, 0)


@pytest.mark.gpu
def test_last_argument_is_the_current_side_stream(recorder):
  dev = torch.cuda.current_device()
  a = torch.zeros(8, device='cuda')
  side = torch.cuda.Stream()
  with torch.cuda.stream(side):
    core._launch('ddsp_b200_add', a, a, a, 8)
  (_, device, args), = recorder.calls
  assert device == dev
  assert args[-1] == side.cuda_stream != torch.cuda.current_stream().cuda_stream


def needs_two_devices():
  if torch.cuda.device_count() < 2:
    pytest.skip('needs two CUDA devices')


@pytest.mark.gpu
def test_launch_goes_to_the_operands_device_and_its_current_stream(recorder):
  needs_two_devices()
  a = torch.zeros(8, device='cuda:1')
  side = torch.cuda.Stream('cuda:1')
  with torch.cuda.stream(side), torch.cuda.device(0):
    core._launch('ddsp_b200_add', a, a, a, 8)
    assert torch.cuda.current_device() == 0
  (_, device, args), = recorder.calls
  assert device == 1
  assert args[-1] == side.cuda_stream


@pytest.mark.gpu
def test_operands_on_two_devices_raise_and_launch_nothing():
  needs_two_devices()
  lib = _lib.load()
  a, out = torch.zeros(8, device='cuda:0'), torch.zeros(8, device='cuda:0')
  b = torch.zeros(8, device='cuda:1')
  before = lib.ddsp_b200_launch_count()
  with pytest.raises(ValueError, match='different devices'):
    core._launch('ddsp_b200_add', a, b, out, 8)
  assert lib.ddsp_b200_launch_count() == before
