"""Host-buffer front end of the decoder: numpy / CPU tensors in, CPU audio out.

The reference's `ProcessorGroup.__call__` is fed numpy arrays and hands back a
tensor the caller reads on the host (processors_test.py:35-42, 80-87).  On a GPU
that round trip is PCIe-bound: at the `ae.gin` shapes a batch item is 668 kB of
network outputs in and 256 kB of audio out, against microseconds of synthesis.
`HostDecoder` therefore cuts the batch into chunks and keeps three streams busy
(host->device copies, the two decoder kernels, device->host copies) through
`ddsp_b200_decoder_forward_host` (include/ddsp_b200.h), so a call costs about
max(H2D, compute, D2H) rather than their sum.  Results are identical to
`ProcessorGroup.__call__` on device tensors.
"""
import ctypes

import numpy as np
import torch

from ddsp_b200 import _lib
from ddsp_b200 import core


def _cpulist(text):
  cpus = set()
  for part in text.strip().split(','):
    if not part:
      continue
    lo, _, hi = part.partition('-')
    cpus.update(range(int(lo), int(hi or lo) + 1))
  return cpus


def bind_to_device_numa_node(device=None):
  """Pins the calling thread to the CPUs of the NUMA node the GPU hangs off
  (Linux sysfs), so that page-locked buffers allocated afterwards are first
  touched - and therefore placed - in memory local to the GPU's PCIe root.  On a
  two-socket host a pinned buffer on the far socket costs the host->device copies
  up to half their bandwidth.  Returns the node id, or None when the topology
  cannot be read (nothing is changed then)."""
  import os
  try:
    index = torch.cuda.current_device() if device is None else torch.device(device).index
    prop = torch.cuda.get_device_properties(index)
    bus = '%04x:%02x:%02x.0' % (prop.pci_domain_id, prop.pci_bus_id, prop.pci_device_id)
    node = int(open('/sys/bus/pci/devices/%s/numa_node' % bus).read().strip())
    if node < 0:
      return None
    cpus = _cpulist(open('/sys/devices/system/node/node%d/cpulist' % node).read())
    cpus &= os.sched_getaffinity(0)
    if not cpus:
      return None
    os.sched_setaffinity(0, cpus)
    return node
  except (OSError, ValueError, AttributeError, RuntimeError):
    return None


def pinned_empty(shape):
  """Page-locked float32 host tensor (asynchronous copies need pinned memory)."""
  return torch.empty(tuple(shape), dtype=torch.float32).pin_memory()


def pin(array):
  """Copy of a numpy array / CPU tensor in page-locked memory."""
  t = torch.as_tensor(array, dtype=torch.float32)
  out = pinned_empty(t.shape)
  out.copy_(t)
  return out


def _host_f32(x, name):
  if isinstance(x, np.ndarray):
    x = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
  if not isinstance(x, torch.Tensor):
    x = torch.as_tensor(x, dtype=torch.float32)
  if x.is_cuda:
    raise ValueError(f'HostDecoder input {name!r} is a CUDA tensor; call the '
                     'ProcessorGroup itself for device-resident inputs.')
  if x.dtype != torch.float32 or not x.is_contiguous():
    x = x.to(torch.float32).contiguous()
  return x


class HostDecoder:
  """Runs a decoder `ProcessorGroup` ([Harmonic, FilteredNoise, Add], scale_fn =
  exp_sigmoid - the `ae.gin` DAG) on host buffers through the chunked copy /
  compute pipeline.

    dec = HostDecoder(group, max_batch=32, n_frames=1000, n_harmonics=100,
                      n_bands=65)
    audio = dec(inputs)          # dict of numpy / pinned CPU tensors -> [B, N]
  """

  def __init__(self, group, max_batch, n_frames, n_harmonics, n_bands,
               n_chunks=8, device=None, bind_numa=True):
    pat = group._decoder_pattern()  # pylint: disable=protected-access
    if pat is None:
      raise ValueError('HostDecoder needs the decoder DAG [Harmonic, '
                       'FilteredNoise, Add(harmonic/signal, filtered_noise/signal)].')
    self.harm, self.noise, self.h_keys, self.n_keys = pat
    if (self.harm.scale_fn is not core.exp_sigmoid or
        self.noise.scale_fn is not core.exp_sigmoid):
      raise NotImplementedError('HostDecoder fuses exp_sigmoid scaling; other '
                                'scale_fn values take the device path.')
    if self.harm.amp_resample_method not in core.AMP_METHODS:
      raise NotImplementedError(self.harm.amp_resample_method)
    if len(self.h_keys) != 3 or len(self.n_keys) != 1:
      raise ValueError('HostDecoder: unexpected DAG input keys.')
    self.n_samples = int(self.harm.n_samples)
    self.max_batch, self.n_frames = int(max_batch), int(n_frames)
    self.n_harmonics, self.n_bands = int(n_harmonics), int(n_bands)
    self.n_chunks = int(n_chunks)
    self.device = torch.device('cuda', torch.cuda.current_device()
                               if device is None else torch.device(device).index)
    self._handle = ctypes.c_void_p()
    # Page-locked buffers made after this point (pinned_empty / pin, the `out`
    # of __call__) land on the GPU's own NUMA node; bind_numa=False leaves the
    # calling thread's CPU affinity alone.
    self.numa_node = bind_to_device_numa_node(self.device) if bind_numa else None
    with torch.cuda.device(self.device):
      _lib.check(_lib.load().ddsp_b200_host_pipeline_create(
          ctypes.byref(self._handle), self.max_batch, self.n_frames,
          self.n_harmonics, self.n_bands, self.n_samples, self.n_chunks))

  def close(self):
    if getattr(self, '_handle', None) is not None and self._handle.value:
      _lib.load().ddsp_b200_host_pipeline_destroy(self._handle)
      self._handle = ctypes.c_void_p()

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint: disable=broad-except
      pass

  def __call__(self, inputs, out=None, sync=True):
    """inputs: the ProcessorGroup's inputs dict, values numpy arrays or CPU
    float32 tensors (pinned for full overlap).  Returns the [B, n_samples] audio
    as a pinned CPU tensor (or `out`).  sync=False returns right after queueing;
    the audio is valid once the current stream has completed."""
    outputs = {'inputs': inputs}
    outputs.update(inputs)
    amps, hd, f0 = [_host_f32(core.nested_lookup(k, outputs), k) for k in self.h_keys]
    mags = _host_f32(core.nested_lookup(self.n_keys[0], outputs), self.n_keys[0])
    if hd.dim() != 3 or mags.dim() != 3:
      raise ValueError(f'decoder inputs must be 3-D, got {tuple(hd.shape)} and '
                       f'{tuple(mags.shape)}.')
    b, f, k = hd.shape
    if (tuple(amps.shape) != (b, f, 1) or tuple(f0.shape) != (b, f, 1) or
        tuple(mags.shape[:2]) != (b, f)):
      raise ValueError(
          f'decoder inputs disagree: amps {tuple(amps.shape)}, f0_hz '
          f'{tuple(f0.shape)}, harmonic_distribution {tuple(hd.shape)}, '
          f'noise_magnitudes {tuple(mags.shape)}.')
    if (f, k, mags.shape[2]) != (self.n_frames, self.n_harmonics, self.n_bands):
      raise ValueError(
          f'HostDecoder was built for (F, K, nb) = ({self.n_frames}, '
          f'{self.n_harmonics}, {self.n_bands}), got ({f}, {k}, {mags.shape[2]}).')
    if b > self.max_batch:
      raise ValueError(f'batch {b} exceeds max_batch {self.max_batch}.')
    if out is None:
      out = pinned_empty((b, self.n_samples))
    elif (tuple(out.shape) != (b, self.n_samples) or out.dtype != torch.float32
          or out.is_cuda or not out.is_contiguous()):
      raise ValueError('out must be a contiguous CPU float32 [B, n_samples] tensor.')
    flags = _lib.CTL_SCALE | (_lib.CTL_NYQUIST if self.harm.normalize_below_nyquist
                              else 0)
    with torch.cuda.device(self.device):
      stream = torch.cuda.current_stream()
      _lib.check(_lib.load().ddsp_b200_decoder_forward_host(
          self._handle, amps.data_ptr(), hd.data_ptr(), f0.data_ptr(),
          mags.data_ptr(), int(self.noise.seed), int(self.noise.next_offset()),
          out.data_ptr(), b,
          self.n_chunks, float(self.harm.sample_rate),
          core.AMP_METHODS[self.harm.amp_resample_method], flags,
          int(self.noise.window_size), float(self.noise.initial_bias),
          stream.cuda_stream))
      if sync:
        stream.synchronize()
    return out
