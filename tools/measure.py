"""How the timing scripts measure on the GPU: the card record, CUDA-event timing of calls
and of the stages of a step, input rings larger than the L2 cache, alternated rounds with their median, peak memory,
data-sheet peaks and JSON-line results.  Importing this module does not initialise
CUDA, so a script's CPU-only paths still run without a GPU."""
import json
import math
import os
import statistics
import subprocess

import torch

# NVIDIA's H100 SXM data sheet, for a card allowed up to 700 W: HBM3 bandwidth and dense
# FP32 rate.  A card set to a lower power limit may not reach them.
HBM_BYTES_PER_S = 3.35e12
FP32_FLOPS_PER_S = 67e12


def card():
  """The current device's name, and nvidia-smi's name and power limit for it ('' when the
  query fails), so every measured number carries what it was measured on."""
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader',
                        '-i', str(torch.cuda.current_device())],
                       capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    q = ''
  return {'device': torch.cuda.get_device_name(), 'nvidia_smi': q}


def require_cuda(script):
  """Exits with one message, instead of a traceback, when there is no CUDA device."""
  if not torch.cuda.is_available():
    raise SystemExit('%s needs a CUDA device' % script)


def event_ms(fn, iters, warmup, inputs=None):
  """Mean ms per call of `iters` calls of fn between two CUDA events, after `warmup`
  untimed calls and a synchronise.  With `inputs`, the i-th warm-up call and the i-th
  timed call are both fn(inputs[i % len(inputs)])."""
  def call(i):
    return fn() if inputs is None else fn(inputs[i % len(inputs)])

  for i in range(warmup):
    call(i)
  torch.cuda.synchronize()
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for i in range(iters):
    call(i)
  stop.record()
  torch.cuda.synchronize()
  return start.elapsed_time(stop) / iters


class StageEvents:
  """Device time of the named stages of a step: begin(name) and end(name) record CUDA
  events around a stage (a stage may recur within a step), and mean_ms(steps) gives
  {name: ms per step} over every stage recorded since the last clear()."""

  def __init__(self):
    self._open, self._log = {}, []

  def _record(self):
    event = torch.cuda.Event(enable_timing=True)
    event.record()
    return event

  def begin(self, name):
    self._open[name] = self._record()

  def end(self, name):
    self._log.append((name, self._open.pop(name), self._record()))

  def clear(self):
    self._open, self._log = {}, []

  def mean_ms(self, steps):
    torch.cuda.synchronize()
    totals = {}
    for name, start, stop in self._log:
      totals[name] = totals.get(name, 0.0) + start.elapsed_time(stop) / steps
    return totals


def l2_bytes():
  return torch.cuda.get_device_properties(torch.cuda.current_device()).L2_cache_size


def ring_len(set_bytes):
  """How many input sets of `set_bytes` bytes make a ring larger than twice the L2 cache,
  so that no call finds its operands in L2 from an earlier call."""
  return max(2, math.ceil(2 * l2_bytes() / set_bytes) + 1)


def peak_bytes(fn):
  """Bytes of device memory fn's call allocates at its peak above what was allocated
  before it."""
  torch.cuda.synchronize()
  base = torch.cuda.memory_allocated()
  torch.cuda.reset_peak_memory_stats()
  fn()
  torch.cuda.synchronize()
  return torch.cuda.max_memory_allocated() - base


def alternate(fns, rounds, iters, warmup):
  """{name: median over `rounds` of event_ms} for `fns` ({name: fn}).  Each round times
  every fn once, in order, so that a change in the card's state during the run reaches
  all of them.  `iters` and `warmup` are one count for every fn or a {name: count}."""
  def count(c, name):
    return c[name] if isinstance(c, dict) else c

  times = {name: [] for name in fns}
  for _ in range(rounds):
    for name, fn in fns.items():
      times[name].append(event_ms(fn, count(iters, name), count(warmup, name)))
  return {name: statistics.median(t) for name, t in times.items()}


def append_rows(path, rows):
  """Appends one JSON line per row to `path`, creating its directory."""
  os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
  with open(path, 'a') as f:
    for row in rows:
      f.write(json.dumps(row) + '\n')
