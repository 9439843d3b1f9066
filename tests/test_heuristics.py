"""heuristics.py (training/heuristics.py) on the CUDA kernels of csrc/heuristics.cuh:
the binarizers, remove_short, the note table and segment_notes(_batch), against the
float64 restatement tests/heuristics_ref.py, which tests/golden/heuristics.npz pins to
the unmodified reference."""
import os

import numpy as np
import pytest
import torch

from tests import heuristics_ref as ref

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'heuristics.npz'))
TRACKS = (2, 3, 79, 80, 81, 1003)
# decisions closer than this to their threshold may flip between float32 and float64
# statistics, or between NumPy's float32 log and a correctly rounded one
NEAR = 1e-4


def _runs(mask):
  """Run id per frame of the runs of equal values, so that a flip near a threshold is
  charged to the run remove_short spreads it over."""
  m = np.asarray(mask, bool)
  return np.concatenate([[0], np.cumsum(m[1:] != m[:-1])])


def _assert_mask(got, want, margin, near, limit):
  """got == want except in runs (of either) holding a frame within `near` of a threshold;
  at most `limit` such frames."""
  got, want = np.asarray(got, bool), np.asarray(want, bool)
  close = np.asarray(margin) < near
  assert close.sum() <= limit, close.sum()
  bad = got != want
  if bad.any():
    excused = np.zeros_like(bad)
    for runs in (_runs(got), _runs(want)):
      excused |= np.isin(runs, runs[close])
    assert not (bad & ~excused).any(), np.nonzero(bad & ~excused)[0][:10]


# ---- CPU: the restatement against the fixture ----------------------------------------------
@pytest.mark.parametrize('t', TRACKS)
def test_restatement_tracks(t):
  f0, amps = GOLDEN[f'track{t}_f0'][:, 0], GOLDEN[f'track{t}_amps'][:, 0]
  s, ms = ref.strided(f0)
  a, ma = ref.pooled(ref.log32(amps))
  m, mm = ref.midi_heuristic(f0, amps)
  _assert_mask(s, GOLDEN[f'track{t}_strided'], ms, NEAR, 2)
  _assert_mask(a, GOLDEN[f'track{t}_amp_pooled'], ma, NEAR, 2)
  _assert_mask(m, GOLDEN[f'track{t}_midi_heuristic'], mm, NEAR, 2)
  for median in (False, True):
    want = GOLDEN[f'track{t}_{"median" if median else "mean"}_f0_notes']
    got = ref.note_table(m, f0, median)
    assert len(got) == len(want)
    for (start, stop, _, p), row in zip(got, want):
      assert (p, start / 250, stop / 250, 127) == tuple(row)
    assert GOLDEN[f'track{t}_mean_f0_total'] == t / 250


@pytest.mark.parametrize('k', [0, 1])
@pytest.mark.parametrize('pad', ['front', 'center', 'end'])
def test_restatement_pads_and_nonfinite(k, pad):
  amps, f0 = GOLDEN[f'edge{k}_amps'][:, 0], GOLDEN[f'edge{k}_f0'][:, 0]
  a, ma = ref.pooled(ref.log32(amps), 9 + k, 1.5, pad)
  _assert_mask(a, GOLDEN[f'edge{k}_amp_pooled_{pad}'], ma, NEAR, 1)
  s, ms = ref.strided(f0, (3, 6, 2), pad)
  _assert_mask(s, GOLDEN[f'edge{k}_strided_{pad}'], ms, NEAR, 1)


def test_restatement_remove_short_and_even_medians():
  names = [k[len('short_'):-len('_in')] for k in GOLDEN.files
           if k.startswith('short_') and k.endswith('_in')]
  min_samples = {'issue': 3, 'leading_off': 2, 'all_on': 10, 'all_off': 2, 'random': 4}
  for name in names:
    v = GOLDEN[f'short_{name}_in'].astype(bool)
    for glue in (0, 1):
      np.testing.assert_array_equal(ref.remove_short(v, min_samples[name], bool(glue)),
                                    GOLDEN[f'short_{name}_glue{glue}'].astype(bool))
  mask, f0 = GOLDEN['even_mask'].astype(bool), GOLDEN['even_f0'][:, 0]
  for median in (False, True):
    want = GOLDEN[f'even_{"median" if median else "mean"}_f0_notes']
    assert [(p, s / 250, e / 250, 127) for s, e, _, p in ref.note_table(mask, f0, median)] \
        == [tuple(r) for r in want]


def test_fixture_errors():
  assert str(GOLDEN['err_zero_edge']) == 'OverflowError'
  assert str(GOLDEN['err_nan_edge']) == 'ValueError'
  assert str(GOLDEN['err_inf_f0_edge']) == 'OverflowError'
  assert str(GOLDEN['err_t1']) == 'TypeError'
  assert str(GOLDEN['err_power_length']) == 'ValueError'
  f0, amps = GOLDEN['track79_f0'][:, 0], GOLDEN['track79_amps'][:, 0].copy()
  amps[-1] = 0.0
  with pytest.raises(ref.EdgeError):
    ref.midi_heuristic(f0, amps)


def test_torch_helpers_on_cpu():
  from ddsp_b200 import heuristics as h
  np.testing.assert_array_equal(h.pad_for_frame(torch.tensor([-3.7, 1.0, 2.9]), 'center', 4),
                                torch.tensor([-3.0, -3.0, -3.7, 1.0, 2.9, 2.0]))
  with pytest.raises(ValueError):
    h.pad_for_frame(torch.tensor([np.inf, 1.0]), 'front', 3)
  with pytest.raises(ValueError):
    h.pad_for_frame(torch.tensor([1.0]), 'middle', 3)
  c = {'f0_hz': torch.tensor([[1.0], [4.0], [2.0], [3.0], [9.0]]),
       'harmonic': {'controls': {'amplitudes': torch.tensor([[5.0], [1.0], [2.0], [7.0]])}}}
  assert float(h.median_f0(c, 0, 4)) == 2.5          # torch.median would give 2
  assert float(h.median_amps(c, 0, 4)) == 3.5
  assert float(h.mean_f0(c, 1, 3)) == 3.0
  assert torch.isnan(h.median_f0({'f0_hz': torch.tensor([1.0, np.nan])}, 0, 2))
  roll = torch.tensor([[1, 0], [1, 1], [1, 1], [0, 1]])
  np.testing.assert_array_equal(h.get_active_frame_indices(roll), [[0, 0], [1, 1], [2, 2], [0, 3]])
  assert h.get_active_frame_indices(roll.bool()).dtype == torch.bool
  frames = h.window_array(np.arange(10.0), 4, 1.0)
  np.testing.assert_array_equal(frames[0], [0, 0, 1, 2])
  assert frames.shape == (4, 4)
  assert h.DDSP_DEFAULT_FRAME_RATE == 250


# ---- GPU -----------------------------------------------------------------------------------
def _h():
  from ddsp_b200 import heuristics
  return heuristics


def _controls(f0, amps, device='cuda'):
  return {'f0_hz': torch.as_tensor(f0, device=device),
          'harmonic': {'controls': {'amplitudes': torch.as_tensor(amps, device=device)}}}


def _batch(b, t, seed):
  """[B, T, 1] f0 and amplitudes: the fixture's track generator per item."""
  from tests.golden import make_heuristics_golden as mk
  f0, amps = zip(*(mk.track(t, seed + i) for i in range(b)))
  return np.stack(f0), np.stack(amps)


@pytest.mark.gpu
@pytest.mark.parametrize('t', TRACKS)
def test_gpu_tracks_against_fixture(t):
  h = _h()
  f0, amps = GOLDEN[f'track{t}_f0'], GOLDEN[f'track{t}_amps']
  c = _controls(f0, amps)
  _, mm = ref.midi_heuristic(f0[:, 0], amps[:, 0])
  _assert_mask(h.midi_heuristic(c).cpu(), GOLDEN[f'track{t}_midi_heuristic'], mm, NEAR, 2)
  for pick in ('mean_f0', 'median_f0'):
    seq = h.segment_notes(h.midi_heuristic, getattr(h, pick), h.median_amps, c)
    want = GOLDEN[f'track{t}_{pick}_notes']
    assert [(n.pitch, n.start_time, n.end_time, n.velocity) for n in seq.notes] == \
        [tuple(r) for r in want]
    assert seq.total_time == GOLDEN[f'track{t}_{pick}_total']


@pytest.mark.gpu
@pytest.mark.parametrize('b,t', [(1, 2), (3, 81), (64, 1003), (3, 15001), (2, 65536)])
def test_gpu_masks_and_tables_against_restatement(b, t):
  h = _h()
  f0, amps = _batch(b, t, 5000 + t)
  c = _controls(f0, amps)
  mask = h.midi_heuristic(c).cpu().numpy()
  strided = h.strided_freq_change(c).cpu().numpy()
  pooled = h.amp_pooled_outliers(c).cpu().numpy()
  assert mask.shape == strided.shape == pooled.shape == (b, t)
  flips = 0
  for i in range(b):
    s, ms = ref.strided(f0[i, :, 0])
    a, ma = ref.pooled(ref.log32(amps[i, :, 0]))
    m, mm = ref.midi_heuristic(f0[i, :, 0], amps[i, :, 0])
    _assert_mask(strided[i], s, ms, 1e-6, max(2, t // 1000))
    _assert_mask(pooled[i], a, ma, 1e-6, max(2, t // 1000))
    _assert_mask(mask[i], m, mm, 1e-6, max(2, t // 1000))
    flips += int((mask[i] != m).sum())
  # note tables of the kernel's own masks against the restatement's
  for median in (False, True):
    table = h.note_table(torch.as_tensor(mask, device='cuda'), c['f0_hz'],
                         'median' if median else 'mean')
    cap = (t + 1) // 2
    assert table.start.shape == (b, cap) and table.count.shape == (b,)
    start, stop, tf0, pitch, count = (x.cpu().numpy() for x in table)
    for i in range(b):
      want = ref.note_table(mask[i], f0[i, :, 0], median)
      n = int(count[i])
      assert n == len(want)
      np.testing.assert_array_equal(start[i, :n], [w[0] for w in want])
      np.testing.assert_array_equal(stop[i, :n], [w[1] for w in want])
      np.testing.assert_array_equal(tf0[i, :n], np.asarray([w[2] for w in want], np.float32))
      np.testing.assert_array_equal(pitch[i, :n], [w[3] for w in want])
      assert not start[i, n:].any() and not pitch[i, n:].any() and not tf0[i, n:].any()


@pytest.mark.gpu
@pytest.mark.parametrize('k', [0, 1])
@pytest.mark.parametrize('pad', ['front', 'center', 'end'])
def test_gpu_pads_and_nonfinite(k, pad):
  h = _h()
  amps, f0 = GOLDEN[f'edge{k}_amps'], GOLDEN[f'edge{k}_f0']
  a, ma = ref.pooled(ref.log32(amps[:, 0]), 9 + k, 1.5, pad)
  got = h.amp_pooled_outliers(_controls(f0, amps), frame_width=9 + k, num_devs=1.5,
                              pad_mode=pad).cpu()
  _assert_mask(got, a, ma, 1e-6, 1)
  _assert_mask(got, GOLDEN[f'edge{k}_amp_pooled_{pad}'], ma, NEAR, 1)
  s, ms = ref.strided(f0[:, 0], (3, 6, 2), pad)
  got = h.strided_freq_change({'f0_hz': torch.as_tensor(f0, device='cuda')},
                              frame_widths=(3, 6, 2), pad_mode=pad).cpu()
  _assert_mask(got, s, ms, 1e-6, 1)
  _assert_mask(got, GOLDEN[f'edge{k}_strided_{pad}'], ms, NEAR, 1)


@pytest.mark.gpu
def test_gpu_remove_short_and_medians():
  h = _h()
  min_samples = {'issue': 3, 'leading_off': 2, 'all_on': 10, 'all_off': 2, 'random': 4}
  for name, ms in min_samples.items():
    v = GOLDEN[f'short_{name}_in']
    for glue in (0, 1):
      got = h.remove_short(torch.as_tensor(v, device='cuda'), ms, bool(glue))
      np.testing.assert_array_equal(got.cpu(), GOLDEN[f'short_{name}_glue{glue}'].astype(bool))
  mask, f0 = GOLDEN['even_mask'].astype(bool), GOLDEN['even_f0']
  c = {'f0_hz': torch.as_tensor(f0, device='cuda')}
  for pick in ('mean_f0', 'median_f0'):
    # a foreign binarizer with this module's pick: the per-item mask, then the table
    seq = h.segment_notes(lambda _: mask, getattr(h, pick), h.median_amps, c)
    assert [(n.pitch, n.start_time, n.end_time) for n in seq.notes] == \
        [tuple(r[:3]) for r in GOLDEN[f'even_{pick}_notes']]
  # the exact median of long runs, odd and even, with duplicates
  rng = np.random.default_rng(7)
  f = rng.choice(np.float32([100, 200.5, 300, 441, -5, 0]), 40001).astype(np.float32)
  m = np.ones(40001, bool)
  m[20000] = False
  table = h.note_table(torch.as_tensor(m, device='cuda'), torch.as_tensor(f, device='cuda'),
                       'median')
  assert int(table.count) == 2
  np.testing.assert_array_equal(table.f0[:2].cpu(),
                                [ref.median32(f[:20000]), ref.median32(f[20001:])])


@pytest.mark.gpu
def test_gpu_power_against_fixture():
  h = _h()
  audio, f0 = GOLDEN['power_audio'].astype(np.float32), GOLDEN['power_f0']
  c = {'f0_hz': torch.as_tensor(f0, device='cuda'),
       'audio': torch.as_tensor(audio, device='cuda')}
  got = h.midi_heuristic_power(c).cpu().numpy()
  assert got.shape == (201,)
  # float32 power on two platforms: allow a couple of flips at the pooled threshold
  assert (got != GOLDEN['power_midi_heuristic'].astype(bool)).sum() <= 4
  pooled = h.power_pooled_outliers(c).cpu().numpy()
  assert (pooled != GOLDEN['power_pooled'].astype(bool)).sum() <= 4
  with pytest.raises(ValueError, match='must match'):
    h.midi_heuristic_power({'f0_hz': c['f0_hz'][:-1], 'audio': c['audio']})


@pytest.mark.gpu
def test_gpu_segment_notes_batch_fused_and_foreign():
  h = _h()
  b, t = 5, 1003
  f0, amps = _batch(b, t, 6000)
  batch = _controls(f0, amps)
  fused = h.segment_notes_batch(h.midi_heuristic, h.mean_f0, h.median_amps, batch)
  calls = []

  def my_binarize(controls):
    return h.midi_heuristic(controls).cpu().numpy()

  def my_pick(controls, start, stop):
    calls.append((start, stop))
    return np.mean(controls['f0_hz'][start:stop].cpu().numpy().astype(np.float64))

  def my_amps(controls, start, stop):
    calls.append(('amps', start, stop))
    return 0.0

  foreign = h.segment_notes_batch(my_binarize, my_pick, my_amps, batch)
  assert len(fused) == len(foreign) == b
  n_notes = 0
  for x, y in zip(fused, foreign):
    assert [(n.start_time, n.end_time, n.pitch) for n in x.notes] == \
        [(n.start_time, n.end_time, n.pitch) for n in y.notes]
    assert x.total_time == y.total_time == t / 250
    n_notes += len(x.notes)
  assert n_notes > 0 and len(calls) == 2 * n_notes
  mixed = h.segment_notes_batch(h.midi_heuristic, h.median_f0, my_amps, batch)
  assert sum(len(s.notes) for s in mixed) == n_notes


@pytest.mark.gpu
def test_gpu_errors():
  h = _h()
  f0, amps = GOLDEN['track79_f0'], GOLDEN['track79_amps'].copy()
  with pytest.raises(ValueError, match='two frames'):
    h.midi_heuristic(_controls(f0[:1], amps[:1]))
  bad = amps.copy()
  bad[-1] = 0.0
  with pytest.raises(ValueError, match='non-finite'):
    h.midi_heuristic(_controls(f0, bad))
  bad = np.stack([amps, amps])
  bad[1, 0] = np.nan
  with pytest.raises(ValueError, match='item 1'):
    h.amp_pooled_outliers(_controls(np.stack([f0, f0]), bad))
  inf = f0.copy()
  inf[0] = np.inf
  with pytest.raises(ValueError, match='f0_midi'):
    h.strided_freq_change({'f0_hz': torch.as_tensor(inf, device='cuda')})
  with pytest.raises(ValueError, match='pad mode'):
    h.amp_pooled_outliers(_controls(f0, amps), pad_mode='middle')
  with pytest.raises(ValueError):
    h.note_table(torch.ones(5, device='cuda'), torch.ones(6, device='cuda'))
  assert not h.note_heuristic_takes(2**28 + 1) and h.note_heuristic_takes(65536)


@pytest.mark.gpu
def test_gpu_refuses_grad():
  h = _h()
  f0 = torch.full((50, 1), 220.0, device='cuda', requires_grad=True)
  amps = torch.full((50, 1), 0.5, device='cuda')
  with pytest.raises(RuntimeError, match='requires grad'):
    h.midi_heuristic(_controls(f0, amps))
  with pytest.raises(RuntimeError, match='requires grad'):
    h.amp_pooled_outliers(_controls(f0.detach(), amps.requires_grad_()))


@pytest.mark.gpu
def test_gpu_reproducible_streams_graphs_devices():
  h = _h()
  f0, amps = _batch(8, 15001, 7000)
  c = _controls(f0, amps)
  first = h.midi_heuristic(c)
  table = h.note_table(first, c['f0_hz'])
  for _ in range(3):
    assert torch.equal(h.midi_heuristic(c), first)
  s = torch.cuda.Stream()
  with torch.cuda.stream(s):
    other = h.midi_heuristic(c)
    other_table = h.note_table(other, c['f0_hz'], 'mean')
  s.synchronize()
  assert torch.equal(other, first)
  assert all(torch.equal(x, y) for x, y in zip(table, other_table))
  # a CUDA graph around midi_heuristic + note_table
  g = torch.cuda.CUDAGraph()
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    h.note_table(h.midi_heuristic(c), c['f0_hz'])   # warm up on the capture stream
    with torch.cuda.graph(g, stream=side):
      g_mask = h.midi_heuristic(c)
      g_table = h.note_table(g_mask, c['f0_hz'])
  torch.cuda.current_stream().wait_stream(side)
  g.replay()
  torch.cuda.synchronize()
  assert torch.equal(g_mask, first)
  assert all(torch.equal(x, y) for x, y in zip(table, g_table))
  if torch.cuda.device_count() > 1:
    c1 = _controls(f0, amps, 'cuda:1')
    m1 = h.midi_heuristic(c1)
    assert m1.device == torch.device('cuda:1')
    assert torch.equal(m1.cpu(), first.cpu())
    t1 = h.note_table(m1, c1['f0_hz'])
    assert torch.equal(t1.pitch.cpu(), table.pitch.cpu())


@pytest.mark.gpu
def test_gpu_poisoned_and_fenced_memory():
  h = _h()
  f0, amps = _batch(3, 1003, 8000)
  clean = h.midi_heuristic(_controls(f0, amps)).cpu()
  clean_table = [x.cpu() for x in h.note_table(clean.cuda(), torch.as_tensor(f0, device='cuda'))]
  # poison the caching allocator's free blocks, then run on operands fenced by NaN
  junk = torch.full((64 << 20,), -1, dtype=torch.int32, device='cuda')
  del junk
  n = f0.size
  fence = torch.full((3 * n,), float('nan'), device='cuda')
  fence[n:2 * n] = torch.as_tensor(f0.reshape(-1), device='cuda')
  afence = torch.full((3 * n,), float('nan'), device='cuda')
  afence[n:2 * n] = torch.as_tensor(amps.reshape(-1), device='cuda')
  c = _controls(fence[n:2 * n].view(f0.shape), afence[n:2 * n].view(amps.shape))
  got = h.midi_heuristic(c)
  assert torch.equal(got.cpu(), clean)
  table = h.note_table(got, c['f0_hz'])
  assert all(torch.equal(x.cpu(), y) for x, y in zip(table, clean_table))
  assert torch.isnan(fence[:n]).all() and torch.isnan(fence[2 * n:]).all()


@pytest.mark.gpu
def test_gpu_peak_memory():
  h = _h()
  b, t = 32, 15001
  f0, amps = _batch(b, t, 9000)
  c = _controls(f0, amps)
  torch.cuda.synchronize()
  torch.cuda.reset_peak_memory_stats()
  base = torch.cuda.memory_allocated()
  h.segment_notes_batch(h.midi_heuristic, h.median_f0, h.median_amps, c)
  peak = torch.cuda.max_memory_allocated() - base
  # workspace 13 B per frame, the mask, and the 8 B per frame note records
  assert peak <= b * t * 24 + (8 << 20), peak
