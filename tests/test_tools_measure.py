"""The timing scripts tools/*_time.py measure through one module, tools/measure.py: it
alone reads the card, times with CUDA events, sizes input rings past L2, reads peak
memory and holds the data-sheet peaks, and no script borrows another script's helpers."""
import glob
import json
import os
import re

from tools import measure

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEASURE_ONLY = ('torch.cuda.Event(', 'nvidia-smi', 'reset_peak_memory_stats', 'L2_cache_size',
                '3.35e12', '3350', '67e12')


def _scripts():
  """{file name: source} of every timing script."""
  out = {}
  for path in sorted(glob.glob(os.path.join(ROOT, 'tools', '*_time.py'))):
    with open(path) as f:
      out[os.path.basename(path)] = f.read()
  return out


def test_measurement_lives_in_measure_only():
  with open(os.path.join(ROOT, 'tools', 'measure.py')) as f:
    module = f.read()
  scripts = _scripts()
  assert len(scripts) >= 24
  for needle in MEASURE_ONLY:
    if needle != '3350':
      assert needle in module, needle
    assert [name for name, src in scripts.items() if needle in src] == [], needle


def test_no_script_imports_another_script():
  for name, src in _scripts().items():
    assert not re.search(r'\b(from|import)\s+tools\.\w+_time\b', src), name


def test_ring_len_exceeds_twice_l2(monkeypatch):
  monkeypatch.setattr(measure, 'l2_bytes', lambda: 50 << 20)
  assert measure.ring_len(1 << 20) == 101
  assert measure.ring_len(25 << 20) == 5
  assert measure.ring_len(30 << 20) == 5
  assert measure.ring_len(1 << 30) == 2


def test_alternate_takes_the_median_of_its_rounds(monkeypatch):
  times = iter([5.0, 50.0, 1.0, 10.0, 3.0, 30.0, 4.0, 40.0])
  calls = []

  def event_ms(fn, iters, warmup):
    calls.append((fn, iters, warmup))
    return next(times)

  monkeypatch.setattr(measure, 'event_ms', event_ms)
  got = measure.alternate({'a': 'fa', 'b': 'fb'}, 4, {'a': 20, 'b': 5}, 3)
  assert got == {'a': 3.5, 'b': 35.0}
  assert calls == [('fa', 20, 3), ('fb', 5, 3)] * 4
  times = iter([2.0, 1.0, 3.0])
  assert measure.alternate({'a': 'fa'}, 3, 10, 1) == {'a': 2.0}


def test_append_rows_appends_json_lines(tmp_path):
  path = tmp_path / 'new_dir' / 'rows.jsonl'
  measure.append_rows(str(path), [{'x': 1}])
  measure.append_rows(str(path), [{'x': 2, 'card': {'device': 'd'}}])
  assert [json.loads(line) for line in path.read_text().splitlines()] == [
      {'x': 1}, {'x': 2, 'card': {'device': 'd'}}]
