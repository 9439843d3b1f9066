"""Writes tests/golden/routing.npz: outputs of the UNMODIFIED REFERENCE's
core.resample (core.py:573-714), processors.Mix and Crop (processors.py:179-263),
synths.TensorToAudio (synths.py:23-52) and effects.ExpDecayReverb
(effects.py:121-199) on seeded inputs, run on the NumPy TensorFlow shim: float32
(narrow) for the host compositions, float64 (wide) for the restatements of
tests/routing_ref.py.  The reverb's noise is pinned with tf.random.inject_uniform.

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_routing_golden.py          # rewrite the fixture
  python tests/golden/make_routing_golden.py --check  # regenerate in memory and compare

tests/test_routing.py reads the fixture (and regenerates it when the reference is
present); the inputs come from the seeded generators below.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim                        # noqa: E402
from tests.golden.make_golden import _both, compare   # noqa: E402

PATH = os.path.join(HERE, 'routing.npz')

# resample cases whose float32 scale is exact, so TensorFlow's float32 index math and
# the wide shim's float64 one pick the same taps: (F, N, method, add_endpoint)
RESAMPLE = [(8, 64, 'linear', True), (5, 17, 'linear', False), (64, 8, 'linear', True),
            (9, 3, 'linear', False), (8, 64, 'nearest', True), (5, 17, 'nearest', False),
            (64, 16, 'nearest', True), (8, 64, 'cubic', True), (5, 17, 'cubic', False),
            (32, 8, 'cubic', True), (8, 64, 'window', True), (5, 64, 'window', False),
            (1, 16, 'window', True), (1, 8, 'linear', True), (4, 1, 'cubic', True)]
# Mix cases: (B, N, C, mix frames)
MIX = [(2, 64, 3, 8), (3, 100, 1, 100), (2, 128, 2, 1)]
# Crop cases: (frame_size, crop_location, audio rank)
CROP = [(320, 'back', 2), (640, 'front', 3), (960, 'center', 2), (7, 'center', 3),
        (1, 'back', 2), (0, 'center', 2), (1, 'front', 3)]
CROP_N = 2000
# ExpDecayReverb cases: (trainable, add_dry, reverb_length, N)
REVERB = [(False, True, 300, 1000), (False, False, 300, 1000), (True, True, 300, 1000),
          (True, False, 1500, 1000), (False, True, 2, 64), (True, True, 3, 64)]
REVERB_B = 2


def resample_input(case, i):
  F = case[0]
  return np.random.default_rng(600 + i).standard_normal((2, F, 3)).astype(np.float32)


def mix_inputs(i):
  B, N, C, F = MIX[i]
  rng = np.random.default_rng(700 + i)
  return (rng.standard_normal((B, N, C)).astype(np.float32),
          rng.standard_normal((B, N, C)).astype(np.float32),
          (3.0 * rng.standard_normal((B, F, 1))).astype(np.float32))


def crop_input(i):
  rank = CROP[i][2]
  shape = (2, CROP_N, 2) if rank == 3 else (2, CROP_N)
  return np.random.default_rng(800 + i).standard_normal(shape).astype(np.float32)


def reverb_inputs(i):
  """Seeded audio [B, N], raw gain and decay ([B, 1], or the learned [1] values
  2.0 / 4.0 when trainable) and the [1, L] noise row of REVERB case i."""
  trainable, _, L, N = REVERB[i]
  rng = np.random.default_rng(900 + i)
  audio = rng.standard_normal((REVERB_B, N)).astype(np.float32)
  gain = rng.standard_normal((REVERB_B, 1)).astype(np.float32)
  decay = rng.uniform(-2.0, 6.0, (REVERB_B, 1)).astype(np.float32)
  if trainable:
    gain, decay = np.full((1, 1), 2.0, np.float32), np.full((1, 1), 4.0, np.float32)
  noise = rng.uniform(-1.0, 1.0, (1, L)).astype(np.float32)
  return audio, gain, decay, noise


def routing():
  ddsp = ref_on_shim.load()
  tf = ref_on_shim.tf()
  out = {}
  for i, case in enumerate(RESAMPLE):
    F, N, method, add_endpoint = case
    x = resample_input(case, i)
    _, w = _both(lambda: ddsp.core.resample(tf.convert_to_tensor(x), N, method=method,
                                            add_endpoint=add_endpoint))
    out['resample_wide_%02d' % i] = np.asarray(w, np.float64)
  for i in range(len(MIX)):
    s1, s2, logits = mix_inputs(i)
    mix = ddsp.processors.Mix()
    n, w = _both(lambda: mix(s1, s2, logits))
    out['mix_f32_%d' % i], out['mix_wide_%d' % i] = n, np.asarray(w, np.float64)
    level = np.random.default_rng(750 + i).uniform(0.0, 1.0, (s1.shape[0], s1.shape[1], 1))
    level = level.astype(np.float32)
    _, w = _both(lambda: mix.get_signal(*(tf.convert_to_tensor(v) for v in (s1, s2, level))))
    out['mix_signal_wide_%d' % i] = np.asarray(w, np.float64)
  for i, (frame, where, _) in enumerate(CROP):
    out['crop_%d' % i] = ref_on_shim.to_numpy(
        ddsp.processors.Crop(frame_size=frame, crop_location=where)(crop_input(i)))
  samples = np.random.default_rng(850).standard_normal((2, 100, 1)).astype(np.float32)
  out['tensor_to_audio'] = ref_on_shim.to_numpy(ddsp.synths.TensorToAudio()(samples))
  for i, (trainable, add_dry, L, _) in enumerate(REVERB):
    audio, gain, decay, noise = reverb_inputs(i)

    def run():
      tf.random.inject_uniform(noise)
      r = ddsp.effects.ExpDecayReverb(trainable=trainable, reverb_length=L,
                                      add_dry=add_dry)
      if trainable:
        r.build(None)
        return r(audio)
      return r(audio, gain, decay)
    n, w = _both(run)
    out['reverb_f32_%d' % i], out['reverb_wide_%d' % i] = n, np.asarray(w, np.float64)
    tf.random.inject_uniform(noise)
    r = ddsp.effects.ExpDecayReverb(reverb_length=L)
    tf.set_wide(True)
    try:
      ir = ref_on_shim.to_numpy(r._get_ir(tf.convert_to_tensor(gain.astype(np.float64)),
                                          tf.convert_to_tensor(decay.astype(np.float64))))
    finally:
      tf.set_wide(False)
    out['ir_wide_%d' % i] = np.asarray(ir, np.float64)
  return out


if __name__ == '__main__':
  got = routing()
  if '--check' in sys.argv:
    compare('routing', got, np.load(PATH))
    print('ok    routing')
  else:
    np.savez_compressed(PATH, **got)
    print('wrote routing %.0f kB' % (os.path.getsize(PATH) / 1e3))
