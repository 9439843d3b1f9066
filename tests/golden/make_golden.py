"""Writes tests/golden/*.npz: outputs of the UNMODIFIED REFERENCE (magenta/ddsp)
on seeded inputs, for the decoder path.

How: the reference package is imported as it lies and run on the NumPy stand-in
for its TensorFlow primitives (oracle/tf_shim via oracle/ref_on_shim.py) - twice:
"narrow" (float32, the reference's own arithmetic incl. its sequential float32
phase cumsum) and "wide" (the same reference code with every float32 widened to
float64: the exact value of the reference's formulae, which is what the 1e-4
parity gate is measured against; BASELINE.md section 5 gives the distance between
the two - the reference's own phase-accumulation error).

Needs the reference sources (oracle/ref_on_shim.py finds them through
DDSP_REFERENCE_ROOT), so it runs only where they are checked out:

  python tests/golden/make_golden.py          # rewrite every fixture
  python tests/golden/make_golden.py --check  # regenerate in memory and compare
  python -m oracle.run_reference_tests        # the reference's own unit tests on the shim

The tests read the fixtures and never the reference: tests/test_reference_pin.py
and tests/test_reference_fuzz.py (oracle vs fixtures), tests/test_effects.py
(FilteredNoiseReverb composition vs fixture) and tests/test_gpu_golden.py (CUDA
path vs fixtures).  Inputs are
regenerated from their seeds by tests/util.synth_inputs; an input checksum in
every fixture guards against generator drift.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_on_shim               # noqa: E402
from tests.util import synth_inputs          # noqa: E402


def checksum(inp):
  return np.float64(sum(float(np.asarray(v, np.float64).sum()) * (i + 1)
                        for i, v in enumerate(inp[k] for k in sorted(inp))))


def _both(fn):
  """fn() under the narrow and the wide shim -> (narrow, wide) numpy results."""
  tf = ref_on_shim.tf()
  out = []
  for wide in (False, True):
    tf.set_wide(wide)
    try:
      out.append(ref_on_shim.to_numpy(fn()))
    finally:
      tf.set_wide(False)
  return out


def _nyquist_margin(ddsp, inp, n_samples, k, sample_rate=16000):
  """Smallest |f_k(t) - sr/2| of the float32 frequency envelopes: the fixture is
  only meaningful if no oscillator sits within an ulp of the Nyquist decision
  (then narrow and wide would disagree by a whole oscillator at that sample)."""
  hf = ddsp.core.get_harmonic_frequencies(inp['f0_hz'], k)
  fe = ddsp.core.resample(hf, n_samples).numpy().astype(np.float64)
  return float(np.abs(fe - sample_rate / 2.0).min())


def c1_harmonic():
  """BASELINE.json configs[0]: Harmonic only, B=1, 16000 samples, 64 harmonics,
  250 frames (synths.Harmonic defaults: window resampling, Nyquist normalise)."""
  ddsp = ref_on_shim.load()
  seed = 101
  inp = synth_inputs(1, 250, 64, 65, 16000, seed=seed)
  args = (inp['amps'], inp['harmonic_distribution'], inp['f0_hz'])
  assert _nyquist_margin(ddsp, inp, 16000, 64) > 1e-2

  def run(angular):
    h = ddsp.synths.Harmonic(n_samples=16000, use_angular_cumsum=angular)
    return h(*args, return_outputs_dict=True)

  n0, w0 = _both(lambda: run(False))
  n1, _ = _both(lambda: run(True))
  return dict(
      seed=seed, input_checksum=checksum(inp),
      amplitudes=n0['controls']['amplitudes'],
      harmonic_distribution=n0['controls']['harmonic_distribution'],
      audio_ref_f32_cumsum=n0['signal'], audio_ref_f32_angular=n1['signal'],
      audio_ref_wide=w0['signal'].astype(np.float64))


def decoder_small():
  """The ae.gin DAG (ae.gin:47-72) through the reference's ProcessorGroup from raw
  network outputs, B=2, F=25, N=1600, K=100, 65 bands, injected noise."""
  ddsp = ref_on_shim.load()
  tf = ref_on_shim.tf()
  seed = 202
  B, F, K, nb, N = 2, 25, 100, 65, 1600
  inp = synth_inputs(B, F, K, nb, N, seed=seed)
  assert _nyquist_margin(ddsp, inp, N, K) > 1e-2

  def run():
    harm = ddsp.synths.Harmonic(n_samples=N, sample_rate=16000)
    noise = ddsp.synths.FilteredNoise(n_samples=N, window_size=0)
    group = ddsp.processors.ProcessorGroup(dag=[
        (harm, ['amps', 'harmonic_distribution', 'f0_hz']),
        (noise, ['noise_magnitudes']),
        (ddsp.processors.Add(), ['filtered_noise/signal', 'harmonic/signal'])])
    tf.random.inject_uniform(inp['noise'])
    feats = {k: inp[k] for k in ('amps', 'harmonic_distribution', 'f0_hz',
                                 'noise_magnitudes')}
    return group.get_controls(feats)

  n, w = _both(run)
  out = dict(seed=seed, input_checksum=checksum(inp))
  for tag, o in (('f32', n), ('wide', w)):
    out['harmonic_' + tag] = o['harmonic']['signal']
    out['filtered_noise_' + tag] = o['filtered_noise']['signal']
    out['audio_' + tag] = o['out']['signal']
  out['magnitudes'] = n['filtered_noise']['controls']['magnitudes']
  out['harmonic_distribution'] = n['harmonic']['controls']['harmonic_distribution']
  out['amplitudes'] = n['harmonic']['controls']['amplitudes']
  return out


def c2_item():
  """One batch item at the configs[1..4] shapes (F=1000, K=100, 65 bands, 64000
  samples): the reference's harmonic and filtered-noise signals, wide; stored as
  float32 (rounding 6e-8, far inside the 1e-4 gate) to keep the file small."""
  ddsp = ref_on_shim.load()
  tf = ref_on_shim.tf()
  seed = 303
  inp = synth_inputs(1, 1000, 100, 65, 64000, seed=seed)
  assert _nyquist_margin(ddsp, inp, 64000, 100) > 1e-2

  def run():
    harm = ddsp.synths.Harmonic(n_samples=64000, sample_rate=16000)
    noise = ddsp.synths.FilteredNoise(n_samples=64000, window_size=0)
    tf.random.inject_uniform(inp['noise'])
    return {'h': harm(inp['amps'], inp['harmonic_distribution'], inp['f0_hz']),
            'n': noise(inp['noise_magnitudes'])}

  n, w = _both(run)
  return dict(seed=seed, input_checksum=checksum(inp),
              harmonic_wide=w['h'].astype(np.float32),
              filtered_noise_wide=w['n'].astype(np.float32),
              # the reference's own float32 result, decimated: documents its
              # phase-accumulation error at 64000 samples
              harmonic_f32_every16=n['h'][:, ::16].astype(np.float32))


def harmonic_shifts():
  """core.harmonic_synthesis with harmonic_shifts (core.py:1084-1093), 'linear'
  and 'window' amplitudes, B=2, F=50, K=20, N=3200."""
  ddsp = ref_on_shim.load()
  seed = 404
  B, F, K, N = 2, 50, 20, 3200
  inp = synth_inputs(B, F, K, 65, N, seed=seed, f0_lo=100.0, f0_hi=500.0)
  rng = np.random.default_rng(seed)
  shifts = (0.02 * rng.standard_normal((B, F, K))).astype(np.float32)
  amps = np.abs(inp['amps']) * 0.5
  hd = np.abs(inp['harmonic_distribution'])
  hd = (hd / hd.sum(-1, keepdims=True)).astype(np.float32)
  out = dict(seed=seed, shifts=shifts, amplitudes=amps.astype(np.float32),
             harmonic_distribution=hd, f0_hz=inp['f0_hz'])
  for method in ('window', 'linear'):
    n, w = _both(lambda: ddsp.core.harmonic_synthesis(
        inp['f0_hz'], amps, harmonic_shifts=shifts, harmonic_distribution=hd,
        n_samples=N, sample_rate=16000, amp_resample_method=method))
    out['audio_f32_' + method] = n
    out['audio_wide_' + method] = w.astype(np.float64)
  return out


def resample_methods():
  """core.resample (core.py:573-642) for every method, both add_endpoint values,
  3-D and 4-D inputs, up- and down-sampling."""
  ddsp = ref_on_shim.load()
  rng = np.random.default_rng(505)
  x3 = rng.standard_normal((2, 10, 3)).astype(np.float32)
  x4 = rng.standard_normal((2, 10, 4, 3)).astype(np.float32)
  out = dict(x3=x3, x4=x4)
  for method in ('nearest', 'linear', 'cubic', 'window'):
    for ep in (True, False):
      n_up = 90 if not ep else 80      # divisible by 9 intervals / 10 frames
      n, w = _both(lambda: ddsp.core.resample(x3, n_up, method=method, add_endpoint=ep))
      out['up3_%s_%d' % (method, ep)] = n
      out['up3w_%s_%d' % (method, ep)] = w
      if method != 'window':
        out['down3_%s_%d' % (method, ep)] = _both(
            lambda: ddsp.core.resample(x3, 4, method=method, add_endpoint=ep))[0]
        out['up4_%s_%d' % (method, ep)] = _both(
            lambda: ddsp.core.resample(x4, 37, method=method, add_endpoint=ep))[0]
  return out


def angular_cumsum():
  """core.angular_cumsum (core.py:799-866) and tf.cumsum on the same angular
  frequencies, float32: [2, 2500, 3] (so the 1000-sample chunking pads)."""
  ddsp = ref_on_shim.load()
  tf = ref_on_shim.tf()
  rng = np.random.default_rng(606)
  omega = (2 * np.pi * rng.uniform(50.0, 4000.0, (2, 1, 3)) / 16000.0 *
           (1 + 0.01 * rng.standard_normal((2, 2500, 3)))).astype(np.float32)
  n, w = _both(lambda: ddsp.core.angular_cumsum(tf.convert_to_tensor(omega)))
  return dict(omega=omega, phase_f32=n, phase_wide=w.astype(np.float64))


def spectral_loss():
  """losses.SpectralLoss (losses.py:130-243) with the ae.gin weights (L1 on
  magnitudes and log magnitudes, ae.gin:39-41), B=2, N=8000."""
  ddsp = ref_on_shim.load()
  rng = np.random.default_rng(707)
  target = (0.1 * rng.standard_normal((2, 8000))).astype(np.float32)
  t = np.arange(8000) / 16000.0
  audio = (0.3 * np.sin(2 * np.pi * 220.0 * t)[None, :] * np.array([[1.0], [0.5]])
           + 0.05 * rng.standard_normal((2, 8000))).astype(np.float32)
  out = dict(target=target, audio=audio)
  for tag, kw in (('mag', dict(mag_weight=1.0, logmag_weight=0.0)),
                  ('maglog', dict(mag_weight=1.0, logmag_weight=1.0))):
    n, w = _both(lambda: ddsp.losses.SpectralLoss(**kw)(target, audio))
    out['loss_f32_' + tag] = np.float32(n)
    out['loss_wide_' + tag] = np.float64(w)
  return out


IR_CASES = [(65, 0), (65, 257), (65, 63), (65, 64), (100, 51), (100, 50), (513, 257),
            (513, 22), (1025, 257), (16, 257), (65, 3)]


def impulse_responses():
  """core.frequency_impulse_response (core.py:1534-1565) and frequency_filter
  (1628-1655) for even AND odd window sizes: tf.signal.hann_window is periodic
  for even lengths and symmetric for odd ones (window_ops._raised_cosine_window),
  which a restatement gets wrong unless it is checked on an odd window shorter than
  the impulse response (window_size=257 with more than 129 bins, e.g.)."""
  ddsp = ref_on_shim.load()
  rng = np.random.default_rng(808)
  out = {}
  for nb, ws in IR_CASES:
    m = rng.uniform(0.0, 1.0, (2, 3, nb)).astype(np.float32)
    n, w = _both(lambda: ddsp.core.frequency_impulse_response(m, ws))
    out['mags_%d_%d' % (nb, ws)] = m
    out['ir_f32_%d_%d' % (nb, ws)] = n
    out['ir_wide_%d_%d' % (nb, ws)] = w.astype(np.float64)
  noise = rng.uniform(-1.0, 1.0, (2, 960)).astype(np.float32)
  mags = rng.uniform(0.0, 1.0, (2, 20, 513)).astype(np.float32)
  n, w = _both(lambda: ddsp.core.frequency_filter(noise, mags, window_size=257))
  out.update(filter_noise=noise, filter_mags=mags, filter_f32=n,
             filter_wide=w.astype(np.float64))
  return out


def fuzz_cases():
  """The seeded argument sweep around the path's configurations - shapes, paddings,
  delays, odd / even / degenerate filter windows, every amplitude resampling method,
  both phase accumulators, sample rates, optional arguments - checked by
  tests/test_reference_fuzz.py.  Returns {group: [(tag, tol, ref_fn, oracle_fn)]}:
  ref_fn(ddsp, tf) runs the reference, oracle_fn(o) the oracle in float64; both
  return dicts of arrays ('phase' is compared modulo 2 pi).  A ref_fn that raises
  marks a case the oracle must reject too."""
  f64 = lambda x: None if x is None else x.astype(np.float64)  # noqa: E731
  opt = lambda tf, x: None if x is None else tf.convert_to_tensor(x)  # noqa: E731
  groups = {}

  cases = groups['fft_convolve'] = []
  rng = np.random.default_rng(123)
  for _ in range(24):
    b, f = int(rng.integers(1, 3)), int(rng.choice([1, 2, 5, 10, 25]))
    frame, s = int(rng.choice([1, 3, 16, 48, 64])), int(rng.choice([1, 2, 3, 10, 31, 64, 65, 128, 200]))
    pad, dc = str(rng.choice(['same', 'valid'])), int(rng.choice([-1, 0, 1, 5]))
    a = rng.standard_normal((b, f * frame)).astype(np.float32)
    ir = rng.standard_normal((b, f, s)).astype(np.float32)
    cases.append((
        ('fft_convolve', b, f, frame, s, pad, dc), 1e-9,
        lambda ddsp, tf, a=a, ir=ir, pad=pad, dc=dc: {'out': ddsp.core.fft_convolve(
            a, ir, padding=pad, delay_compensation=dc)},
        lambda o, a=a, ir=ir, pad=pad, dc=dc: {'out': o.fft_convolve(
            f64(a), f64(ir), padding=pad, delay_compensation=dc)}))

  cases = groups['frequency_filter'] = []
  rng = np.random.default_rng(124)
  for _ in range(20):
    f, frame = int(rng.choice([1, 4, 10])), int(rng.choice([8, 32, 64]))
    nb = int(rng.choice([2, 3, 9, 16, 33, 65, 100, 129, 130, 257]))
    ws = int(rng.choice([0, 1, 2, 3, 7, 8, 50, 51, 64, 65, 257]))
    a = rng.uniform(-1, 1, (1, f * frame)).astype(np.float32)
    m = rng.uniform(0, 1, (1, f, nb)).astype(np.float32)
    cases.append((
        ('frequency_filter', f, frame, nb, ws), 1e-9,
        lambda ddsp, tf, a=a, m=m, ws=ws: {'out': ddsp.core.frequency_filter(a, m, window_size=ws)},
        lambda o, a=a, m=m, ws=ws: {'out': o.frequency_filter(f64(a), f64(m), window_size=ws)}))

  cases = groups['harmonic_synthesis'] = []
  rng = np.random.default_rng(321)
  for _ in range(14):
    b, f = int(rng.integers(1, 3)), int(rng.choice([2, 5, 10, 25]))
    hop, k = int(rng.choice([4, 16, 64, 100])), int(rng.choice([1, 3, 20, 60]))
    method = str(rng.choice(['window', 'linear', 'nearest', 'cubic']))
    uac, sr = bool(rng.integers(0, 2)), int(rng.choice([16000, 8000, 44100]))
    f0 = rng.uniform(20, sr * 0.45, (b, f, 1)).astype(np.float32)
    amp = rng.uniform(0, 1, (b, f, 1)).astype(np.float32)
    hd = rng.uniform(0, 1, (b, f, k)).astype(np.float32) if rng.integers(0, 4) else None
    shifts = (rng.uniform(-0.05, 0.05, (b, f, k)).astype(np.float32)
              if hd is not None and rng.integers(0, 2) else None)
    kw = dict(n_samples=f * hop, sample_rate=sr, amp_resample_method=method,
              use_angular_cumsum=uac)
    # tensors, so that the wide mode widens every operand (a raw float32 array in
    # `1.0 + harmonic_shifts` would be rounded by NumPy before the shim sees it)
    cases.append((
        ('harmonic_synthesis', b, f, hop, k, method, uac, sr), 2e-7,
        lambda ddsp, tf, f0=f0, amp=amp, hd=hd, shifts=shifts, kw=kw: {
            'out': ddsp.core.harmonic_synthesis(
                opt(tf, f0), opt(tf, amp), harmonic_shifts=opt(tf, shifts),
                harmonic_distribution=opt(tf, hd), **kw)},
        lambda o, f0=f0, amp=amp, hd=hd, shifts=shifts, kw=kw: {
            'out': o.harmonic_synthesis(f64(f0), f64(amp), harmonic_shifts=f64(shifts),
                                        harmonic_distribution=f64(hd), dtype=np.float64,
                                        **kw)}))

  cases = groups['controls_oscillators_streaming_and_scalers'] = []
  rng = np.random.default_rng(999)
  for _ in range(8):                                   # Harmonic.get_controls variants
    f, k = int(rng.choice([3, 10])), int(rng.choice([1, 7, 40]))
    scale, nyq, sr = bool(rng.integers(0, 2)), bool(rng.integers(0, 2)), int(rng.choice([16000, 4000]))
    a = rng.standard_normal((1, f, 1)).astype(np.float32)
    h = rng.standard_normal((1, f, k)).astype(np.float32)
    f0 = rng.uniform(0, sr / 2, (1, f, 1)).astype(np.float32)
    if not scale:
      a, h = np.abs(a), np.abs(h)
    keys = ('amplitudes', 'harmonic_distribution', 'f0_hz')

    def ref_ctl(ddsp, tf, a=a, h=h, f0=f0, f=f, sr=sr, scale=scale, nyq=nyq):
      syn = ddsp.synths.Harmonic(n_samples=f * 8, sample_rate=sr,
                                 scale_fn=ddsp.core.exp_sigmoid if scale else None,
                                 normalize_below_nyquist=nyq)
      c = syn.get_controls(a, h, f0)
      return {key: c[key] for key in keys}

    def oracle_ctl(o, a=a, h=h, f0=f0, sr=sr, scale=scale, nyq=nyq):
      c = o.harmonic_get_controls(f64(a), f64(h), f64(f0), sample_rate=sr, scale=scale,
                                  normalize_below_nyquist=nyq, dtype=np.float64)
      return {key: c[key] for key in keys}
    cases.append((('get_controls', f, k, scale, nyq, sr), 1e-12, ref_ctl, oracle_ctl))
  for _ in range(8):                                   # oscillator_bank
    b, n, k = int(rng.integers(1, 3)), int(rng.choice([50, 1000, 2500])), int(rng.choice([1, 4, 17]))
    sr, ss, uac = int(rng.choice([16000, 8000])), bool(rng.integers(0, 2)), bool(rng.integers(0, 2))
    fe = rng.uniform(0, sr * 0.6, (b, n, k)).astype(np.float32)
    ae = rng.uniform(0, 1, (b, n, k)).astype(np.float32)
    kw = dict(sample_rate=sr, sum_sinusoids=ss, use_angular_cumsum=uac)
    cases.append((
        ('oscillator_bank', b, n, k, sr, ss, uac), 1e-8,
        lambda ddsp, tf, fe=fe, ae=ae, kw=kw: {'out': ddsp.core.oscillator_bank(
            opt(tf, fe), opt(tf, ae), **kw)},
        lambda o, fe=fe, ae=ae, kw=kw: {'out': o.oscillator_bank(
            f64(fe), f64(ae), dtype=np.float64, **kw)}))
  for _ in range(8):                                   # streaming synthesis, carried phase
    b, f, hop = int(rng.integers(1, 3)), int(rng.choice([1, 4, 10])), int(rng.choice([16, 64]))
    k = int(rng.choice([1, 5, 30]))
    f0 = rng.uniform(50, 2000, (b, f, 1)).astype(np.float32)
    amp = rng.uniform(0, 1, (b, f, 1)).astype(np.float32)
    hd = rng.uniform(0, 1, (b, f, k)).astype(np.float32) if rng.integers(0, 3) else None
    ph = rng.uniform(0, 6.28, (b, 1, 1)).astype(np.float32) if rng.integers(0, 2) else None
    method = str(rng.choice(['linear', 'window']))
    kw = dict(n_samples=f * hop, sample_rate=16000, amp_resample_method=method)

    def ref_stream(ddsp, tf, f0=f0, amp=amp, hd=hd, ph=ph, kw=kw):
      audio, phase = ddsp.core.streaming_harmonic_synthesis(
          opt(tf, f0), opt(tf, amp), opt(tf, hd), opt(tf, ph), **kw)
      return {'out': audio, 'phase': phase}

    def oracle_stream(o, f0=f0, amp=amp, hd=hd, ph=ph, kw=kw):
      audio, phase = o.streaming_harmonic_synthesis(f64(f0), f64(amp), f64(hd), f64(ph),
                                                    dtype=np.float64, **kw)
      return {'out': audio, 'phase': phase}
    cases.append((('streaming', b, f, hop, k, method), 1e-8, ref_stream, oracle_stream))
  for _ in range(5):                                   # scaling functions
    x = (4 * rng.standard_normal((2, 5, 7))).astype(np.float32)
    ex, mv, th = float(rng.choice([10.0, 2.0, 5.0])), float(rng.choice([2.0, 1.0])), float(rng.choice([1e-7, 1e-3]))
    cases.append((
        ('exp_sigmoid', ex, mv, th), 1e-12,
        lambda ddsp, tf, x=x, a=(ex, mv, th): {'out': ddsp.core.exp_sigmoid(opt(tf, x), *a)},
        lambda o, x=x, a=(ex, mv, th): {'out': o.exp_sigmoid(f64(x), *a, dtype=np.float64)}))
    depth = int(rng.choice([1, 8, 64]))
    fr = rng.standard_normal((2, 5, 3 * depth)).astype(np.float32)
    for name in ('frequencies_sigmoid', 'frequencies_softmax'):
      cases.append((
          (name, depth), 1e-9,
          lambda ddsp, tf, fr=fr, d=depth, name=name: {'out': getattr(ddsp.core, name)(
              opt(tf, fr), depth=d)},
          lambda o, fr=fr, d=depth, name=name: {'out': getattr(o, name)(
              f64(fr), depth=d, dtype=np.float64)}))
  for _ in range(4):                                   # Sinusoidal
    f, k, hop = int(rng.choice([5, 10])), int(rng.choice([1, 4, 9])), int(rng.choice([16, 64]))
    a = rng.standard_normal((1, f, k)).astype(np.float32)
    fr = rng.standard_normal((1, f, k)).astype(np.float32)
    method = str(rng.choice(['window', 'linear']))

    def ref_sin(ddsp, tf, a=a, fr=fr, n=f * hop, method=method):
      syn = ddsp.synths.Sinusoidal(n_samples=n, sample_rate=16000, amp_resample_method=method)
      return {'out': syn(opt(tf, a), opt(tf, fr))}

    def oracle_sin(o, a=a, fr=fr, n=f * hop, method=method):
      c = o.sinusoidal_get_controls(f64(a), f64(fr), dtype=np.float64)
      return {'out': o.sinusoidal_get_signal(c['amplitudes'], c['frequencies'], n,
                                             amp_resample_method=method, dtype=np.float64)}
    cases.append((('sinusoidal', f, k, hop, method), 1e-8, ref_sin, oracle_sin))
  return groups


def reference_fuzz():
  """The reference's wide results on every case of fuzz_cases(), float64; '<key>_raises'
  marks a case the reference rejects."""
  ddsp = ref_on_shim.load()
  tf = ref_on_shim.tf()
  out = {}
  for group, cases in fuzz_cases().items():
    for i, (_, _, ref_fn, _) in enumerate(cases):
      key = '%s_%03d' % (group, i)
      tf.set_wide(True)
      try:
        res = ref_on_shim.to_numpy(ref_fn(ddsp, tf))
      except Exception:  # pylint: disable=broad-except
        out[key + '_raises'] = np.bool_(True)
        continue
      finally:
        tf.set_wide(False)
      for k, v in res.items():
        out['%s_%s' % (key, k)] = np.asarray(v, np.float64)
  return out


REVERB = dict(B=2, N=3000, L=1920, F=40, NB=16, WS=257)


def reverb_inputs(trainable):
  """Seeded audio, magnitudes (one learned row when trainable) and noise of the
  FilteredNoiseReverb composition check."""
  rng = np.random.default_rng(5)
  audio = rng.standard_normal((REVERB['B'], REVERB['N'])).astype(np.float32)
  mags = rng.standard_normal((1 if trainable else REVERB['B'], REVERB['F'],
                              REVERB['NB'])).astype(np.float32)
  noise = rng.uniform(-1, 1, (mags.shape[0], REVERB['L'])).astype(np.float32)
  return audio, mags, noise


def reverb_composition():
  """effects.FilteredNoiseReverb (effects.py:202-278) of the reference, float32,
  with its random draw pinned to reverb_inputs' noise: fixed magnitudes and the
  trainable (single learned response) variant."""
  ddsp = ref_on_shim.load()
  tf = ref_on_shim.tf()
  out = {}
  uniform = tf.random.uniform
  for trainable in (False, True):
    audio, mags, noise = reverb_inputs(trainable)
    tf.random.uniform = lambda shape, minval=0, maxval=1, noise=noise, **kw: tf.constant(noise)
    try:
      r = ddsp.effects.FilteredNoiseReverb(
          trainable=trainable, reverb_length=REVERB['L'], window_size=REVERB['WS'],
          n_frames=REVERB['F'], n_filter_banks=REVERB['NB'])
      if trainable:
        r.build(None)
        r._magnitudes = tf.constant(mags[0])
        want = ref_on_shim.to_numpy(r(audio))
      else:
        want = ref_on_shim.to_numpy(r(audio, mags))
    finally:
      tf.random.uniform = uniform
    out['out_trainable_%d' % trainable] = np.asarray(want, np.float32)
  return out


WINDOW_CASES = [(128, 0, False), (128, 257, False), (128, 64, False), (128, 63, False),
                (30, 257, False), (2048, 257, True), (100, 51, True), (100, 50, False),
                (4, 0, False)]
CROP_CASES = [(64192, 64000, 128, 'same', -1), (64192, 64000, 128, 'valid', -1),
              (1009, 1000, 10, 'same', 0), (109, 10, 100, 'same', -1),
              (4095, 1000, 3000, 'same', 0), (3999, 1000, 3000, 'valid', -1)]


def host_helper_inputs():
  """Seeded impulse responses for WINDOW_CASES and audio for CROP_CASES."""
  rng = np.random.default_rng(0)
  irs = [rng.standard_normal((2, 3, size)).astype(np.float32) for size, _, _ in WINDOW_CASES]
  audio = [rng.standard_normal((2, c[0])).astype(np.float32) for c in CROP_CASES]
  return irs, audio


def host_helpers():
  """core.apply_window_to_impulse_response (core.py:1477-1531) of the reference on
  WINDOW_CASES, float32, and where core.crop_and_compensate_delay (1338-1379) cuts
  each CROP_CASES input: its output is exactly audio[:, start : start + length]."""
  ddsp = ref_on_shim.load()
  irs, audio = host_helper_inputs()
  out = {}
  for i, ((_, ws, causal), ir) in enumerate(zip(WINDOW_CASES, irs)):
    out['window_%d' % i] = ref_on_shim.to_numpy(
        ddsp.core.apply_window_to_impulse_response(ir, ws, causal)).astype(np.float32)
  for i, ((_, n, s, pad, dc), a) in enumerate(zip(CROP_CASES, audio)):
    cut = ref_on_shim.to_numpy(ddsp.core.crop_and_compensate_delay(a, n, s, pad, dc))
    starts = [j for j in range(a.shape[1] - cut.shape[1] + 1)
              if np.array_equal(a[:, j:j + cut.shape[1]], cut)] if cut.size else [0]
    assert len(starts) == 1, (CROP_CASES[i], starts)
    out['crop_%d' % i] = np.array([starts[0], cut.shape[1]], np.int64)
  return out


FIXTURES = dict(c1_harmonic=c1_harmonic, decoder_small=decoder_small, c2_item=c2_item,
                harmonic_shifts=harmonic_shifts, resample_methods=resample_methods,
                angular_cumsum=angular_cumsum, spectral_loss=spectral_loss,
                impulse_responses=impulse_responses, reference_fuzz=reference_fuzz,
                reverb_composition=reverb_composition, host_helpers=host_helpers)


def compare(name, got, want, atol=0.0):
  assert set(want.files) == set(got), (name, sorted(set(want.files) ^ set(got)))
  for k in want.files:
    np.testing.assert_allclose(np.asarray(got[k], np.float64),
                               np.asarray(want[k], np.float64), rtol=0, atol=atol,
                               err_msg='%s/%s' % (name, k))


if __name__ == '__main__':
  check = '--check' in sys.argv
  only = [a for a in sys.argv[1:] if not a.startswith('--')]
  for name, fn in FIXTURES.items():
    if only and name not in only:
      continue
    path = os.path.join(HERE, name + '.npz')
    got = fn()
    if check:
      compare(name, got, np.load(path))
      print('ok   ', name)
    else:
      np.savez_compressed(path, **got)
      print('wrote', name, '%.0f kB' % (os.path.getsize(path) / 1e3))
