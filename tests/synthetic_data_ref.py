"""Host float64 restatement of numpy's legacy RandomState stream (MT19937) and of
generate_notes_v2's walk over it (training/data_preparation/synthetic_data.py).

`Stream` replays np.random.RandomState word for word: init_genrand seeding, a
vectorised twist, the 53-bit double of two words, the polar Gaussian with its cached
second value, and masked rejection for random_integers.  `notes_v2` walks it in the
reference's draw order and returns the reference's float64 arrays before its TF steps
(harm_amp, harm_dist, f0_midi, mags, and the harm_amp divisor).  numpy does the
elementwise arithmetic as the reference's numpy does it, and the scalar log / sqrt of
the Gaussians are libm's, as in numpy's C code, so the arrays are the reference's bits.
"""
import math

import numpy as np

N, M = 624, 397
_UPPER, _LOWER, _MATRIX_A = np.uint32(0x80000000), np.uint32(0x7fffffff), np.uint32(0x9908b0df)


def init_genrand(seed):
  key = np.empty(N, np.uint32)
  x = int(seed) & 0xffffffff
  key[0] = x
  for i in range(1, N):
    x = (1812433253 * (x ^ (x >> 30)) + i) & 0xffffffff
    key[i] = x
  return key


def twist(key):
  """The next 624 raw words, in three dependent vectorised phases."""
  def mix(lo, hi):
    y = (lo & _UPPER) | (hi & _LOWER)
    return (y >> np.uint32(1)) ^ np.where(y & np.uint32(1), _MATRIX_A, np.uint32(0))
  y = mix(key, np.roll(key, -1))
  new = np.empty(N, np.uint32)
  new[:N - M] = key[M:] ^ y[:N - M]
  new[N - M:2 * (N - M)] = new[:N - M] ^ y[N - M:2 * (N - M)]
  new[2 * (N - M):N - 1] = new[N - M:M - 1] ^ y[2 * (N - M):N - 1]
  new[N - 1] = new[M - 1] ^ mix(key[N - 1:], new[:1])[0]
  return new


def temper(y):
  y = y ^ (y >> np.uint32(11))
  y = y ^ ((y << np.uint32(7)) & np.uint32(0x9d2c5680))
  y = y ^ ((y << np.uint32(15)) & np.uint32(0xefc60000))
  return y ^ (y >> np.uint32(18))


class Stream:
  """np.random.RandomState's legacy stream from (key, pos, has_gauss, gauss)."""

  def __init__(self, key, pos=N, has_gauss=0, gauss=0.0):
    self.blocks = [np.asarray(key, np.uint32).copy()]
    self.words = [temper(self.blocks[0])]
    self.pos = int(pos)
    self.has_gauss = bool(has_gauss)
    self.gauss = float(gauss)

  @classmethod
  def seeded(cls, seed):
    return cls(init_genrand(seed))

  @classmethod
  def from_numpy(cls, state):
    _, key, pos, has_gauss, gauss = state
    return cls(key, pos, has_gauss, gauss)

  def state(self):
    """(key, pos, has_gauss, gauss) as numpy's get_state() reports them."""
    return self.blocks[0].copy(), self.pos, int(self.has_gauss), self.gauss

  def peek(self, n):
    while len(self.blocks) * N - self.pos < n:
      self.blocks.append(twist(self.blocks[-1]))
      self.words.append(temper(self.blocks[-1]))
    return np.concatenate(self.words)[self.pos:self.pos + n]

  def take(self, n):
    self.pos += n
    while self.pos > N:   # numpy twists lazily: pos stays N until the next word
      self.pos -= N
      self.blocks.pop(0)
      self.words.pop(0)

  @staticmethod
  def _doubles(w):
    a, b = w[0::2] >> np.uint32(5), w[1::2] >> np.uint32(6)
    return (a.astype(np.float64) * 67108864.0 + b) / 9007199254740992.0

  def rand(self, n):
    d = self._doubles(self.peek(2 * n))
    self.take(2 * n)
    return d

  def uniform(self, low=0.0, high=1.0):
    low, high = float(low), float(high)
    return low + (high - low) * float(self.rand(1)[0])

  def random_integers(self, low, high):
    rng = int(high) - int(low)
    if rng < 0:
      raise ValueError('low > high')
    if rng == 0:
      return int(low)
    mask = (1 << rng.bit_length()) - 1
    while True:
      v = int(self.peek(1)[0]) & mask
      self.take(1)
      if v <= rng:
        return int(low) + v

  def randn(self, *shape):
    n = int(np.prod(shape))
    out = np.empty(n)
    done = 0
    if n and self.has_gauss:
      out[0], self.has_gauss, self.gauss, done = self.gauss, False, 0.0, 1
    while done < n:
      pairs = (n - done + 1) // 2
      tries = int(pairs * 1.3) + 8
      d = self._doubles(self.peek(4 * tries))
      x1, x2 = 2.0 * d[0::2] - 1.0, 2.0 * d[1::2] - 1.0
      r2 = x1 * x1 + x2 * x2
      ok = np.nonzero(~((r2 >= 1.0) | (r2 == 0.0)))[0][:pairs]
      f = np.array([math.sqrt(-2.0 * math.log(r) / r) for r in r2[ok]])
      vals = np.empty(2 * len(ok))
      vals[0::2], vals[1::2] = f * x2[ok], f * x1[ok]
      if len(ok) < pairs:
        self.take(4 * tries)
        out[done:done + len(vals)] = vals
        done += len(vals)
        continue
      self.take(4 * (int(ok[-1]) + 1))
      take = n - done
      out[done:] = vals[:take]
      if take < len(vals):
        self.has_gauss, self.gauss = True, float(vals[take])
      done = n
    return out.reshape(shape)


def _random_blend(s, length, env_start=1.0, env_end=0.0, exp_max=2.0):
  e = s.uniform(-exp_max, exp_max)
  v = np.linspace(1.0, 0.0, length) ** (2.0 ** e)
  return env_start * v + env_end * (1.0 - v)


def _random_harm_dist(s, n, low_pass, rand_phase):
  nc = s.random_integers(1, 20)
  smoothness = s.uniform(1.0, 10.0)
  coeffs = s.rand(nc)
  freqs = s.rand(nc) * n / smoothness
  comps = [coeffs[i] * np.cos(np.linspace(0.0, 2.0 * np.pi * freqs[i], n) +
                              s.uniform(0.0, np.pi * 2.0 * rand_phase)) for i in range(nc)]
  if low_pass:
    lp = []
    for c in comps:
      end = s.uniform(0.0, 0.5)
      lp.append(c * np.linspace(1.0, end, n) ** s.uniform(0.5, 2.0))
    comps = lp
  return np.sum(np.stack(comps), axis=0)


def _distribution(s, width, length):
  low_pass = s.uniform() <= 0.8
  rand_phase = s.uniform(0.0, 0.4)
  start = _random_harm_dist(s, width, low_pass, rand_phase)[np.newaxis, :]
  end = _random_harm_dist(s, width, low_pass, rand_phase)[np.newaxis, :]
  blend = _random_blend(s, length, 1.0, 0.0)[:, np.newaxis]
  return start * blend + end * (1.0 - blend)


def notes_v2(s, n_batch=1, n_timesteps=125, n_harmonics=100, n_mags=65, min_note_length=5,
             max_note_length=25, p_silent=0.1, p_vibrato=0.5, get_controls=True):
  """generate_notes_v2's float64 arrays drawn from Stream s: harm_amp [B, T],
  harm_dist [B, T, K], f0_midi [B, T], mags [B, T, M], and the divisor (None without
  get_controls)."""
  T = n_timesteps
  harm_amp = np.zeros([n_batch, T])
  harm_dist = np.zeros([n_batch, T, n_harmonics])
  f0_midi = np.zeros([n_batch, T])
  mags = np.zeros([n_batch, T, n_mags])
  for b in range(n_batch):
    t0 = 0
    while t0 < T:
      t1 = min(t0 + s.random_integers(min_note_length, max_note_length), T)
      length = t1 - t0
      if s.uniform() <= p_silent:
        harm_amp[b, t0:t1] -= 10.0
      else:
        a0 = s.uniform(-1.0, 3.0)
        a1 = s.uniform(-1.0, 3.0)
        harm_amp[b, t0:t1] += _random_blend(s, length, a0, a1)
        harm_amp[b, t0:t1] += s.uniform(0.0, 0.1) * s.randn(length)
        harm_dist[b, t0:t1] += _distribution(s, n_harmonics, length)
        harm_dist[b, t0:t1] += s.uniform(0.0, 0.5) * s.randn(length, n_harmonics)
        f0 = s.uniform(24.0, 84.0)
        if s.uniform() <= p_vibrato:
          v0 = s.uniform(0.0, 1.0)
          v1 = s.uniform(0.0, 1.0)
          periods = s.uniform(0.0, length * 2.0 / min_note_length)
          vib = _random_blend(s, length, v0, v1) * np.sin(
              np.linspace(0.0, 2.0 * np.pi * periods, length))
          note = f0 + vib
        else:
          note = f0 * np.ones([length])
        f0_midi[b, t0:t1] += note
        f0_midi[b, t0:t1] += s.uniform(0.0, 0.1) * s.randn(length)
      mags[b, t0:t1] += _distribution(s, n_mags, length)
      mags[b, t0:t1] += s.uniform(0.0, 0.2) * s.randn(length, n_mags)
      mags[b, t0:t1] -= s.uniform(1.0, 10.0)
      t0 = t1
  divisor = None
  if get_controls:
    inner = s.uniform(2.0, 10.0)
    wide = s.uniform() <= 0.2
    divisor = s.uniform(1.0, inner if wide else 2.0)
  return harm_amp, harm_dist, f0_midi, mags, divisor


def seeded_v2(seed, **kwargs):
  """np.random.seed(seed); generate_notes_v2(n_batch=1, **kwargs), restated."""
  return notes_v2(Stream.seeded(seed), 1, **kwargs)
