// The self-supervised training data of InverseSynthesis (training/data_preparation/
// synthetic_data.py, generate_notes_v2): piecewise notes of harmonic amplitude,
// harmonic distribution, f0 and noise magnitudes, drawn from numpy's legacy
// RandomState.
//
// The reference draws every value from np.random's MT19937 stream, one scalar or one
// array call at a time, and the note-level control flow (note lengths, silences,
// component counts, vibrato) reads draws that come after each Gaussian block.  So one
// CTA walks one stream in the reference's order:
//   * the MT state lives in shared memory as a window of two 624-word blocks, the
//     current one (numpy's `key`) and the next; `pos` indexes the window, so any draw
//     of up to 624 words reads without a twist in the middle.  Crossing into the next
//     block twists a new one out of place, in three dependent phases.
//   * scalar draws (uniform doubles, masked-rejection integers) are taken by every
//     thread alike from the shared words: the walk's control flow stays uniform.
//   * Gaussian blocks run numpy's legacy polar method, one attempt (4 words) per
//     thread per round; a block ballot and prefix count map the k-th accepted attempt
//     to outputs 2k and 2k + 1 of the block, and the attempt that completes the block
//     fixes how many words it consumed.  An odd block leaves its last value cached.
// Elementary float64 arithmetic is numpy's, rounded step by step (__dmul_rn /
// __dadd_rn: never contracted into FMA); cos, sin, pow, log and sqrt are CUDA's.
// Integer decisions read only uniforms and integers, so they are exact.  No atomics.
#pragma once
#include <math_constants.h>
#include <stdint.h>

#include "common.cuh"

namespace ddsp {
namespace synth_ {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kN = 624;             // MT19937 state words
constexpr int kM = 397;
constexpr int kWindow = 2 * kN;     // the current block and the next one
constexpr int kMaxComponents = 20;  // random_harm_dist: uniform_int(1, 20)

struct Params {
  const int64_t* seeds;  // [B] seeds mode: one stream per item (NULL in state mode)
  uint32_t* key;         // [624] state mode: numpy's key, in and out
  int* pos;              // [2] state mode: pos and has_gauss, in and out
  double* gauss;         // [1] state mode: the cached Gaussian, in and out
  double* harm_amp;      // [B, T]
  double* harm_dist;     // [B, T, K]
  double* f0_midi;       // [B, T]
  double* mags;          // [B, T, M]
  double* divisor;       // [B] the harm_amp divisor (get_controls only)
  int B, T, K, M, min_len, max_len, get_controls;
  double p_silent, p_vibrato;
};

// The shared-memory layout of one CTA (dynamic, sized by T and max(K, M)):
//   ring [kWindow] raw MT words: block `base` is current, the other one next;
//   wcount [kWarps] accepted polar attempts per warp; last [1] the attempt that
//   completed a Gaussian block and cache [1] the value it leaves cached;
//   comp [5 kMaxComponents] random_harm_dist's per-component draws;
//   dist_a, dist_b [max(K, M)] a note's start and end distributions; blend [T].
// The offsets are constants or depend on max(K, M) alone, so no pointer stays live.
extern __shared__ __align__(16) unsigned char smem_raw[];
constexpr int kWcountOff = kWindow * 4;
constexpr int kCacheOff = kWcountOff + 56;
constexpr int kCompOff = kCacheOff + 8;
constexpr int kDistOff = kCompOff + 5 * kMaxComponents * 8;

struct Smem {
  int nk;  // max(K, M)
  __device__ uint32_t* ring() const { return reinterpret_cast<uint32_t*>(smem_raw); }
  __device__ int* wcount() const { return reinterpret_cast<int*>(smem_raw + kWcountOff); }
  __device__ int* last() const { return wcount() + kWarps; }
  __device__ double* cache() const { return reinterpret_cast<double*>(smem_raw + kCacheOff); }
  __device__ double* comp() const { return reinterpret_cast<double*>(smem_raw + kCompOff); }
  __device__ double* dist_a() const { return reinterpret_cast<double*>(smem_raw + kDistOff); }
  __device__ double* dist_b() const { return dist_a() + nk; }
  __device__ double* blend() const { return dist_a() + 2 * nk; }
};

__host__ __device__ inline size_t smem_bytes(int T, int K, int M) {
  const int nk = K > M ? K : M;
  return (size_t)kDistOff + (2 * (size_t)nk + T) * 8;
}

__device__ __forceinline__ uint32_t temper(uint32_t y) {
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= y >> 18;
  return y;
}

__device__ __forceinline__ uint32_t twist_word(uint32_t lo_src, uint32_t hi_src, uint32_t m) {
  const uint32_t y = (lo_src & 0x80000000u) | (hi_src & 0x7fffffffu);
  return m ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}

// np.linspace(start, stop, n)[j]: j * step + start, the last element stop, and
// (j / (n - 1)) * delta + start when the step is 0.
__device__ inline double linspace(double start, double stop, int n, int j) {
  if (n == 1) return start;
  if (j == n - 1) return stop;
  const double delta = __dsub_rn(stop, start);
  const double step = __ddiv_rn(delta, (double)(n - 1));
  if (step == 0.0) return __dadd_rn(__dmul_rn(__ddiv_rn((double)j, (double)(n - 1)), delta), start);
  return __dadd_rn(__dmul_rn((double)j, step), start);
}

// One MT19937 stream walked by a whole CTA.  pos, base and the Gaussian cache are
// registers that every thread keeps alike.
struct Walk {
  Smem s;
  int pos;       // next word, 0..kWindow; <= kN between draws (numpy's pos)
  int base;      // 0 or kN: where the current block starts in the ring
  bool has_gauss;
  double gauss;

  __device__ uint32_t word(int j) const {
    int i = base + j;
    if (i >= kWindow) i -= kWindow;
    return temper(s.ring()[i]);
  }
  // numpy's 53-bit double from two words: (a >> 5, b >> 6), exact.
  __device__ double dbl(int j) const {
    const uint32_t a = word(j) >> 5, b = word(j + 1) >> 6;
    return ((double)a * 67108864.0 + (double)b) * (1.0 / 9007199254740992.0);
  }

  // Twists the next block out of the current one.  Collective.
  __device__ void twist_next() {
    const uint32_t* cur = s.ring() + base;
    uint32_t* nxt = s.ring() + (kN - base);
    __syncthreads();  // nobody still reads the block being replaced
    for (int i = threadIdx.x; i < kN - kM; i += kThreads)
      nxt[i] = twist_word(cur[i], cur[i + 1], cur[i + kM]);
    __syncthreads();
    for (int i = kN - kM + threadIdx.x; i < 2 * (kN - kM); i += kThreads)
      nxt[i] = twist_word(cur[i], cur[i + 1], nxt[i - (kN - kM)]);
    __syncthreads();
    for (int i = 2 * (kN - kM) + threadIdx.x; i < kN; i += kThreads)
      nxt[i] = i < kN - 1 ? twist_word(cur[i], cur[i + 1], nxt[i - (kN - kM)])
                          : twist_word(cur[i], nxt[0], nxt[kM - 1]);
    __syncthreads();
  }
  // Makes the next block current once every word of the current one is used.
  __device__ void settle() {
    if (pos > kN) {
      pos -= kN;
      base = kN - base;
      twist_next();
    }
  }
  __device__ double uniform(double lo, double hi) {
    settle();
    const double d = dbl(pos);
    pos += 2;
    return __dadd_rn(lo, __dmul_rn(__dsub_rn(hi, lo), d));
  }
  __device__ bool flip(double p) { return uniform(0.0, 1.0) <= p; }
  // random_integers(lo, hi): masked rejection on single words; no draw when lo == hi.
  __device__ int integer(int lo, int hi) {
    const uint32_t rng = (uint32_t)(hi - lo);
    if (rng == 0) return lo;
    uint32_t mask = rng;
    mask |= mask >> 1;
    mask |= mask >> 2;
    mask |= mask >> 4;
    mask |= mask >> 8;
    mask |= mask >> 16;
    for (;;) {
      settle();
      const uint32_t v = word(pos) & mask;
      ++pos;
      if (v <= rng) return lo + (int)v;
    }
  }

  // np.random.randn(n), element e handed to emit(e, value) by the thread that has it.
  template <class Emit>
  __device__ void gaussians(int64_t n, Emit&& emit) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int64_t done = 0;
    if (n > 0 && has_gauss) {
      if (tid == 0) emit((int64_t)0, gauss);
      has_gauss = false;
      gauss = 0.0;
      done = 1;
    }
    while (done < n) {
      settle();
      const int avail = (kWindow - pos) / 4;
      const int attempts = avail < kThreads ? avail : kThreads;
      double x1 = 0.0, x2 = 0.0, r2 = 0.0;
      bool ok = false;
      if (tid < attempts) {
        const int j = pos + 4 * tid;
        x1 = __dsub_rn(2.0 * dbl(j), 1.0);
        x2 = __dsub_rn(2.0 * dbl(j + 2), 1.0);
        r2 = __dadd_rn(__dmul_rn(x1, x1), __dmul_rn(x2, x2));
        ok = !(r2 >= 1.0 || r2 == 0.0);
      }
      const unsigned vote = __ballot_sync(0xffffffffu, ok);
      if (lane == 0) s.wcount()[warp] = __popc(vote);
      __syncthreads();
      int rank = __popc(vote & ((1u << lane) - 1u)), total = 0;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) {
        const int c = s.wcount()[w];
        rank += w < warp ? c : 0;
        total += c;
      }
      const int64_t pairs = (n - done + 1) / 2;
      if (ok && rank < pairs) {
        const double f = sqrt(__ddiv_rn(-2.0 * log(r2), r2));
        const int64_t e = done + 2 * (int64_t)rank;
        emit(e, __dmul_rn(f, x2));
        if (e + 1 < n) emit(e + 1, __dmul_rn(f, x1));
        else *s.cache() = __dmul_rn(f, x1);
        if (rank == pairs - 1) *s.last() = tid;
      }
      __syncthreads();
      if (total >= pairs) {
        pos += 4 * (*s.last() + 1);
        if ((n - done) & 1) {
          has_gauss = true;
          gauss = *s.cache();
        }
        done = n;
      } else {
        pos += 4 * attempts;
        done += 2 * (int64_t)total;
      }
      __syncthreads();  // wcount, last and cache are read
    }
  }

  // random_blend's draw: the exponent 2 ** uniform(-2, 2), and the blend of a and b
  // over L frames into the blend row.
  __device__ void blend(int L, double a, double b) {
    const double p = pow(2.0, uniform(-2.0, 2.0));
    __syncthreads();  // the previous blend is read
    for (int j = threadIdx.x; j < L; j += kThreads) {
      const double v = pow(linspace(1.0, 0.0, L, j), p);
      s.blend()[j] = __dadd_rn(__dmul_rn(a, v), __dmul_rn(b, __dsub_rn(1.0, v)));
    }
    __syncthreads();
  }

  // random_harm_dist(n, low_pass, rand_phase) into out[n].
  __device__ void harm_dist(int n, bool low_pass, double rand_phase, double* out) {
    const int nc = integer(1, kMaxComponents);
    const double smooth = uniform(1.0, 10.0);
    settle();
    double* coeff = s.comp();
    double* freq = coeff + kMaxComponents;
    double* phase = freq + kMaxComponents;
    double* end = phase + kMaxComponents;
    double* expo = end + kMaxComponents;
    const double phase_hi = __dmul_rn(2.0 * CUDART_PI, rand_phase);
    __syncthreads();  // the previous distribution's draws are read
    const int i = threadIdx.x;
    // rand(nc), rand(nc), nc phases, then (low_pass) nc (end, exponent) pairs: at most
    // 10 nc words <= 200, all inside the window.
    if (i < nc) {
      coeff[i] = dbl(pos + 2 * i);
      freq[i] = __ddiv_rn(__dmul_rn(dbl(pos + 2 * nc + 2 * i), (double)n), smooth);
      phase[i] = __dadd_rn(0.0, __dmul_rn(phase_hi, dbl(pos + 4 * nc + 2 * i)));
      if (low_pass) {
        end[i] = __dadd_rn(0.0, __dmul_rn(0.5, dbl(pos + 6 * nc + 4 * i)));
        expo[i] = __dadd_rn(0.5, __dmul_rn(1.5, dbl(pos + 6 * nc + 4 * i + 2)));
      }
    }
    pos += (low_pass ? 10 : 6) * nc;
    __syncthreads();
    for (int j = threadIdx.x; j < n; j += kThreads) {
      double acc = 0.0;
      for (int c = 0; c < nc; ++c) {
        const double arg = __dadd_rn(linspace(0.0, __dmul_rn(2.0 * CUDART_PI, freq[c]), n, j),
                                     phase[c]);
        double v = __dmul_rn(coeff[c], cos(arg));
        if (low_pass) v = __dmul_rn(v, pow(linspace(1.0, end[c], n, j), expo[c]));
        acc = c == 0 ? v : __dadd_rn(acc, v);
      }
      out[j] = acc;
    }
    __syncthreads();
  }
};

// The distribution of a note: both ends, their blend and the noise block, into rows
// [t0, t0 + L) of dst [., width]; the rows are (0 + blend) + scale * noise.
__device__ void distribution(Walk& w, double* dst, int t0, int L, int width, double noise_hi) {
  const bool low_pass = w.flip(0.8);
  const double rand_phase = w.uniform(0.0, 0.4);
  w.harm_dist(width, low_pass, rand_phase, w.s.dist_a());
  w.harm_dist(width, low_pass, rand_phase, w.s.dist_b());
  w.blend(L, 1.0, 0.0);
  const double scale = w.uniform(0.0, noise_hi);
  const Smem s = w.s;
  double* rows = dst + (int64_t)t0 * width;
  w.gaussians((int64_t)L * width, [&](int64_t e, double z) {
    const int r = (int)(e / width), c = (int)(e - (int64_t)r * width);
    const double bl = s.blend()[r];
    const double v = __dadd_rn(__dmul_rn(s.dist_a()[c], bl),
                               __dmul_rn(s.dist_b()[c], __dsub_rn(1.0, bl)));
    rows[e] = __dadd_rn(__dadd_rn(0.0, v), __dmul_rn(scale, z));
  });
}

// generate_notes_v2's rows of one item, drawn from w.
__device__ void render_item(Walk& w, const Params& p, int64_t b) {
  const int T = p.T, K = p.K, M = p.M;
  double* ha = p.harm_amp + b * T;
  double* hd = p.harm_dist + b * (int64_t)T * K;
  double* f0m = p.f0_midi + b * T;
  double* mg = p.mags + b * (int64_t)T * M;
  const Smem s = w.s;
  for (int t0 = 0; t0 < T;) {
    int L = w.integer(p.min_len, p.max_len);
    const int t1 = L < T - t0 ? t0 + L : T;
    L = t1 - t0;
    if (w.flip(p.p_silent)) {
      for (int64_t e = threadIdx.x; e < (int64_t)L * K; e += kThreads)
        hd[(int64_t)t0 * K + e] = 0.0;
      for (int j = threadIdx.x; j < L; j += kThreads) {
        ha[t0 + j] = -10.0;
        f0m[t0 + j] = 0.0;
      }
    } else {
      // Amplitudes: a blend between two levels, plus noise.
      const double a0 = w.uniform(-1.0, 3.0);
      const double a1 = w.uniform(-1.0, 3.0);
      w.blend(L, a0, a1);
      const double amp_noise = w.uniform(0.0, 0.1);
      w.gaussians(L, [&](int64_t e, double z) {
        ha[t0 + e] = __dadd_rn(__dadd_rn(0.0, s.blend()[e]), __dmul_rn(amp_noise, z));
      });
      // Harmonic distribution.
      distribution(w, hd, t0, L, K, 0.5);
      // Fundamental frequency, with or without vibrato.
      const double f0 = w.uniform(24.0, 84.0);
      const bool vibrato = w.flip(p.p_vibrato);
      double periods = 0.0;
      if (vibrato) {
        const double v0 = w.uniform(0.0, 1.0);
        const double v1 = w.uniform(0.0, 1.0);
        periods = w.uniform(0.0, __ddiv_rn((double)L * 2.0, (double)p.min_len));
        w.blend(L, v0, v1);
      }
      const double top = __dmul_rn(2.0 * CUDART_PI, periods);
      const double f0_noise = w.uniform(0.0, 0.1);
      w.gaussians(L, [&](int64_t e, double z) {
        const int j = (int)e;
        const double note =
            vibrato ? __dadd_rn(f0, __dmul_rn(s.blend()[j], sin(linspace(0.0, top, L, j)))) : f0;
        f0m[t0 + j] = __dadd_rn(__dadd_rn(0.0, note), __dmul_rn(f0_noise, z));
      });
    }
    // Filtered noise; its level is drawn after its noise block, so the rows are
    // finished once it exists.
    distribution(w, mg, t0, L, M, 0.2);
    const double level = w.uniform(1.0, 10.0);
    __syncthreads();  // the noise block's rows are written
    for (int64_t e = threadIdx.x; e < (int64_t)L * M; e += kThreads) {
      double* m = mg + (int64_t)t0 * M + e;
      *m = __dsub_rn(*m, level);
    }
    t0 = t1;
  }
}

// uniform_float(1.0, [2.0, uniform_float(2.0, 10.0)][flip(0.2)]): the inner uniform,
// the flip, then the outer uniform.
__device__ inline double final_divisor(Walk& w) {
  const double inner = w.uniform(2.0, 10.0);
  const bool wide = w.flip(0.2);
  return w.uniform(1.0, wide ? inner : 2.0);
}

// Seeds mode: CTA b runs np.random.seed(seeds[b]); generate_notes_v2(n_batch=1).
// State mode (seeds == NULL, one CTA): generate_notes_v2(n_batch=B) from numpy's state.
__global__ void __launch_bounds__(kThreads, 1) synthetic_notes_kernel(Params p) {
  Walk w;
  w.s.nk = p.K > p.M ? p.K : p.M;
  w.base = 0;
  const bool seeds = p.seeds != nullptr;
  if (seeds) {
    if (threadIdx.x == 0) {  // init_genrand
      uint32_t x = (uint32_t)p.seeds[blockIdx.x];
      w.s.ring()[0] = x;
      for (int i = 1; i < kN; ++i) {
        x = 1812433253u * (x ^ (x >> 30)) + (uint32_t)i;
        w.s.ring()[i] = x;
      }
    }
    w.pos = kN;
    w.has_gauss = false;
    w.gauss = 0.0;
  } else {
    for (int i = threadIdx.x; i < kN; i += kThreads) w.s.ring()[i] = p.key[i];
    w.pos = p.pos[0];
    w.has_gauss = p.pos[1] != 0;
    w.gauss = p.gauss[0];
  }
  w.twist_next();
  const int64_t b0 = seeds ? blockIdx.x : 0, b1 = seeds ? b0 + 1 : p.B;
  for (int64_t b = b0; b < b1; ++b) render_item(w, p, b);
  if (p.get_controls) {
    const double d = final_divisor(w);
    for (int64_t b = b0 + threadIdx.x; b < b1; b += kThreads) p.divisor[b] = d;
  }
  if (!seeds) {
    w.settle();
    __syncthreads();
    for (int i = threadIdx.x; i < kN; i += kThreads) p.key[i] = w.s.ring()[w.base + i];
    if (threadIdx.x == 0) {
      p.pos[0] = w.pos;
      p.pos[1] = w.has_gauss ? 1 : 0;
      p.gauss[0] = w.gauss;
    }
  }
}

}  // namespace synth_
}  // namespace ddsp
