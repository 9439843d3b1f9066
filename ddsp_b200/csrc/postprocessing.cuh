// Adjusting controls for tone transfer (training/postprocessing.py and the tuning helpers
// of colab/colab_utils.py): detect_notes and smooth, the quantile fit and transform of
// QuantileTransformer, get_tuning_factor and auto_tune.
//
// The reference runs these in numpy and scipy on the host, with one tf.nn.conv1d.  Each
// kernel here repeats its numpy operation sequence step by step, so that the results are
// the reference's bits where numpy's are defined bit for bit:
//   * no contraction into FMA where numpy rounds a product before adding it
//     (__dmul_rn / __dadd_rn, __fmul_rn / __fadd_rn);
//   * float32 steps of the reference stay float32 steps here (the inputs arrive as
//     doubles widened exactly from float32, and a flag rounds every step back);
//   * reductions whose order numpy fixes (axis-0 means: row by row) keep that order.
// Every kernel is forward only and uses no atomics: results are bit-reproducible.
#pragma once
#include <float.h>
#include <math_constants.h>

#include "common.cuh"

namespace ddsp {
namespace post_ {

constexpr int kThreads = 256;
constexpr int kPartials = 1024;        // most partial sums of detect_notes' global mean
constexpr int64_t kMinChunk = 4096;    // fewest frames per partial sum

// ---- detect_notes / smooth -----------------------------------------------------------
struct DetectParams {
  const double* loud;    // [n] loudness (dB), widened from float32 or float64
  const double* conf;    // [n] f0 confidence (or smooth's input)
  double* ratio;         // [n] out: note_on_ratio, or the smoothed signal
  uint8_t* mask;         // [n] out: ratio >= note_threshold (not in smooth mode)
  double* partial;       // workspace [kPartials]: sums of loudness over fixed chunks
  float* powed;          // workspace [n]: float32(conf ** exponent), smooth's input
  int64_t n, chunk;
  int T, k, n_partials, flags;
  double exponent, weight, min_db, note_threshold;
};

// numpy's x ** e for a float array and a Python scalar exponent: its fast paths for
// 2, 0.5, 1, -1 and 0, else pow.  In float32 (f32) or float64.
__device__ __forceinline__ double np_power(double x, double e, bool f32) {
  if (f32) {
    const float v = (float)x;
    if (e == 2.0) return __fmul_rn(v, v);
    if (e == 0.5) return __fsqrt_rn(v);
    if (e == 1.0) return v;
    if (e == -1.0) return __frcp_rn(v);
    if (e == 0.0) return 1.0f;
    return (float)pow((double)v, e);
  }
  if (e == 2.0) return __dmul_rn(x, x);
  if (e == 0.5) return __dsqrt_rn(x);
  if (e == 1.0) return x;
  if (e == -1.0) return __drcp_rn(x);
  if (e == 0.0) return 1.0;
  return pow(x, e);
}

// Pass 1: smooth's float32 input and the loudness sum of each fixed chunk (thread-strided
// double sums, then a fixed tree).
__global__ void __launch_bounds__(kThreads) detect_prepare_kernel(DetectParams p) {
  __shared__ double red[kThreads];
  const bool smooth_only = p.flags & DDSP_B200_DETECT_SMOOTH_ONLY;
  const bool conf_f32 = p.flags & DDSP_B200_DETECT_CONF_F32;
  const int64_t lo = (int64_t)blockIdx.x * p.chunk;
  const int64_t hi = min(p.n, lo + p.chunk);
  double s = 0.0;
  for (int64_t i = lo + threadIdx.x; i < hi; i += kThreads) {
    const double c = p.conf[i];
    p.powed[i] = smooth_only ? (float)c : (float)np_power(c, p.exponent, conf_f32);
    if (!smooth_only) s = __dadd_rn(s, p.loud[i]);
  }
  if (smooth_only) return;
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = kThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + w]);
    __syncthreads();
  }
  if (threadIdx.x == 0) p.partial[blockIdx.x] = red[0];
}

// Pass 2: every CTA reduces the partial sums in the same fixed order (so all agree on the
// mean), then each frame's box filter (TF 'SAME': (k-1)/2 zero taps on the left) in
// float32, tap by tap, and its ratio.
__global__ void __launch_bounds__(kThreads) detect_notes_kernel(DetectParams p) {
  __shared__ double red[kThreads];
  const bool smooth_only = p.flags & DDSP_B200_DETECT_SMOOTH_ONLY;
  const bool loud_f32 = p.flags & DDSP_B200_DETECT_LOUD_F32;
  double mean = 0.0;
  if (!smooth_only) {
    double s = 0.0;
    for (int i = threadIdx.x; i < p.n_partials; i += kThreads) s = __dadd_rn(s, p.partial[i]);
    red[threadIdx.x] = s;
    __syncthreads();
    for (int w = kThreads / 2; w > 0; w >>= 1) {
      if (threadIdx.x < w) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + w]);
      __syncthreads();
    }
    mean = __ddiv_rn(red[0], (double)p.n);
  }
  const float w = __fdiv_rn(1.0f, (float)p.k);
  const int left = (p.k - 1) / 2;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < p.n;
       i += (int64_t)gridDim.x * kThreads) {
    const int t = (int)(i % p.T);
    const float* row = p.powed + (i - t);
    float s = 0.0f;
    for (int j = 0; j < p.k; ++j) {
      const int c = t - left + j;
      const float v = (c >= 0 && c < p.T) ? row[c] : 0.0f;
      s = __fadd_rn(s, __fmul_rn(v, w));
    }
    if (smooth_only) {
      p.ratio[i] = s;
      continue;
    }
    bool on;
    if (loud_f32) {
      const float md = (float)p.min_db;
      const float thr = __fmul_rn(__fsub_rn((float)mean, md), (float)p.weight);
      const float r = __fdiv_rn(__fmul_rn(s, __fsub_rn((float)p.loud[i], md)), thr);
      p.ratio[i] = r;
      on = r >= (float)p.note_threshold;
    } else {
      const double thr = __dmul_rn(__dsub_rn(mean, p.min_db), p.weight);
      const double r = __ddiv_rn(__dmul_rn((double)s, __dsub_rn(p.loud[i], p.min_db)), thr);
      p.ratio[i] = r;
      on = r >= p.note_threshold;
    }
    p.mask[i] = on;
  }
}

// ---- QuantileTransformer: fit ----------------------------------------------------------
// np.nanpercentile(col, references * 100) by numpy 2.3's linear method on a sorted
// column of n non-NaN values: virtual index (n - 1) q, neighbours floor / floor + 1
// (both n - 1 at or past the end, where numpy's gamma is v - (-1)), and _lerp: b - a in
// the input dtype, a + d t, or b - d (1 - t) where t >= 0.5, in float64.  Then
// np.maximum.accumulate down the column.
struct FitParams {
  const double* sorted;   // [F, n_rows] each column ascending, NaN last
  const int64_t* counts;  // [F] non-NaN values per column
  const double* q;        // [nq] references_ (percent / 100, as numpy forms it)
  double* quantiles;      // [nq, F] out
  int64_t n_rows;
  int F, nq, f32;
};

__global__ void __launch_bounds__(kThreads) quantile_fit_kernel(FitParams p) {
  const int f = blockIdx.x;
  const double* col = p.sorted + (int64_t)f * p.n_rows;
  const int64_t n = p.counts[f];
  for (int i = threadIdx.x; i < p.nq; i += kThreads) {
    double r;
    if (n == 0) {
      r = __longlong_as_double(0x7ff8000000000000ll);
    } else {
      const double v = __dmul_rn((double)(n - 1), p.q[i]);
      double prev = floor(v);
      int64_t ia, ib;
      if (v >= (double)(n - 1)) {
        prev = -1.0;
        ia = ib = n - 1;
      } else if (v < 0.0) {
        prev = 0.0;
        ia = ib = 0;
      } else {
        ia = (int64_t)prev;
        ib = ia + 1;
      }
      const double t = __dsub_rn(v, prev);
      const double a = col[ia], b = col[ib];
      const double d = p.f32 ? (double)__fsub_rn((float)b, (float)a) : __dsub_rn(b, a);
      r = t >= 0.5 ? __dsub_rn(b, __dmul_rn(d, __dsub_rn(1.0, t)))
                   : __dadd_rn(a, __dmul_rn(d, t));
    }
    p.quantiles[(int64_t)i * p.F + f] = r;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double m = p.quantiles[f];
    for (int i = 1; i < p.nq; ++i) {
      double* x = p.quantiles + (int64_t)i * p.F + f;
      // np.maximum(m, x): m where m > x or m is NaN, else x (x on ties, so -0 / +0
      // resolve as numpy's do)
      m = (m > *x || isnan(m)) ? m : *x;
      *x = m;
    }
  }
}

// ---- QuantileTransformer: transform ----------------------------------------------------
struct TransformParams {
  const double* x;          // [n, F]
  const double* quantiles;  // [nq, F]
  const double* references; // [nq]
  double* out;              // [n, F]
  int64_t n;
  int F, nq, inverse, normal, f32;
};

// np.interp(x, xp, fp) for non-NaN x (numpy's arr_interp with left / right defaults):
// j is the last knot with xp[j] <= x; an exactly hit knot and the last knot give fp[j];
// otherwise slope (x - xp[j]) + fp[j], retried from the right knot when that is NaN, and
// fp[j] when both are NaN and fp[j] == fp[j + 1].  With `flip` the knots are (-xp, -fp)
// reversed, as _transform_col's descending pass passes them.
__device__ double np_interp(double x, const double* xp0, const double* fp0, int m, bool flip) {
  auto xp = [&](int j) { return flip ? -xp0[m - 1 - j] : xp0[j]; };
  auto fp = [&](int j) { return flip ? -fp0[m - 1 - j] : fp0[j]; };
  if (m == 1) return fp(0);   // left, right and the knot's value are all fp[0]
  if (x > xp(m - 1)) return fp(m - 1);
  if (x < xp(0)) return fp(0);
  int lo = 0, hi = m;
  while (lo < hi) {
    const int mid = lo + ((hi - lo) >> 1);
    if (x >= xp(mid)) lo = mid + 1;
    else hi = mid;
  }
  // NaN knots (a column fitted on no values) compare false everywhere: numpy's search
  // then lands on an inner knot, whose NaN slope gives NaN below
  const int j = max(lo - 1, 0);
  if (j == m - 1) return fp(j);
  const double xj = xp(j), fj = fp(j), xj1 = xp(j + 1), fj1 = fp(j + 1);
  if (xj == x) return fj;
  const double slope = __ddiv_rn(__dsub_rn(fj1, fj), __dsub_rn(xj1, xj));
  double r = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, xj)), fj);
  if (isnan(r)) {
    r = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, xj1)), fj1);
    if (isnan(r) && fj == fj1) r = fj;
  }
  return r;
}

// _transform_col for element (row, column): the bounds tests on the input, the
// interpolation (forward: the mean of the ascending and the negated descending pass),
// the bounds, and for 'normal' the norm.ppf / norm.cdf and the clip.
__global__ void __launch_bounds__(kThreads) quantile_transform_kernel(TransformParams p) {
  extern __shared__ double sm[];
  const int f = blockIdx.y;
  double* qs = sm;
  double* refs = sm + p.nq;
  for (int i = threadIdx.x; i < p.nq; i += kThreads) {
    qs[i] = p.quantiles[(int64_t)i * p.F + f];
    refs[i] = p.references[i];
  }
  __syncthreads();
  const double q0 = qs[0], qn = qs[p.nq - 1];
  const double thr = 1e-7;
  // the 'normal' clip: norm.ppf(1e-7 - eps) and norm.ppf(1 - (1e-7 - eps))
  const double clip_min = normcdfinv(__dsub_rn(thr, DBL_EPSILON));
  const double clip_max = normcdfinv(__dsub_rn(1.0, __dsub_rn(thr, DBL_EPSILON)));
  for (int64_t r = (int64_t)blockIdx.x * kThreads + threadIdx.x; r < p.n;
       r += (int64_t)gridDim.x * kThreads) {
    double x = p.x[r * p.F + f];
    double y;
    bool lo, hi;
    if (!p.inverse) {
      if (p.normal) {
        if (p.f32) {   // float32 x_col -/+ 1e-7 (a weak Python float), compared in double
          lo = (double)__fsub_rn((float)x, (float)thr) < q0;
          hi = (double)__fadd_rn((float)x, (float)thr) > qn;
        } else {
          lo = __dsub_rn(x, thr) < q0;
          hi = __dadd_rn(x, thr) > qn;
        }
      } else {
        lo = x == q0;
        hi = x == qn;
      }
      y = x;
      if (!isnan(x)) {
        y = __dmul_rn(0.5, __dsub_rn(np_interp(x, qs, refs, p.nq, false),
                                     np_interp(-x, qs, refs, p.nq, true)));
        if (p.f32) y = (float)y;   // written back into the float32 column
      }
      if (hi) y = 1.0;
      if (lo) y = 0.0;
      if (p.normal) {
        // scipy's norm.ppf: -inf at 0, inf at 1, NaN outside [0, 1]; then np.clip
        // (scipy's float32 loop of ndtri rounds to float32)
        y = (y > 0.0 && y < 1.0) ? (p.f32 ? (double)(float)normcdfinv(y) : normcdfinv(y))
            : y == 0.0 ? -CUDART_INF : y == 1.0 ? CUDART_INF : CUDART_NAN;
        if (!isnan(y)) y = fmin(fmax(y, clip_min), clip_max);
      }
    } else {
      if (p.normal) {
        x = isnan(x) ? x : x == -CUDART_INF ? 0.0 : x == CUDART_INF ? 1.0 : normcdf(x);
        lo = __dsub_rn(x, thr) < 0.0;
        hi = __dadd_rn(x, thr) > 1.0;
      } else {
        lo = x == 0.0;
        hi = x == 1.0;
      }
      y = isnan(x) ? x : np_interp(x, refs, qs, p.nq, false);
      if (hi) y = qn;
      if (lo) y = q0;
    }
    p.out[r * p.F + f] = y;
  }
}

// ---- get_tuning_factor -----------------------------------------------------------------
// numpy's float64 `a % 1.0`: fmod (exact here as a - trunc(a)), + 1 where negative, +0
// where zero.
__device__ __forceinline__ double np_mod1(double a) {
  double m = __dsub_rn(a, trunc(a));
  if (m != 0.0) {
    if (m < 0.0) m = __dadd_rn(m, 1.0);
  } else {
    m = 0.0;
  }
  return m;
}

__device__ __forceinline__ float np_mod1f(float a) {
  float m = __fsub_rn(a, truncf(a));
  if (m != 0.0f) {
    if (m < 0.0f) m = __fadd_rn(m, 1.0f);
  } else {
    m = 0.0f;
  }
  return m;
}

// midi_diffs of one frame and factor: (f0 - factor) % 1, less 1 above 0.5.
__device__ __forceinline__ double midi_diff(double f0, double factor) {
  double d = np_mod1(__dsub_rn(f0, factor));
  return d > 0.5 ? __dsub_rn(d, 1.0) : d;
}

struct TuningParams {
  const double* f0;        // [N] f0_midi[mask_on]
  const double* conf;      // [N] f0_confidence[mask_on]
  const double* factors;   // [n_factors]
  double* costs;           // [2, n_factors] out: cost_diffs, cost_deltas
  int* index;              // [1] out: np.argmin of the normalised cost
  int64_t N;
  int n_factors;
};

// One CTA per factor: each chunk's terms in parallel, then summed row by row in one
// thread (numpy's axis-0 mean adds the rows in order).
__global__ void __launch_bounds__(kThreads) tuning_costs_kernel(TuningParams p) {
  __shared__ double term_d[kThreads], term_w[kThreads];
  const double factor = p.factors[blockIdx.x];
  double sum_d = 0.0, sum_w = 0.0;
  for (int64_t base = 0; base < p.N; base += kThreads) {
    const int64_t i = base + threadIdx.x;
    if (i < p.N) {
      const double f = p.f0[i], w = p.conf[i];
      const double d = midi_diff(f, factor);
      term_d[threadIdx.x] = __dmul_rn(w, fabs(d));
      if (i + 1 < p.N) {
        const double f1 = p.f0[i + 1];
        const double at = __dsub_rn(f, d), at1 = __dsub_rn(f1, midi_diff(f1, factor));
        term_w[threadIdx.x] = __dmul_rn(w, __dsub_rn(at1, at) != 0.0 ? 1.0 : 0.0);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const int64_t len = min((int64_t)kThreads, p.N - base);
      const int64_t len_w = min((int64_t)kThreads, p.N - 1 - base);
      for (int j = 0; j < len; ++j) sum_d = __dadd_rn(sum_d, term_d[j]);
      for (int j = 0; j < len_w; ++j) sum_w = __dadd_rn(sum_w, term_w[j]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    p.costs[blockIdx.x] = __ddiv_rn(sum_d, (double)p.N);
    p.costs[p.n_factors + blockIdx.x] = __ddiv_rn(sum_w, (double)max(p.N - 1, (int64_t)0));
  }
}

// numpy's pairwise sum of n <= 128 doubles: below 8 in order, else eight strided
// accumulators combined as ((0+1)+(2+3))+((4+5)+(6+7)), then the tail in order.
__device__ double np_pairwise_sum(const double* x, int n) {
  if (n < 8) {
    double s = -0.0;
    for (int i = 0; i < n; ++i) s = __dadd_rn(s, x[i]);
    return s;
  }
  double r[8];
  for (int j = 0; j < 8; ++j) r[j] = x[j];
  int i = 8;
  for (; i < n - (n % 8); i += 8)
    for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], x[i + j]);
  double s = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                       __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < n; ++i) s = __dadd_rn(s, x[i]);
  return s;
}

// (x - mean(x)) / std(x) into y, numpy's mean and population std.
__device__ void np_normalise(const double* x, double* y, double* tmp, int n) {
  const double mean = __ddiv_rn(np_pairwise_sum(x, n), (double)n);
  for (int i = 0; i < n; ++i) {
    const double d = __dsub_rn(x[i], mean);
    tmp[i] = __dmul_rn(d, d);
  }
  const double sd = __dsqrt_rn(__ddiv_rn(np_pairwise_sum(tmp, n), (double)n));
  for (int i = 0; i < n; ++i) y[i] = __ddiv_rn(__dsub_rn(x[i], mean), sd);
}

// np.argmin: the first minimum, or the first NaN.
__device__ __forceinline__ int np_argmin(const double* x, int n) {
  int best = 0;
  double m = x[0];
  if (isnan(m)) return 0;
  for (int i = 1; i < n; ++i) {
    if (isnan(x[i])) return i;
    if (x[i] < m) {
      m = x[i];
      best = i;
    }
  }
  return best;
}

__global__ void tuning_argmin_kernel(TuningParams p) {
  __shared__ double a[DDSP_B200_TUNING_MAX_FACTORS], b[DDSP_B200_TUNING_MAX_FACTORS],
      tmp[DDSP_B200_TUNING_MAX_FACTORS];
  if (threadIdx.x != 0) return;
  const int n = p.n_factors;
  np_normalise(p.costs + n, a, tmp, n);   // cost_deltas
  np_normalise(p.costs, b, tmp, n);       // cost_diffs
  for (int i = 0; i < n; ++i) a[i] = __dadd_rn(a[i], b[i]);
  p.index[0] = np_argmin(a, n);
}

// ---- auto_tune -------------------------------------------------------------------------
// The major scales: note n of scale s is 12 (n / 7) + {0,2,4,5,7,9,11}[n % 7] + s.
__device__ __forceinline__ double scale_note(int s, int n) {
  const int steps[7] = {0, 2, 4, 5, 7, 9, 11};
  return (double)(12 * (n / 7) + steps[n % 7] + s);
}

struct AutoTuneParams {
  const double* f0;        // [T] f0_midi
  const double* f0_on;     // [N] f0_midi[mask_on] (scale mode)
  double* scale_cost;      // [12] out: mean over the masked frames of the distance
  int* scale_index;        // [1] out: np.argmin(scale_cost)
  double* out;             // [T] out
  int64_t T, N;
  double tuning_factor, amount;
  int chromatic, f32;
};

// Distance of f0 to the nearest note of scale s (NaN propagates, as np.min does).
__device__ __forceinline__ double scale_distance(double f, int s) {
  double m = fabs(__dsub_rn(f, scale_note(s, 0)));
  for (int n = 1; n < DDSP_B200_SCALE_NOTES; ++n) {
    const double d = fabs(__dsub_rn(f, scale_note(s, n)));
    m = (isnan(m) || m < d) ? m : d;
  }
  return m;
}

// One CTA per scale: the masked frames' distances, summed frame by frame.
__global__ void __launch_bounds__(kThreads) scale_costs_kernel(AutoTuneParams p) {
  __shared__ double term[kThreads];
  const int s = blockIdx.x;
  double sum = 0.0;
  for (int64_t base = 0; base < p.N; base += kThreads) {
    const int64_t i = base + threadIdx.x;
    if (i < p.N) term[threadIdx.x] = scale_distance(p.f0_on[i], s);
    __syncthreads();
    if (threadIdx.x == 0) {
      const int64_t len = min((int64_t)kThreads, p.N - base);
      for (int j = 0; j < len; ++j) sum = __dadd_rn(sum, term[j]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) p.scale_cost[s] = __ddiv_rn(sum, (double)p.N);
}

// Every frame: chromatic, (f0 - tuning_factor) % 1 less 1 above 0.5; else the
// difference to its nearest note (the first on ties) of the scale with the smallest
// cost.  Then f0 - amount * midi_diff.
__global__ void __launch_bounds__(kThreads) auto_tune_kernel(AutoTuneParams p) {
  int s = 0;
  if (!p.chromatic) {
    s = np_argmin(p.scale_cost, 12);
    if (blockIdx.x == 0 && threadIdx.x == 0) p.scale_index[0] = s;
  }
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < p.T;
       i += (int64_t)gridDim.x * kThreads) {
    const double f = p.f0[i];
    if (p.chromatic && p.f32) {
      const float ff = (float)f;
      float d = np_mod1f(__fsub_rn(ff, (float)p.tuning_factor));
      if (d > 0.5f) d = __fsub_rn(d, 1.0f);
      p.out[i] = __fsub_rn(ff, __fmul_rn((float)p.amount, d));
      continue;
    }
    double d;
    if (p.chromatic) {
      d = midi_diff(f, p.tuning_factor);
    } else {
      int best = 0;
      double m = fabs(__dsub_rn(f, scale_note(s, 0)));
      for (int n = 1; n < DDSP_B200_SCALE_NOTES; ++n) {
        const double a = fabs(__dsub_rn(f, scale_note(s, n)));
        if (!isnan(m) && (isnan(a) || a < m)) {
          m = a;
          best = n;
        }
      }
      d = __dsub_rn(f, scale_note(s, best));
    }
    p.out[i] = __dsub_rn(f, __dmul_rn(p.amount, d));
  }
}

}  // namespace post_
}  // namespace ddsp
