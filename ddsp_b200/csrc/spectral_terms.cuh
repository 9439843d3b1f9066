// Every spectrogram term of losses.SpectralLoss (losses.py:194-234) for one FFT
// size, 'L1' or 'L2', in one pass over the target and value STFTs [B, T, F]:
//   mag          m                        [B, T,   F]
//   delta_time   core.diff(m, axis=1)     [B, T-1, F]
//   delta_freq   core.diff(m, axis=2)     [B, T,   F-1]
//   cumsum_freq  cumsum(m, axis=2)        [B, T,   F]
//   logmag       safe_log(m)              [B, T,   F]
// Each active term adds its sum of |d| (L1) or d^2 (L2), d = target - value, to its
// float64 slot of `sums`, and its share of the gradient of
//   sum_term weight_term * mean(term)
// w.r.t. X_v goes to `grad`, pre-scaled for an unnormalised inverse rfft
// (spectral_l1's irfft_size = -1).
//
// Layout: a CTA owns `rows` consecutive whole frames of one item (at least one,
// about kTileBins bins).  It stages both magnitude rows in shared memory, plus one
// halo frame on each side when delta_time is active, so the frame differences at
// its edges need no second kernel.  delta_freq and cumsum_freq are row-local; the
// cumsum is a segmented block scan of m_t - m_v, and its gradient a segmented
// suffix scan of the per-bin derivative.  The halo frames belong to neighbouring
// CTAs, so with delta_time the gradient must not overwrite either STFT; without
// it every element is read before the same CTA writes it, and grad may be X_v.
//
// Conventions of spectral_l1: |X| = sqrtf(re^2 + im^2); a bin with |X_v| = 0 gets
// no gradient; safe_log(m) = log(m <= 0 ? 1e-5 : m), with no gradient there.
// Summation: each thread adds its terms in double, a CTA reduces them in a fixed
// order and adds one double atomic per term, as spectral_l1 does; only the order of
// those CTA partials varies between runs.  The gradient uses no atomics.
#pragma once
#include <algorithm>

#include "common.cuh"

namespace ddsp {
namespace st_ {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kTileBins = 4096;
constexpr int kMaxBins = DDSP_B200_SPECTRAL_TERMS_MAX_BINS;
constexpr float kEps = 1e-5f;   // core.safe_log

enum {
  kMag = DDSP_B200_TERM_MAG,
  kDeltaTime = DDSP_B200_TERM_DELTA_TIME,
  kDeltaFreq = DDSP_B200_TERM_DELTA_FREQ,
  kCumsumFreq = DDSP_B200_TERM_CUMSUM_FREQ,
  kLogmag = DDSP_B200_TERM_LOGMAG,
  kAllTerms = 31
};

// Per-term weight / element count, indexed by the term's bit.
struct Coeffs {
  float c[5];
};

// d loss / d value of one element, before the weight / count
template <bool L2>
__device__ __forceinline__ float dphi(float d) {
  if (L2) return 2.f * d;
  return (d > 0.f) ? 1.f : (d < 0.f ? -1.f : 0.f);
}
template <bool L2>
__device__ __forceinline__ double err(float d) {
  return L2 ? (double)(d * d) : (double)fabsf(d);
}

// In-place inclusive scan of a[0, n) in segments of F elements (each frame row);
// REV scans every segment from its end.  Thread i scans one contiguous chunk; the
// chunks' (starts-a-segment, total) pairs are combined across the block.  Fixed
// order throughout.
template <bool REV>
__device__ void segmented_scan(float* a, int n, int F) {
  __shared__ float w_tot[kWarps];
  __shared__ int w_flag[kWarps];
  const int per = (n + kThreads - 1) / kThreads;
  const int lo = threadIdx.x * per, hi = min(n, lo + per);
  // position j of this chunk in scan order is element REV ? n-1-j : j
  float run = 0.f;
  int flag = 0;
  for (int j = lo; j < hi; ++j) {
    const int i = REV ? n - 1 - j : j;
    const bool start = REV ? (i + 1) % F == 0 : i % F == 0;
    if (start) { run = 0.f; flag = 1; }
    run += a[i];
    a[i] = run;
  }
  // exclusive segmented scan of (flag, run) over threads
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float v = run;
  int f = flag;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float pv = __shfl_up_sync(0xffffffffu, v, o);
    const int pf = __shfl_up_sync(0xffffffffu, f, o);
    if (lane >= o) {
      if (!f) v += pv;
      f |= pf;
    }
  }
  if (lane == 31) { w_tot[warp] = v; w_flag[warp] = f; }
  __syncthreads();
  // carry into this warp from the warps before it
  float carry = 0.f;
  for (int w = warp - 1; w >= 0; --w) {
    carry += w_tot[w];
    if (w_flag[w]) break;
  }
  // exclusive value for this thread: inclusive of lane-1, plus the warp carry unless
  // a segment started earlier in this warp
  float ex = __shfl_up_sync(0xffffffffu, v, 1);
  int exf = __shfl_up_sync(0xffffffffu, f, 1);
  if (lane == 0) { ex = 0.f; exf = 0; }
  if (!exf) ex += carry;
  for (int j = lo; j < hi; ++j) {
    const int i = REV ? n - 1 - j : j;
    const bool start = REV ? (i + 1) % F == 0 : i % F == 0;
    if (start) break;
    a[i] += ex;
  }
  __syncthreads();
}

template <int TERMS, bool L2>
__global__ void __launch_bounds__(kThreads)
spectral_terms_kernel(const float2* __restrict__ xt, const float2* xv, float2* grad,
                      double* __restrict__ sums, int T, int F, int rows, Coeffs k) {
  constexpr bool MAG = TERMS & kMag, DT = TERMS & kDeltaTime, DF = TERMS & kDeltaFreq,
                 CS = TERMS & kCumsumFreq, LOG = TERMS & kLogmag;
  extern __shared__ float smem[];
  // local row r + 1 holds frame t0 + r; rows 0 and nr + 1 are the halo frames
  float* mt = smem;
  float* mv = mt + (size_t)(rows + 2) * F;
  float* cs = mv + (size_t)(rows + 2) * F;
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * rows;
  const int nr = min(rows, T - t0);
  const size_t item = (size_t)b * T * F;

  const int e_lo = DT ? 0 : F, e_hi = (nr + (DT ? 2 : 1)) * F;
  for (int e = e_lo + threadIdx.x; e < e_hi; e += kThreads) {
    const int t = t0 - 1 + e / F;
    float a = 0.f, c = 0.f;
    if (t >= 0 && t < T) {
      const size_t g = item + (size_t)t * F + (e % F);
      const float2 p = xt[g], q = xv[g];
      a = sqrtf(p.x * p.x + p.y * p.y);
      c = sqrtf(q.x * q.x + q.y * q.y);
    }
    mt[e] = a;
    mv[e] = c;
  }
  __syncthreads();

  const int n = nr * F;
  double acc[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  if (CS) {
    for (int i = threadIdx.x; i < n; i += kThreads) cs[i] = mt[F + i] - mv[F + i];
    __syncthreads();
    segmented_scan<false>(cs, n, F);
    for (int i = threadIdx.x; i < n; i += kThreads) {
      const float d = cs[i];
      acc[3] += err<L2>(d);
      cs[i] = -k.c[3] * dphi<L2>(d);
    }
    __syncthreads();
    segmented_scan<true>(cs, n, F);
  }

  for (int i = threadIdx.x; i < n; i += kThreads) {
    const int r = i / F, f = i - r * F, t = t0 + r;
    const int e = F + i;
    const float a = mt[e], c = mv[e];
    float dm = 0.f;   // d loss / d m_v
    if (MAG) {
      const float d = a - c;
      acc[0] += err<L2>(d);
      dm -= k.c[0] * dphi<L2>(d);
    }
    if (DT) {
      if (t + 1 < T) {
        const float d = (mt[e + F] - a) - (mv[e + F] - c);
        acc[1] += err<L2>(d);
        dm += k.c[1] * dphi<L2>(d);
      }
      if (t > 0) dm -= k.c[1] * dphi<L2>((a - mt[e - F]) - (c - mv[e - F]));
    }
    if (DF) {
      if (f + 1 < F) {
        const float d = (mt[e + 1] - a) - (mv[e + 1] - c);
        acc[2] += err<L2>(d);
        dm += k.c[2] * dphi<L2>(d);
      }
      if (f > 0) dm -= k.c[2] * dphi<L2>((a - mt[e - 1]) - (c - mv[e - 1]));
    }
    if (CS) dm += cs[i];
    if (LOG) {
      const float d = logf(a <= 0.f ? kEps : a) - logf(c <= 0.f ? kEps : c);
      acc[4] += err<L2>(d);
      if (c > 0.f) dm -= k.c[4] * dphi<L2>(d) / c;
    }
    // d/dX_v = dm X_v / |X_v|, halved off DC and Nyquist for the unnormalised irfft
    const size_t g = item + (size_t)t0 * F + i;
    const float2 q = xv[g];
    float s = 0.f;
    if (c > 0.f) s = dm / c * ((f == 0 || f == F - 1) ? 1.f : 0.5f);
    grad[g] = make_float2(s * q.x, s * q.y);
  }

  __shared__ double red[5][kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    if (!(TERMS & (1 << j))) continue;
    double s = acc[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[j][warp] = s;
  }
  __syncthreads();
  if (threadIdx.x < 5 && (TERMS & (1 << threadIdx.x))) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += red[threadIdx.x][w];
    atomicAdd(sums + threadIdx.x, s);
  }
}

using Kernel = void (*)(const float2*, const float2*, float2*, double*, int, int, int, Coeffs);

// The instantiation for one set of terms (1..kAllTerms) and loss type.
template <int TERMS>
Kernel pick(int terms, bool l2) {
  if (terms == TERMS) return l2 ? spectral_terms_kernel<TERMS, true> : spectral_terms_kernel<TERMS, false>;
  if constexpr (TERMS < kAllTerms) return pick<TERMS + 1>(terms, l2);
  return nullptr;
}

// Frames per CTA for F bins, and the shared memory it stages.
inline int tile_rows(int T, int F) { return std::max(1, std::min(T, kTileBins / F)); }
inline size_t tile_smem(int rows, int F, int terms) {
  return sizeof(float) * (size_t)F * (2 * (rows + 2) + ((terms & kCumsumFreq) ? rows : 0));
}

}  // namespace st_
}  // namespace ddsp
