// core.harmonic_oscillator_bank (core.py:966-1025): one audio-rate f0 [B, N] drives K
// harmonics with amplitude envelopes [B, N, K] and a carried phase,
//   phi_t = init + (2 pi / sr) sum_{u<=t} f_u,   y_t = sum_k a_{t,k} sin(k phi_t),
// with no Nyquist mask (the reference has none here).
//
// The phase is the oscillator bank's: 64-bit fixed-point turns, each sample's
// turns_to_fix64(f / sr) added with wrapping (exact) adds, plus the initial phase as
// harmonic.cuh's streaming kernel adds it.  Harmonic k's phase is the wrapping integer
// product k P, so it wraps exactly modulo one turn, and sin is fix64_sin's.  Wrapping sums
// are exact in any order, so every kernel below gets the same P_t however it splits time.
// Neither direction needs a workspace.
//
// Forward, one launch: a CTA per span of samples (at most kMaxSpans spans per item) sums the
// terms of all earlier samples itself (f is read again from L2: about kMaxSpans / 2 reads
// of f per sample, against K of the amplitudes), then scans its span kChunk samples at a
// time into shared memory; its warps walk the rows with lanes over k, so the amplitude
// reads are coalesced rows, and there is one phase scan per item, not per harmonic.  The
// last span's CTA writes final_phase; for use_angular_cumsum=False it also counts whole
// turns (term128), so the unwrapped sum is exact before its one rounding.
//
// Backward (TensorFlow's gradients; floormod passes gradient 1), with
// c_t = g_t sum_k k a_{t,k} cos(k phi_t):
//   d a_{t,k} = g_t sin(k phi_t),   d f_t = (2 pi / sr) (sum_{u>=t} c_u + g_phi),
//   d init = sum_u c_u + g_phi.
// One cluster of kCl CTAs per item, as oscbank_backward: its kCl * kBwWarps warps split
// time into contiguous segments, exchange phase totals (so d a is the gradient of the audio
// that was produced) and then totals of c in double, through shared and distributed shared
// memory in a fixed order.  Each warp walks its segment forward (d a, c_t) and, for d f,
// back again: c_t is the exact double product of g_t and a float row sum, which the first
// walk parks in d f's own element.  No atomics and no memset: every output is
// bit-reproducible.  Outputs that are not asked for are not computed (neither d f nor
// d init: no cosine and no exchange of c).
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"

namespace ddsp {
namespace hob_ {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kChunk = 1024;                 // samples one scan puts in shared memory
constexpr int kPer = kChunk / kThreads;      // consecutive samples per thread in a scan
constexpr int kMaxSpans = 128;               // forward CTAs per item at most
constexpr int kBwWarps = 16;
constexpr int kCl = 8;                       // the portable cluster size
constexpr int kSegs = kBwWarps * kCl;        // backward time segments per item

typedef unsigned __int128 u128;

// The samples each forward CTA covers (a multiple of kChunk), and the CTAs per item: at
// most kMaxSpans, none of them empty.
__host__ __device__ inline int span_len(int N) {
  const int chunks = (N + kChunk - 1) / kChunk;
  return (chunks + kMaxSpans - 1) / kMaxSpans * kChunk;
}
__host__ __device__ inline int n_spans(int N) {
  const int len = span_len(N);
  return (N + len - 1) / len;
}

// One sample's phase increment f / sr in turns, exactly as a 128-bit fixed-point number
// (2^64 = one turn): whole turns in the high word, turns_to_fix64's fraction below.
__device__ __forceinline__ u128 term128(float f, double inv_sr) {
  const double x = (double)f * inv_sr;
  const long long whole = __double2ll_rn(rint(x));
  return ((u128)(unsigned long long)whole << 64) +
         (u128)(__int128)(long long)turns_to_fix64(x);
}

__device__ __forceinline__ unsigned long long term64(float f, double inv_sr) {
  return turns_to_fix64((double)f * inv_sr);
}

__device__ __forceinline__ u128 shfl_xor128(u128 v, int o) {
  const unsigned long long lo = __shfl_xor_sync(0xffffffffu, (unsigned long long)v, o);
  const unsigned long long hi = __shfl_xor_sync(0xffffffffu, (unsigned long long)(v >> 64), o);
  return ((u128)hi << 64) | lo;
}

// Sum over the CTA (wrapping adds: exact in any order); every thread gets it.
__device__ __forceinline__ u128 block_sum128(u128 v, u128* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += shfl_xor128(v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  u128 s = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) s += red[w];
  return s;
}

__device__ __forceinline__ unsigned long long init_fix64(const float* init, int b) {
  return init ? turns_to_fix64((double)init[b] * 0.15915494309189535) : 0ull;
}

// The phase (base included) of samples [t0, t1), t1 - t0 <= kChunk, into sP; returns
// the phase after t1 - 1 to every thread.
__device__ __forceinline__ unsigned long long scan_chunk(const float* __restrict__ fb, int t0,
                                                         int t1, unsigned long long base,
                                                         double inv_sr, unsigned long long* sP,
                                                         unsigned long long* wtot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int s0 = t0 + kPer * threadIdx.x;
  unsigned long long incl[kPer];
  unsigned long long run = 0;
#pragma unroll
  for (int j = 0; j < kPer; ++j) {
    if (s0 + j < t1) run += term64(__ldg(fb + s0 + j), inv_sr);
    incl[j] = run;
  }
  unsigned long long scan = run;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long up = __shfl_up_sync(0xffffffffu, scan, o);
    if (lane >= o) scan += up;
  }
  __syncthreads();                       // the previous chunk's rows are done with sP
  if (lane == 31) wtot[warp] = scan;
  __syncthreads();
  unsigned long long before = base + scan - run, total = base;
  for (int w = 0; w < kWarps; ++w) {
    if (w < warp) before += wtot[w];
    total += wtot[w];
  }
#pragma unroll
  for (int j = 0; j < kPer; ++j)
    if (s0 + j < t1) sP[s0 + j - t0] = before + incl[j];
  __syncthreads();
  return total;
}

// audio [B, N]; final_phase [B] (or nullptr).  grid (B, n_spans(N)): the batch rides on x,
// so any B that fits in memory is taken.
__global__ void __launch_bounds__(kThreads)
hob_forward(const float* __restrict__ f, const float* __restrict__ a,
            const float* __restrict__ init, float* __restrict__ audio,
            float* __restrict__ final_phase, int N, int K, double inv_sr, int unwrapped) {
  __shared__ unsigned long long sP[kChunk];
  __shared__ u128 red[kWarps];
  __shared__ unsigned long long wtot[kWarps];
  const int b = blockIdx.x, sp = blockIdx.y, spans = gridDim.y;
  const int len = span_len(N);
  const int t_begin = sp * len, t_end = min(N, t_begin + len);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* fb = f + (size_t)b * N;
  // the earlier samples' phase; the last span counts whole turns too when final_phase
  // needs the unwrapped sum
  const bool last = sp == spans - 1;
  const bool wide = last && final_phase != nullptr && unwrapped;
  u128 before = 0;
  if (wide) {
    for (int t = threadIdx.x; t < t_begin; t += kThreads) before += term128(__ldg(fb + t), inv_sr);
  } else {
    unsigned long long acc = 0;
    for (int t = threadIdx.x; t < t_begin; t += kThreads) acc += term64(__ldg(fb + t), inv_sr);
    before = acc;
  }
  before = block_sum128(before, red);
  const unsigned long long p_init = init_fix64(init, b);
  unsigned long long P0 = p_init + (unsigned long long)before;
  u128 own = 0;                          // this span's terms, whole turns included (wide)
  for (int t0 = t_begin; t0 < t_end; t0 += kChunk) {
    const int t1 = min(t_end, t0 + kChunk);
    const unsigned long long P1 = scan_chunk(fb, t0, t1, P0, inv_sr, sP, wtot);
    for (int t = t0 + warp; t < t1; t += kWarps) {
      const unsigned long long P = sP[t - t0];
      const float* ar = a + ((size_t)b * N + t) * K;
      float acc = 0.f;
      for (int k = lane; k < K; k += 32)
        acc = fmaf(__ldg(ar + k), fix64_sin((unsigned long long)(k + 1) * P), acc);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) audio[(size_t)b * N + t] = acc;
    }
    P0 = P1;
  }
  if (!last || final_phase == nullptr) return;
  if (wide) {
    for (int t = t_begin + threadIdx.x; t < t_end; t += kThreads) own += term128(__ldg(fb + t), inv_sr);
    own = block_sum128(own, red);
  }
  if (threadIdx.x == 0) {
    // use_angular_cumsum: the wrapped sum in [0, 2 pi), else the unwrapped one; both plus
    // the initial phase (core.py:1003-1013)
    double turns = (double)(P0 - p_init) * 5.421010862427522e-20;   // 2^-64
    if (wide) {
      const u128 tot = before + own;
      turns = (double)(unsigned long long)tot * 5.421010862427522e-20 +
              (double)(long long)(unsigned long long)(tot >> 64);
    }
    const double init_rad = init ? (double)init[b] : 0.0;
    final_phase[b] = (float)(turns * 6.283185307179586 + init_rad);
  }
}

// Backward: one cluster of kCl CTAs per item (grid (kCl, B)).  g_phi, d f, d a and d init
// may each be nullptr.
__global__ void __cluster_dims__(kCl, 1, 1) __launch_bounds__(kBwWarps * 32)
hob_backward(const float* __restrict__ f, const float* __restrict__ a,
             const float* __restrict__ init, const float* __restrict__ g,
             const float* __restrict__ g_phi, float* __restrict__ df, float* __restrict__ da,
             float* __restrict__ d_init, int N, int K, double inv_sr, double scale) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  __shared__ unsigned long long ph_seg[kBwWarps], ph_cta;
  __shared__ double s_seg[kBwWarps], s_cta;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int rank = (int)cluster.block_rank();
  const int b = blockIdx.y;
  const int len = (N + kSegs - 1) / kSegs;
  const int t0 = min(N, (rank * kBwWarps + w) * len);
  const int t1 = t0 + min(len, N - t0);
  const size_t row0 = (size_t)b * N;
  const bool phase = df != nullptr || d_init != nullptr;

  // 1. the phase before the segment
  unsigned long long tot = 0;
  for (int t = t0 + lane; t < t1; t += 32) tot += term64(f[row0 + t], inv_sr);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
  if (lane == 0) ph_seg[w] = tot;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long c = 0;
    for (int v = 0; v < kBwWarps; ++v) c += ph_seg[v];
    ph_cta = c;
  }
  cluster.sync();
  unsigned long long ph = init_fix64(init, b);
  for (int q = 0; q < rank; ++q) ph += *cluster.map_shared_rank(&ph_cta, q);
  for (int v = 0; v < w; ++v) ph += ph_seg[v];

  // 2. forward walk: d a, c_t and the segment's total of c
  double seg = 0.0;
  for (int t = t0; t < t1; ++t) {
    const size_t row = row0 + t;
    ph += term64(f[row], inv_sr);
    const float gt = g[row];
    const float* ar = a + row * K;
    float acc = 0.f;
    for (int k = lane; k < K; k += 32) {
      const unsigned long long pk = (unsigned long long)(k + 1) * ph;
      if (da != nullptr) da[row * K + k] = gt * fix64_sin(pk);
      if (phase) acc = fmaf((float)(k + 1) * __ldg(ar + k), fix64_cos(pk), acc);
    }
    if (!phase) continue;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    seg += (double)gt * (double)acc;       // exact product
    if (df != nullptr && lane == 0) df[row] = acc;
  }
  if (!phase) {
    cluster.sync();                      // no CTA leaves while another reads its ph_cta
    return;
  }

  // 3. the later segments' totals, nearest last, then the walk back
  if (lane == 0) s_seg[w] = seg;
  __syncthreads();
  if (threadIdx.x == 0) {
    double c = 0.0;
    for (int v = 0; v < kBwWarps; ++v) c += s_seg[v];
    s_cta = c;
  }
  cluster.sync();
  double suf = g_phi != nullptr ? (double)g_phi[b] : 0.0;
  for (int q = kCl - 1; q > rank; --q) suf += *cluster.map_shared_rank(&s_cta, q);
  for (int v = kBwWarps - 1; v > w; --v) suf += s_seg[v];
  if (d_init != nullptr && rank == 0 && w == 0 && lane == 0) d_init[b] = (float)(suf + seg);
  if (df != nullptr && lane == 0) {
    for (int t = t1 - 1; t >= t0; --t) {
      const size_t row = row0 + t;
      suf += (double)g[row] * (double)df[row];
      df[row] = (float)(scale * suf);
    }
  }
  cluster.sync();                        // no CTA leaves while another reads its s_cta
}

}  // namespace hob_
}  // namespace ddsp
