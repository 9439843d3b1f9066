// core.oscillator_bank (core.py:911-962) as a stand-alone op on audio-rate
// envelopes [B, N, K] (what synths.Sinusoidal feeds it; SURVEY.md 8f-4).
//   amp = 0 where f >= sr/2; omega = f * 2 pi / sr; phi = cumsum_t(omega);
//   out = amp * sin(phi)  ([B,N,K]) or its sum over k ([B,N]).
// The cumsum is an exact wrapping sum of 64-bit fixed-point turns, done as a
// three-pass chunked scan (chunk = 128 samples): per-chunk totals, a scan of the
// totals per (b, k), then the running phase inside each chunk.  Threads run over
// k (the contiguous axis), so every global access is coalesced; the path is
// HBM-bound: f is read twice, amp once.
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"

namespace ddsp {

constexpr int kObChunk = 128;
constexpr int kObThreads = 128;

// pass 1: chunk totals.  grid (n_chunks, B), threads over k.
__global__ void __launch_bounds__(kObThreads)
oscbank_chunk_sums(const float* __restrict__ f, unsigned long long* __restrict__ sums,
                   int N, int K, int n_chunks, double inv_sr) {
  const int b = blockIdx.y, ch = blockIdx.x;
  const int t0 = ch * kObChunk, t1 = min(N, t0 + kObChunk);
  for (int k = threadIdx.x; k < K; k += kObThreads) {
    const float* fp = f + ((size_t)b * N + t0) * K + k;
    unsigned long long acc = 0;
    for (int t = t0; t < t1; ++t, fp += K) acc += turns_to_fix64((double)(*fp) * inv_sr);
    sums[((size_t)b * n_chunks + ch) * K + k] = acc;
  }
}

// pass 2: exclusive scan of the chunk totals along the chunk axis, in place.
__global__ void __launch_bounds__(kObThreads)
oscbank_scan_chunks(unsigned long long* __restrict__ sums, int K, int n_chunks,
                    int64_t BK) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= BK) return;
  const int64_t b = i / K;
  const int k = (int)(i - b * K);
  unsigned long long run = 0;
  unsigned long long* p = sums + (size_t)b * n_chunks * K + k;
  for (int ch = 0; ch < n_chunks; ++ch, p += K) {
    const unsigned long long v = *p;
    *p = run;
    run += v;
  }
}

// pass 3: running phase inside the chunk, sin, mask, optional sum over k.
template <bool SUM>
__global__ void __launch_bounds__(kObThreads)
oscbank_apply(const float* __restrict__ f, const float* __restrict__ a,
              const unsigned long long* __restrict__ offs, float* __restrict__ out,
              int N, int K, int n_chunks, double inv_sr, float nyquist) {
  __shared__ float partial[kObChunk][kObThreads / 32 + 1];
  const int b = blockIdx.y, ch = blockIdx.x;
  const int t0 = ch * kObChunk, t1 = min(N, t0 + kObChunk);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (SUM) {
    for (int i = threadIdx.x; i < kObChunk * (kObThreads / 32 + 1); i += kObThreads)
      (&partial[0][0])[i] = 0.f;
    __syncthreads();
  }
  for (int kb = 0; kb < K; kb += kObThreads) {
    const int k = kb + threadIdx.x;
    const bool live = k < K;
    unsigned long long ph = live ? offs[((size_t)b * n_chunks + ch) * K + k] : 0ull;
    const size_t base = ((size_t)b * N + t0) * K + (live ? k : 0);
    const float* fp = f + base;
    const float* ap = a + base;
    for (int t = t0; t < t1; ++t, fp += K, ap += K) {
      float v = 0.f;
      if (live) {
        const float fv = *fp;
        ph += turns_to_fix64((double)fv * inv_sr);
        const float s = fix64_sin(ph);
        v = (fv >= nyquist) ? 0.f : (*ap) * s;
        if (!SUM) out[((size_t)b * N + t) * K + k] = v;
      }
      if (SUM) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) partial[t - t0][warp] += v;
      }
    }
  }
  if (SUM) {
    __syncthreads();
    for (int i = threadIdx.x; i < t1 - t0; i += kObThreads) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < kObThreads / 32; ++w) s += partial[i][w];
      out[(size_t)b * N + t0 + i] = s;
    }
  }
}

// core.angular_cumsum (core.py:799-866) done exactly: pass 3 variant that writes
// the wrapped phase itself, in radians in [0, float32(2 pi)] (f is then the angular
// frequency in rad/sample and inv_sr = 1 / (2 pi)).
__global__ void __launch_bounds__(kObThreads)
oscbank_phase_out(const float* __restrict__ f, const unsigned long long* __restrict__ offs,
                  float* __restrict__ out, int N, int K, int n_chunks, double inv_sr) {
  const int b = blockIdx.y, ch = blockIdx.x;
  const int t0 = ch * kObChunk, t1 = min(N, t0 + kObChunk);
  for (int k = threadIdx.x; k < K; k += kObThreads) {
    unsigned long long ph = offs[((size_t)b * n_chunks + ch) * K + k];
    const size_t base = ((size_t)b * N + t0) * K + k;
    const float* fp = f + base;
    float* op = out + base;
    for (int t = t0; t < t1; ++t, fp += K, op += K) {
      ph += turns_to_fix64((double)(*fp) * inv_sr);
      *op = (float)((double)ph * 5.421010862427522e-20 * 6.283185307179586);   // 2^-64 turns -> rad
    }
  }
}

// ---- backward (TensorFlow's gradients of core.py:911-962 and 799-866) ----------
//   phi_t = (2 pi / sr) sum_{u<=t} f_u  (the forward's exact fixed-point phase),
//   m = [f < sr/2] (the forward's float32 decision; the mask passes no gradient):
//   d a[t,k] = g m sin(phi),   d f[t,k] = (2 pi / sr) sum_{u>=t} g_u a_u m_u cos(phi_u);
//   angular_cumsum: d omega[t] = sum_{u>=t} g_u (floormod has derivative 1).
// One cluster of kObbCluster CTAs per (b, tile of 32 oscillators); lane = oscillator,
// so every access is a coalesced row of 32 floats.  The cluster's 128 warps split time
// into contiguous segments, one per warp, in (rank, warp) order.  Segment totals cross
// warps through shared memory and CTAs through distributed shared memory, each added in
// a fixed order, so no workspace, atomic or memset is needed and the result is
// bit-reproducible:
//   1. the segment's fixed-point phase total (u64, exact); exchange -> phase at the
//      segment start;
//   2. walk forward: d a, and the segment total of g a m cos(phi) in double;
//      exchange -> suffix of the later segments;
//   3. walk backward from the segment's end phase (ph -= fix(f) is exact), adding
//      g a m cos(phi) in double; d f = float((2 pi / sr) * suffix), rounded once.
// The phase is the forward's: the same turns_to_fix64 terms, rounded to 2^-32 turn, and
// sin(phi) is the forward's sinpif, so d a is the gradient of the audio it produced and
// does not depend on whether d f is asked for.  Without d f, step 2's sum and step 3
// are skipped (no cosine); without d a, nothing is written in step 2.  KIND: SUM (g is [B, N]),
// FULL (g is [B, N, K]) or CUMSUM (angular_cumsum: no phase, d omega is written as d f).
constexpr int kObbLanes = 32;
constexpr int kObbWarps = 16;
constexpr int kObbCluster = 8;                       // the portable cluster size
constexpr int kObbSegs = kObbWarps * kObbCluster;    // time segments per (b, tile)
enum { kObbSum = 0, kObbFull = 1, kObbCumsum = 2 };

template <int KIND>
__global__ void __cluster_dims__(kObbCluster, 1, 1) __launch_bounds__(kObbLanes * kObbWarps)
oscbank_backward(const float* __restrict__ f, const float* __restrict__ a,
                 const float* __restrict__ g, float* __restrict__ df,
                 float* __restrict__ da, int N, int K, double inv_sr, float nyquist,
                 double scale) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  __shared__ unsigned long long ph_seg[kObbWarps][kObbLanes], ph_cta[kObbLanes];
  __shared__ double s_seg[kObbWarps][kObbLanes], s_cta[kObbLanes];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int rank = (int)cluster.block_rank();
  const int b = blockIdx.y;
  const int k = (blockIdx.x / kObbCluster) * kObbLanes + lane;
  const bool live = k < K;
  const int len = (N + kObbSegs - 1) / kObbSegs;
  const int t0 = min(N, (rank * kObbWarps + w) * len);
  const int t1 = t0 + min(len, N - t0);
  const size_t row0 = (size_t)b * N;
  // the term of d f at sample t, with the phase ph (inclusive of t)
  auto term = [&](int t, unsigned long long ph) -> double {
    const size_t i = (row0 + t) * K + k;
    const float gv = g[KIND == kObbSum ? row0 + t : i];
    if (KIND == kObbCumsum) return (double)gv;
    const float fv = f[i];
    const float c = fix64_cos(ph);
    return (fv >= nyquist) ? 0.0 : (double)(gv * (a[i] * c));
  };

  unsigned long long ph = 0;     // phase before the segment, then after it
  if (KIND != kObbCumsum) {
    unsigned long long tot = 0;
    if (live)
      for (int t = t0; t < t1; ++t)
        tot += turns_to_fix64((double)f[(row0 + t) * K + k] * inv_sr);
    ph_seg[w][lane] = tot;
    __syncthreads();
    if (w == 0) {
      unsigned long long c = 0;
      for (int v = 0; v < kObbWarps; ++v) c += ph_seg[v][lane];
      ph_cta[lane] = c;
    }
    cluster.sync();
    for (int q = 0; q < rank; ++q) ph += cluster.map_shared_rank(&ph_cta[0], q)[lane];
    for (int v = 0; v < w; ++v) ph += ph_seg[v][lane];
  }

  double tot = 0.0;
  if (live) {
    if (KIND == kObbCumsum) {
      for (int t = t0; t < t1; ++t) tot += term(t, 0);
    } else if (da != nullptr || df != nullptr) {
      for (int t = t0; t < t1; ++t) {
        const size_t i = (row0 + t) * K + k;
        ph += turns_to_fix64((double)f[i] * inv_sr);
        if (da != nullptr) {
          const float s = fix64_sin(ph);
          da[i] = (f[i] >= nyquist) ? 0.f : g[KIND == kObbSum ? row0 + t : i] * s;
        }
        if (df != nullptr) tot += term(t, ph);
      }
    }
  }
  if (df == nullptr) {
    cluster.sync();              // no CTA leaves while another reads its ph_cta
    return;
  }

  s_seg[w][lane] = tot;
  __syncthreads();
  if (w == 0) {
    double c = 0.0;
    for (int v = 0; v < kObbWarps; ++v) c += s_seg[v][lane];
    s_cta[lane] = c;
  }
  cluster.sync();
  double acc = 0.0;              // the later segments, nearest last
  for (int q = kObbCluster - 1; q > rank; --q)
    acc += cluster.map_shared_rank(&s_cta[0], q)[lane];
  for (int v = kObbWarps - 1; v > w; --v) acc += s_seg[v][lane];
  if (live) {
    for (int t = t1 - 1; t >= t0; --t) {
      const size_t i = (row0 + t) * K + k;
      acc += term(t, ph);
      df[i] = (float)(acc * scale);
      if (KIND != kObbCumsum) ph -= turns_to_fix64((double)f[i] * inv_sr);
    }
  }
  cluster.sync();                // no CTA leaves while another reads its s_cta
}

// Debug mode `tf_sequential`: the reference's own float32 arithmetic, in its own
// order - one thread per (b, k) walks the time axis.  mode 1: tf.cumsum
// (core.py:955); mode 2: angular_cumsum with its chunking (core.py:836-866).
// in_is_hz: the input is a frequency in Hz and omega = f * 2 pi / sr is formed
// first, as two float32 ops (core.py:947-948).  With `amp` the output is
// amp * sin(phase) with the Nyquist mask (core.py:942, 958-959), else the phase.
__device__ __forceinline__ float tf_floormod(float x, float y) {
  float r = fmodf(x, y);
  if (r != 0.0f && ((r < 0.0f) != (y < 0.0f))) r += y;
  return r;
}

__global__ void __launch_bounds__(128)
tf_sequential_cumsum(const float* __restrict__ in, const float* __restrict__ amp,
                     float* __restrict__ out, int B, int N, int K, int mode,
                     int chunk_size, int in_is_hz, float sample_rate) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * K) return;
  const int b = (int)(i / K), k = (int)(i % K);
  const float two_pi = 6.2831853071795864769f;      // float32(2 pi), as 2.0 * np.pi cast by TF
  const float nyq = sample_rate * 0.5f;
  const float* ip = in + (size_t)b * N * K + k;
  const float* ap = amp ? amp + (size_t)b * N * K + k : nullptr;
  float* op = out + (size_t)b * N * K + k;
  float run = 0.f;          // running sum inside the chunk (or over everything)
  float raw_off = 0.f;      // sequential cumsum of the chunk-end remainders
  float off = 0.f;          // offset of the current chunk
  for (int t = 0; t < N; ++t) {
    const float x = ip[(size_t)t * K];
    float w = x;
    if (in_is_hz) w = __fdiv_rn(__fmul_rn(x, two_pi), sample_rate);
    if (mode == 2 && t > 0 && t % chunk_size == 0) {
      raw_off = __fadd_rn(raw_off, tf_floormod(run, two_pi));
      off = tf_floormod(raw_off, two_pi);
      run = 0.f;
    }
    run = __fadd_rn(run, w);
    float ph = run;
    if (mode == 2) ph = tf_floormod(__fadd_rn(run, off), two_pi);
    float v = ph;
    if (ap) {
      const float a = (in_is_hz && x >= nyq) ? 0.f : ap[(size_t)t * K];
      v = __fmul_rn(a, sinf(ph));
    }
    op[(size_t)t * K] = v;
  }
}

}  // namespace ddsp
