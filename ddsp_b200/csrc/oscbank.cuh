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
        const uint32_t p32 = (uint32_t)((ph + 0x80000000ull) >> 32);
        const float s = sinpif((float)(int)p32 * 4.656612873077393e-10f);
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
