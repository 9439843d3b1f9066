// Filtered noise, generic (any nb / window_size / frame size) building blocks:
//   ir_kernel   - core.frequency_impulse_response (core.py:1534-1565) with
//                 apply_window_to_impulse_response (core.py:1477-1531) as one
//                 closed-form cosine sum per tap (SURVEY.md A.5).
//   fir_kernel  - core.fft_convolve (core.py:1382-1473) restated as the
//                 equivalent direct-form time-varying FIR (SURVEY.md A.6):
//                   y_full[q] = sum_m h_{fr(q-m)}[m] x[q-m],  fr(p) = p / frame
//                   out[o]    = y_full[o + start]
//                 (the IR is chosen by the INPUT sample's frame).
// The fused fast path for the decoder regime lives in noise_fused.cuh.
#pragma once
#include "common.cuh"

namespace ddsp {

// Geometry of the windowed causal IR (host + device).
struct IrGeom {
  int nb;      // number of magnitude bins
  int S0;      // irfft length 2 (nb - 1)
  int ws;      // effective window size
  int half;    // (ws + 1) / 2 when padded
  int S;       // output taps
  int shift;   // tap j <-> zero-phase offset n = j - shift
  int padded;  // ws < S0
};

__host__ __device__ inline IrGeom make_ir_geom(int nb, int window_size) {
  IrGeom g;
  g.nb = nb;
  g.S0 = 2 * (nb - 1);
  g.ws = (window_size <= 0 || window_size > g.S0) ? g.S0 : window_size;
  g.padded = (g.S0 - g.ws) > 0;
  if (g.padded) {
    g.half = (g.ws + 1) / 2;
    g.S = 2 * g.half - 1;      // ws if odd, ws - 1 if even (core_test.py:825-855)
    g.shift = g.half - 2;
  } else {
    g.half = 0;
    g.S = g.S0;
    g.shift = g.S0 / 2;
  }
  return g;
}

// Window value and zero-phase index of causal tap j (core.py:1494-1529).
__device__ __forceinline__ void ir_tap(const IrGeom& g, int j, int* idx_out,
                                       float* w_out) {
  int n = j - g.shift;
  int idx = n % g.S0;
  if (idx < 0) idx += g.S0;
  float w;
  if (g.padded) {
    // tf.signal.hann_window(ws): 0.5 - 0.5 cos(2 pi k / d) with d = ws for even ws and
    // d = ws - 1 for odd ws (window_ops._raised_cosine_window: an odd length gives the
    // symmetric window whatever `periodic` says); a window of one sample is 1.
    const float d = (float)((g.ws & 1) ? g.ws - 1 : g.ws);
    if (g.ws == 1) {
      w = (idx >= g.S0 - g.half) ? 1.0f : 0.f;
    } else if (idx < g.ws - g.half) {
      w = 0.5f - 0.5f * cospif(2.0f * (float)(g.half + idx) / d);
    } else if (idx >= g.S0 - g.half) {
      w = 0.5f - 0.5f * cospif(2.0f * (float)(idx - (g.S0 - g.half)) / d);
    } else {
      w = 0.f;
    }
  } else {
    w = 0.5f - 0.5f * cospif(2.0f * (float)j / (float)g.S0);
  }
  *idx_out = idx;
  *w_out = w;
}

constexpr int kIrThreads = 256;
constexpr int kIrFrames = 8;  // frames per CTA

// mags [BF, nb] -> ir [BF, S].  smem: cos table S0 + kIrFrames * nb mags.
__global__ void __launch_bounds__(kIrThreads)
ir_kernel(const float* __restrict__ mags, float* __restrict__ ir, int64_t BF,
          IrGeom g) {
  extern __shared__ __align__(16) float sm[];
  float* sCos = sm;               // [S0]
  float* sM = sm + g.S0;          // [kIrFrames][nb]
  const int tid = threadIdx.x;
  const int64_t f0 = (int64_t)blockIdx.x * kIrFrames;
  const int nf = (int)min((int64_t)kIrFrames, BF - f0);
  for (int i = tid; i < g.S0; i += kIrThreads)
    sCos[i] = cospif(2.0f * (float)i / (float)g.S0);
  for (int i = tid; i < nf * g.nb; i += kIrThreads)
    sM[i] = mags[f0 * g.nb + i];
  __syncthreads();
  const float inv = 1.0f / (float)g.S0;
  for (int e = tid; e < nf * g.S; e += kIrThreads) {
    const int fr = e / g.S, j = e - fr * g.S;
    int idx; float w;
    ir_tap(g, j, &idx, &w);
    const float* m = sM + fr * g.nb;
    float acc = m[0] + ((idx & 1) ? -m[g.nb - 1] : m[g.nb - 1]);
    int ph = 0;                         // (k * idx) mod S0
    // double accumulator: a float32 sum over thousands of bins drifts past 1e-6 of
    // the taps (1.5e-6 at 5000 bins)
    double acc2 = 0.0;
    for (int k = 1; k < g.nb - 1; ++k) {
      ph += idx;
      if (ph >= g.S0) ph -= g.S0;
      acc2 = fma((double)m[k], (double)sCos[ph], acc2);
    }
    ir[(f0 + fr) * g.S + j] = w * (float)((double)acc + 2.0 * acc2) * inv;
  }
}

constexpr int kFirThreads = 256;

// Direct-form time-varying FIR.  One thread per output sample; the input window
// of the CTA is staged in shared memory, IR taps come through L1/L2.
__global__ void __launch_bounds__(kFirThreads)
fir_kernel(const float* __restrict__ x, const float* __restrict__ ir,
           float* out, int N, int F, int S, int frame, int ir_batch_stride,
           int start, int out_len, int accumulate) {
  extern __shared__ __align__(16) float sx[];   // [kFirThreads + S - 1]
  const int b = blockIdx.y;
  const int o0 = blockIdx.x * kFirThreads;
  const int tid = threadIdx.x;
  const float* xb = x + (size_t)b * N;
  const float* irb = ir + (size_t)b * ir_batch_stride;
  const int q0 = o0 + start;                 // y_full index of the CTA's first output
  const int p_lo = q0 - (S - 1);             // first input sample needed
  const int win = kFirThreads + S - 1;
  for (int i = tid; i < win; i += kFirThreads) {
    int p = p_lo + i;
    sx[i] = (p >= 0 && p < N) ? xb[p] : 0.f;
  }
  __syncthreads();
  const int o = o0 + tid;
  if (o >= out_len) return;
  const int q = q0 + tid;
  // valid taps: 0 <= q - m < N
  const int m_lo = max(0, q - (N - 1));
  const int m_hi = min(S - 1, q);
  float acc = 0.f;
  for (int m = m_lo; m <= m_hi; ++m) {
    const int p = q - m;
    const int fr = p / frame;
    acc = fmaf(irb[(size_t)fr * S + m], sx[p - p_lo], acc);
  }
  float* ob = out + (size_t)b * out_len;
  if (accumulate) acc += ob[o];
  ob[o] = acc;
}

// tf.random.uniform([B, N], -1, 1) stand-in (synths.py:192-193): Philox4x32-10.
__global__ void __launch_bounds__(256)
uniform_noise_kernel(float* __restrict__ out, int B, int N, uint64_t seed,
                     uint64_t offset) {
  const int n4 = (N + 3) >> 2;
  const int64_t total = (int64_t)B * n4;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < total; i += stride) {
    const int b = (int)(i / n4);
    const int q = (int)(i - (int64_t)b * n4);
    const float4 v = noise4((uint32_t)q, (uint32_t)b, seed, offset);
    float* o = out + (size_t)b * N + 4 * (size_t)q;
    const int rem = N - 4 * q;
    o[0] = v.x;
    if (rem > 1) o[1] = v.y;
    if (rem > 2) o[2] = v.z;
    if (rem > 3) o[3] = v.w;
  }
}

}  // namespace ddsp
