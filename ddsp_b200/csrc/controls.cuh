// get_controls prologues (synths.py:94-121, 165-179) and processors.Add.
#pragma once
#include "common.cuh"

namespace ddsp {

// The Nyquist decision of Harmonic.get_controls for harmonic number k1 = 1..K:
// get_harmonic_frequencies is f0 * linspace(1..K) in float32 (core.py:1042-1044),
// silent at or above sr/2 (core.py:888-890).  The forward and both backward kernels
// (controls_bwd.cuh) decide with this one expression.
__device__ __forceinline__ bool harmonic_above_nyquist(float f0, int k1, float nyquist) {
  return __fmul_rn(f0, (float)k1) >= nyquist;
}

// Harmonic.get_controls: one warp per (b, f) row of harmonic_distribution.
//   hd = exp_sigmoid(hd)                    (synths.py:110-112, core.py:386-404)
//   hd[k] = 0 where f0 * k >= sr/2          (core.py:894-901, 888-890)
//   hd /= sum(hd), 0 denominator -> 1e-7    (core.py:903-906, 207-210)
__global__ void __launch_bounds__(256)
harmonic_controls_kernel(const float* amps_in, const float* hd_in,
                         const float* __restrict__ f0, float* amps_out,
                         float* hd_out, int rows, int K,
                         float nyquist, int flags) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const bool scale = flags & DDSP_B200_CTL_SCALE;
  const bool nyq = flags & DDSP_B200_CTL_NYQUIST;
  const float f = f0[warp];
  const float* in = hd_in + (size_t)warp * K;
  float* out = hd_out + (size_t)warp * K;
  float sum = 0.f;
  for (int c = lane; c < K; c += 32) {
    float v = in[c];
    if (scale) v = exp_sigmoid_f(v);
    if (nyq && harmonic_above_nyquist(f, c + 1, nyquist)) v = 0.f;
    out[c] = v;
    sum += v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float denom = (sum == 0.0f) ? 1e-7f : sum;
  for (int c = lane; c < K; c += 32) out[c] = __fdiv_rn(out[c], denom);
  if (lane == 0) {
    float a = amps_in[warp];
    amps_out[warp] = scale ? exp_sigmoid_f(a) : a;
  }
}

// FilteredNoise.get_controls: exp_sigmoid(x + initial_bias) (synths.py:176-177)
__global__ void __launch_bounds__(256)
noise_controls_kernel(const float* in, float* out,
                      int64_t n, float bias, int apply_scale) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    float v = in[i];
    out[i] = apply_scale ? exp_sigmoid_f(v + bias) : v;
  }
}

// processors.Add.get_signal (processors.py:174-176)
__global__ void __launch_bounds__(256)
add_kernel(const float* a, const float* b, float* out, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) out[i] = a[i] + b[i];
}

// core.resample / core.upsample_with_windows (core.py:573-714) as a stand-alone
// op: [B, F, C] -> [B, N, C].  method 0 = 'window' (Hann overlap-add ==
// two-tap raised cosine, SURVEY A.2), 1 = 'linear' (tf v1 bilinear,
// align_corners = !add_endpoint), 2 = 'nearest', 3 = 'cubic' (tf v1 bicubic).  Index math follows TF's
// float32 scale * index for linear / nearest; the window method needs an integer
// hop (checked by the caller, core.py:687-693).
__global__ void __launch_bounds__(256)
resample_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int F,
                int C, int N, int method, int add_endpoint) {
  const int64_t total = (int64_t)B * N * C;
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const float scale = (!add_endpoint && N > 1) ? (float)(F - 1) / (float)(N - 1)
                                               : (float)F / (float)N;
  const int hop = add_endpoint ? N / max(F, 1) : N / max(F - 1, 1);
  for (; idx < total; idx += stride) {
    const int c = (int)(idx % C);
    const int64_t bt = idx / C;
    const int t = (int)(bt % N);
    const int b = (int)(bt / N);
    const float* x = in + (size_t)b * F * C + c;
    float v;
    if (method == 0) {
      const int i = t / hop, r = t - i * hop;
      const int i1 = min(i + 1, F - 1);            // add_endpoint: frame F := F-1
      const float w1 = 0.5f - 0.5f * cospif((float)r / (float)hop);
      v = x[(size_t)i * C] * (1.0f - w1) + x[(size_t)i1 * C] * w1;
    } else if (method == 1) {
      const float src = (float)t * scale;
      const float fl = floorf(src);
      const int lo = max((int)fl, 0);
      const int hi = min((int)ceilf(src), F - 1);
      const float top = x[(size_t)min(lo, F - 1) * C], bot = x[(size_t)hi * C];
      v = __fadd_rn(top, __fmul_rn(__fsub_rn(bot, top), src - fl));
    } else if (method == 2) {
      const float src = (float)t * scale;
      const int i = min((int)(add_endpoint ? floorf(src) : roundf(src)), F - 1);
      v = x[(size_t)i * C];
    } else {
      // 'cubic': TensorFlow's legacy bicubic kernel (resize_bicubic_op.cc, Keys
      // A = -0.75, no half-pixel centres).  Its weights come from a 1025-entry
      // float32 table indexed by lrintf(delta * 1024); the same entries are
      // evaluated here in double and rounded to float32.
      const float src = (float)t * scale;
      const float fl = floorf(src);
      const int loc = (int)fl;
      const int off = (int)lrintf((src - fl) * 1024.0f);
      const double A = -0.75;
      const double xa = off * (1.0 / 1024.0), xb = (1024 - off) * (1.0 / 1024.0);
      const float w1 = (float)(((A + 2) * xa - (A + 3)) * xa * xa + 1);
      const float w2 = (float)(((A + 2) * xb - (A + 3)) * xb * xb + 1);
      const double ya = xa + 1.0, yb = xb + 1.0;
      const float w0 = (float)(((A * ya - 5 * A) * ya + 8 * A) * ya - 4 * A);
      const float w3 = (float)(((A * yb - 5 * A) * yb + 8 * A) * yb - 4 * A);
      const float v0 = x[(size_t)min(max(loc - 1, 0), F - 1) * C];
      const float v1 = x[(size_t)min(max(loc, 0), F - 1) * C];
      const float v2 = x[(size_t)min(max(loc + 1, 0), F - 1) * C];
      const float v3 = x[(size_t)min(max(loc + 2, 0), F - 1) * C];
      v = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(v0, w0), __fmul_rn(v1, w1)),
                              __fmul_rn(v2, w2)), __fmul_rn(v3, w3));
    }
    out[idx] = v;
  }
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
