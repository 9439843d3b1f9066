// get_controls prologues (synths.py:94-121, 165-179).
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

}  // namespace ddsp
