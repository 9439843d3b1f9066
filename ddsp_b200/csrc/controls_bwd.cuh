// Backward of the frame-rate controls (synths.Harmonic.get_controls,
// synths.py:94-121; synths.FilteredNoise.get_controls, synths.py:165-179) - the
// pieces that let the C4 training step (decoder forward + backward through
// SpectralLoss) run from RAW network outputs without a single frame-rate torch
// op.  The reference gets them from TF autodiff through core.exp_sigmoid
// (core.py:386-404) and core.normalize_harmonics (core.py:894-907).
#pragma once
#include "common.cuh"

namespace ddsp {

// exp_sigmoid(x) = 2 sigmoid(x)^ln10 + 1e-7 and its derivative
//   y' = (y - 1e-7) ln10 (1 - sigmoid(x)),  1 - sigmoid(x) = t / (1 + t), t = e^-x
// (t = inf, x << 0, is taken as the limit 1).
__device__ __forceinline__ float exp_sigmoid_grad(float x, float* y_out) {
  const float kLog2e = 1.4426950408889634f;
  const float kLn10 = 2.302585092994046f;
  const float t = ex2_approx(-x * kLog2e);
  float l;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(1.0f + t));
  const float core = 2.0f * ex2_approx(-kLn10 * l);          // y - 1e-7
  *y_out = core + 1e-7f;
  const float one_minus_sig = (t < 1e30f) ? t * __frcp_rn(1.0f + t) : 1.0f;
  return core * kLn10 * one_minus_sig;
}

// One warp per (b, i) row.
//   dha[k]   = g0[i,k] + g1[i-1,k] (i > 0) + g1[F-1,k] (i == F-1)      (harmonic_backward.cuh)
//   n        = e / sum(e), e = exp_sigmoid(hd_raw) on the live prefix (f0 k < sr/2)
//   d amp    = sum_k dha[k] n[k];   d n[k] = dha[k] amp
//   d e[k]   = (d n[k] - sum_j d n[j] n[j]) / sum(e)
//   d hd_raw = d e * exp_sigmoid'(hd_raw);  d amps_raw = d amp * exp_sigmoid'(amps_raw)
// flags: DDSP_B200_CTL_SCALE (exp_sigmoid applied), DDSP_B200_CTL_NYQUIST.
__global__ void __launch_bounds__(256)
harmonic_controls_backward_kernel(const float* __restrict__ amps_raw,
                                  const float* __restrict__ hd_raw,
                                  const float* __restrict__ f0,
                                  const float* __restrict__ g0,
                                  const float* __restrict__ g1,
                                  float* __restrict__ d_amps_raw,
                                  float* __restrict__ d_hd_raw, int rows, int F, int K,
                                  float nyquist, int flags) {
  const int row = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int i = row % F;
  const bool scale = flags & DDSP_B200_CTL_SCALE;
  const float f = f0[row];
  int live = K;
  if ((flags & DDSP_B200_CTL_NYQUIST) && f > 0.f) {
    int k = (int)fminf(nyquist / f, (float)K);
    while (k < K && __fmul_rn(f, (float)(k + 1)) < nyquist) ++k;
    while (k > 0 && !(__fmul_rn(f, (float)k) < nyquist)) --k;
    live = k;
  }
  const float* hr = hd_raw + (size_t)row * K;
  const float* g0r = g0 + (size_t)row * K;
  const float* g1p = (i > 0) ? g1 + (size_t)(row - 1) * K : nullptr;
  const float* g1l = (i == F - 1) ? g1 + (size_t)row * K : nullptr;
  float* dr = d_hd_raw + (size_t)row * K;

  float amp = amps_raw[row], damp_dx = 1.0f;
  if (scale) damp_dx = exp_sigmoid_grad(amp, &amp);

  // pass 1: sum(e), sum(dha e)
  float se = 0.f, sde = 0.f;
  for (int k = lane; k < live; k += 32) {
    float e = hr[k];
    if (scale) e = exp_sigmoid_f(e);
    float d = g0r[k];
    if (g1p) d += g1p[k];
    if (g1l) d += g1l[k];
    se += e;
    sde = fmaf(d, e, sde);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    se += __shfl_xor_sync(0xffffffffu, se, o);
    sde += __shfl_xor_sync(0xffffffffu, sde, o);
  }
  const float denom = (se == 0.0f) ? 1e-7f : se;          // safe_divide, core.py:207-210
  const float inv = 1.0f / denom;
  const float dot = sde * inv;                             // sum_k dha[k] n[k] = d amp
  // with the safe denominator a constant (se == 0) there is no coupling term
  const float couple = (se == 0.0f) ? 0.f : dot;
  // pass 2
  for (int k = lane; k < K; k += 32) {
    float out = 0.f;
    if (k < live) {
      float y = hr[k], dy = 1.0f;
      if (scale) dy = exp_sigmoid_grad(y, &y);
      float d = g0r[k];
      if (g1p) d += g1p[k];
      if (g1l) d += g1l[k];
      out = amp * (d - couple) * inv * dy;
    }
    dr[k] = out;
  }
  if (lane == 0) d_amps_raw[row] = dot * damp_dx;
}

// FilteredNoise.get_controls backward: magnitudes = exp_sigmoid(raw + bias).
__global__ void __launch_bounds__(256)
noise_controls_backward_kernel(const float* __restrict__ mags_raw,
                               const float* __restrict__ dmags, float* __restrict__ d_raw,
                               int64_t n, float bias) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    float y;
    const float dy = exp_sigmoid_grad(mags_raw[i] + bias, &y);
    d_raw[i] = dmags[i] * dy;
  }
}

}  // namespace ddsp
