// Backward of the frame-rate controls (synths.Harmonic.get_controls,
// synths.py:94-121; synths.FilteredNoise.get_controls, synths.py:165-179) - the
// pieces that let the C4 training step (decoder forward + backward through
// SpectralLoss) run from RAW network outputs without a single frame-rate torch
// op.  The reference gets them from TF autodiff through core.exp_sigmoid
// (core.py:386-404) and core.normalize_harmonics (core.py:894-907).
#pragma once
#include "common.cuh"
#include "controls.cuh"

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

// Harmonics 1..live of a row are below Nyquist and the rest are masked: the forward's
// own float32 decision (harmonic_above_nyquist; f0 * k rounds monotonically in k), found
// from the quotient instead of by testing all K.  f0 <= 0 masks nothing; without
// DDSP_B200_CTL_NYQUIST every harmonic is live.
__device__ __forceinline__ int harmonic_live_prefix(float f, int K, float nyquist,
                                                    int flags) {
  if (!(flags & DDSP_B200_CTL_NYQUIST) || !(f > 0.f)) return K;
  int k = (int)fminf(nyquist / f, (float)K);
  while (k < K && !harmonic_above_nyquist(f, k + 1, nyquist)) ++k;
  while (k > 0 && harmonic_above_nyquist(f, k, nyquist)) --k;
  return k;
}

// The vector-Jacobian product of one row of core.normalize_harmonics after the scaling,
// by one warp in two passes over the row.  With e = exp_sigmoid(hd_raw) (hd_raw itself
// without `scale`) on the live prefix, s = sum(e), n = e / s and an upstream gradient
// gain * up(k) on n[k]:
//   d e[k]      = gain * (up(k) - sum_j up(j) n[j]) / s    (k < live; 0 above)
//   d hd_raw[k] = d e[k] * exp_sigmoid'(hd_raw[k])
// s == 0 takes safe_divide's constant 1e-7 denominator (core.py:207-210) and has no
// coupling term.  Writes all K elements of dr; returns sum_j up(j) n[j] to every lane.
template <class Up>
__device__ __forceinline__ float harmonic_row_vjp(const float* __restrict__ hr,
                                                  float* __restrict__ dr, int K, int live,
                                                  bool scale, int lane, float gain, Up up) {
  // pass 1: sum(e), sum(up e)
  float se = 0.f, sde = 0.f;
  for (int k = lane; k < live; k += 32) {
    float e = hr[k];
    if (scale) e = exp_sigmoid_f(e);
    se += e;
    sde = fmaf(up(k), e, sde);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    se += __shfl_xor_sync(0xffffffffu, se, o);
    sde += __shfl_xor_sync(0xffffffffu, sde, o);
  }
  const float denom = (se == 0.0f) ? 1e-7f : se;          // safe_divide, core.py:207-210
  const float inv = 1.0f / denom;
  const float dot = sde * inv;
  // with the safe denominator a constant (se == 0) there is no coupling term
  const float couple = (se == 0.0f) ? 0.f : dot;
  // pass 2
  for (int k = lane; k < K; k += 32) {
    float out = 0.f;
    if (k < live) {
      float y = hr[k], dy = 1.0f;
      if (scale) dy = exp_sigmoid_grad(y, &y);
      out = gain * (up(k) - couple) * inv * dy;
    }
    dr[k] = out;
  }
  return dot;
}

// Backward of Harmonic.get_controls fused with the recombination of the synthesizer's
// g0 / g1, one warp per (b, i) row:
//   dha[k]   = g0[i,k] + g1[i-1,k] (i > 0) + g1[F-1,k] (i == F-1)      (harmonic_backward.cuh)
//   d amp    = sum_k dha[k] n[k];   d n[k] = dha[k] amp
// then harmonic_row_vjp with up = dha and gain = amp, and
//   d amps_raw = d amp * exp_sigmoid'(amps_raw).
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
  const int live = harmonic_live_prefix(f0[row], K, nyquist, flags);
  const float* g0r = g0 + (size_t)row * K;
  const float* g1p = (i > 0) ? g1 + (size_t)(row - 1) * K : nullptr;
  const float* g1l = (i == F - 1) ? g1 + (size_t)row * K : nullptr;

  float amp = amps_raw[row], damp_dx = 1.0f;
  if (scale) damp_dx = exp_sigmoid_grad(amp, &amp);

  const float dot = harmonic_row_vjp(
      hd_raw + (size_t)row * K, d_hd_raw + (size_t)row * K, K, live, scale, lane, amp,
      [=](int k) {
        float d = g0r[k];
        if (g1p) d += g1p[k];
        if (g1l) d += g1l[k];
        return d;
      });
  if (lane == 0) d_amps_raw[row] = dot * damp_dx;
}

// The vector-Jacobian product of Harmonic.get_controls for any upstream gradient, one
// warp per (b, i) row: d_amplitudes [rows] on the scaled amplitudes and d_hd [rows, K]
// on the normalised distribution, either NULL for zeros (and then not read).
//   d hd_raw   = harmonic_row_vjp(up = d_hd)
//   d amps_raw = d_amplitudes * exp_sigmoid'(amps_raw)       (d_amplitudes without scale)
// f0 gets nothing: the mask is piecewise constant (tf.where).  Bound by HBM traffic:
// hd_raw and d_hd are read in both passes (the second from L2 for rows that fit),
// d_hd_raw is written once.
__global__ void __launch_bounds__(256)
harmonic_controls_vjp_kernel(const float* __restrict__ amps_raw,
                             const float* __restrict__ hd_raw,
                             const float* __restrict__ f0,
                             const float* __restrict__ d_amplitudes,
                             const float* __restrict__ d_hd,
                             float* __restrict__ d_amps_raw,
                             float* __restrict__ d_hd_raw, int rows, int K,
                             float nyquist, int flags) {
  const int row = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const bool scale = flags & DDSP_B200_CTL_SCALE;
  float* dr = d_hd_raw + (size_t)row * K;
  if (d_hd) {
    const float* ur = d_hd + (size_t)row * K;
    harmonic_row_vjp(hd_raw + (size_t)row * K, dr, K,
                     harmonic_live_prefix(f0[row], K, nyquist, flags), scale, lane, 1.0f,
                     [=](int k) { return ur[k]; });
  } else {
    for (int k = lane; k < K; k += 32) dr[k] = 0.f;
  }
  if (lane == 0) {
    float d = 0.f;
    if (d_amplitudes) {
      d = d_amplitudes[row];
      float y;
      if (scale) d *= exp_sigmoid_grad(amps_raw[row], &y);
    }
    d_amps_raw[row] = d;
  }
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
