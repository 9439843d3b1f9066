// Modulated delay: core.variable_length_delay (core.py:1285-1314, on
// core.linear_lookup, 1168-1214) and effects.ModDelay.get_signal
// (effects.py:328-394), forward and backward.
//
// The reference frames the padded audio with frame_step = 1 into [B, N, L],
// reverses the frames, appends column 0 as a wrap column and interpolates over all
// L + 1 columns.  Only two of them carry weight, so per output sample t, with
// pos = phase(t) * L:
//
//   out(t) = sum_{j=0..L} relu(1 - |pos - j|) v_j,
//   v_j = x[t - j] for j < L (0 before the start),  v_L = x[t]   (the wrap column)
//
// i.e. taps j0 = floor(pos) and j0 + 1 with weights 1 - frac and frac; taps outside
// [0, L] read nothing.  phase(t) = raw(t) * scale + offset in float32 (two roundings,
// as ModDelay's host arithmetic), pos in double: exact for L < 2^29, so j0 and frac
// are exact and so is the knot test of the backward pass.
//
// Gradients are TensorFlow's subgradients of that formula (abs'(0) = relu'(0) = 0):
// d pos = v_{j0+1} - v_{j0} off the knots and 0 where pos is an integer.
//
// Forward: one thread per output, the taps read through L2 (one code path for every
// L; neighbouring outputs read neighbouring inputs, so the gathers coalesce for any
// smooth phase).  Backward: a CTA owns an INPUT tile [s0, s0 + kTile) and walks the
// only outputs that reach it, t in [s0, s0 + kTile + L - 2]; each warp accumulates
// the taps that land in the tile into a private shared buffer, lanes with equal
// targets summed in lane order, and the warp buffers are summed in warp order, so
// d audio is written once per element, without atomics, bit-reproducibly.  The CTA
// also writes d gain and d phase of the outputs inside its tile.
#pragma once
#include "taps.cuh"

namespace ddsp {
namespace md_ {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kTile = 1024;      // backward input tile (per-warp buffers: 32 KB)

__host__ __device__ constexpr size_t backward_smem_bytes() {
  return sizeof(float) * (size_t)kWarps * kTile;
}

struct Taps {
  int j0;       // lower tap; j0 + 1 is the upper one
  float w0;     // weight of j0 (1 - frac)
  float w1;     // weight of j0 + 1 (frac)
  bool knot;    // pos is an integer: the subgradient of the position is 0
};

__device__ __forceinline__ Taps taps(float raw, float scale, float offset, int L) {
  const float phase = __fadd_rn(__fmul_rn(raw, scale), offset);   // no FMA
  const double pos = (double)phase * (double)L;
  Taps tp;
  if (!(pos > -2.0 && pos < (double)L + 2.0)) {   // no tap in [0, L] (or NaN)
    tp.j0 = -2;
    tp.w0 = tp.w1 = 0.f;
    tp.knot = true;
    return tp;
  }
  const double fl = floor(pos);
  const double frac = pos - fl;                   // exact
  tp.j0 = (int)fl;
  tp.w0 = (float)(1.0 - frac);
  tp.w1 = (float)frac;
  tp.knot = frac == 0.0;
  return tp;
}

// the input index tap j of output t reads, or -1 when it reads nothing
__device__ __forceinline__ int tap_source(int j, int t, int L) {
  if (j < 0 || j > L) return -1;
  return j == L ? t : t - j;      // t - j < 0: the causal zero padding
}

__device__ __forceinline__ float tap_value(const float* __restrict__ x, int j, int t,
                                           int L) {
  const int s = tap_source(j, t, L);
  return s >= 0 ? __ldg(x + s) : 0.f;
}

// out[t] = (add_dry ? x[t] : 0) + gain[t] * delay(x)[t]   (gain NULL: 1)
__global__ void __launch_bounds__(kThreads)
mod_delay_forward_kernel(const float* __restrict__ audio, const float* __restrict__ phase,
                         const float* __restrict__ gain, float* __restrict__ out, int N,
                         int L, float scale, float offset, int add_dry) {
  const int b = blockIdx.y;
  const int t = blockIdx.x * kThreads + threadIdx.x;
  if (t >= N) return;
  const size_t row = (size_t)b * N;
  const float* x = audio + row;
  const Taps tp = taps(__ldg(phase + row + t), scale, offset, L);
  const float v0 = tap_value(x, tp.j0, t, L);
  const float v1 = tap_value(x, tp.j0 + 1, t, L);
  float wet = __fadd_rn(__fmul_rn(tp.w0, v0), __fmul_rn(tp.w1, v1));
  if (gain != nullptr) wet = __fmul_rn(wet, __ldg(gain + row + t));
  out[row + t] = add_dry ? __fadd_rn(wet, x[t]) : wet;
}

// d audio (optional), d gain (optional, needs gain) and d phase (optional) of
// out = [add_dry] x + gain * delay(x; raw * scale + offset), for upstream gradient g.
// d phase is with respect to `raw` (times scale).
__global__ void __launch_bounds__(kThreads)
mod_delay_backward_kernel(const float* __restrict__ audio, const float* __restrict__ phase,
                          const float* __restrict__ gain, const float* __restrict__ grad,
                          float* __restrict__ d_audio, float* __restrict__ d_gain,
                          float* __restrict__ d_phase, int N, int L, float scale,
                          float offset, int add_dry) {
  extern __shared__ float md_buf[];                   // [kWarps][kTile]
  __shared__ float stage[kWarps][32];
  const int b = blockIdx.y;
  const int s0 = blockIdx.x * kTile;
  const int tile = min(kTile, N - s0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t row = (size_t)b * N;
  const float* x = audio + row;
  const float* ph = phase + row;
  const float* g = grad + row;
  const float* gn = gain ? gain + row : nullptr;
  float* buf = md_buf + warp * kTile;

  if (d_audio != nullptr) {
    for (int i = lane; i < tile; i += 32) buf[i] = 0.f;
    __syncwarp();
  }
  // outputs reaching the tile: t in [s0, s0 + tile + L - 2] (tap j reads t - j,
  // j <= L - 1; the wrap tap reads t itself)
  const int t_end = d_audio != nullptr ? (int)min((long long)N, (long long)s0 + tile + L - 1)
                                       : s0 + tile;
  for (int base = s0 + warp * 32; base < t_end; base += kThreads) {   // warp-uniform
    const int t = base + lane;
    const bool live = t < t_end;
    float c = 0.f;
    Taps tp;
    tp.j0 = -2; tp.w0 = tp.w1 = 0.f; tp.knot = true;
    if (live) {
      const float gt = __ldg(g + t);
      const float gain_t = gn ? __ldg(gn + t) : 1.f;
      tp = taps(__ldg(ph + t), scale, offset, L);
      c = gt * gain_t;
      if (t < s0 + tile && (d_gain != nullptr || d_phase != nullptr)) {
        const float v0 = tap_value(x, tp.j0, t, L);
        const float v1 = tap_value(x, tp.j0 + 1, t, L);
        if (d_gain != nullptr)
          d_gain[row + t] = gt * __fadd_rn(__fmul_rn(tp.w0, v0), __fmul_rn(tp.w1, v1));
        if (d_phase != nullptr)
          d_phase[row + t] = tp.knot ? 0.f : c * ((float)L * (v1 - v0)) * scale;
      }
    }
    if (d_audio != nullptr) {
      const int s_lo = tap_source(tp.j0, t, L), s_hi = tap_source(tp.j0 + 1, t, L);
      scatter_tap(buf, stage[warp], s_lo, c * tp.w0, live && s_lo >= s0 && s_lo < s0 + tile,
                  s0, lane);
      scatter_tap(buf, stage[warp], s_hi, c * tp.w1, live && s_hi >= s0 && s_hi < s0 + tile,
                  s0, lane);
    }
  }
  if (d_audio == nullptr) return;
  __syncthreads();
  for (int i = threadIdx.x; i < tile; i += kThreads) {
    float acc = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) acc += md_buf[w * kTile + i];
    if (add_dry) acc += g[s0 + i];
    d_audio[row + s0 + i] = acc;
  }
}

}  // namespace md_
}  // namespace ddsp
