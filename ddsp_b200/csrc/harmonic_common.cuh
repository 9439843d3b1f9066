// Shared pieces of the fused harmonic kernels (hop % 64 == 0): the 256-entry
// sin / cos table, the 64-bit fixed-point phase, the
// per-sample oscillator state (two Reinsch chains over the harmonics, odd / even,
// in one f32x2), the exact per-oscillator slow path for f0 < 1 Hz, and the
// get_controls rows for wide harmonic distributions.  Used by harmonic_v4.cuh
// (forward), harmonic_bwd2.cuh / backward.cuh (backward).
//
// Derivations (closed-form phase, Reinsch recurrence, per-row accumulators,
// live-count Nyquist culling) are in DESIGN.md section 3.1.
#pragma once
#include <cmath>
#include <cstdlib>

#include "harmonic.cuh"

namespace ddsp {

constexpr int kSinTabBits = 8;
constexpr int kSinTab = 1 << kSinTabBits;  // 256-entry (sin, cos) table

__device__ __forceinline__ float2 bc2(float x) { return make_float2(x, x); }

// Slow, exact per-oscillator evaluation of one sample (frames with f0 < 1 Hz,
// where the live-count shortcut is not valid).
__device__ __noinline__ float harmonic_sample_exact(const float* x0,
                                                    const float* x1, float w0,
                                                    float w1, uint32_t p32,
                                                    float f_lo, float f_hi,
                                                    float frac, int K,
                                                    float nyq) {
  float acc = 0.f;
  uint32_t pk = 0;
  for (int k = 1; k <= K; ++k) {
    pk += p32;
    if (!(ref_harmonic_freq(f_lo, f_hi, frac, k) < nyq)) continue;
    float a = x0[k - 1] * w0 + x1[k - 1] * w1;
    acc = fmaf(a, sinpif((float)(int)pk * 4.656612873077393e-10f), acc);
  }
  return acc;
}

// The fused kernels need whole 64-sample chunks per frame.
inline bool harmonic_fused_supported(const HarmonicParams& p) {
  return (p.hop % 64 == 0) && p.hop <= 8192 && p.K <= 1024;
}

namespace hcm {

__device__ const float2 g_sincos256[kSinTab] = {
#include "sincos_tab.inc"
};

// top 32 bits of P + c1 * A + c2 * D (mod 2^64); P already carries the +2^31
// rounding offset.  4 IMADs.
__device__ __forceinline__ uint32_t phase32(unsigned long long P, unsigned long long A,
                                            unsigned long long D, uint32_t c1,
                                            uint32_t c2) {
  unsigned long long acc = P + (unsigned long long)(uint32_t)A * c1;
  uint32_t hi = (uint32_t)(acc >> 32) + (uint32_t)(A >> 32) * c1;
  acc = (((unsigned long long)hi << 32) | (uint32_t)acc) +
        (unsigned long long)(uint32_t)D * c2;
  return (uint32_t)(acc >> 32) + (uint32_t)(D >> 32) * c2;
}

// Oscillator state of ONE sample: .x = odd-harmonic chain sin((1+2j) phi),
// .y = even-harmonic chain sin((2+2j) phi); both step by the angle 2 phi reduced
// to [-pi/2, pi/2] (sigma = -1 where it was shifted by half a turn: every other
// step then flips sign, hence the accumulators split by step parity e / o).
struct Osc {
  float2 v, d, na;
  float sigma;
  float2 a0e, a0o, a1e, a1o;    // row x0 / x1, step parity
};

__device__ __forceinline__ void osc_init(Osc& st, uint32_t p,
                                         const float2* __restrict__ tab) {
  const uint32_t i = (p + (1u << (31 - kSinTabBits))) >> (32 - kSinTabBits);
  const int r = (int)(p - (i << (32 - kSinTabBits)));
  const float2 t = tab[i & (kSinTab - 1)];
  const float eps = (float)r * 1.4629180792671596e-9f;           // 2 pi / 2^32
  const float e2 = eps * eps;
  const float ce = fmaf(e2, -0.5f, 1.0f);
  const float se = eps * fmaf(e2, -0.16666667f, 1.0f);
  const float s1 = fmaf(t.y, se, t.x * ce);
  const float c1 = fmaf(-t.x, se, t.y * ce);
  const float ss = s1 * s1, cc = c1 * c1;
  const bool flip = ss > cc;                                     // cos(2 phi) < 0
  const float s2 = (s1 + s1) * c1;                               // sin(2 phi)
  const float na = -4.0f * fminf(ss, cc);
  st.v = make_float2(s1, s2);
  st.d = make_float2(flip ? 0.0f : s1 + s1, s2);
  st.na = make_float2(na, na);
  st.sigma = flip ? -1.0f : 1.0f;
  st.a0e = st.a0o = st.a1e = st.a1o = make_float2(0.f, 0.f);
}

// Four harmonics (k+1 .. k+4) of one sample: two chain steps.
__device__ __forceinline__ void osc_group(Osc& st, const float4& X0, const float4& X1) {
  st.a0e = ffma2(make_float2(X0.x, X0.y), st.v, st.a0e);
  st.a1e = ffma2(make_float2(X1.x, X1.y), st.v, st.a1e);
  st.d = ffma2(st.na, st.v, st.d);
  st.v = fadd2(st.v, st.d);
  st.a0o = ffma2(make_float2(X0.z, X0.w), st.v, st.a0o);
  st.a1o = ffma2(make_float2(X1.z, X1.w), st.v, st.a1o);
  st.d = ffma2(st.na, st.v, st.d);
  st.v = fadd2(st.v, st.d);
}

__device__ __forceinline__ float4 mask4(const float4& X, int k, int ks) {
  // harmonic numbers k+1 .. k+4 live iff number <= ks
  return make_float4(k + 1 <= ks ? X.x : 0.f, k + 2 <= ks ? X.y : 0.f,
                     k + 3 <= ks ? X.z : 0.f, k + 4 <= ks ? X.w : 0.f);
}

__device__ __forceinline__ float osc_finish(const Osc& st, float w0, float w1) {
  const float r0 = fmaf(st.sigma, st.a0o.x + st.a0o.y, st.a0e.x + st.a0e.y);
  const float r1 = fmaf(st.sigma, st.a1o.x + st.a1o.y, st.a1e.x + st.a1e.y);
  return fmaf(r1, w1, r0 * w0);
}

// Frame record and oscillator seed of the (odd, even)-chain layout: the backward
// kernel (harmonic_bwd2.cuh) keeps the third forward generation's records; the
// forward kernel is harmonic_v4.cuh.
constexpr int kBwdWarps = 4;     // warps per CTA of the backward kernel
struct __align__(16) FrameRec {
  unsigned long long P, A;       // P carries the +2^31 rounding offset
  unsigned long long D;
  int kca, kcb;                  // live counts at r = 0 / r = hop-1; kca < 0: exact path
  float f_lo, f_hi, amp0, amp1;
};
static_assert(sizeof(FrameRec) == 48, "FrameRec must be three 16-byte words");

// osc_init without zeroing the accumulators.
__device__ __forceinline__ void osc_seed(Osc& st, uint32_t p,
                                         const float2* __restrict__ tab) {
  const uint32_t i = (p + (1u << (31 - kSinTabBits))) >> (32 - kSinTabBits);
  const int r = (int)(p - (i << (32 - kSinTabBits)));
  const float2 t = tab[i & (kSinTab - 1)];
  const float eps = (float)r * 1.4629180792671596e-9f;           // 2 pi / 2^32
  const float e2 = eps * eps;
  const float ce = fmaf(e2, -0.5f, 1.0f);
  const float se = eps * fmaf(e2, -0.16666667f, 1.0f);
  const float s1 = fmaf(t.y, se, t.x * ce);
  const float c1 = fmaf(-t.x, se, t.y * ce);
  const float ss = s1 * s1, cc = c1 * c1;
  const bool flip = ss > cc;                                     // cos(2 phi) < 0
  const float s2 = (s1 + s1) * c1;                               // sin(2 phi)
  const float na = -4.0f * fminf(ss, cc);
  st.v = make_float2(s1, s2);
  st.d = make_float2(flip ? 0.0f : s1 + s1, s2);
  st.na = make_float2(na, na);
  st.sigma = flip ? -1.0f : 1.0f;
}


// Harmonic.get_controls for up to four rows (r0 .. r0+3 of this warp's block) in
// shared memory, 8 lanes per row: exp_sigmoid on the live prefix, zeros above it,
// row normalisation with safe_divide (synths.py:110-117, core.py:894-907).  The
// frame-rate live count of each row (f0*k < sr/2 in float32) was computed once
// per row by the caller.
__device__ __forceinline__ void controls_rows(float* __restrict__ sXw,
                                              const int* __restrict__ sLive, int r0,
                                              int nrows, int Kp, bool raw_scale,
                                              int lane) {
  const int K4 = Kp >> 2;
  const int sub = lane >> 3, l8 = lane & 7;
  const int r = r0 + sub;
  const bool row_ok = r < nrows;
  float4* row4 = reinterpret_cast<float4*>(sXw + (row_ok ? r : r0) * Kp);
  const int live = sLive[row_ok ? r : r0];
  float sum = 0.f;
  if (row_ok) {
    for (int c4 = l8; c4 < K4; c4 += 8) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (4 * c4 < live) {
        v = row4[c4];
        float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          float w = e[u];
          if (raw_scale) w = exp_sigmoid_f(w);
          if (4 * c4 + u >= live) w = 0.f;
          e[u] = w;
          sum += w;
        }
        v = make_float4(e[0], e[1], e[2], e[3]);
      }
      row4[c4] = v;
    }
  }
  sum += __shfl_xor_sync(0xffffffffu, sum, 4);
  sum += __shfl_xor_sync(0xffffffffu, sum, 2);
  sum += __shfl_xor_sync(0xffffffffu, sum, 1);
  const float inv = 1.0f / ((sum == 0.0f) ? 1e-7f : sum);
  if (row_ok) {
    for (int c4 = l8; 4 * c4 < live; c4 += 8) {
      float4 v = row4[c4];
      v.x *= inv; v.y *= inv; v.z *= inv; v.w *= inv;
      row4[c4] = v;
    }
  }
}

}  // namespace hcm
}  // namespace ddsp
