// harmonic_v4: fourth generation of the fused harmonic kernel (hop % 64 == 0).
// The mathematics is that of the earlier generations (closed-form phase, Reinsch
// chains over the harmonics with angle 2 phi, per-row accumulators, live-count
// Nyquist culling, get_controls fused into the slab staging - DESIGN.md 3.1).
// In the third generation the oscillator loop was about a quarter of the warp
// instructions per 64-sample frame; everything else was overhead at one issue
// slot each.  What changed:
//
//   * the f32x2 lanes hold the SAME chain of the lane's TWO samples (r, r + 32),
//     not the (odd, even) chains of one sample.  Harmonic amplitudes enter as
//     broadcast scalar operands; the seeds (table look-up, rotation,
//     double-angle, Reinsch constants), the weights and the final combination
//     are f32x2 over the two samples: no cross-half sums, eight accumulator
//     registers less;
//   * the per-sample phase is 4 IMADs on the 64-bit fixed-point frame phase
//     (hcm::phase32);
//   * get_controls writes each row once: exp_sigmoid on the live prefix, zeros
//     above it, and the row's 1 / sum goes into the frame amplitude (amp / sum),
//     not into a second pass over the row;
//   * frame-rate zeros make the Nyquist mask free: when every sample of a frame
//     has live count kc, row x0 is zero above kc by construction and row x1 is
//     zero above its own count; if that is <= kc the frame runs ceil(kc / 4)
//     unmasked groups.  Only the other frames take a masked group.
//
// On sm_90a (each f32x2 operation is two scalar instructions) the group loops run
// pairs of groups on one 32-bit shared address (2 loop instructions per group,
// 9 before), the first group of a uniform frame writes the accumulators instead
// of zeroing them, and a CTA is four warps over 32 frames: one record warp builds
// the 32 frame records while the other three transform the 33 rows, so that one
// prologue serves 32 frames and the two run side by side (DESIGN.md 3.1, 4).
#pragma once
#include "harmonic_common.cuh"

namespace ddsp {

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

namespace hv4 {

constexpr int NW = 4;            // warps per CTA
constexpr int NT = NW * 32;
constexpr int MIN_CTAS = 6;      // per SM: 24 warps, 80 registers

// -DDDSP_HV4_TIMING: per-SM totals of each warp's clock() cycles by kernel phase,
// summed over every CTA the SM ran (tools/harm_timing.py reads them back through
// ddsp_b200_debug_harm_timing); measurement builds only.
#ifdef DDSP_HV4_TIMING
constexpr int kTimingPhases = 8;     // + 1 slot: warps counted
__device__ unsigned long long g_hv4_timing[kMaxSMs * (kTimingPhases + 1)];
#define HV4_TIMING_DECL                                                                 \
  unsigned tacc__[kTimingPhases] = {0, 0, 0, 0, 0, 0, 0, 0};                            \
  unsigned tprev__ = (unsigned)clock()
#define HV4_LAP(i)                                                                      \
  do {                                                                                  \
    const unsigned n__ = (unsigned)clock();                                             \
    tacc__[i] += n__ - tprev__;                                                         \
    tprev__ = n__;                                                                      \
  } while (0)
#define HV4_TIMING_FLUSH()                                                              \
  do {                                                                                  \
    if (lane == 0) {                                                                    \
      unsigned smid__;                                                                  \
      asm volatile("mov.u32 %0, %%smid;" : "=r"(smid__));                               \
      unsigned long long* t__ = g_hv4_timing + (smid__ % kMaxSMs) * (kTimingPhases + 1); \
      for (int i__ = 0; i__ < kTimingPhases; ++i__) atomicAdd(t__ + i__, (unsigned long long)tacc__[i__]); \
      atomicAdd(t__ + kTimingPhases, 1ull);                                             \
    }                                                                                   \
  } while (0)
#else
#define HV4_TIMING_DECL
#define HV4_LAP(i)
#define HV4_TIMING_FLUSH()
#endif

struct __align__(16) FrameRec {
  unsigned long long P, A;       // P carries the +2^31 rounding and +2^-9 turn offsets
  unsigned long long D;
  int ng;                        // > 0: uniform frame, ng unmasked groups; 0: per-sample
                                 // live counts; < 0: exact path (f0 < 1 Hz)
  int rem;                       // uniform frame: harmonics of the masked last group
  float f_lo, f_hi, amp0, amp1;  // amp = amplitude / row sum
};
static_assert(sizeof(FrameRec) == 48, "FrameRec must be three 16-byte words");

struct Smem {
  size_t off_mbar, off_sin, off_cos, off_x, off_w, off_red, off_inv, off_rec, off_live, total;
};

__host__ __device__ inline Smem smem_layout(int FW, int Kp, int hop) {
  Smem s;
  const size_t FT = (size_t)FW * NW;
  size_t o = 0;
  s.off_mbar = o; o += 16;
  s.off_sin = o;  o += sizeof(float) * kSinTab;
  s.off_cos = o;  o += sizeof(float) * kSinTab;
  s.off_x = o;    o += sizeof(float) * (FT + 1) * Kp;                 // 16 B aligned
  s.off_w = o;    o += (hop == 64) ? 0 : sizeof(float) * hop;
  o = (o + 15) & ~(size_t)15;
  s.off_red = o;  o += 16 * NW;                                       // double + u64 per warp
  s.off_rec = o;  o += sizeof(FrameRec) * FT;
  s.off_inv = o;  o += sizeof(float) * (FT + 1);
  s.off_live = o; o += sizeof(int) * (FT + 1);
  s.total = (o + 15) & ~(size_t)15;
  return s;
}

using hcm::phase32;

// 16-byte shared-memory load at a 32-bit shared address: the group loops step one
// such address (ptxas otherwise keeps a generic pointer and an index beside it)
__device__ __forceinline__ float4 lds128(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "r"(a));
  return v;
}

__device__ __forceinline__ float2 bffma2(float x, float2 v, float2 acc) {
  return ffma2(make_float2(x, x), v, acc);
}
__device__ __forceinline__ float2 bfmul2(float x, float2 v) {
  return fmul2(make_float2(x, x), v);
}

// Harmonic.get_controls for up to four rows (r0 .. r0+3 of this warp's block) in
// shared memory, 8 lanes per row (synths.py:110-117, core.py:894-907): exp_sigmoid
// on the live prefix, zeros above it, ONE store per element; the row's 1 / sum
// (safe_divide: a zero sum counts as 1e-7) goes to sInv[r] and is folded into the
// frame amplitude by the caller.
__device__ __forceinline__ void controls_rows4(float* __restrict__ sXw,
                                               const int* __restrict__ sLive,
                                               float* __restrict__ sInv, int r0,
                                               int nrows, int Kp, bool raw_scale,
                                               int lane) {
  const int K4 = Kp >> 2;
  const int sub = lane >> 3, l8 = lane & 7;
  const int r = r0 + sub;
  const bool row_ok = r < nrows;
  float4* row4 = reinterpret_cast<float4*>(sXw + (row_ok ? r : r0) * Kp);
  const int live = row_ok ? sLive[r] : 0;
  const int live4 = (live + 3) >> 2;                 // float4 groups with a live element
  float sum = 0.f;
  int c4 = l8;
  for (; c4 < live4; c4 += 8) {
    float4 x = row4[c4];
    if (raw_scale) {
      x.x = exp_sigmoid_f(x.x); x.y = exp_sigmoid_f(x.y);
      x.z = exp_sigmoid_f(x.z); x.w = exp_sigmoid_f(x.w);
    }
    const int k = 4 * c4;
    if (k + 1 >= live) x.y = 0.f;
    if (k + 2 >= live) x.z = 0.f;
    if (k + 3 >= live) x.w = 0.f;
    sum += (x.x + x.y) + (x.z + x.w);
    row4[c4] = x;
  }
  if (row_ok) {
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    for (; c4 < K4; c4 += 8) row4[c4] = z;
  }
  sum += __shfl_xor_sync(0xffffffffu, sum, 4);
  sum += __shfl_xor_sync(0xffffffffu, sum, 2);
  sum += __shfl_xor_sync(0xffffffffu, sum, 1);
  if (row_ok && l8 == 0) sInv[r] = __fdividef(1.0f, (sum == 0.0f) ? 1e-7f : sum);
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

// Frame-rate live count of a row (f0 * k < sr/2 in float32, core.py:888).
__device__ __forceinline__ int row_live_count(float fq, int K, float nyquist, bool nyq) {
  int live = K;
  if (nyq && fq > 0.f) {
    int k = (int)fminf(nyquist / fq, (float)K);
    while (k < K && __fmul_rn(fq, (float)(k + 1)) < nyquist) ++k;
    while (k > 0 && !(__fmul_rn(fq, (float)k) < nyquist)) --k;
    live = k;
  }
  return live;
}

// The exact per-oscillator slow path (f0 < 1 Hz) behind one call.
__device__ __noinline__ float sample_exact(const float* x0, int row_stride, float w0,
                                           float w1, uint32_t p32, float f_lo, float f_hi,
                                           float frac, int K, float nyq) {
  return harmonic_sample_exact(x0, x0 + row_stride, w0, w1, p32, f_lo, f_hi, frac, K, nyq);
}

// Oscillator state of the lane's TWO samples (.x = sample r, .y = sample r + 32):
// vo = sin((1+2j) phi), ve = sin((2+2j) phi); both chains step by the angle 2 phi
// reduced to [-pi/2, pi/2] (sg = -1 where it was shifted by half a turn: every
// other step then flips sign, hence the accumulators split by step parity e / o).
struct Osc2 {
  float2 vo, ve, dlo, dle, na, sg;
  float2 s0e, s0o, s1e, s1o;     // row x0 / x1, step parity: odd-harmonic chain
  float2 t0e, t0o, t1e, t1o;     // ... even-harmonic chain
};

// q = 2^32 * (phase + 2^-9) mod 2^32 for both samples.
__device__ __forceinline__ void osc_seed2(Osc2& st, uint32_t qa, uint32_t qb,
                                          const float* __restrict__ sSin,
                                          const float* __restrict__ sCos) {
  const uint32_t ia = qa >> (32 - kSinTabBits), ib = qb >> (32 - kSinTabBits);
  const float2 tx = make_float2(sSin[ia], sSin[ib]);
  const float2 ty = make_float2(sCos[ia], sCos[ib]);
  constexpr uint32_t kLow = (1u << (32 - kSinTabBits)) - 1u;
  constexpr float kC = 1.4629180792671596e-9f;                    // 2 pi / 2^32
  constexpr float kOff = -(float)(1u << (31 - kSinTabBits)) * kC;
  const float2 eps = ffma2(make_float2((float)(qa & kLow), (float)(qb & kLow)),
                                make_float2(kC, kC), make_float2(kOff, kOff));
  const float2 e2 = fmul2(eps, eps);
  const float2 ce = ffma2(e2, make_float2(-0.5f, -0.5f), make_float2(1.f, 1.f));
  const float2 se = fmul2(eps, ffma2(e2, make_float2(-0.16666667f, -0.16666667f),
                                               make_float2(1.f, 1.f)));
  const float2 nse = make_float2(-se.x, -se.y);
  const float2 s1 = ffma2(ty, se, fmul2(tx, ce));
  const float2 c1 = ffma2(tx, nse, fmul2(ty, ce));
  const float2 ss = fmul2(s1, s1), cc = fmul2(c1, c1);
  const float2 s2 = fmul2(fadd2(s1, s1), c1);           // sin(2 phi)
  st.sg = make_float2(ss.x > cc.x ? -1.0f : 1.0f, ss.y > cc.y ? -1.0f : 1.0f);
  st.na = fmul2(make_float2(fminf(ss.x, cc.x), fminf(ss.y, cc.y)),
                     make_float2(-4.0f, -4.0f));
  st.vo = s1;
  st.ve = s2;
  st.dlo = ffma2(s1, st.sg, s1);                             // 2 s1, or 0 if shifted
  st.dle = s2;
}

__device__ __forceinline__ void osc_step(Osc2& st) {
  st.dlo = ffma2(st.na, st.vo, st.dlo);
  st.dle = ffma2(st.na, st.ve, st.dle);
  st.vo = fadd2(st.vo, st.dlo);
  st.ve = fadd2(st.ve, st.dle);
}

// Four harmonics (k+1 .. k+4) of both samples: two chain steps.  Each of the
// eight accumulators takes ONE f32x2 FMA per group (two back-to-back updates of one
// accumulator made ptxas rotate registers through MOVs at the loop edge).
__device__ __forceinline__ void osc_group(Osc2& st, const float4& X0, const float4& X1) {
  st.s0e = bffma2(X0.x, st.vo, st.s0e);
  st.s1e = bffma2(X1.x, st.vo, st.s1e);
  st.t0e = bffma2(X0.y, st.ve, st.t0e);
  st.t1e = bffma2(X1.y, st.ve, st.t1e);
  osc_step(st);
  st.s0o = bffma2(X0.z, st.vo, st.s0o);
  st.s1o = bffma2(X1.z, st.vo, st.s1o);
  st.t0o = bffma2(X0.w, st.ve, st.t0o);
  st.t1o = bffma2(X1.w, st.ve, st.t1o);
  osc_step(st);
}

// First four harmonics: the accumulators are written, not accumulated into.
__device__ __forceinline__ void osc_group_first(Osc2& st, const float4& X0,
                                                const float4& X1) {
  st.s0e = bfmul2(X0.x, st.vo);
  st.s1e = bfmul2(X1.x, st.vo);
  st.t0e = bfmul2(X0.y, st.ve);
  st.t1e = bfmul2(X1.y, st.ve);
  osc_step(st);
  st.s0o = bfmul2(X0.z, st.vo);
  st.s1o = bfmul2(X1.z, st.vo);
  st.t0o = bfmul2(X0.w, st.ve);
  st.t1o = bfmul2(X1.w, st.ve);
  osc_step(st);
}

// Four harmonics with per-sample live counts (ka, kb): the sines are masked.
__device__ __forceinline__ void osc_group_masked(Osc2& st, const float4& X0,
                                                 const float4& X1, int k, int ka,
                                                 int kb) {
  float2 mo = make_float2(k + 1 <= ka ? st.vo.x : 0.f, k + 1 <= kb ? st.vo.y : 0.f);
  float2 me = make_float2(k + 2 <= ka ? st.ve.x : 0.f, k + 2 <= kb ? st.ve.y : 0.f);
  st.s0e = bffma2(X0.x, mo, st.s0e);
  st.s1e = bffma2(X1.x, mo, st.s1e);
  st.t0e = bffma2(X0.y, me, st.t0e);
  st.t1e = bffma2(X1.y, me, st.t1e);
  osc_step(st);
  mo = make_float2(k + 3 <= ka ? st.vo.x : 0.f, k + 3 <= kb ? st.vo.y : 0.f);
  me = make_float2(k + 4 <= ka ? st.ve.x : 0.f, k + 4 <= kb ? st.ve.y : 0.f);
  st.s0o = bffma2(X0.z, mo, st.s0o);
  st.s1o = bffma2(X1.z, mo, st.s1o);
  st.t0o = bffma2(X0.w, me, st.t0o);
  st.t1o = bffma2(X1.w, me, st.t1o);
  osc_step(st);
}

__device__ __forceinline__ float4 mask4u(const float4& X, int rem) {
  return make_float4(X.x, rem > 1 ? X.y : 0.f, rem > 2 ? X.z : 0.f, 0.f);
}

struct LaneConst {
  uint32_t c1a, c2a, c1b, c2b;   // r + 1, r (r + 1) / 2 for the lane's two samples
  float2 w1;                     // amplitude weight of row x1 (Hann or linear)
};

template <bool WINDOW>
__device__ __forceinline__ LaneConst lane_const(int r0, int lane, float inv_hop,
                                                const float* __restrict__ sW) {
  LaneConst c;
  const uint32_t ra = r0 + lane, rb = ra + 32;
  c.c1a = ra + 1; c.c2a = (ra * (ra + 1)) >> 1;
  c.c1b = rb + 1; c.c2b = (rb * (rb + 1)) >> 1;
  // keep the constants in registers: ptxas otherwise re-derives them (and their
  // integer feeds) in every frame
  asm volatile("" : "+r"(c.c1a), "+r"(c.c2a), "+r"(c.c1b), "+r"(c.c2b));
  if (sW != nullptr) {
    c.w1 = make_float2(sW[ra], sW[rb]);
  } else {
    const float fa = (float)ra * inv_hop, fb = (float)rb * inv_hop;
    c.w1 = make_float2(WINDOW ? (0.5f - 0.5f * cospif(fa)) : fa,
                       WINDOW ? (0.5f - 0.5f * cospif(fb)) : fb);
  }
  asm volatile("" : "+f"(c.w1.x), "+f"(c.w1.y));
  return c;
}

// 64 samples of one frame (samples r0 + lane and r0 + lane + 32) by one warp.
// x0 = sX + xoff is the frame's own row, x1 = x0 + Kp the next one; `out` points at
// the lane's first sample.
__device__ __forceinline__ void frame_chunk(
    const float* __restrict__ sX, int xoff, int Kp, const FrameRec* __restrict__ rec,
    const LaneConst& lc, int r0, float inv_hop, const float* __restrict__ sSin,
    const float* __restrict__ sCos, int K, float nyquist, int lane,
    float* __restrict__ out, int accumulate) {
  const float* __restrict__ x0 = sX + xoff;
  const uint32_t kp4 = (uint32_t)Kp << 2;               // bytes from row x0 to row x1
  const ulonglong2 PA = *reinterpret_cast<const ulonglong2*>(&rec->P);
  const uint4 Dk = *reinterpret_cast<const uint4*>(&rec->D);
  const float4 fa = *reinterpret_cast<const float4*>(&rec->f_lo);
  const unsigned long long D = ((unsigned long long)Dk.y << 32) | Dk.x;
  const int ng = (int)Dk.z, rem = (int)Dk.w;
  const uint32_t qa = phase32(PA.x, PA.y, D, lc.c1a, lc.c2a);
  const uint32_t qb = phase32(PA.x, PA.y, D, lc.c1b, lc.c2b);
  // (1 - w1) amp0, w1 amp1
  const float2 w0 = ffma2(make_float2(-lc.w1.x, -lc.w1.y), make_float2(fa.z, fa.z),
                               make_float2(fa.z, fa.z));
  const float2 w1 = bfmul2(fa.w, lc.w1);
  float2 y;
  if (ng < 0) {              // f0 < 1 Hz somewhere: exact per-oscillator path
    constexpr uint32_t kRound = 1u << (31 - kSinTabBits);
    int ra = r0 + lane, xo = xoff;
    asm volatile("" : "+r"(ra), "+r"(xo));      // nothing of this path runs ahead of the branch
    const float fra = (float)ra * inv_hop, frb = (float)(ra + 32) * inv_hop;
    y.x = sample_exact(sX + xo, Kp, w0.x, w1.x, qa - kRound, fa.x, fa.y, fra, K, nyquist);
    y.y = sample_exact(sX + xo, Kp, w0.y, w1.y, qb - kRound, fa.x, fa.y, frb, K, nyquist);
  } else {
    Osc2 st;
    osc_seed2(st, qa, qb, sSin, sCos);
    if (ng > 0) {
      // every sample of the frame has the same live count: ng unmasked groups,
      // then (rem != 0) one group masked with warp-uniform predicates.  The
      // first group writes the accumulators (no zeroing); an even count runs
      // its second group alone; the loop runs pairs of groups on one 32-bit
      // shared address into row x0 (row x1 is that address plus 4 Kp).  The
      // harmonics stay in order, so the sums are those of one group at a time.
      uint32_t a = smem_u32(x0);
      const uint32_t a_end = a + (ng << 4);         // ng >= 1
      osc_group_first(st, lds128(a), lds128(a + kp4));
      a += 16;
      if ((ng & 1) == 0) {
        osc_group(st, lds128(a), lds128(a + kp4));
        a += 16;
      }
#pragma unroll 1
      while (a != a_end) {
        osc_group(st, lds128(a), lds128(a + kp4));
        osc_group(st, lds128(a + 16), lds128(a + kp4 + 16));
        a += 32;
      }
      if (rem != 0) osc_group(st, mask4u(lds128(a), rem), mask4u(lds128(a + kp4), rem));
    } else {                 // live count changes inside this frame (or is < 4)
      int ra = r0 + lane;
      asm volatile("" : "+r"(ra));
      const float fra = (float)ra * inv_hop, frb = (float)(ra + 32) * inv_hop;
      const int ka = live_harmonics(fa.x, fa.y, fra, K, nyquist);
      const int kb = live_harmonics(fa.x, fa.y, frb, K, nyquist);
      const int kmin = __reduce_min_sync(0xffffffffu, min(ka, kb));
      const int kmax = __reduce_max_sync(0xffffffffu, max(ka, kb));
      st.s0e = st.s0o = st.s1e = st.s1o = make_float2(0.f, 0.f);
      st.t0e = st.t0o = st.t1e = st.t1o = make_float2(0.f, 0.f);
      // the groups every sample keeps whole, addressed as in the uniform loop
      uint32_t a = smem_u32(x0);
      const uint32_t a_main = a + ((kmin & ~3) << 2);
      if (kmin & 4) {
        osc_group(st, lds128(a), lds128(a + kp4));
        a += 16;
      }
#pragma unroll 1
      while (a != a_main) {
        osc_group(st, lds128(a), lds128(a + kp4));
        osc_group(st, lds128(a + 16), lds128(a + kp4 + 16));
        a += 32;
      }
      for (int k = kmin & ~3; k < kmax; k += 4, a += 16)
        osc_group_masked(st, lds128(a), lds128(a + kp4), k, ka, kb);
    }
    const float2 t0 = ffma2(st.sg, fadd2(st.s0o, st.t0o), fadd2(st.s0e, st.t0e));
    const float2 t1 = ffma2(st.sg, fadd2(st.s1o, st.t1o), fadd2(st.s1e, st.t1e));
    y = ffma2(t1, w1, fmul2(t0, w0));
  }
  if (accumulate) {
    y.x += out[0];
    y.y += out[32];
  }
  out[0] = y.x;
  out[32] = y.y;
}

template <bool WINDOW, int HOPT>
__global__ void __launch_bounds__(NT, MIN_CTAS)
harmonic_v4_kernel(HarmonicParams p, int use_tma, int FW) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int hop = HOPT ? HOPT : p.hop;
  const int Kp = p.Kp, K = p.K, F = p.F;
  const int FT = FW * NW;
  const Smem L = smem_layout(FW, Kp, hop);
  void* mbar = (void*)(smem_raw + L.off_mbar);
  float* sSin = (float*)(smem_raw + L.off_sin);
  float* sCos = (float*)(smem_raw + L.off_cos);
  float* sX = (float*)(smem_raw + L.off_x);
  float* sW = (HOPT == 64) ? nullptr : (float*)(smem_raw + L.off_w);
  double* sRedD = (double*)(smem_raw + L.off_red);                        // [NW]
  unsigned long long* sWarpTot = (unsigned long long*)(smem_raw + L.off_red) + NW;
  float* sInv = (float*)(smem_raw + L.off_inv);                           // [FT + 1]
  FrameRec* sRec = (FrameRec*)(smem_raw + L.off_rec);                     // [FT]
  int* sLive = (int*)(smem_raw + L.off_live);                             // [FT + 1]

  const int b = blockIdx.y;
  const int i0 = blockIdx.x * FT;
  const int nfr = min(FT, F - i0);
  const int rows_in = min(nfr + 1, F - i0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* f0b = p.f0 + (size_t)b * F;
  const float* ampb = p.amps + (size_t)b * F;

  // Programmatic dependent launch: the noise kernel of the decoder may start
  // its prologue on SMs this grid has vacated.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  HV4_TIMING_DECL;
  // ---- 0. the frame slab: one TMA bulk copy, issued before anything else ----
  if (use_tma && tid == 0) {
    mbar_init(mbar, 1);
    const uint32_t bytes = (uint32_t)rows_in * (uint32_t)K * 4u;
    mbar_expect_tx(mbar, bytes);
    tma_bulk_g2s(sX, p.hd + ((size_t)b * F + i0) * K, bytes, mbar);
  }

  // ---- 1. every global load of the prologue is issued here, back to back: the
  //         f0 values before the tile (prefix sum, 16-byte loads where the item's
  //         row is aligned), the table, the tile's frames, the two frequencies of
  //         the closed-form tile phase.  One memory round trip instead of up to ten
  //         dependent ones (the prologue was 8 % of the instructions and 23 % of
  //         the warp time in the first capture of this kernel).
  //         RECORD WARPS: the per-frame quantities are computed with lane = frame
  //         by the first ceil(FT / 32) warps for the whole tile (every warp doing
  //         it for its own FW frames ran the same 300 instructions NW times).
  const int n_rec = (FT + 31) >> 5;                     // record warps
  const bool rec_warp = warp < n_rec;
  const int fr = warp * 32 + lane;                      // tile frame of a record lane
  const int cnt = max(0, min(32, nfr - warp * 32));     // frames of this record warp
  const bool raw_scale = p.ctl_flags & DDSP_B200_CTL_SCALE;
  //         CONTROLS WARPS: get_controls rows are split over the warps that build
  //         no records (over all warps when every warp builds records), so that
  //         the transform runs while the records are built.
  const int n_ctl = (NW > n_rec) ? NW - n_rec : NW;
  const int cw = (NW > n_rec) ? warp - n_rec : warp;  // < 0: no rows
  const int rw = (nfr + n_ctl - 1) / n_ctl;
  const int c0 = cw * rw;                               // first row of the warp
  const int ncr = (cw < 0) ? 0 : max(0, min(rw, nfr - c0));
  const bool c_last = ncr > 0 && c0 + ncr == nfr;
  const int nrows = ncr + ((c_last && rows_in > nfr) ? 1 : 0);   // + the real row after the tile
  const float f_row = (lane < nrows) ? f0b[min(i0 + c0 + lane, F - 1)] : 0.f;
  float f = 0.f, a = 0.f, f_tile = 0.f, f_first = 0.f;
  float f_x = 0.f, a_x = 0.f;      // lane 31 of a full record warp: the frame after its range
  if (rec_warp && cnt > 0) {
    if (lane <= cnt) {
      const int g = min(i0 + fr, F - 1);                // frame F := frame F-1
      f = f0b[g];
      a = ampb[g];
    }
    if (lane == 31 && cnt == 32) {
      const int g = min(i0 + fr + 1, F - 1);
      f_x = f0b[g];
      a_x = ampb[g];
    }
    f_tile = f0b[i0];
    f_first = f0b[0];
  }
  constexpr int TPT = kSinTab / NT;                     // table entries per thread
  static_assert(TPT * NT == kSinTab, "the table splits evenly over the CTA");
  float2 tab[TPT];
#pragma unroll
  for (int u = 0; u < TPT; ++u) tab[u] = hcm::g_sincos256[tid + u * NT];
  double part = 0.0;
  if ((reinterpret_cast<uintptr_t>(f0b) & 15) == 0) {
    const float4* f4 = reinterpret_cast<const float4*>(f0b);
    const int n4 = i0 >> 2;
    float4 v[4];
    int j = tid;
    for (; j + 3 * NT < n4; j += 4 * NT) {
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = f4[j + u * NT];
#pragma unroll
      for (int u = 0; u < 4; ++u)
        part += ((double)v[u].x + (double)v[u].y) + ((double)v[u].z + (double)v[u].w);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u)
      v[u] = (j + u * NT < n4) ? f4[j + u * NT] : make_float4(0.f, 0.f, 0.f, 0.f);
    const float tail = (tid < (i0 & 3)) ? f0b[4 * n4 + tid] : 0.f;   // i0 % 4 frames
#pragma unroll
    for (int u = 0; u < 4; ++u)
      part += ((double)v[u].x + (double)v[u].y) + ((double)v[u].z + (double)v[u].w);
    part += (double)tail;
  } else {
#pragma unroll 4
    for (int j = tid; j < i0; j += NT) part += (double)f0b[j];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if (lane == 0) sRedD[warp] = part;
#pragma unroll
  for (int u = 0; u < TPT; ++u) {
    sSin[tid + u * NT] = tab[u].x;
    sCos[tid + u * NT] = tab[u].y;
  }
  const float inv_hop = 1.0f / (float)hop;
  if (HOPT != 64) {
    for (int r = tid; r < hop; r += NT) {
      const float frac = (float)r * inv_hop;
      sW[r] = WINDOW ? (0.5f - 0.5f * cospif(frac)) : frac;
    }
  }
  if (!use_tma) {
    if (p.hd != nullptr) {
      const float* hdb = p.hd + ((size_t)b * F + i0) * K;
      for (int idx = tid; idx < rows_in * Kp; idx += NT) {
        int r = idx / Kp, c = idx - r * Kp;
        sX[idx] = (c < K) ? hdb[r * K + c] : 0.f;
      }
    } else {
      for (int idx = tid; idx < rows_in * Kp; idx += NT)
        sX[idx] = (idx % Kp == 0) ? 1.0f : 0.f;
    }
  }
  HV4_LAP(0);
  __syncthreads();            // tables, mbarrier init, partial sums, (LDG slab)
  HV4_LAP(1);

  // ---- 2. frame records (record warps, lane = frame) ----
  const bool have_ctl = (p.ctl_flags != 0) && (p.hd != nullptr);
  // rows are zero above their frame-rate live count (get_controls did it here)
  const bool zero_ok = have_ctl && (p.ctl_flags & DDSP_B200_CTL_NYQUIST);
  unsigned long long excl = 0;            // wrapping sum of the record warp's earlier frame totals
  if (rec_warp && cnt > 0) {
    if (raw_scale && lane <= cnt) a = exp_sigmoid_f(a);   // synths.py:110-111
    const float f_next = __shfl_down_sync(0xffffffffu, f, 1);
    const float a_next = __shfl_down_sync(0xffffffffu, a, 1);
    // lane 31 of a full record warp needs frame 32 of the NEXT record warp's range
    float f_n = f_next, a_n = a_next;
    if (lane == 31 && cnt == 32) {
      f_n = f_x;
      a_n = raw_scale ? exp_sigmoid_f(a_x) : a_x;
    }
    unsigned long long tot = 0;
    double a0 = 0.0, dd = 0.0;
    if (lane < cnt) {
      a0 = (double)f * p.inv_sr;
      const double a1 = (double)f_n * p.inv_sr;
      dd = (a1 - a0) * (1.0 / (double)hop);
      tot = frame_total_fix64(a0, a1, hop);
    }
    const unsigned long long incl = warp_scan_frame_totals(tot, lane);
    excl = incl - tot;
    if (lane == 31) sWarpTot[warp] = incl;             // total of the record warp's frames
    const bool nyq = p.ctl_flags & DDSP_B200_CTL_NYQUIST;
    const int live = row_live_count(f, K, p.nyquist, nyq);
    int live_next = __shfl_down_sync(0xffffffffu, live, 1);
    if (lane == 31 && cnt == 32) live_next = row_live_count(f_n, K, p.nyquist, nyq);
    int ng = -1, rem = 0;                              // exact slow path
    if (lane < cnt && f >= 1.0f && f_n >= 1.0f) {
      const int kca = live_harmonics(f, f_n, 0.0f, K, p.nyquist);
      const int kcb = live_harmonics(f, f_n, (float)(hop - 1) * inv_hop, K, p.nyquist);
      ng = 0;                                          // per-sample live counts
      if (kca == kcb) {
        if (zero_ok && live == kca && live_next <= kca) {
          ng = max(1, (kca + 3) >> 2);                 // zeros above kca in both rows
        } else {
          ng = kca >> 2;                               // (0: the general path)
          rem = kca & 3;
        }
      }
    }
    if (lane < cnt) {
      FrameRec r;
      r.P = 0; r.A = turns_to_fix64(a0); r.D = turns_to_fix64(dd);
      r.ng = ng; r.rem = rem;
      r.f_lo = f; r.f_hi = f_n; r.amp0 = a; r.amp1 = a_n;
      sRec[fr] = r;
    }
    // the record warps' totals (sWarpTot) are shared among the record warps only
    const int n_act = (nfr + 31) >> 5;
    if (n_act > 1) asm volatile("bar.sync 1, %0;" ::"r"(32 * n_act) : "memory");
    HV4_LAP(2);

    // phase at the start of the tile, then the record warp's offset
    double base_sum = 0.0;
#pragma unroll
    for (int w = 0; w < NW; ++w) base_sum += sRedD[w];
    const double a_tile = (double)f_tile * p.inv_sr;
    const double a_first = (double)f_first * p.inv_sr;
    unsigned long long P0 = tile_phase_base(base_sum, a_first, a_tile, hop, p.inv_sr);
    for (int w = 0; w < warp; ++w) P0 += sWarpTot[w];
    if (lane < cnt) {
      const unsigned long long Pf = P0 + excl;         // exact frame phase, 2^64 = 1 turn
      sRec[fr].P = Pf + 0x80000000ull + (1ull << (63 - kSinTabBits));
    }
  }
  HV4_LAP(3);

  // ---- 3. get_controls on the controls warp's rows (synths.py:110-117) ----
  if (ncr > 0) {
    float* sXw = sX + (size_t)c0 * Kp;
    if (have_ctl) {
      const bool nyq = p.ctl_flags & DDSP_B200_CTL_NYQUIST;
      for (int r = lane; r < nrows; r += 32)
        sLive[c0 + r] = row_live_count(r == lane ? f_row : f0b[min(i0 + c0 + r, F - 1)], K,
                                       p.nyquist, nyq);
      __syncwarp();
    }
    if (use_tma) mbar_wait(mbar, 0);
    HV4_LAP(4);
    if (have_ctl) {
      if (Kp <= 128) {
        for (int r0 = 0; r0 < nrows; r0 += 4)
          controls_rows4(sXw, sLive + c0, sInv + c0, r0, nrows, Kp, raw_scale, lane);
      } else {
        for (int r0 = 0; r0 < nrows; r0 += 4)
          controls_rows(sXw, sLive + c0, r0, nrows, Kp, raw_scale, lane);
        for (int r = lane; r < nrows; r += 32) sInv[c0 + r] = 1.0f;
      }
    } else {
      for (int r = lane; r < nrows; r += 32) sInv[c0 + r] = 1.0f;
    }
    if (c_last && rows_in < nfr + 1) {                  // frame F := frame F-1
      __syncwarp();
      for (int c = lane; c < Kp; c += 32) sXw[ncr * Kp + c] = sXw[(ncr - 1) * Kp + c];
      if (lane == 0) sInv[c0 + ncr] = sInv[c0 + ncr - 1];
    }
  }
  HV4_LAP(5);
  __syncthreads();   // the records, the transformed rows and their 1 / sum
  HV4_LAP(6);

  // ---- 4. samples: the warp's own FW frames ----
  const int w0f = warp * FW;
  const int nfw = max(0, min(FW, nfr - w0f));
  if (nfw > 0) {
    FrameRec* rec = sRec + w0f;
    if (lane < nfw) {                                   // amp / row sum
      rec[lane].amp0 *= sInv[w0f + lane];
      rec[lane].amp1 *= sInv[w0f + lane + 1];
    }
    __syncwarp();
    float* o = p.audio + (size_t)b * p.N + (size_t)(i0 + w0f) * hop + lane;
    int xoff = w0f * Kp;
    if (HOPT == 64) {
      const LaneConst lc = lane_const<WINDOW>(0, lane, inv_hop, nullptr);
#pragma unroll 1
      for (int li = 0; li < nfw; ++li, ++rec, xoff += Kp, o += 64) {
        frame_chunk(sX, xoff, Kp, rec, lc, 0, inv_hop, sSin, sCos, K, p.nyquist, lane, o,
                    p.accumulate);
      }
    } else {
      for (int li = 0; li < nfw; ++li, ++rec, xoff += Kp) {
        for (int r0 = 0; r0 < hop; r0 += 64, o += 64) {
          const LaneConst lc = lane_const<WINDOW>(r0, lane, inv_hop, sW);
          frame_chunk(sX, xoff, Kp, rec, lc, r0, inv_hop, sSin, sCos, K, p.nyquist, lane, o,
                      p.accumulate);
        }
      }
    }
  }
  HV4_LAP(7);
  HV4_TIMING_FLUSH();
}

}  // namespace hv4

// Returns 0 on success, negative on error, 1 if the tile cannot fit shared memory
// (the caller then takes the generic kernel).
int launch_harmonic_v4(HarmonicParams p, cudaStream_t st) {
  using namespace hv4;
  p.Kp = (p.K + 3) & ~3;
  // Four warps per CTA and 8 frames per warp: one full record warp for the 32-frame
  // tile while the other three transform its 33 rows.  Small grids shrink the tile
  // until every SM has one.
  int FW = 8;
  const long long want_ctas = 8ll * num_sms();                   // 32 warps per SM
  while (FW > 4 && (long long)p.B * ((p.F + FW * NW - 1) / (FW * NW)) < want_ctas) FW = (FW + 1) >> 1;
  while (FW > 1 && (long long)p.B * ((p.F + FW * NW - 1) / (FW * NW)) < num_sms()) FW = (FW + 1) >> 1;
  FW =std::max(1, std::min(FW, (p.F + NW - 1) / NW));
  while (FW > 1 && smem_layout(FW, p.Kp, p.hop).total > 64 * 1024) FW = (FW + 1) / 2;
  const size_t smem = smem_layout(FW, p.Kp, p.hop).total;
  if (smem > kMaxDynSmem) return 1;
  const int use_tma = (p.hd != nullptr) && (p.K % 4 == 0) &&
                      (((uintptr_t)p.hd & 15) == 0);
  dim3 grid((p.F + FW * NW - 1) / (FW * NW), p.B);
  const bool win = p.amp_method == DDSP_B200_AMP_WINDOW;
  auto kern = p.hop == 64 ? (win ? harmonic_v4_kernel<true, 64> : harmonic_v4_kernel<false, 64>)
                          : (win ? harmonic_v4_kernel<true, 0> : harmonic_v4_kernel<false, 0>);
  return launch("harmonic_forward(v4)", kern, grid, NT, smem, st, p, use_tma, FW);
}

}  // namespace ddsp
