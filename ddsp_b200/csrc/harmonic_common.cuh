// Base of the harmonic kernel family: the parameters and the entry points' checks
// of them, the reference's float32 Nyquist decision, the 256-entry sin / cos table
// and the 64-bit fixed-point phase arithmetic, which a backward kernel shares
// with its forward to reproduce the forward's phase.  Derivations (closed-form phase, Reinsch
// recurrence, per-row accumulators, live-count Nyquist culling): DESIGN.md 3.1.
#pragma once
#include <cmath>

#include "common.cuh"

namespace ddsp {

struct HarmonicParams {
  const float* __restrict__ f0;    // [B,F]
  const float* __restrict__ amps;  // [B,F]
  const float* __restrict__ hd;    // [B,F,K] or nullptr (K == 1, hd == 1)
  float* __restrict__ audio;       // [B,N]
  int B, F, K, N, hop;
  int FT;          // frames per CTA tile
  int Kp;          // smem row stride (floats)
  float sample_rate;
  float nyquist;
  double inv_sr;
  int amp_method;
  int accumulate;
  // 0: amps / hd are synthesizer CONTROLS (outputs of get_controls).
  // DDSP_B200_CTL_*: they are raw network outputs; Harmonic.get_controls
  // (synths.py:94-121) is applied while the frame slab is staged (fast path).
  int ctl_flags;
  // Streaming synthesis (core.harmonic_oscillator_bank, core.py:966-1025):
  const float* init_phase;   // [B] radians added to the phase, or nullptr
  float* final_phase;        // [B] phase after the last sample (radians), or nullptr
  int mask_nyquist;          // 0: no audio-rate Nyquist mask (streaming bank has none)
};

// The reference's float32 evaluation of the k-th harmonic's audio-rate
// frequency: hf = f0 * k (core.py:1044), then v1 bilinear
// lo + (hi - lo) * frac (core.py:617-620).  Explicit _rn intrinsics forbid FMA
// contraction so the Nyquist decision (core.py:888-890) matches op for op.
__device__ __forceinline__ float ref_harmonic_freq(float f_lo, float f_hi,
                                                   float frac, int k) {
  float kf = (float)k;
  float lo = __fmul_rn(f_lo, kf);
  float hi = __fmul_rn(f_hi, kf);
  return __fadd_rn(lo, __fmul_rn(__fsub_rn(hi, lo), frac));
}

// Number of harmonics k = 1..count that stay below Nyquist at this sample,
// assuming f_k(t) is non-decreasing in k (true whenever both frame f0 >= 1 Hz).
__device__ __forceinline__ int live_harmonics(float f_lo, float f_hi,
                                              float frac, int K, float nyq) {
  float ft = f_lo + (f_hi - f_lo) * frac;
  int k = (int)fminf(nyq / fmaxf(ft, 1e-3f), (float)K);
  k = max(0, min(k, K));
  while (k < K && ref_harmonic_freq(f_lo, f_hi, frac, k + 1) < nyq) ++k;
  while (k > 0 && !(ref_harmonic_freq(f_lo, f_hi, frac, k) < nyq)) --k;
  return k;
}

constexpr int kSinTabBits = 8;
constexpr int kSinTab = 1 << kSinTabBits;  // 256-entry (sin, cos) table

// The fused kernels need whole 64-sample chunks per frame.
inline bool harmonic_fused_supported(const HarmonicParams& p) {
  return (p.hop % 64 == 0) && p.hop <= 8192 && p.K <= 1024;
}

// The fused forward's launcher, defined in harmonic_v4.cuh and compiled in
// harmonic.cu only; the decoder in noise.cu launches the kernel through it.
int launch_harmonic_v4(HarmonicParams p, cudaStream_t st);

// The checks every harmonic entry point makes; `name` prefixes the messages.
static int harm_check(const char* name, int B, int F, int K, int N, int amp_method,
                      float sample_rate) {
  DDSP_REQUIRE(B >= 0 && F >= 1 && K >= 1 && N >= 1, DDSP_B200_E_INVALID,
               "%s: bad shape B=%d F=%d K=%d N=%d", name, B, F, K, N);
  DDSP_REQUIRE(amp_method == DDSP_B200_AMP_WINDOW || amp_method == DDSP_B200_AMP_LINEAR,
               DDSP_B200_E_INVALID, "%s: bad amp_method %d", name, amp_method);
  DDSP_REQUIRE(sample_rate > 0.f, DDSP_B200_E_INVALID,
               "%s: sample_rate must be positive", name);
  return 0;
}

// HarmonicParams of a harmonic entry point.  The caller sets the fields in which it
// differs: accumulate, ctl_flags, the phase pointers, mask_nyquist and Kp.
static HarmonicParams harm_params(const float* f0, const float* amps, const float* hd,
                                  float* audio, int B, int F, int K, int N,
                                  float sample_rate, int amp_method) {
  HarmonicParams p;
  p.f0 = f0; p.amps = amps; p.hd = hd; p.audio = audio;
  p.B = B; p.F = F; p.K = K; p.N = N; p.hop = N / F;
  p.sample_rate = sample_rate; p.nyquist = sample_rate * 0.5f;
  p.inv_sr = 1.0 / (double)sample_rate;
  p.amp_method = amp_method; p.accumulate = 0; p.ctl_flags = 0;
  p.init_phase = nullptr; p.final_phase = nullptr; p.mask_nyquist = 1;
  p.Kp = (K + 3) & ~3;
  return p;
}

// Fixed-point phase (2^64 = one turn) of a frame where a = f / sr goes linearly
// from a0 to a1: its total and its slope D = (a1 - a0) / hop.  harmonic_v4_kernel
// alone forms D as (a1 - a0) * (1.0 / hop), equal for power-of-two hops; at hop
// 192 the v4 forward's D and the backward's may differ in the last bit.
__device__ __forceinline__ unsigned long long frame_total_fix64(double a0, double a1, int hop) {
  return turns_to_fix64((double)hop * a0 + (a1 - a0) * (0.5 * (hop - 1)));
}
__device__ __forceinline__ unsigned long long frame_slope_fix64(double a0, double a1, int hop) {
  return turns_to_fix64((a1 - a0) / (double)hop);
}

// Phase at a tile's start: the telescoped sum of the earlier frames' totals in
// one double evaluation (2^-38 turn resolution).  base_sum sums their f0;
// a_first and a_tile, f / sr of frame 0 and of the tile's first frame, are
// formed by each caller in its own order.  v4 sums base_sum in float4 groups
// ((x + y) + (z + w)), the backward kernel strided over its threads: the sums can
// differ in the last bit, and the forward and backward phases then by about 2^-37
// turns.
__device__ __forceinline__ unsigned long long tile_phase_base(
    double base_sum, double a_first, double a_tile, int hop, double inv_sr) {
  return turns_to_fix64((double)hop * (base_sum * inv_sr) +
                        0.5 * (hop - 1) * (a_tile - a_first));
}

// Inclusive prefix over the warp of the lanes' frame totals (wrapping adds: exact).
__device__ __forceinline__ unsigned long long warp_scan_frame_totals(unsigned long long tot,
                                                                     int lane) {
  unsigned long long incl = tot;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long up = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += up;
  }
  return incl;
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

}  // namespace hcm
}  // namespace ddsp
