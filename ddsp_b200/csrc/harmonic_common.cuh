// Shared pieces of the fused harmonic kernels (hop % 64 == 0): the 256-entry
// sin / cos table and the 64-bit fixed-point phase.  Used by harmonic_v4.cuh
// (forward) and harmonic_bwd2.cuh (backward); backward.cuh takes the table size.
//
// Derivations (closed-form phase, Reinsch recurrence, per-row accumulators,
// live-count Nyquist culling) are in DESIGN.md section 3.1.
#pragma once
#include <cmath>

#include "harmonic.cuh"

namespace ddsp {

constexpr int kSinTabBits = 8;
constexpr int kSinTab = 1 << kSinTabBits;  // 256-entry (sin, cos) table

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

}  // namespace hcm
}  // namespace ddsp
