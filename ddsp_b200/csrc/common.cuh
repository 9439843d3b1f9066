// Shared helpers for libddsp_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <atomic>
#include <stdint.h>
#include <stdio.h>

#include "../../include/ddsp_b200.h"

namespace ddsp {

// ---- error reporting (thread-local string, no global mutable state) --------
void set_error(const char* fmt, ...);
void count_launch();

#define DDSP_REQUIRE(cond, code, ...)  \
  do {                                 \
    if (!(cond)) {                     \
      ::ddsp::set_error(__VA_ARGS__);  \
      return (code);                   \
    }                                  \
  } while (0)

#define DDSP_CHECK_LAUNCH(name)                                         \
  do {                                                                  \
    ::ddsp::count_launch();                                             \
    cudaError_t e__ = cudaGetLastError();                               \
    if (e__ != cudaSuccess) {                                           \
      ::ddsp::set_error("%s: CUDA error: %s", name,                     \
                        cudaGetErrorString(e__));                       \
      return DDSP_B200_E_CUDA;                                          \
    }                                                                   \
  } while (0)

// Dynamic shared memory one CTA may reserve (of 227 KB usable per CTA).
constexpr size_t kMaxDynSmem = 200 * 1024;

// Allows `kernel` to launch with `bytes` of dynamic shared memory (past the default
// 48 KB), or reports E_CUDA with `name` in front of the message.
template <typename K>
int set_smem(K kernel, size_t bytes, const char* name) {
  if (bytes > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(
        kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();   // reported here, not by the next launch check
      set_error("%s: cannot reserve %zu B of shared memory: %s", name, bytes,
                cudaGetErrorString(e));
      return DDSP_B200_E_CUDA;
    }
  }
  return 0;
}

// Reserves `smem`, launches `kern` and checks the launch: how every kernel of the
// library starts (noise_ring.cuh's programmatic dependent launch aside).  Returns 0, or
// E_CUDA with `name` in front of the message.
template <typename... KArgs, typename... Args>
int launch(const char* name, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem,
           cudaStream_t st, Args&&... args) {
  int rc = set_smem(kern, smem, name);
  if (rc) return rc;
  kern<<<grid, block, smem, st>>>(static_cast<Args&&>(args)...);
  DDSP_CHECK_LAUNCH(name);
  return 0;
}

// Upper bound on the SM count, for per-SM debug arrays (H100 SXM has 132).
constexpr int kMaxSMs = 256;

// SM count of the current device (132 on H100 SXM, 114 on H100 PCIe), queried
// once per device: persistent grids and grid caps are sized by it.
inline int num_sms() {
  static std::atomic<int> cache[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0) dev = 0;
  std::atomic<int>* slot = dev < 64 ? &cache[dev] : nullptr;
  int n = slot ? slot->load(std::memory_order_relaxed) : 0;
  if (n > 0) return n;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
    n = 132;   // the error surfaces at the launch that follows
  if (n > kMaxSMs) n = kMaxSMs;
  if (slot) slot->store(n, std::memory_order_relaxed);
  return n;
}

// ---- f32x2 arithmetic -------------------------------------------------------
// Two float lanes computed as two scalar round-to-nearest operations (Hopper has
// no packed f32x2 FMA).  The _rn intrinsics are never contracted or reassociated,
// so every lane is rounded exactly as the packed instruction would round it.
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) {
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}

// ---- fixed-point phase ------------------------------------------------------
// Phase is kept in *turns* as a 64-bit fixed-point fraction (2^64 == 1 turn).
// Wrapping integer addition is exact modular arithmetic, so the phase of the
// k-th harmonic is the wrapping product k * phase - no accumulation error, no
// large-argument sin.  This is the intent of core.angular_cumsum
// (core.py:799-866) carried out exactly.
__device__ __forceinline__ unsigned long long turns_to_fix64(double turns) {
  double fr = turns - rint(turns);  // [-0.5, 0.5]
  return (unsigned long long)__double2ll_rn(fr * 18446744073709551616.0);
}

// sin and cos of a fixed-point phase, rounded to 2^-32 turn: how every oscillator-bank
// kernel evaluates its oscillators (a backward recomputes the forward's bits).
__device__ __forceinline__ float fix64_pi31(unsigned long long ph) {
  const uint32_t p32 = (uint32_t)((ph + 0x80000000ull) >> 32);
  return (float)(int)p32 * 4.656612873077393e-10f;   // 2^-31: [-1, 1) half turns
}
__device__ __forceinline__ float fix64_sin(unsigned long long ph) {
  return sinpif(fix64_pi31(ph));
}
__device__ __forceinline__ float fix64_cos(unsigned long long ph) {
  return cospif(fix64_pi31(ph));
}

// core.exp_sigmoid (core.py:386-404): 2 * sigmoid(x)^ln(10) + 1e-7, evaluated
// as 2 * 2^(-ln10 * log2(1 + e^-x)) + 1e-7 on the SFU (3 MUFU ops): both limits
// are exact (x -> -inf: 1e-7, x -> +inf: 2 + 1e-7) and nothing overflows to NaN.
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float exp_sigmoid_f(float x) {
  const float kLog2e = 1.4426950408889634f;
  const float kLn10 = 2.302585092994046f;
  const float t = ex2_approx(-x * kLog2e);          // e^-x  (inf for x << 0)
  float l;                                           // log2(1 + e^-x), arg >= 1
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(1.0f + t));
  return fmaf(2.0f, ex2_approx(-kLn10 * l), 1e-7f);
}

// ---- Philox4x32-10 (Salmon et al., SC'11) ----------------------------------
struct Philox4 {
  uint32_t x, y, z, w;
};

__device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1,
                                                 uint32_t c2, uint32_t c3,
                                                 uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
  const uint32_t W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
    uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0;
    uint32_t n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += W0; k1 += W1;
  }
  return Philox4{c0, c1, c2, c3};
}

// 23 mantissa bits -> [1, 2) -> 2x - 3 in [-1, 1).
__device__ __forceinline__ float u32_to_pm1(uint32_t r) {
  return 2.0f * __uint_as_float((r >> 9) | 0x3F800000u) - 3.0f;
}

// Four consecutive noise samples (index 4*q .. 4*q+3) of batch item b.
__device__ __forceinline__ float4 noise4(uint32_t q, uint32_t b, uint64_t seed,
                                         uint64_t offset) {
  Philox4 r = philox4x32_10(q, b, (uint32_t)offset, (uint32_t)(offset >> 32),
                            (uint32_t)seed, (uint32_t)(seed >> 32));
  return make_float4(u32_to_pm1(r.x), u32_to_pm1(r.y), u32_to_pm1(r.z),
                     u32_to_pm1(r.w));
}

// --- mbarrier / TMA bulk copy (PTX) -----------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(void* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(void* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(
                   smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src,
                                             uint32_t bytes, void* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void mbar_wait(void* bar, uint32_t phase) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(phase)
      : "memory");
}

__device__ __forceinline__ void mbar_arrive(void* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar))
               : "memory");
}
// Named barrier over a subset of the CTA (ids 1..15; 0 is __syncthreads).
__device__ __forceinline__ void named_bar(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

}  // namespace ddsp
