// Device helpers of the routing and modulated-delay kernels that the wavetable
// kernels share: resample_kernel's taps (routing.cuh) and the warp scatter of
// mod_delay.cuh's backward.  Kernels stay in their families' headers, so
// wavetable.cuh includes this one instead of theirs.
#pragma once
#include "common.cuh"

namespace ddsp {
namespace rt_ {

struct ResampleGeom {
  int F, N, method, add_endpoint;
  float scale;   // the forward's float32 index scale
  int hop;       // 'window' only
};

__host__ __device__ inline ResampleGeom resample_geom(int F, int N, int method,
                                                       int add_endpoint) {
  ResampleGeom g;
  g.F = F; g.N = N; g.method = method; g.add_endpoint = add_endpoint;
  g.scale = (!add_endpoint && N > 1) ? (float)(F - 1) / (float)(N - 1)
                                     : (float)F / (float)N;
  const int den = add_endpoint ? (F > 1 ? F : 1) : (F - 1 > 1 ? F - 1 : 1);
  g.hop = N / den;
  return g;
}

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }

// The frames sample t reads, and their weights, exactly as resample_kernel
// computes them.  Returns the tap count (1, 2 or 4).
__device__ __forceinline__ int resample_taps(const ResampleGeom& g, int t, int* idx,
                                             float* w) {
  if (g.method == 0) {
    const int i = t / g.hop, r = t - i * g.hop;
    const float w1 = 0.5f - 0.5f * cospif((float)r / (float)g.hop);
    idx[0] = i; w[0] = 1.0f - w1;
    idx[1] = min(i + 1, g.F - 1); w[1] = w1;
    return 2;
  }
  const float src = (float)t * g.scale;
  const float fl = floorf(src);
  if (g.method == 1) {
    idx[0] = min(max((int)fl, 0), g.F - 1); w[0] = 1.0f - (src - fl);
    idx[1] = min((int)ceilf(src), g.F - 1); w[1] = src - fl;
    return 2;
  }
  if (g.method == 2) {
    idx[0] = min((int)(g.add_endpoint ? floorf(src) : roundf(src)), g.F - 1);
    w[0] = 1.0f;
    return 1;
  }
  const int loc = (int)fl;
  const int off = (int)lrintf((src - fl) * 1024.0f);
  const double A = -0.75;
  const double xa = off * (1.0 / 1024.0), xb = (1024 - off) * (1.0 / 1024.0);
  const double ya = xa + 1.0, yb = xb + 1.0;
  w[0] = (float)(((A * ya - 5 * A) * ya + 8 * A) * ya - 4 * A);
  w[1] = (float)(((A + 2) * xa - (A + 3)) * xa * xa + 1);
  w[2] = (float)(((A + 2) * xb - (A + 3)) * xb * xb + 1);
  w[3] = (float)(((A * yb - 5 * A) * yb + 8 * A) * yb - 4 * A);
#pragma unroll
  for (int k = 0; k < 4; ++k) idx[k] = clampi(loc - 1 + k, 0, g.F - 1);
  return 4;
}

// lowest / highest frame sample t reads (non-decreasing in t)
__device__ __forceinline__ int resample_lo(const ResampleGeom& g, int t) {
  if (g.method == 0) return t / g.hop;
  const float src = (float)t * g.scale;
  if (g.method == 1) return min(max((int)floorf(src), 0), g.F - 1);
  if (g.method == 2) return min((int)(g.add_endpoint ? floorf(src) : roundf(src)), g.F - 1);
  return clampi((int)floorf(src) - 1, 0, g.F - 1);
}
__device__ __forceinline__ int resample_hi(const ResampleGeom& g, int t) {
  if (g.method == 0) return min(t / g.hop + 1, g.F - 1);
  const float src = (float)t * g.scale;
  if (g.method == 1) return min((int)ceilf(src), g.F - 1);
  if (g.method == 2) return min((int)(g.add_endpoint ? floorf(src) : roundf(src)), g.F - 1);
  return clampi((int)floorf(src) + 2, 0, g.F - 1);
}

// first t in [0, N) with hi(t) >= j (use_hi) or lo(t) > j (!use_hi); N if none
__device__ __forceinline__ int resample_bound(const ResampleGeom& g, int j, bool use_hi) {
  int a = 0, b = g.N;
  while (a < b) {
    const int m = a + ((b - a) >> 1);
    const bool past = use_hi ? resample_hi(g, m) >= j : resample_lo(g, m) > j;
    if (past) b = m; else a = m + 1;
  }
  return a;
}

}  // namespace rt_

namespace md_ {

// Adds `val` of every lane whose `target` lies in the tile to buf[target - s0].
// Fast path: valid targets strictly increasing over the lanes (every smooth phase),
// so no two lanes share one.  Otherwise lanes with one target are summed by the
// lowest of them, in lane order.  Both give the same bits: a lone lane adds its own
// value either way.
__device__ __forceinline__ void scatter_tap(float* buf, float* stage, int target,
                                            float val, bool valid, int s0, int lane) {
  int prev = valid ? target : -1;                 // inclusive max scan of valid targets
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, prev, o);
    if (lane >= o) prev = max(prev, u);
  }
  int below = __shfl_up_sync(0xffffffffu, prev, 1);
  if (lane == 0) below = -1;
  if (__all_sync(0xffffffffu, !valid || target > below)) {
    if (valid) buf[target - s0] += val;
    return;
  }
  stage[lane] = val;
  __syncwarp();
  const unsigned peers = __match_any_sync(0xffffffffu, valid ? target : -1);
  if (valid && (peers & ((1u << lane) - 1u)) == 0u) {
    float sum = 0.f;
    for (unsigned m = peers; m != 0u; m &= m - 1u) sum += stage[__ffs(m) - 1];
    buf[target - s0] += sum;
  }
  __syncwarp();
}

}  // namespace md_
}  // namespace ddsp
