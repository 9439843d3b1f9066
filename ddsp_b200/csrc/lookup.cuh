// core.linear_lookup (core.py:1168-1214) as a stand-alone op: phase [B, N] reads tables
// [B, W] (one per item) or [B, N, W] (one per sample) with the reference's own formula,
//   out_t = sum_{j=0..W} relu(1 - |phase_t - lin_j| W) T_t[j mod W],
// lin = float32 linspace(0, 1, W + 1) as TensorFlow builds it (delta = 1 / W, lin_j =
// delta j, lin_W = 1), every step in float32.  A phase outside [0, 1] is not wrapped: it
// gets partial weights or none.  Only columns within one grid step of phase W carry weight,
// so each sample evaluates the four candidates floor(phase W) - 1 .. + 2 (the float32 grid
// is off by far less than a step for W <= DDSP_B200_LOOKUP_MAX_W) and never the other W - 3.
//
// Gradients are TensorFlow's (abs'(0) = relu'(0) = 0), as wavetable.cuh and mod_delay.cuh
// take them:
//   d phase_t = -W g_t sum_j [1 - d_j > 0] sign(phase_t - lin_j) T_t[j mod W],
//   d T_t[j mod W] += g_t w_j.
// d phase is exactly 0 on a grid point of a power-of-two W.  Per-sample tables get their
// gradient written densely, one warp per row.  Per-item tables reduce over time as
// wavetable.cuh's wt_bwd_table does, on its column tiles: per-warp shared column buffers
// filled with taps.cuh's scatter_tap and added in warp order; the time segments of one
// table are the CTAs of one cluster, added in rank order through distributed shared
// memory, so no workspace is needed.  No atomics and no memset: every gradient is
// bit-reproducible.
#pragma once
#include <cooperative_groups.h>

#include "wavetable.cuh"

namespace ddsp {
namespace ll_ {

constexpr int kThreads = 256;
constexpr int kCand = 4;              // candidate columns per sample
constexpr int kCl = 8;                // CTAs (time segments) per table in the [B, W] backward

struct Cand {
  int j[kCand];       // column of the extended table (W is column 0 again), -1: none
  float w[kCand];     // relu(1 - d_j)
  float s[kCand];     // sign(phase - lin_j) where 1 - d_j > 0, else 0
};

__device__ __forceinline__ Cand candidates(float phase, int W) {
  Cand c;
  const double pos = (double)phase * (double)W;
  const bool near = pos > -2.0 && pos < (double)W + 2.0;   // false for NaN too
  const int j0 = near ? (int)floor(pos) - 1 : -8;
  const float Wf = (float)W;
  const float delta = __fdiv_rn(1.0f, Wf);
#pragma unroll
  for (int i = 0; i < kCand; ++i) {
    const int j = j0 + i;
    c.j[i] = -1;
    c.w[i] = 0.f;
    c.s[i] = 0.f;
    if (j < 0 || j > W) continue;
    const float lin = j == W ? 1.0f : __fmul_rn(delta, (float)j);
    const float diff = __fsub_rn(phase, lin);
    const float one_minus = __fsub_rn(1.0f, __fmul_rn(fabsf(diff), Wf));
    c.j[i] = j;
    if (one_minus > 0.f) {
      c.w[i] = one_minus;
      c.s[i] = diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f);
    }
  }
  return c;
}

__device__ __forceinline__ int col(int j, int W) { return j == W ? 0 : j; }

// out_t (BWD = false) or d phase_t (BWD = true) of one sample per thread, over the
// rows = B N samples.  grid ceil(rows / kThreads); tab is [B, W] or, PER_SAMPLE, [B, N, W].
template <bool PER_SAMPLE, bool BWD>
__global__ void __launch_bounds__(kThreads)
ll_samples(const float* __restrict__ phase, const float* __restrict__ tab,
           const float* __restrict__ g, float* __restrict__ out, int64_t rows, int N, int W) {
  const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (i >= rows) return;
  const float* tr = tab + (size_t)(PER_SAMPLE ? i : i / N) * W;
  const Cand c = candidates(__ldg(phase + i), W);
  float acc = 0.f;
#pragma unroll
  for (int q = 0; q < kCand; ++q) {
    if (c.j[q] < 0) continue;
    const float v = __ldg(tr + col(c.j[q], W));
    acc = BWD ? __fadd_rn(acc, __fmul_rn(c.s[q], v)) : __fadd_rn(acc, __fmul_rn(c.w[q], v));
  }
  out[i] = BWD ? __fmul_rn(__fmul_rn(-(float)W, __ldg(g + i)), acc) : acc;
}

// d tables [B, N, W]: one warp per row writes the whole row.
__global__ void __launch_bounds__(kThreads)
ll_dtab_rows(const float* __restrict__ phase, const float* __restrict__ g,
             float* __restrict__ d_tab, int64_t rows, int W) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = ((int64_t)blockIdx.x * kThreads + threadIdx.x) >> 5; r < rows;
       r += ((int64_t)gridDim.x * kThreads) >> 5) {
    const Cand c = candidates(__ldg(phase + r), W);
    const float gt = __ldg(g + r);
    float* dr = d_tab + (size_t)r * W;
    for (int j = lane; j < W; j += 32) {
      float v = 0.f;
#pragma unroll
      for (int q = 0; q < kCand; ++q)
        if (c.j[q] >= 0 && col(c.j[q], W) == j) v = __fadd_rn(v, __fmul_rn(gt, c.w[q]));
      dr[j] = v;
    }
  }
}

// d tables [B, W]: one cluster of kCl CTAs per (item, column tile) (wavetable.cuh's
// tiles), grid (kCl * n_ct, min(B, 65535)); a cluster takes items blockIdx.y,
// + gridDim.y, ...  CTA `rank` scatters the samples of time segment `rank` into per-warp
// shared buffers and adds them in warp order into its first buffer; then each CTA adds
// one slice of the columns over the cluster's CTAs in rank order, through distributed
// shared memory.
__global__ void __cluster_dims__(kCl, 1, 1) __launch_bounds__(wt_::kTabWarps * 32)
ll_dtab_items(const float* __restrict__ phase, const float* __restrict__ g,
              float* __restrict__ d_tab, int B, int N, int W) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ float ll_buf[];                    // [kTabWarps][cols]
  __shared__ float stage[wt_::kTabWarps][32];
  const int rank = (int)cluster.block_rank();
  const int ct = blockIdx.x / kCl;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = ct * wt_::kTabCols, cols = min(wt_::kTabCols, W - c0);
  float* buf = ll_buf + warp * cols;
  const int a = (int)((long long)N * rank / kCl), e = (int)((long long)N * (rank + 1) / kCl);
  const int j0 = (int)((long long)cols * rank / kCl), j1 = (int)((long long)cols * (rank + 1) / kCl);
  for (int b = blockIdx.y; b < B; b += gridDim.y) {    // cluster-uniform
    for (int j = lane; j < cols; j += 32) buf[j] = 0.f;
    __syncwarp();
    const size_t row = (size_t)b * N;
    for (int base = a + warp * 32; base < e; base += wt_::kTabWarps * 32) {   // warp-uniform
      const int t = base + lane;
      const bool live = t < e;
      Cand c;
      float gt = 0.f;
      if (live) {
        c = candidates(__ldg(phase + row + t), W);
        gt = __ldg(g + row + t);
      } else {
#pragma unroll
        for (int q = 0; q < kCand; ++q) { c.j[q] = -1; c.w[q] = 0.f; }
      }
#pragma unroll
      for (int q = 0; q < kCand; ++q) {
        const int j = c.j[q] < 0 ? -1 : col(c.j[q], W);
        md_::scatter_tap(buf, stage[warp], j, __fmul_rn(gt, c.w[q]),
                         j >= c0 && j < c0 + cols, c0, lane);
      }
    }
    __syncthreads();
    for (int j = threadIdx.x; j < cols; j += wt_::kTabWarps * 32) {
      float acc = 0.f;
#pragma unroll
      for (int w = 0; w < wt_::kTabWarps; ++w) acc += ll_buf[w * cols + j];
      ll_buf[j] = acc;
    }
    cluster.sync();
    for (int j = j0 + threadIdx.x; j < j1; j += wt_::kTabWarps * 32) {
      float acc = 0.f;
      for (int q = 0; q < kCl; ++q) acc += cluster.map_shared_rank(ll_buf, q)[j];
      d_tab[(size_t)b * W + c0 + j] = acc;
    }
    cluster.sync();                     // no CTA refills or leaves while another reads it
  }
}

}  // namespace ll_
}  // namespace ddsp
