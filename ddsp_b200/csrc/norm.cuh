// nn.Normalize followed by a ReLU, as every site of nn.ResNet runs them (nn.py:699-839):
//   y = max(0, xh * scale[c] + shift[c]),  xh = (x - mean_g) * rstd_g,
// over x [B, HW, C] channels-last (NHWC with H and W flattened), with the C channels in
// G groups of C / G (G = 1 'layer', 32 'group', C 'instance') and each (item, group)
// normalized over HW and its channels by its mean and population variance:
// rstd = 1 / sqrt(var + eps).  The backward recomputes xh and the ReLU mask from x with
// the forward's arithmetic, so only the per-(item, group) mean and rstd are saved.
//
// Geometry.  One cluster of kNormCluster CTAs per item; CTA `rank` owns a contiguous
// range of rows (positions of HW) across all C channels.  Thread t works on the channel
// quad q = t % (C / 4) and the row lane r = t / (C / 4): rows r, r + R, ... of its range,
// R = kNormThreads / (C / 4) lanes, one float4 per row.
//   Forward: per-thread Welford moments of its 4 channels; Chan merges over the row lanes
//   (a tree in shared memory), then over each group's channels (a tree); the group
//   moments of the 8 CTAs are merged in rank order by every CTA through distributed
//   shared memory; a second pass over the CTA's rows (from L2) writes y.
//   Backward: per-channel sums A = sum dv xh and S = sum dv (dv = dy where the forward's
//   ReLU passed), added over the row lanes by a tree; the CTA's per-channel sums go to a
//   partial buffer for dscale and dshift; scaled by scale[c] and added over each group's
//   channels and then over the cluster's 8 CTAs in rank order, they give the group means
//   of g = dv scale and g xh, and a second pass writes
//   dx = rstd (g - mean(g) - xh mean(g xh)).  A second, small launch adds the partials
//   over items and ranks in order: dscale and dshift.
// Every sum runs in a fixed order with no atomics: results are bit-reproducible, and an
// item's y and dx depend on that item alone.
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"

namespace ddsp {

constexpr int kNormCluster = DDSP_B200_NORM_CLUSTER;   // CTAs per item
constexpr int kNormThreads = 512;
constexpr int kNormMaxChannels = 4 * kNormThreads;   // one quad per thread at least

// Row lanes of a CTA for C channels.
__host__ __device__ inline int norm_lanes(int C) { return kNormThreads / (C / 4); }

// Dynamic shared memory: per-lane per-channel statistics (3 arrays in the forward, 2 in
// the backward) and two per-group values.
__host__ __device__ inline size_t norm_smem_bytes(int C, int G, bool backward) {
  return sizeof(float) * ((size_t)(backward ? 2 : 3) * norm_lanes(C) * C + 2 * (size_t)G);
}

// Rows [r0, r1) of HW that CTA `rank` owns.
__device__ __forceinline__ void norm_rows(int HW, int rank, int& r0, int& r1) {
  const int per = (HW + kNormCluster - 1) / kNormCluster;
  r0 = min(HW, rank * per);
  r1 = min(HW, r0 + per);
}

// Chan et al.'s merge of the moments (nb, mb, Mb) into (n, m, M): count, mean and sum of
// squared deviations.  An empty side leaves the other as it is.
__device__ __forceinline__ void chan_merge(float& n, float& m, float& M, float nb, float mb,
                                           float Mb) {
  if (nb == 0.0f) return;
  if (n == 0.0f) {
    n = nb, m = mb, M = Mb;
    return;
  }
  const float nt = n + nb, d = mb - m, f = nb / nt;
  m = fmaf(d, f, m);
  M = M + Mb + d * d * (n * f);
  n = nt;
}

__device__ __forceinline__ float norm_relu(float v) { return v <= 0.0f ? 0.0f : v; }

// x, y [B, HW, C]; scale, shift [C]; mean, rstd [B, G].  Grid: kNormCluster B CTAs.
__global__ void __cluster_dims__(kNormCluster, 1, 1) __launch_bounds__(kNormThreads, 2)
    norm_relu_forward_kernel(const float* __restrict__ x, const float* __restrict__ scale,
                             const float* __restrict__ shift, float* __restrict__ y,
                             float* __restrict__ mean, float* __restrict__ rstd, int HW, int C,
                             int G, float eps) {
  namespace cg = cooperative_groups;
  extern __shared__ float4 norm_smem4[];
  float* sm = reinterpret_cast<float*>(norm_smem4);
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int b = blockIdx.x / kNormCluster;
  const int nq = C / 4, R = norm_lanes(C), L = R * C, cpg = C / G;
  float* sn = sm;              // [R][C] counts
  float* smu = sm + L;         // [R][C] means
  float* sM = sm + 2 * L;      // [R][C] sums of squared deviations
  float* gmean = sm + 3 * L;   // [G]
  float* grstd = gmean + G;    // [G]
  const int t = threadIdx.x, q = t % nq, r = t / nq;
  const bool active = r < R;
  int r0, r1;
  norm_rows(HW, rank, r0, r1);
  const float* xb = x + (int64_t)b * HW * C + 4 * q;

  if (active) {
    float n = 0.0f, m[4] = {0.0f, 0.0f, 0.0f, 0.0f}, M[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll 4
    for (int row = r0 + r; row < r1; row += R) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(xb + (int64_t)row * C));
      const float xv[4] = {v.x, v.y, v.z, v.w};
      n += 1.0f;
      const float inv = 1.0f / n;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float d = xv[k] - m[k];
        m[k] = fmaf(d, inv, m[k]);
        M[k] = fmaf(d, xv[k] - m[k], M[k]);
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int e = r * C + 4 * q + k;
      sn[e] = n, smu[e] = m[k], sM[e] = M[k];
    }
  }
  __syncthreads();
  for (int s = 1; s < R; s *= 2) {   // row lanes: lane r takes lane r + s
    for (int e = t; e < L; e += kNormThreads) {
      const int rr = e / C;
      if (rr % (2 * s) == 0 && rr + s < R)
        chan_merge(sn[e], smu[e], sM[e], sn[e + s * C], smu[e + s * C], sM[e + s * C]);
    }
    __syncthreads();
  }
  for (int s = 1; s < cpg; s *= 2) {   // a group's channels: channel k takes k + s
    for (int c = t; c < C; c += kNormThreads) {
      const int k = c % cpg;
      if (k % (2 * s) == 0 && k + s < cpg)
        chan_merge(sn[c], smu[c], sM[c], sn[c + s], smu[c + s], sM[c + s]);
    }
    __syncthreads();
  }
  cluster.sync();   // every CTA's group moments are in its row 0
  for (int g = t; g < G; g += kNormThreads) {
    float n = 0.0f, m = 0.0f, M = 0.0f;
    for (int k = 0; k < kNormCluster; ++k) {
      const float* rs = cluster.map_shared_rank(sm, k);
      const int c = g * cpg;
      chan_merge(n, m, M, rs[c], rs[L + c], rs[2 * L + c]);
    }
    const float rs = 1.0f / sqrtf(M / n + eps);
    gmean[g] = m, grstd[g] = rs;
    if (rank == 0) mean[(int64_t)b * G + g] = m, rstd[(int64_t)b * G + g] = rs;
  }
  cluster.sync();   // no CTA leaves while another reads its moments; gmean is visible

  if (!active) return;
  float mu[4], rsd[4], sc[4], sh[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int c = 4 * q + k, g = c / cpg;
    mu[k] = gmean[g], rsd[k] = grstd[g], sc[k] = scale[c], sh[k] = shift[c];
  }
  float* yb = y + (int64_t)b * HW * C + 4 * q;
#pragma unroll 4
  for (int row = r0 + r; row < r1; row += R) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(xb + (int64_t)row * C));
    const float xv[4] = {v.x, v.y, v.z, v.w};
    float o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k] = norm_relu(fmaf((xv[k] - mu[k]) * rsd[k], sc[k], sh[k]));
    *reinterpret_cast<float4*>(yb + (int64_t)row * C) = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// dy, dx [B, HW, C]; partial [B, kNormCluster, 2, C] receives each CTA's per-channel
// sums of dv xh (row 0) and dv (row 1).  Grid: kNormCluster B CTAs.
__global__ void __cluster_dims__(kNormCluster, 1, 1) __launch_bounds__(kNormThreads, 2)
    norm_relu_backward_kernel(const float* __restrict__ x, const float* __restrict__ scale,
                              const float* __restrict__ shift, const float* __restrict__ mean,
                              const float* __restrict__ rstd, const float* __restrict__ dy,
                              float* __restrict__ dx, float* __restrict__ partial, int HW,
                              int C, int G) {
  namespace cg = cooperative_groups;
  extern __shared__ float4 norm_smem4[];
  float* sm = reinterpret_cast<float*>(norm_smem4);
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int b = blockIdx.x / kNormCluster;
  const int nq = C / 4, R = norm_lanes(C), L = R * C, cpg = C / G;
  float* sA = sm;              // [R][C] sums of dv xh
  float* sS = sm + L;          // [R][C] sums of dv
  float* gS1 = sm + 2 * L;     // [G] mean of g
  float* gS2 = gS1 + G;        // [G] mean of g xh
  const int t = threadIdx.x, q = t % nq, r = t / nq;
  const bool active = r < R;
  int r0, r1;
  norm_rows(HW, rank, r0, r1);
  const int64_t base = (int64_t)b * HW * C + 4 * q;
  // The thread's per-channel constants, read again for the second pass rather than held
  // in registers across the reductions.
  float mu[4], rsd[4], sc[4], sh[4];
  auto constants = [&] {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = 4 * q + k, g = c / cpg;
      mu[k] = mean[(int64_t)b * G + g], rsd[k] = rstd[(int64_t)b * G + g];
      sc[k] = scale[c], sh[k] = shift[c];
    }
  };
  if (active) {
    constants();
    float A[4] = {0.0f, 0.0f, 0.0f, 0.0f}, S[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll 1
    for (int row = r0 + r; row < r1; row += R) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(x + base + (int64_t)row * C));
      const float4 u = __ldg(reinterpret_cast<const float4*>(dy + base + (int64_t)row * C));
      const float xv[4] = {v.x, v.y, v.z, v.w}, gv[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float xh = (xv[k] - mu[k]) * rsd[k];
        const float dv = fmaf(xh, sc[k], sh[k]) > 0.0f ? gv[k] : 0.0f;
        A[k] = fmaf(dv, xh, A[k]);
        S[k] += dv;
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) sA[r * C + 4 * q + k] = A[k], sS[r * C + 4 * q + k] = S[k];
  }
  __syncthreads();
  for (int s = 1; s < R; s *= 2) {
    for (int e = t; e < L; e += kNormThreads) {
      const int rr = e / C;
      if (rr % (2 * s) == 0 && rr + s < R) sA[e] += sA[e + s * C], sS[e] += sS[e + s * C];
    }
    __syncthreads();
  }
  float* pb = partial + ((int64_t)b * kNormCluster + rank) * 2 * C;
  for (int c = t; c < C; c += kNormThreads) {
    pb[c] = sA[c], pb[C + c] = sS[c];
    sA[c] *= scale[c], sS[c] *= scale[c];   // sums of g xh and g
  }
  __syncthreads();
  for (int s = 1; s < cpg; s *= 2) {
    for (int c = t; c < C; c += kNormThreads) {
      const int k = c % cpg;
      if (k % (2 * s) == 0 && k + s < cpg) sA[c] += sA[c + s], sS[c] += sS[c + s];
    }
    __syncthreads();
  }
  cluster.sync();
  const float inv_n = 1.0f / ((float)HW * (float)cpg);
  for (int g = t; g < G; g += kNormThreads) {
    float a = 0.0f, s = 0.0f;
    for (int k = 0; k < kNormCluster; ++k) {
      const float* rs = cluster.map_shared_rank(sm, k);
      a += rs[g * cpg], s += rs[L + g * cpg];
    }
    gS1[g] = s * inv_n, gS2[g] = a * inv_n;
  }
  cluster.sync();

  if (!active) return;
  constants();
  float m1[4], m2[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int g = (4 * q + k) / cpg;
    m1[k] = gS1[g], m2[k] = gS2[g];
  }
#pragma unroll 1
  for (int row = r0 + r; row < r1; row += R) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(x + base + (int64_t)row * C));
    const float4 u = __ldg(reinterpret_cast<const float4*>(dy + base + (int64_t)row * C));
    const float xv[4] = {v.x, v.y, v.z, v.w}, gv[4] = {u.x, u.y, u.z, u.w};
    float o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float xh = (xv[k] - mu[k]) * rsd[k];
      const float g = fmaf(xh, sc[k], sh[k]) > 0.0f ? gv[k] * sc[k] : 0.0f;
      o[k] = rsd[k] * (g - fmaf(xh, m2[k], m1[k]));
    }
    *reinterpret_cast<float4*>(dx + base + (int64_t)row * C) = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// dscale[c] and dshift[c]: partial's rows 0 and 1 of channel c added over the P = B
// kNormCluster CTAs in order.
__global__ void __launch_bounds__(256) norm_relu_param_grad_kernel(
    const float* __restrict__ partial, float* __restrict__ dscale, float* __restrict__ dshift,
    int P, int C) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * C) return;
  const int which = i / C, c = i % C;
  float s = 0.0f;
  for (int p = 0; p < P; ++p) s += partial[((int64_t)p * 2 + which) * C + c];
  (which ? dshift : dscale)[c] = s;
}

}  // namespace ddsp
