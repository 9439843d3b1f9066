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
// The residual site of nn.DilatedConvStack (nn.py:1287-1323) runs on the same geometry
// and the same statistics pass (norm_group_moments), over the convolution's output y:
//   x_next = x + xh s + h,  r = relu(x_next),  xh = normalize(y) (or y for no norm),
// with s and h per channel or read per row from a FiLM Dense output.  Its backward sums
// g = gx + gr 1[x_next > 0] and g s per channel by the same lane, group and cluster
// reductions (norm_lane_sums, norm_group_means).
// Every sum runs in a fixed order with no atomics: results are bit-reproducible, and an
// item's outputs depend on that item alone.
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

// The forward's statistics of one item: every thread of the cluster's CTAs calls it.
// Welford moments of the CTA's rows [r0, r1) of xb (the item's first row, offset to the
// thread's quad), Chan merges over the row lanes and a group's channels, then the 8
// CTAs' group moments merged in rank order through distributed shared memory.  Leaves
// the group means and rstds in gmean, grstd [G] of every CTA's shared memory (visible
// on return) and writes them to mean_b, rstd_b [G] from rank 0.
__device__ __forceinline__ void norm_group_moments(const float* __restrict__ xb, int r0, int r1,
                                                   int C, int G, float eps, float* mean_b,
                                                   float* rstd_b) {
  namespace cg = cooperative_groups;
  extern __shared__ float4 norm_smem4[];
  float* sm = reinterpret_cast<float*>(norm_smem4);
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int nq = C / 4, R = norm_lanes(C), L = R * C, cpg = C / G;
  float* sn = sm;              // [R][C] counts
  float* smu = sm + L;         // [R][C] means
  float* sM = sm + 2 * L;      // [R][C] sums of squared deviations
  float* gmean = sm + 3 * L;   // [G]
  float* grstd = gmean + G;    // [G]
  const int t = threadIdx.x, q = t % nq, r = t / nq;

  if (r < R) {
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
    if (rank == 0) mean_b[g] = m, rstd_b[g] = rs;
  }
  cluster.sync();   // no CTA leaves while another reads its moments; gmean is visible
}

// x, y [B, HW, C]; scale, shift [C]; mean, rstd [B, G].  Grid: kNormCluster B CTAs.
__global__ void __cluster_dims__(kNormCluster, 1, 1) __launch_bounds__(kNormThreads, 2)
    norm_relu_forward_kernel(const float* __restrict__ x, const float* __restrict__ scale,
                             const float* __restrict__ shift, float* __restrict__ y,
                             float* __restrict__ mean, float* __restrict__ rstd, int HW, int C,
                             int G, float eps) {
  namespace cg = cooperative_groups;
  extern __shared__ float4 norm_smem4[];
  float* sm = reinterpret_cast<float*>(norm_smem4);
  const int rank = (int)cg::this_cluster().block_rank();
  const int b = blockIdx.x / kNormCluster;
  const int nq = C / 4, R = norm_lanes(C), L = R * C, cpg = C / G;
  const float* gmean = sm + 3 * L;
  const float* grstd = gmean + G;
  const int t = threadIdx.x, q = t % nq, r = t / nq;
  int r0, r1;
  norm_rows(HW, rank, r0, r1);
  const float* xb = x + (int64_t)b * HW * C + 4 * q;
  norm_group_moments(xb, r0, r1, C, G, eps, mean + (int64_t)b * G, rstd + (int64_t)b * G);

  if (r >= R) return;
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

// The backward's sums over a CTA's row lanes: sA[r][c] and sS[r][c] (2 R C floats at
// the start of shared memory) added by a tree into row 0, in a fixed order.  Every
// thread calls it after storing its lane's sums.
__device__ __forceinline__ void norm_lane_sums(int C) {
  extern __shared__ float4 norm_smem4[];
  float* sA = reinterpret_cast<float*>(norm_smem4);
  const int R = norm_lanes(C), L = R * C, t = threadIdx.x;
  float* sS = sA + L;
  __syncthreads();
  for (int s = 1; s < R; s *= 2) {
    for (int e = t; e < L; e += kNormThreads) {
      const int rr = e / C;
      if (rr % (2 * s) == 0 && rr + s < R) sA[e] += sA[e + s * C], sS[e] += sS[e + s * C];
    }
    __syncthreads();
  }
}

// From the per-channel sums of u xh (sA row 0) and u (sS row 0) of every CTA of the
// cluster: each group's mean of u and u xh over its HW cpg elements, in gS1 and gS2 [G]
// after the 2 R C lane sums.  The channels of a group are added by a tree, then the 8
// CTAs' group sums in rank order through distributed shared memory.  Every thread of the
// cluster calls it; the means are visible on return.
__device__ __forceinline__ void norm_group_means(int HW, int C, int G) {
  namespace cg = cooperative_groups;
  extern __shared__ float4 norm_smem4[];
  float* sm = reinterpret_cast<float*>(norm_smem4);
  cg::cluster_group cluster = cg::this_cluster();
  const int R = norm_lanes(C), L = R * C, cpg = C / G, t = threadIdx.x;
  float* sA = sm;
  float* sS = sm + L;
  float* gS1 = sm + 2 * L;
  float* gS2 = gS1 + G;
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
  norm_lane_sums(C);
  float* pb = partial + ((int64_t)b * kNormCluster + rank) * 2 * C;
  for (int c = t; c < C; c += kNormThreads) {
    pb[c] = sA[c], pb[C + c] = sS[c];
    sA[c] *= scale[c], sS[c] *= scale[c];   // sums of g xh and g
  }
  __syncthreads();
  norm_group_means(HW, C, G);

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

// ---- The residual site of nn.DilatedConvStack ---------------------------------------
// The per-row s and h of the thread's quad, whose first elements are at offset fr of
// scale and shift: s = 1 where scale is null (shift_only), and h is read unless sh is
// null (the backward needs s alone).
__device__ __forceinline__ void norm_row_affine(const float* __restrict__ scale,
                                                const float* __restrict__ shift, int64_t fr,
                                                float sc[4], float* sh) {
  if (sh) {
    const float4 h = __ldg(reinterpret_cast<const float4*>(shift + fr));
    sh[0] = h.x, sh[1] = h.y, sh[2] = h.z, sh[3] = h.w;
  }
  if (scale) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(scale + fr));
    sc[0] = v.x, sc[1] = v.y, sc[2] = v.z, sc[3] = v.w;
  } else {
    sc[0] = sc[1] = sc[2] = sc[3] = 1.0f;
  }
}

// x_next = x + xh s + h and, when r is not null, r = relu(x_next), over y, x, x_next, r
// [B, T, C], with xh = (y - mean_g) rstd_g (the statistics pass of normalize_relu, on y)
// when kNorm, else xh = y.  s = scale[c] and h = shift[c] (nn.Normalize), or with kRow
// item b's row t reads them at (b T + t) ld of scale and shift (a FiLM Dense output read
// in place; a null scale is s = 1).  mean, rstd [B, G] when kNorm.  Grid: kNormCluster B
// CTAs.
template <bool kNorm, bool kRow>
__global__ void __cluster_dims__(kNormCluster, 1, 1) __launch_bounds__(kNormThreads, 2)
    norm_residual_forward_kernel(const float* __restrict__ y, const float* __restrict__ x,
                                 const float* __restrict__ scale,
                                 const float* __restrict__ shift, int ld,
                                 float* __restrict__ x_next, float* __restrict__ r_out,
                                 float* __restrict__ mean, float* __restrict__ rstd, int T,
                                 int C, int G, float eps) {
  namespace cg = cooperative_groups;
  extern __shared__ float4 norm_smem4[];
  const float* sm = reinterpret_cast<const float*>(norm_smem4);
  const int rank = (int)cg::this_cluster().block_rank();
  const int b = blockIdx.x / kNormCluster;
  const int nq = C / 4, R = norm_lanes(C);
  const int t = threadIdx.x, q = t % nq, r = t / nq;
  int r0, r1;
  norm_rows(T, rank, r0, r1);
  const int64_t base = (int64_t)b * T * C + 4 * q;
  float mu[4] = {0.0f, 0.0f, 0.0f, 0.0f}, rsd[4] = {1.0f, 1.0f, 1.0f, 1.0f};
  if (kNorm) {
    norm_group_moments(y + base, r0, r1, C, G, eps, mean + (int64_t)b * G,
                       rstd + (int64_t)b * G);
    const float* gmean = sm + 3 * R * C;
    const int cpg = C / G;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int g = (4 * q + k) / cpg;
      mu[k] = gmean[g], rsd[k] = gmean[G + g];
    }
  }
  if (r >= R) return;
  float sc[4], sh[4];
  if (!kRow) {
#pragma unroll
    for (int k = 0; k < 4; ++k) sc[k] = scale[4 * q + k], sh[k] = shift[4 * q + k];
  }
#pragma unroll 2
  for (int row = r0 + r; row < r1; row += R) {
    if (kRow)
      norm_row_affine(scale, shift, ((int64_t)b * T + row) * ld + 4 * q, sc, sh);
    const int64_t e = base + (int64_t)row * C;
    const float4 v = __ldg(reinterpret_cast<const float4*>(y + e));
    const float4 u = __ldg(reinterpret_cast<const float4*>(x + e));
    const float yv[4] = {v.x, v.y, v.z, v.w}, xv[4] = {u.x, u.y, u.z, u.w};
    float o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float xh = kNorm ? (yv[k] - mu[k]) * rsd[k] : yv[k];
      o[k] = xv[k] + fmaf(xh, sc[k], sh[k]);
    }
    *reinterpret_cast<float4*>(x_next + e) = make_float4(o[0], o[1], o[2], o[3]);
    if (r_out)
      *reinterpret_cast<float4*>(r_out + e) =
          make_float4(norm_relu(o[0]), norm_relu(o[1]), norm_relu(o[2]), norm_relu(o[3]));
  }
}

// The site's backward.  g = gx + gr 1[x_next > 0] (gr may be null) is written to dx,
// and u = g s.  dy = rstd (u - mean_g(u) - xh mean_g(u xh)) when kNorm (the group means
// from the cluster's sums, then a second pass that reads g back from dx), else dy = u.
// Per channel (!kRow): each CTA's per-channel sums of g xh and g go to partial
// [B, kNormCluster, 2, C] for norm_relu_param_grad_kernel.  Per row: g xh and g are
// written at the forward's offsets and stride ld to dscale (unless it is null, as scale
// is for shift_only) and dshift.  Grid: kNormCluster B CTAs.
template <bool kNorm, bool kRow>
__global__ void __cluster_dims__(kNormCluster, 1, 1) __launch_bounds__(kNormThreads, 2)
    norm_residual_backward_kernel(const float* __restrict__ y, const float* __restrict__ scale,
                                  int ld,
                                  const float* __restrict__ x_next,
                                  const float* __restrict__ mean,
                                  const float* __restrict__ rstd, const float* __restrict__ gx,
                                  const float* __restrict__ gr, float* __restrict__ dy,
                                  float* __restrict__ dx, float* __restrict__ dscale,
                                  float* __restrict__ dshift, float* __restrict__ partial,
                                  int T, int C, int G) {
  constexpr bool kChannel = !kRow;
  namespace cg = cooperative_groups;
  extern __shared__ float4 norm_smem4[];
  float* sm = reinterpret_cast<float*>(norm_smem4);
  const int rank = (int)cg::this_cluster().block_rank();
  const int b = blockIdx.x / kNormCluster;
  const int nq = C / 4, R = norm_lanes(C), L = R * C;
  const int t = threadIdx.x, q = t % nq, r = t / nq;
  const bool active = r < R;
  int r0, r1;
  norm_rows(T, rank, r0, r1);
  const int64_t base = (int64_t)b * T * C + 4 * q;
  float mu[4] = {0.0f, 0.0f, 0.0f, 0.0f}, rsd[4] = {1.0f, 1.0f, 1.0f, 1.0f};
  float sc[4] = {1.0f, 1.0f, 1.0f, 1.0f};
  // The thread's per-channel constants, read again for the second pass rather than held
  // in registers across the reductions.
  auto constants = [&] {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = 4 * q + k;
      if (kNorm) {
        const int g = c / (C / G);
        mu[k] = mean[(int64_t)b * G + g], rsd[k] = rstd[(int64_t)b * G + g];
      }
      if (kChannel) sc[k] = scale[c];
    }
  };
  if (active) {
    constants();
    float A[4] = {0.0f, 0.0f, 0.0f, 0.0f}, S[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll 1
    for (int row = r0 + r; row < r1; row += R) {
      const int64_t e = base + (int64_t)row * C;
      const int64_t fr = ((int64_t)b * T + row) * ld + 4 * q;
      if (!kChannel) norm_row_affine(scale, nullptr, fr, sc, nullptr);
      const float4 w = __ldg(reinterpret_cast<const float4*>(gx + e));
      float g[4] = {w.x, w.y, w.z, w.w};
      if (gr) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(gr + e));
        const float4 n = __ldg(reinterpret_cast<const float4*>(x_next + e));
        const float av[4] = {a.x, a.y, a.z, a.w}, nv[4] = {n.x, n.y, n.z, n.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) g[k] += nv[k] > 0.0f ? av[k] : 0.0f;
      }
      *reinterpret_cast<float4*>(dx + e) = make_float4(g[0], g[1], g[2], g[3]);
      const float4 v = __ldg(reinterpret_cast<const float4*>(y + e));
      const float yv[4] = {v.x, v.y, v.z, v.w};
      float gxh[4], u[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float xh = kNorm ? (yv[k] - mu[k]) * rsd[k] : yv[k];
        gxh[k] = g[k] * xh;
        u[k] = g[k] * sc[k];
        if (kChannel) {
          A[k] = fmaf(g[k], xh, A[k]), S[k] += g[k];
        } else if (kNorm) {
          A[k] = fmaf(u[k], xh, A[k]), S[k] += u[k];
        }
      }
      if (!kChannel) {
        if (dscale)
          *reinterpret_cast<float4*>(dscale + fr) = make_float4(gxh[0], gxh[1], gxh[2], gxh[3]);
        *reinterpret_cast<float4*>(dshift + fr) = make_float4(g[0], g[1], g[2], g[3]);
      }
      if (!kNorm)
        *reinterpret_cast<float4*>(dy + e) = make_float4(u[0], u[1], u[2], u[3]);
    }
    if (kChannel || kNorm) {
#pragma unroll
      for (int k = 0; k < 4; ++k) sm[r * C + 4 * q + k] = A[k], sm[L + r * C + 4 * q + k] = S[k];
    }
  }
  if (!kChannel && !kNorm) return;
  norm_lane_sums(C);
  if (kChannel) {
    float* pb = partial + ((int64_t)b * kNormCluster + rank) * 2 * C;
    for (int c = t; c < C; c += kNormThreads) {
      pb[c] = sm[c], pb[C + c] = sm[L + c];
      if (kNorm) sm[c] *= scale[c], sm[L + c] *= scale[c];   // sums of u xh and u
    }
    __syncthreads();
  }
  if (!kNorm) return;
  norm_group_means(T, C, G);

  if (!active) return;
  constants();
  const float* gS1 = sm + 2 * L;
  float m1[4], m2[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int g = (4 * q + k) / (C / G);
    m1[k] = gS1[g], m2[k] = gS1[G + g];
  }
#pragma unroll 1
  for (int row = r0 + r; row < r1; row += R) {
    const int64_t e = base + (int64_t)row * C;
    if (!kChannel)
      norm_row_affine(scale, nullptr, ((int64_t)b * T + row) * ld + 4 * q, sc,
                               nullptr);
    const float4 v = __ldg(reinterpret_cast<const float4*>(y + e));
    const float4 w = *reinterpret_cast<const float4*>(dx + e);   // g, this thread's write
    const float yv[4] = {v.x, v.y, v.z, v.w}, gv[4] = {w.x, w.y, w.z, w.w};
    float o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float xh = (yv[k] - mu[k]) * rsd[k];
      o[k] = rsd[k] * (gv[k] * sc[k] - fmaf(xh, m2[k], m1[k]));
    }
    *reinterpret_cast<float4*>(dy + e) = make_float4(o[0], o[1], o[2], o[3]);
  }
}

}  // namespace ddsp
