// The sequential part of the Keras GRU (tf.keras.layers.GRU, reset_after=True, gate
// columns z | r | h) that decoders.RnnFcDecoder runs over every frame: the forward
// recurrence and its backpropagation through time, each one persistent launch over all
// T steps.  The parallel GEMMs (x W + b, and the weight and input gradients) stay on
// cuBLAS through torch.
//
// Geometry.  One cluster of kGruCluster (8, the portable size) CTAs per batch slice of
// BS items.  CTA `rank` owns hidden units [rank Hc, (rank + 1) Hc), Hc = H / 8, and
// keeps the columns of U (recurrent_kernel [H, 3H]) those units need for the whole
// launch: 3 H^2 / 8 floats, in shared memory and, for H >= 384, partly in registers.
// Thread p = j Q + q works for unit j on chunk q of the contraction (Q chunks of R rows
// in the forward, of 3R columns in the backward); the Q partial sums of a unit are
// added by an xor butterfly in registers, which gives every lane of the unit the same
// bits.  Lane q < BS then does item q's elementwise step and sends its result to every
// CTA of the cluster through distributed shared memory; one cluster.sync() per step
// orders those writes.  Clusters never wait for each other.
//
//   H        Q   R = H/Q   threads   rows of U in registers (forward / backward)
//   32..256  16  2..32     2H        0 / 0
//   288..352 8   36..44    H         0 / 0
//   384..512 4   96..128   H/2       64 / 66
//
// Arithmetic is FP32 in a fixed order (no atomics, no TF32), so results are
// bit-reproducible, and item b's results depend on item b alone whatever the slice.
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"

namespace ddsp {

constexpr int kGruCluster = 8;         // CTAs per cluster: the portable maximum
constexpr int kGruMaxSlice = 4;        // items per cluster (BS)
constexpr int kGruRegRowsFwd = 64;     // rows of U per thread in registers, H >= 384
constexpr int kGruRegRowsBwd = 66;
constexpr size_t kGruMaxSmem = 227 * 1024;   // all a Hopper CTA may reserve

// Chunks of the contraction per unit (see the table above).
__host__ __device__ inline int gru_chunks(int H) { return H <= 256 ? 16 : H <= 352 ? 8 : 4; }

// Stride of one chunk of n (even) values in a shared vector: n/2 odd keeps the float2
// reads of the Q chunk lanes of a warp on distinct banks.
__host__ __device__ inline int gru_pad(int n) { return 2 * ((n / 2) | 1); }

// Shared-memory slot of entry e of a vector cut into chunks of n with stride s.
__host__ __device__ inline int gru_slot(int e, int n, int s) { return (e / n) * s + e % n; }

__device__ __forceinline__ float gru_sigmoid(float a) { return 1.0f / (1.0f + expf(-a)); }

// Packs recurrent_kernel U [H, 3H] into both per-CTA layouts, then copies c [3H]:
//   forward,  rank block [R][3][P]:  U[q R + i][g H + rank Hc + j]
//   backward, rank block [3R][P]:    U[rank Hc + j][q 3R + i]
// with p = j Q + q.  A thread's register rows come first in its block, the rest is
// copied to shared memory as one contiguous range.
__global__ void __launch_bounds__(256) gru_pack_kernel(const float* __restrict__ U,
                                                       const float* __restrict__ c,
                                                       float* __restrict__ pack, int H) {
  const int Q = gru_chunks(H), R = H / Q, Hc = H / kGruCluster, P = Q * Hc;
  const int64_t n = 3LL * H * H, blk = 3LL * R * P;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < 2 * n + 3 * H;
       idx += (int64_t)gridDim.x * blockDim.x) {
    float v;
    if (idx < n) {
      const int rank = (int)(idx / blk), rem = (int)(idx % blk);
      const int i = rem / (3 * P), g = (rem / P) % 3, p = rem % P;
      v = U[(int64_t)((p % Q) * R + i) * 3 * H + g * H + rank * Hc + p / Q];
    } else if (idx < 2 * n) {
      const int64_t e = idx - n;
      const int rank = (int)(e / blk), rem = (int)(e % blk);
      const int i = rem / P, p = rem % P;
      v = U[(int64_t)(rank * Hc + p / Q) * 3 * H + (p % Q) * 3 * R + i];
    } else {
      v = c[idx - 2 * n];
    }
    pack[idx] = v;
  }
}

// Dynamic shared memory of a launch: U's shared rows and the double-buffered vector
// (h in the forward, d_rec in the backward) of BS items.
__host__ __device__ inline size_t gru_smem_bytes(int H, int BS, bool backward) {
  const int Q = gru_chunks(H), R = H / Q, P = Q * (H / kGruCluster);
  const int rr = Q == 4 ? (backward ? kGruRegRowsBwd : kGruRegRowsFwd) : 0;
  const int vec = backward ? 3 * R : R;
  return sizeof(float) * ((size_t)3 * (R - rr) * P + (size_t)2 * BS * Q * gru_pad(vec));
}

// Forward: gates [B, T, 4H] holds x W + b in its first 3H columns and receives
// z | r | h~ | (h U_h + c_h); states [B, T + 1, H] holds h_0 in row 0 and receives
// h_1 .. h_T.  pack: the forward blocks, c at 6 H^2.
template <int RR, int BS>
__global__ void __cluster_dims__(kGruCluster, 1, 1) __launch_bounds__(RR ? 256 : 512, 1)
    gru_forward_kernel(const float* __restrict__ pack, float* __restrict__ gates,
                       float* __restrict__ states, int B, int T, int H) {
  namespace cg = cooperative_groups;
  extern __shared__ float4 gru_smem4[];
  float* sm = reinterpret_cast<float*>(gru_smem4);
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int Q = gru_chunks(H), R = H / Q, Hc = H / kGruCluster, P = Q * Hc;
  const int S = gru_pad(R), HB = Q * S;
  const int p = threadIdx.x, q = p % Q, j = p / Q, u = rank * Hc + j;
  const int n_sm = 3 * (R - RR) * P;
  float* Us = sm;
  float* hs = sm + n_sm;                       // [2][BS][HB]
  const float* blk = pack + (int64_t)rank * 3 * R * P;

  float w[RR > 0 ? RR : 1][3];
#pragma unroll
  for (int i = 0; i < RR; ++i)
#pragma unroll
    for (int g = 0; g < 3; ++g) w[i][g] = blk[(i * 3 + g) * P + p];
  const float4* src = reinterpret_cast<const float4*>(blk + 3 * RR * P);
  for (int i = p; i < n_sm / 4; i += P) reinterpret_cast<float4*>(Us)[i] = src[i];
  for (int i = p; i < 2 * BS * HB; i += P) hs[i] = 0.0f;
  __syncthreads();
  const int b0 = (blockIdx.x / kGruCluster) * BS;
  for (int e = p; e < BS * H; e += P) {
    const int bb = e / H, k = e % H;
    if (b0 + bb < B) hs[bb * HB + gru_slot(k, R, S)] = states[(int64_t)(b0 + bb) * (T + 1) * H + k];
  }
  const bool act = q < BS && b0 + q < B;
  const int b = b0 + q;
  const float* c = pack + 6LL * H * H;
  const float cz = c[u], cr = c[H + u], ch = c[2 * H + u];
  const int su = gru_slot(u, R, S);
  cluster.sync();   // every CTA's buffers are ready before the first remote write

  for (int t = 0; t < T; ++t) {
    const int cur = t & 1;
    float* g4 = gates + ((int64_t)(act ? b : 0) * T + t) * 4 * H;
    float xz = 0.0f, xr = 0.0f, xh = 0.0f;
    if (act) {   // issued first: the loads complete under the matrix-vector product
      xz = g4[u];
      xr = g4[H + u];
      xh = g4[2 * H + u];
    }
    const float* hb = hs + cur * BS * HB + q * S;
    float acc[3][BS];
#pragma unroll
    for (int g = 0; g < 3; ++g)
#pragma unroll
      for (int bb = 0; bb < BS; ++bb) acc[g][bb] = 0.0f;
#pragma unroll
    for (int i = 0; i < RR; i += 2) {
#pragma unroll
      for (int bb = 0; bb < BS; ++bb) {
        const float2 h2 = *reinterpret_cast<const float2*>(hb + bb * HB + i);
#pragma unroll
        for (int g = 0; g < 3; ++g) {
          acc[g][bb] = fmaf(w[i][g], h2.x, acc[g][bb]);
          acc[g][bb] = fmaf(w[i + 1][g], h2.y, acc[g][bb]);
        }
      }
    }
    const float* us = Us + p;
#pragma unroll 2
    for (int i = RR; i < R; i += 2, us += 6 * P) {
      float a[6];
#pragma unroll
      for (int m = 0; m < 6; ++m) a[m] = us[m * P];
#pragma unroll
      for (int bb = 0; bb < BS; ++bb) {
        const float2 h2 = *reinterpret_cast<const float2*>(hb + bb * HB + i);
#pragma unroll
        for (int g = 0; g < 3; ++g) {
          acc[g][bb] = fmaf(a[g], h2.x, acc[g][bb]);
          acc[g][bb] = fmaf(a[3 + g], h2.y, acc[g][bb]);
        }
      }
    }
    for (int m = 1; m < Q; m <<= 1)
#pragma unroll
      for (int g = 0; g < 3; ++g)
#pragma unroll
        for (int bb = 0; bb < BS; ++bb)
          acc[g][bb] += __shfl_xor_sync(0xffffffffu, acc[g][bb], m);
    float hz = 0.0f, hr = 0.0f, hh = 0.0f;
#pragma unroll
    for (int bb = 0; bb < BS; ++bb)
      if (q == bb) {
        hz = acc[0][bb];
        hr = acc[1][bb];
        hh = acc[2][bb];
      }
    if (act) {
      const float z = gru_sigmoid(xz + (hz + cz));
      const float r = gru_sigmoid(xr + (hr + cr));
      const float hu = hh + ch;
      const float hc = tanhf(xh + r * hu);
      const float hp = hs[cur * BS * HB + q * HB + su];
      const float hn = z * hp + (1.0f - z) * hc;
      g4[u] = z;
      g4[H + u] = r;
      g4[2 * H + u] = hc;
      g4[3 * H + u] = hu;
      states[((int64_t)b * (T + 1) + t + 1) * H + u] = hn;
      float* nxt = hs + (cur ^ 1) * BS * HB + q * HB + su;
#pragma unroll
      for (int r2 = 0; r2 < kGruCluster; ++r2) *cluster.map_shared_rank(nxt, r2) = hn;
    }
    cluster.sync();
  }
}

// Backward through time: grad_out [B, T, H] (dL/dh_1 .. h_T) -> d_pre [B, T, 3H], the
// gradient of x W + b, and d_rec [B, T + 1, 3H], of h U + c in rows 0 .. T-1 and zeros in
// row T, so that row b (T + 1) + t of d_rec and of states [B, T + 1, H] are the same step
// and dU = states^T d_rec is one GEMM over the flat buffers:
//   dh = grad_out_t + dh_carry,  dz = dh (h_prev - h~),  da_h = dh (1 - z)(1 - h~^2),
//   d_pre = [dz z(1-z), da_h hu r(1-r), da_h],  d_rec = [.., .., da_h r],
//   dh_carry(t-1) = dh z + d_rec U^T.
// pack: the backward blocks at 3 H^2.
template <int RR, int BS>
__global__ void __cluster_dims__(kGruCluster, 1, 1) __launch_bounds__(RR ? 256 : 512, 1)
    gru_backward_kernel(const float* __restrict__ pack, const float* __restrict__ gates,
                        const float* __restrict__ states, const float* __restrict__ grad_out,
                        float* __restrict__ d_pre, float* __restrict__ d_rec, int B, int T,
                        int H) {
  namespace cg = cooperative_groups;
  extern __shared__ float4 gru_smem4[];
  float* sm = reinterpret_cast<float*>(gru_smem4);
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int Q = gru_chunks(H), R = H / Q, Hc = H / kGruCluster, P = Q * Hc;
  const int R3 = 3 * R, S = gru_pad(R3), HB = Q * S;
  const int p = threadIdx.x, q = p % Q, j = p / Q, u = rank * Hc + j;
  const int n_sm = 3 * (R - RR) * P;
  float* Us = sm;
  float* ds = sm + n_sm;                       // [2][BS][HB]
  const float* blk = pack + 3LL * H * H + (int64_t)rank * 3 * R * P;

  float w[RR > 0 ? 3 * RR : 1];
#pragma unroll
  for (int i = 0; i < 3 * RR; ++i) w[i] = blk[i * P + p];
  const float4* src = reinterpret_cast<const float4*>(blk + 3 * RR * P);
  for (int i = p; i < n_sm / 4; i += P) reinterpret_cast<float4*>(Us)[i] = src[i];
  for (int i = p; i < 2 * BS * HB; i += P) ds[i] = 0.0f;
  const int b0 = (blockIdx.x / kGruCluster) * BS;
  const bool act = q < BS && b0 + q < B;
  const int b = b0 + q;
  const int sz = gru_slot(u, R3, S), sr = gru_slot(H + u, R3, S), sh = gru_slot(2 * H + u, R3, S);
  float go = 0.0f, z = 0.0f, r = 0.0f, hc = 0.0f, hu = 0.0f, hp = 0.0f, carry = 0.0f;
  auto fetch = [&](int t) {
    const float* g4 = gates + ((int64_t)b * T + t) * 4 * H;
    go = grad_out[((int64_t)b * T + t) * H + u];
    z = g4[u];
    r = g4[H + u];
    hc = g4[2 * H + u];
    hu = g4[3 * H + u];
    hp = states[((int64_t)b * (T + 1) + t) * H + u];
  };
  if (act) {
    fetch(T - 1);
    float* last = d_rec + ((int64_t)b * (T + 1) + T) * 3 * H;
    last[u] = 0.0f;
    last[H + u] = 0.0f;
    last[2 * H + u] = 0.0f;
  }
  cluster.sync();   // every CTA's buffers are ready before the first remote write

  for (int t = T - 1;; --t) {
    const int cur = t & 1;
    if (act) {
      const float dh = go + carry;
      const float dz = dh * (hp - hc);
      const float dah = dh * (1.0f - z) * (1.0f - hc * hc);
      const float daz = dz * (z * (1.0f - z));
      const float dar = dah * hu * (r * (1.0f - r));
      const float drh = dah * r;
      const int64_t o = ((int64_t)b * T + t) * 3 * H, o1 = o + (int64_t)b * 3 * H;
      d_pre[o + u] = daz;
      d_pre[o + H + u] = dar;
      d_pre[o + 2 * H + u] = dah;
      d_rec[o1 + u] = daz;
      d_rec[o1 + H + u] = dar;
      d_rec[o1 + 2 * H + u] = drh;
      carry = dh * z;
      float* base = ds + cur * BS * HB + q * HB;
#pragma unroll
      for (int r2 = 0; r2 < kGruCluster; ++r2) {
        *cluster.map_shared_rank(base + sz, r2) = daz;
        *cluster.map_shared_rank(base + sr, r2) = dar;
        *cluster.map_shared_rank(base + sh, r2) = drh;
      }
      if (t > 0) fetch(t - 1);   // completes under the matrix-vector product
    }
    cluster.sync();
    if (t == 0) break;
    const float* db = ds + cur * BS * HB + q * S;
    float acc[BS];
#pragma unroll
    for (int bb = 0; bb < BS; ++bb) acc[bb] = 0.0f;
#pragma unroll
    for (int i = 0; i < 3 * RR; i += 2) {
#pragma unroll
      for (int bb = 0; bb < BS; ++bb) {
        const float2 d2 = *reinterpret_cast<const float2*>(db + bb * HB + i);
        acc[bb] = fmaf(w[i], d2.x, acc[bb]);
        acc[bb] = fmaf(w[i + 1], d2.y, acc[bb]);
      }
    }
    const float* us = Us + p;
#pragma unroll 4
    for (int i = 3 * RR; i < R3; i += 2, us += 2 * P) {
      const float a0 = us[0], a1 = us[P];
#pragma unroll
      for (int bb = 0; bb < BS; ++bb) {
        const float2 d2 = *reinterpret_cast<const float2*>(db + bb * HB + i);
        acc[bb] = fmaf(a0, d2.x, acc[bb]);
        acc[bb] = fmaf(a1, d2.y, acc[bb]);
      }
    }
    for (int m = 1; m < Q; m <<= 1)
#pragma unroll
      for (int bb = 0; bb < BS; ++bb) acc[bb] += __shfl_xor_sync(0xffffffffu, acc[bb], m);
#pragma unroll
    for (int bb = 0; bb < BS; ++bb)
      if (q == bb) carry += acc[bb];
  }
}

}  // namespace ddsp
