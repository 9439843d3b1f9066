// Note segmentation and note pooling (training/nn.py:375-557): get_note_mask,
// get_note_mask_from_onset, get_note_moments and pool_over_notes, with the gradient of
// the moments and the pooled values to x.
//
// Mask.  One CTA per item walks the frames in chunks of kMaskThreads, one frame per
// thread.  A block scan of the edges, carried across chunks, gives each frame's region
// index.  For get_note_mask with note_on_only a first pass decides, per region, whether
// the reference's float32 mask-weighted sum of q over all T frames is > 0, in float64:
// a segmented block scan sums q over the region, and a region is off when any frame
// outside it is non-finite (its 0 * inf or 0 * NaN term makes the reference's sum NaN).
// The decisions go to a workspace byte per region (B * min(R, T) bytes), and a second
// pass writes the dense [T_out, R] rows once, a warp per row, lanes over the columns.
//
// Moments and pool.  x [B,T,D] and an arbitrary float mask m [B,T,N]:
//   L_n = sum_t m_tn,  Ls_n = L_n or 1e-7 where L_n == 0 (safe_divide),
//   mu_nd = sum_t m_tn x_td / Ls_n,  v_nd = sum_t ((x_td - mu_nd) m_tn)^2 / Ls_n,
//   sigma_nd = sqrt(v_nd),  Pmu_td = sum_n m_tn mu_nd,  Psigma_td = sum_n m_tn sigma_nd.
// The variance takes a second pass over t with the finished mean (never E[x^2] - mu^2).
// Contractions over t run on CTA tiles of kTile notes by kDTile dims; contractions over n
// on tiles of kTile frames by kDTile dims.  Each thread owns 4 rows by 2 columns of its
// tile and sums its chunk of kTile terms serially, then adds the chunk to its total: a
// fixed order, no atomics, bit-reproducible.
//
// Backward to x, from the total upstream gradients
//   Gmu_nd = gmu_nd + sum_t m_tn gPmu_td,  Gsigma_nd = gsigma_nd + sum_t m_tn gPsigma_td:
//   Gv = Gsigma 0.5 / sigma,  GQ = Gv / Ls,  Gmu' = Gmu - 2 GQ sum_t m_tn r_tnd,
//   dx_td = sum_n m_tn (Gmu'_nd / Ls_n + 2 GQ_nd r_tnd),  r_tnd = (x_td - mu_nd) m_tn.
// A first launch (over t) writes A = Gmu' / Ls and C = 2 GQ to the workspace [B,N,D]
// each, a second (over n) sums dx.  Without a gradient through sigma the C term is
// skipped, so a std output nobody uses cannot turn 0 * inf into NaN.  With one, v = 0
// gives NaN through the whole (b, d), as float64 autograd of the reference does.
#pragma once
#include "common.cuh"

namespace ddsp {
namespace notes_ {

constexpr int kMaskThreads = 512;
constexpr int kMaskWarps = kMaskThreads / 32;
constexpr int kThreads = 256;   // 8 warps: ty = warp owns 4 rows, tx = lane 2 columns
constexpr int kTile = 32;       // notes (over-t kernels) or frames (over-n kernels) per CTA
constexpr int kDTile = 64;      // dims per CTA
constexpr int kChunk = 32;      // terms staged per step of the summed index

// ---- mask -----------------------------------------------------------------------------
struct MaskParams {
  const float* q;       // [B, T]
  const float* onset;   // [B, T] (onset rule only)
  uint8_t* on;          // [B, Rf] region decisions (edge rule with note_on_only)
  int T, T_out, R, Rf, note_on_only;
};

// Edge of frame t (0 <= t < T): 1 opens a region.
template <bool kOnset>
__device__ __forceinline__ int edge(const MaskParams& p, const float* q, const float* on,
                                    int t) {
  if (t == 0) return 1;
  if (kOnset) return (int)on[t];   // truncation toward zero
  return t <= p.T - 2 && fabsf(q[t] - q[t - 1]) > 0.f;
}

// Inclusive block sum-scan of one int per thread, plus `carry`; `tot` holds kMaskWarps + 1
// ints.  Unsigned adds: onset counts wrap as TensorFlow's int32 cumsum does.
__device__ __forceinline__ int scan_int(int v, int carry, int* tot, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned s = (unsigned)v;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned y = __shfl_up_sync(0xffffffffu, s, o);
    if (lane >= o) s += y;
  }
  if (lane == 31) tot[warp] = (int)s;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned run = (unsigned)carry;
    for (int w = 0; w < kMaskWarps; ++w) {
      const unsigned x = (unsigned)tot[w];
      tot[w] = (int)run;
      run += x;
    }
    tot[kMaskWarps] = (int)run;
  }
  __syncthreads();
  const int out = (int)(s + (unsigned)tot[warp]);
  if (total) *total = tot[kMaskWarps];
  __syncthreads();
  return out;
}

struct Seg {
  double s;   // sum of q over the segment
  int nf;     // non-finite frames in it
  int head;   // the segment holds a region start
};

__device__ __forceinline__ Seg seg_join(const Seg& a, const Seg& b) {
  return b.head ? b : Seg{a.s + b.s, a.nf + b.nf, a.head};
}

// Inclusive segmented scan of one Seg per thread, continuing `carry` (the open region of
// the chunks before); returns this frame's region-so-far and updates `carry`.
__device__ __forceinline__ Seg scan_seg(Seg v, Seg* carry, Seg* tot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    Seg y;
    y.s = __shfl_up_sync(0xffffffffu, v.s, o);
    y.nf = __shfl_up_sync(0xffffffffu, v.nf, o);
    y.head = __shfl_up_sync(0xffffffffu, v.head, o);
    if (lane >= o) v = seg_join(y, v);
  }
  if (lane == 31) tot[warp] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    Seg run = *carry;
    for (int w = 0; w < kMaskWarps; ++w) {
      const Seg x = tot[w];
      tot[w] = run;
      run = seg_join(run, x);
    }
    *carry = run;
  }
  __syncthreads();
  const Seg out = seg_join(tot[warp], v);
  __syncthreads();
  return out;
}

template <bool kOnset>
__global__ void __launch_bounds__(kMaskThreads)
note_mask_kernel(MaskParams p, float* __restrict__ mask) {
  __shared__ int itot[kMaskWarps + 1];
  __shared__ Seg stot[kMaskWarps];
  __shared__ Seg carry;
  __shared__ int cols[kMaskThreads];
  const int64_t b = blockIdx.x;
  const float* q = p.q + b * p.T;
  const float* on = kOnset ? p.onset + b * p.T : nullptr;
  uint8_t* flags = p.on + b * p.Rf;
  const bool decide = !kOnset && p.note_on_only;

  if (decide) {
    // every frame's 0 * q term enters every region's sum: count the non-finite frames
    int nf_total = 0;
    for (int t0 = 0; t0 < p.T; t0 += kMaskThreads) {
      const int t = t0 + threadIdx.x;
      const int nf = t < p.T && !isfinite(q[t]);
      int total;
      scan_int(nf, nf_total, itot, &total);
      nf_total = total;
    }
    if (threadIdx.x == 0) carry = Seg{0.0, 0, 0};
    int count = 0;
    for (int t0 = 0; t0 < p.T; t0 += kMaskThreads) {
      const int t = t0 + threadIdx.x;
      const bool in = t < p.T;
      const int e = in ? edge<false>(p, q, on, t) : 0;
      int total;
      const int idx = scan_int(e, count, itot, &total) - 1;
      count = total;
      const float qt = in ? q[t] : 0.f;
      const Seg r = scan_seg(Seg{(double)qt, in && !isfinite(qt), e}, &carry, stot);
      const bool last = in && (t == p.T - 1 || edge<false>(p, q, on, t + 1));
      if (last && idx < p.Rf) flags[idx] = r.s > 0.0 && r.nf == nf_total;
    }
    __syncthreads();   // the decisions are visible to the whole CTA
  }

  int count = 0;
  for (int t0 = 0; t0 < p.T_out; t0 += kMaskThreads) {
    const int t = t0 + threadIdx.x;
    // T = 1 gives two rows of region 0 (the edge rule pads one frame at each end)
    const int tq = t < p.T ? t : p.T - 1;
    const int e = t < p.T ? edge<kOnset>(p, q, on, t) : 0;
    int total;
    const int idx = scan_int(e, count, itot, &total) - 1;
    count = total;
    int col = -1;
    if (t < p.T_out && idx >= 0 && idx < p.R) {
      bool keep = true;
      if (p.note_on_only) keep = kOnset ? q[tq] > 0.f : flags[idx] != 0;
      col = keep ? idx : -1;
    }
    cols[threadIdx.x] = col;
    __syncthreads();
    const int rows = min(kMaskThreads, p.T_out - t0);
    const int lane = threadIdx.x & 31;
    for (int row = threadIdx.x >> 5; row < rows; row += kMaskWarps) {
      float* dst = mask + ((b * p.T_out) + t0 + row) * (int64_t)p.R;
      const int c = cols[row];
      for (int n = lane; n < p.R; n += 32) dst[n] = n == c ? 1.f : 0.f;
    }
    __syncthreads();
  }
}

// ---- moments, pool and backward ----------------------------------------------------------
struct Params {
  const float* x;   // [B, T, D]
  const float* m;   // [B, T, N]
  int T, N, D;
  int tiles_r, tiles_d;   // tiles of the output rows (n or t) and of d per item
};

struct Tile {
  int64_t b;
  int r0, d0;
};

__device__ __forceinline__ Tile tile_of(const Params& p) {
  const int64_t per_item = (int64_t)p.tiles_r * p.tiles_d;
  const int64_t blk = blockIdx.x;
  Tile t;
  t.b = blk / per_item;
  const int64_t rem = blk - t.b * per_item;
  t.r0 = (int)(rem / p.tiles_d) * kTile;
  t.d0 = (int)(rem % p.tiles_d) * kDTile;
  return t;
}

// Stages mask rows t0 .. t0 + kChunk of the notes n0 .. n0 + kTile as ms[t][n], and the
// [kChunk, kDTile] block at dims d0.. of each [B,T,D] operand v0, v1, v2 that is not
// null into vs[0], vs[1], vs[2], zeros outside the shapes.
__device__ __forceinline__ void stage_block(const Params& p, const Tile& tl, int t0,
                                            const float* v, float (*vs)[kDTile]) {
  for (int k = threadIdx.x; k < kChunk * kDTile; k += kThreads) {
    const int tt = k / kDTile, dd = k % kDTile;
    const int t = t0 + tt, d = tl.d0 + dd;
    vs[tt][dd] = t < p.T && d < p.D ? v[(tl.b * p.T + t) * p.D + d] : 0.f;
  }
}

__device__ __forceinline__ void stage_over_t(const Params& p, const Tile& tl, int t0,
                                             float (*ms)[kTile], float (*vs)[kChunk][kDTile],
                                             const float* v0, const float* v1 = nullptr,
                                             const float* v2 = nullptr) {
  for (int k = threadIdx.x; k < kChunk * kTile; k += kThreads) {
    const int tt = k / kTile, nn = k % kTile;
    const int t = t0 + tt, n = tl.r0 + nn;
    ms[tt][nn] = t < p.T && n < p.N ? p.m[(tl.b * p.T + t) * p.N + n] : 0.f;
  }
  if (v0) stage_block(p, tl, t0, v0, vs[0]);
  if (v1) stage_block(p, tl, t0, v1, vs[1]);
  if (v2) stage_block(p, tl, t0, v2, vs[2]);
  __syncthreads();
}

// Loads the [B,N,D] operand `a` at this thread's 4 notes and 2 dims.
__device__ __forceinline__ void load_nd(const Params& p, const Tile& tl, const float* a,
                                        float (&out)[4][2]) {
  const int ty = threadIdx.x >> 5, tx = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int n = tl.r0 + ty * 4 + i, d = tl.d0 + tx + 32 * j;
      out[i][j] = a && n < p.N && d < p.D ? a[(tl.b * p.N + n) * p.D + d] : 0.f;
    }
}

__device__ __forceinline__ void store_nd(const Params& p, const Tile& tl, float* a,
                                         const float (&v)[4][2]) {
  const int ty = threadIdx.x >> 5, tx = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int n = tl.r0 + ty * 4 + i, d = tl.d0 + tx + 32 * j;
      if (n < p.N && d < p.D) a[(tl.b * p.N + n) * p.D + d] = v[i][j];
    }
}

__device__ __forceinline__ float safe_len(float l) { return l == 0.f ? 1e-7f : l; }

// mean and, with kStd, std [B,N,D]: two passes over t.
template <bool kStd>
__global__ void __launch_bounds__(kThreads, 1)
note_moments_kernel(Params p, float* __restrict__ mean, float* __restrict__ stdev) {
  __shared__ __align__(16) float ms[kChunk][kTile];
  __shared__ float xs[1][kChunk][kDTile];
  const Tile tl = tile_of(p);
  const int ty = threadIdx.x >> 5, tx = threadIdx.x & 31;
  float len[4] = {0.f, 0.f, 0.f, 0.f}, s[4][2] = {};
  for (int t0 = 0; t0 < p.T; t0 += kChunk) {
    stage_over_t(p, tl, t0, ms, xs, p.x);
    float cl[4] = {0.f, 0.f, 0.f, 0.f}, cs[4][2] = {};
#pragma unroll 8
    for (int tt = 0; tt < kChunk; ++tt) {
      const float4 m4 = *reinterpret_cast<const float4*>(&ms[tt][ty * 4]);
      const float mv[4] = {m4.x, m4.y, m4.z, m4.w};
      const float xv[2] = {xs[0][tt][tx], xs[0][tt][tx + 32]};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        cl[i] += mv[i];
#pragma unroll
        for (int j = 0; j < 2; ++j) cs[i][j] = fmaf(mv[i], xv[j], cs[i][j]);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      len[i] += cl[i];
#pragma unroll
      for (int j = 0; j < 2; ++j) s[i][j] += cs[i][j];
    }
    __syncthreads();
  }
  float mu[4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) mu[i][j] = s[i][j] / safe_len(len[i]);
  store_nd(p, tl, mean, mu);
  if (!kStd) return;
  float q[4][2] = {};
  for (int t0 = 0; t0 < p.T; t0 += kChunk) {
    stage_over_t(p, tl, t0, ms, xs, p.x);
    float cq[4][2] = {};
#pragma unroll 8
    for (int tt = 0; tt < kChunk; ++tt) {
      const float4 m4 = *reinterpret_cast<const float4*>(&ms[tt][ty * 4]);
      const float mv[4] = {m4.x, m4.y, m4.z, m4.w};
      const float xv[2] = {xs[0][tt][tx], xs[0][tt][tx + 32]};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float r = (xv[j] - mu[i][j]) * mv[i];
          cq[i][j] = fmaf(r, r, cq[i][j]);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) q[i][j] += cq[i][j];
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) q[i][j] = sqrtf(q[i][j] / safe_len(len[i]));
  store_nd(p, tl, stdev, q);
}

// Contraction over n on a tile of kTile frames by kDTile dims, from [B,N,D] operands.
enum Mode {
  kPoolMean,   // out0 = sum_n m mu
  kPoolBoth,   // and out1 = sum_n m sigma
  kDxMean,     // dx = sum_n m A
  kDxBoth      // dx = sum_n m (A + C (x - mu) m)
};

struct OverN {
  const float* a;    // mu or A
  const float* c;    // sigma or C
  const float* mu;   // mu (kDxBoth)
};

template <int kMode>
__global__ void __launch_bounds__(kThreads, 1)
note_over_n_kernel(Params p, OverN o, float* __restrict__ out0, float* __restrict__ out1) {
  constexpr bool kTwo = kMode == kPoolBoth || kMode == kDxBoth;
  __shared__ float ms[kTile][kChunk + 1];   // [t][n]
  __shared__ float as[kChunk][kDTile];
  __shared__ float cs[kTwo ? kChunk : 1][kDTile];
  __shared__ float us[kMode == kDxBoth ? kChunk : 1][kDTile];
  const Tile tl = tile_of(p);
  const int ty = threadIdx.x >> 5, tx = threadIdx.x & 31;
  float xv[4][2] = {};
  if (kMode == kDxBoth) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int t = tl.r0 + ty * 4 + i, d = tl.d0 + tx + 32 * j;
        xv[i][j] = t < p.T && d < p.D ? p.x[(tl.b * p.T + t) * p.D + d] : 0.f;
      }
  }
  float s0[4][2] = {}, s1[4][2] = {};
  for (int n0 = 0; n0 < p.N; n0 += kChunk) {
    for (int k = threadIdx.x; k < kTile * kChunk; k += kThreads) {
      const int tt = k / kChunk, nn = k % kChunk;
      const int t = tl.r0 + tt, n = n0 + nn;
      ms[tt][nn] = t < p.T && n < p.N ? p.m[(tl.b * p.T + t) * p.N + n] : 0.f;
    }
    for (int k = threadIdx.x; k < kChunk * kDTile; k += kThreads) {
      const int nn = k / kDTile, dd = k % kDTile;
      const int n = n0 + nn, d = tl.d0 + dd;
      const bool in = n < p.N && d < p.D;
      const int64_t at = (tl.b * p.N + n) * p.D + d;
      as[nn][dd] = in ? o.a[at] : 0.f;
      if (kTwo) cs[nn][dd] = in ? o.c[at] : 0.f;
      if (kMode == kDxBoth) us[nn][dd] = in ? o.mu[at] : 0.f;
    }
    __syncthreads();
    float c0[4][2] = {}, c1[4][2] = {};
#pragma unroll 4
    for (int nn = 0; nn < kChunk; ++nn) {
      float av[2], cv[2], uv[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        av[j] = as[nn][tx + 32 * j];
        if (kTwo) cv[j] = cs[nn][tx + 32 * j];
        if (kMode == kDxBoth) uv[j] = us[nn][tx + 32 * j];
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float mv = ms[ty * 4 + i][nn];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          if (kMode == kDxBoth) {
            const float r = (xv[i][j] - uv[j]) * mv;
            c0[i][j] = fmaf(mv, fmaf(cv[j], r, av[j]), c0[i][j]);
          } else {
            c0[i][j] = fmaf(mv, av[j], c0[i][j]);
            if (kMode == kPoolBoth) c1[i][j] = fmaf(mv, cv[j], c1[i][j]);
          }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        s0[i][j] += c0[i][j];
        if (kMode == kPoolBoth) s1[i][j] += c1[i][j];
      }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int t = tl.r0 + ty * 4 + i, d = tl.d0 + tx + 32 * j;
      if (t < p.T && d < p.D) {
        const int64_t at = (tl.b * p.T + t) * p.D + d;
        out0[at] = s0[i][j];
        if (kMode == kPoolBoth) out1[at] = s1[i][j];
      }
    }
}

struct Grads {
  const float* mean;     // [B,N,D] forward mean
  const float* stdev;    // [B,N,D] forward std (kStd)
  const float* gmu;      // [B,N,D] or null
  const float* gsd;      // [B,N,D] or null
  const float* gpmu;     // [B,T,D] or null
  const float* gpsd;     // [B,T,D] or null
};

// A = Gmu' / Ls and, with kStd, C = 2 GQ, [B,N,D] each: one pass over t.
template <bool kStd>
__global__ void __launch_bounds__(kThreads, 1)
note_moments_backward_kernel(Params p, Grads g, float* __restrict__ A, float* __restrict__ C) {
  __shared__ __align__(16) float ms[kChunk][kTile];
  __shared__ float vs[3][kChunk][kDTile];   // x, gPmu, gPsigma
  const Tile tl = tile_of(p);
  const int ty = threadIdx.x >> 5, tx = threadIdx.x & 31;
  // x (for r, with a std gradient) and the pooled gradients present
  const bool pooled_mean = g.gpmu != nullptr, pooled_std = kStd && g.gpsd != nullptr;
  float mu[4][2];
  load_nd(p, tl, g.mean, mu);
  float len[4] = {0.f, 0.f, 0.f, 0.f}, pm[4][2] = {}, ps[4][2] = {}, sr[4][2] = {};
  for (int t0 = 0; t0 < p.T; t0 += kChunk) {
    stage_over_t(p, tl, t0, ms, vs, kStd ? p.x : nullptr, g.gpmu,
                 kStd ? g.gpsd : nullptr);
    float cl[4] = {0.f, 0.f, 0.f, 0.f}, cpm[4][2] = {}, cps[4][2] = {}, csr[4][2] = {};
#pragma unroll 4
    for (int tt = 0; tt < kChunk; ++tt) {
      const float4 m4 = *reinterpret_cast<const float4*>(&ms[tt][ty * 4]);
      const float mv[4] = {m4.x, m4.y, m4.z, m4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) cl[i] += mv[i];
      if (pooled_mean) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float gv = vs[1][tt][tx + 32 * j];
#pragma unroll
          for (int i = 0; i < 4; ++i) cpm[i][j] = fmaf(mv[i], gv, cpm[i][j]);
        }
      }
      if (pooled_std) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float gv = vs[2][tt][tx + 32 * j];
#pragma unroll
          for (int i = 0; i < 4; ++i) cps[i][j] = fmaf(mv[i], gv, cps[i][j]);
        }
      }
      if (kStd) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float xv = vs[0][tt][tx + 32 * j];
#pragma unroll
          for (int i = 0; i < 4; ++i) csr[i][j] = fmaf(mv[i], (xv - mu[i][j]) * mv[i], csr[i][j]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      len[i] += cl[i];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        pm[i][j] += cpm[i][j];
        ps[i][j] += cps[i][j];
        sr[i][j] += csr[i][j];
      }
    }
    __syncthreads();
  }
  float gmu[4][2], a[4][2], c[4][2];
  load_nd(p, tl, g.gmu, gmu);
  if (kStd) {
    float sd[4][2], gsd[4][2];
    load_nd(p, tl, g.stdev, sd);
    load_nd(p, tl, g.gsd, gsd);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const float ls = safe_len(len[i]);
        const float gv = (gsd[i][j] + ps[i][j]) * (0.5f / sd[i][j]);
        const float gq = gv / ls;
        c[i][j] = 2.f * gq;
        a[i][j] = ((gmu[i][j] + pm[i][j]) - c[i][j] * sr[i][j]) / ls;
      }
    store_nd(p, tl, C, c);
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) a[i][j] = (gmu[i][j] + pm[i][j]) / safe_len(len[i]);
  }
  store_nd(p, tl, A, a);
}

}  // namespace notes_
}  // namespace ddsp
