// Windowed-sinc filter design and filtering: core.sinc_impulse_response and
// core.sinc_filter (core.py:1568-1625, 1658-1690).  With S = 2 (window_size / 2) + 1
// taps, half = S / 2, n = m - half and the cutoff c (already scaled by 2 / sample_rate):
//   u[m] = w[m] sinc(c n),  w[m] = 0.54 - 0.46 cos(2 pi m / (S - 1))   (Hamming, odd S)
//   h[m] = u[m] / |Sum_m u[m]|,  and delta[m - half] - h[m] for the high-pass.
// sinc(x) = sin(pi x) / (pi x), with |x| < 1e-20 replaced by 1e-20 (core.py:1571): the
// value there is 1 and its gradient 0.  A frame's taps depend on one scalar, so every
// kernel here builds them in shared memory; none writes them to global memory except
// sinc_ir_kernel, whose output they are.
//
// sinc_filter is fft_convolve with automatic delay compensation (start = half - 1) and
// the taps of each INPUT sample's frame, fr(p) = p / frame (SURVEY.md A.6):
//   y[o] = Sum_p h_{fr(p)}[o + start - p] x[p]                    sinc_filter_kernel
// Its backward separates by frame j.  With G[q] = g[q - start] (0 outside the crop),
// A[p] = Sum_m u_j[m] G[p + m], A'[p] = Sum_m u'_j[m] G[p + m], u' = du/dc, S' = Sum u',
// s = sign(Sum u) and inv = 1 / |Sum u|:
//   dx[p] = inv A[p]          (G[p + half] - inv A[p] for the high-pass)
//   dc_j  = inv (Sum_{p in j} x[p] A'[p] - s S' inv Sum_{p in j} x[p] A[p])
// (negated for the high-pass), both from sinc_filter_backward_kernel.  Every sum runs
// in a fixed order and there are no atomics, so all outputs are bit-reproducible.
#pragma once
#include "common.cuh"

namespace ddsp {

constexpr int kSincThreads = 256;
constexpr float kSincPi = 3.14159265358979323846f;

__device__ __forceinline__ float sinc_window(int m, int S) {
  return S == 1 ? 1.0f : 0.54f - 0.46f * cospif((float)(2 * m) / (float)(S - 1));
}

// u[m] = w sinc(c n) and, when du is set, du/dc = w n sinc'(c n), where
// sinc'(x) = (cos(pi x) - sinc(x)) / x; a series below |x| = 1/4, where the difference
// cancels (its first omitted term is under 1e-9 relative there).
__device__ __forceinline__ float sinc_tap(float c, int m, int S, float* du) {
  const int half = S / 2;
  const float w = sinc_window(m, S);
  const float n = (float)(m - half);
  const float x = __fmul_rn(c, n);
  if (fabsf(x) < 1e-20f) {
    if (du) *du = 0.f;
    return w;
  }
  const float s = sinpif(x) / (kSincPi * x);
  if (du) {
    float d;
    if (fabsf(x) < 0.25f) {
      const float t = (kSincPi * x) * (kSincPi * x);
      const float poly =
          1.f - t * (1.f / 10.f - t * (1.f / 280.f - t * (1.f / 15120.f - t * (1.f / 1330560.f))));
      d = -(kSincPi * kSincPi / 3.f) * x * poly;
    } else {
      d = (cospif(x) - s) / x;
    }
    *du = w * n * d;
  }
  return w * s;
}

// Sums of kN values over the CTA: a butterfly within each warp (every lane ends with
// the same bits, since a + b == b + a), then the warps' sums in warp order.  `red`
// holds kN * (kSincThreads / 32) floats.  Contains two __syncthreads.
template <int kN>
__device__ __forceinline__ void sinc_block_sum(float (&v)[kN], float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < kN; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < kN; ++k) red[k * (kSincThreads / 32) + warp] = v[k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kN; ++k) {
    float t = 0.f;
    for (int w = 0; w < kSincThreads / 32; ++w) t += red[k * (kSincThreads / 32) + w];
    v[k] = t;
  }
  __syncthreads();
}

// ---- core.sinc_impulse_response: one CTA per cutoff --------------------------------
__global__ void __launch_bounds__(kSincThreads)
sinc_ir_kernel(const float* __restrict__ cutoff, float* __restrict__ ir, int S,
               float scale, int high_pass) {
  __shared__ float red[kSincThreads / 32];
  const long long row = blockIdx.x;
  const float c = __fmul_rn(cutoff[row], scale);
  float* h = ir + row * S;
  float sum[1] = {0.f};
  for (int m = threadIdx.x; m < S; m += kSincThreads) sum[0] += sinc_tap(c, m, S, nullptr);
  sinc_block_sum<1>(sum, red);
  const float inv = 1.0f / fabsf(sum[0]);
  const int half = S / 2;
  for (int m = threadIdx.x; m < S; m += kSincThreads) {
    const float v = sinc_tap(c, m, S, nullptr) * inv;
    h[m] = high_pass ? (m == half ? 1.f : 0.f) - v : v;
  }
}

// d cutoff of sinc_impulse_response: d_c = scale inv (Sum dh u' - s S' inv Sum dh u),
// negated for the high-pass.
__global__ void __launch_bounds__(kSincThreads)
sinc_ir_backward_kernel(const float* __restrict__ cutoff, const float* __restrict__ d_ir,
                        float* __restrict__ d_cutoff, int S, float scale, int high_pass) {
  __shared__ float red[4 * (kSincThreads / 32)];
  const long long row = blockIdx.x;
  const float c = __fmul_rn(cutoff[row], scale);
  const float* dh = d_ir + row * S;
  float v[4] = {0.f, 0.f, 0.f, 0.f};   // Sum u, Sum u', Sum dh u, Sum dh u'
  for (int m = threadIdx.x; m < S; m += kSincThreads) {
    float du;
    const float u = sinc_tap(c, m, S, &du);
    const float d = dh[m];
    v[0] += u;
    v[1] += du;
    v[2] = fmaf(d, u, v[2]);
    v[3] = fmaf(d, du, v[3]);
  }
  sinc_block_sum<4>(v, red);
  if (threadIdx.x == 0) {
    const float inv = 1.0f / fabsf(v[0]);
    const float s = v[0] < 0.f ? -1.f : 1.f;
    const float dc = inv * (v[3] - s * v[1] * inv * v[2]);
    d_cutoff[row] = (high_pass ? -dc : dc) * scale;
  }
}

// ---- core.sinc_filter forward -------------------------------------------------------
// A CTA owns kSincTile outputs of one item; thread t the four consecutive outputs
// q0 + 4t .. q0 + 4t + 3 (q = o + start).  For every frame whose input samples reach
// the tile, the CTA builds the frame's unnormalised taps u in shared memory, padded by
// kSincPad zeros on both sides, and each warp runs over the inputs of that frame that
// reach its 128 outputs, four at a time: one LDS.128 of taps and one broadcast LDS.128
// of audio feed 16 FMAs.  The frame's partial sums are scaled by its 1 / |Sum u| into
// the outputs, so the normalised taps are never formed.
constexpr int kSincR = 4;
constexpr int kSincTile = kSincThreads * kSincR;   // 1024 outputs
constexpr int kSincPad = 128;                      // one warp's span of outputs

struct SincFilterParams {
  const float* __restrict__ x;        // [B, N]
  const float* __restrict__ cutoff;   // [cutoff_batch, F]
  float* out;                         // [B, out_len]
  int N, F, frame, S, cutoff_stride;  // cutoff_stride: F, or 0 for a shared cutoff
  float scale;
  int high_pass, start, out_len, accumulate;
};

__host__ __device__ inline int sinc_round4(int v) { return (v + 3) & ~3; }
// x window offset: a multiple of 4 of at least S + 3 samples before q0
__host__ __device__ inline int sinc_xoff(int S) { return sinc_round4(S + 3); }
__host__ __device__ inline int sinc_hs_len(int S) { return 2 * kSincPad + sinc_round4(S) + 8; }
__host__ __device__ inline size_t sinc_filter_smem(int S) {
  return sizeof(float) * ((size_t)sinc_hs_len(S) + sinc_xoff(S) + kSincTile + 4);
}

__global__ void __launch_bounds__(kSincThreads)
sinc_filter_kernel(SincFilterParams p) {
  extern __shared__ __align__(16) float sm[];
  __shared__ float red[kSincThreads / 32];
  const int S = p.S;
  const int hs_len = sinc_hs_len(S);
  float* hs = sm;                          // [hs_len]  taps u at kSincPad + m
  float* xs = sm + hs_len;                 // [xoff + kSincTile + 4]  x[xbase + i]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.y;
  const int o0 = blockIdx.x * kSincTile;
  const int q0 = o0 + p.start;
  const int xoff = sinc_xoff(S);
  const int xbase = q0 - xoff;
  const float* xb = p.x + (size_t)b * p.N;
  for (int i = tid; i < xoff + kSincTile + 4; i += kSincThreads) {
    const int q = xbase + i;
    xs[i] = (q >= 0 && q < p.N) ? xb[q] : 0.f;
  }
  for (int i = tid; i < hs_len; i += kSincThreads)
    if (i < kSincPad || i >= kSincPad + S) hs[i] = 0.f;
  const int p_first = max(0, q0 - S + 1);
  const int p_last = min(p.N - 1, q0 + kSincTile - 1);
  const int qw = q0 + warp * 32 * kSincR;
  const int qt = qw + lane * kSincR;
  const int w_lo = max(qw - S + 1, p_first);
  const int w_hi = min(qw + 32 * kSincR - 1, p_last);
  const float* cb = p.cutoff + (size_t)b * p.cutoff_stride;
  float acc[kSincR];
#pragma unroll
  for (int r = 0; r < kSincR; ++r) acc[r] = 0.f;
  for (int j = p_first / p.frame; j <= p_last / p.frame; ++j) {
    const float c = __fmul_rn(cb[j], p.scale);
    __syncthreads();                       // the previous frame's taps are consumed
    float sum[1] = {0.f};
    for (int m = tid; m < S; m += kSincThreads) {
      const float u = sinc_tap(c, m, S, nullptr);
      hs[kSincPad + m] = u;
      sum[0] += u;
    }
    sinc_block_sum<1>(sum, red);           // also publishes hs
    const int P0 = max(j * p.frame, w_lo);
    const int P1 = min((j + 1) * p.frame - 1, w_hi);
    if (P0 > P1) continue;
    const float inv = 1.0f / fabsf(sum[0]);
    float facc[kSincR];
#pragma unroll
    for (int r = 0; r < kSincR; ++r) facc[r] = 0.f;
    const int pb0 = P0 - (((P0 - q0) % 4 + 4) % 4);   // pb = q0 (mod 4): aligned loads
    float4 hi = *reinterpret_cast<const float4*>(hs + kSincPad + qt - pb0);
    for (int pb = pb0; pb <= P1; pb += 4) {
      // taps h[qt + r - pb - i] = t[4 + r - i] with t = h[qt - pb - 4 .. qt - pb + 3]
      const float4 lo = *reinterpret_cast<const float4*>(hs + kSincPad + qt - pb - 4);
      float4 xv = *reinterpret_cast<const float4*>(xs + pb - xbase);
      if (pb < P0 || pb + 3 > P1) {        // inputs of other frames
        if (pb + 0 < P0 || pb + 0 > P1) xv.x = 0.f;
        if (pb + 1 < P0 || pb + 1 > P1) xv.y = 0.f;
        if (pb + 2 < P0 || pb + 2 > P1) xv.z = 0.f;
        if (pb + 3 < P0 || pb + 3 > P1) xv.w = 0.f;
      }
      const float t[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
      const float xi[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int r = 0; r < kSincR; ++r) facc[r] = fmaf(t[4 + r - i], xi[i], facc[r]);
      }
      hi = lo;
    }
#pragma unroll
    for (int r = 0; r < kSincR; ++r) acc[r] = fmaf(inv, facc[r], acc[r]);
  }
  const int half = S / 2;
  float* ob = p.out + (size_t)b * p.out_len;
#pragma unroll
  for (int r = 0; r < kSincR; ++r) {
    const int o = o0 + tid * kSincR + r;
    if (o >= p.out_len) continue;
    // high-pass: delta[m - half] - h, i.e. the input half taps back minus the low-pass
    const float y = p.high_pass ? xs[qt + r - half - xbase] - acc[r] : acc[r];
    ob[o] = p.accumulate ? ob[o] + y : y;
  }
}

// ---- core.sinc_filter backward --------------------------------------------------------
// Tiles are whole frames (kSincBwdTile / frame of them) when frames are at most
// kSincBwdTile samples, and segments of one frame otherwise (fir_dir_kernel's split).  A
// CTA stages its tile's window of G once, then per frame builds u and u', and all
// threads share the frame's correlation: nPB blocks of four inputs times nMC chunks of
// taps, whose partial sums are added in chunk order.  One LDS.128 of G and two
// broadcast LDS.128 of u and u' feed 32 FMAs.  d cutoff of a frame goes straight to its
// output when the frame is one tile of a per-item cutoff, and to partial sums that
// sinc_dc_reduce adds in segment, then item order otherwise.
constexpr int kSincBwdTile = 1024;

struct SincBwdParams {
  const float* __restrict__ x;        // [B, N]
  const float* __restrict__ cutoff;   // [cutoff_batch, F]
  const float* __restrict__ g;        // [B, out_len]
  float* dx;                          // [B, N] or null
  float* dc;                          // [B * F * n_seg] partial sums, or [B, F]
  int N, F, frame, S, cutoff_stride;
  float scale;
  int high_pass, start, out_len;
  int fpt, n_seg, seg, tiles;         // frames per tile, segments per frame, tiles per item
};

// Tiles of the backward: kSincBwdTile / frame whole frames per tile, or n_seg segments
// of `seg` samples per frame.
__host__ __device__ inline void sinc_bwd_tiles(int N, int F, int frame, int* fpt, int* n_seg,
                                               int* seg, int* tiles) {
  (void)N;
  if (frame <= kSincBwdTile) {
    *fpt = kSincBwdTile / frame; *n_seg = 1; *seg = frame;
    *tiles = (F + *fpt - 1) / *fpt;
  } else {
    *fpt = 1; *n_seg = (frame + kSincBwdTile - 1) / kSincBwdTile;
    *seg = (frame + *n_seg - 1) / *n_seg;
    *tiles = F * *n_seg;
  }
}

__host__ __device__ inline int sinc_gs_len(int S) { return kSincBwdTile + sinc_round4(S) + 8; }
__host__ __device__ inline size_t sinc_bwd_smem(int S) {
  // G window, u and u' (zero padded to a multiple of 4, plus one float4), partial sums
  return sizeof(float) * ((size_t)sinc_gs_len(S) + 2 * ((size_t)sinc_round4(S) + 4) +
                          2 * (size_t)kSincBwdTile);
}

template <bool kDc>
__global__ void __launch_bounds__(kSincThreads)
sinc_filter_backward_kernel(SincBwdParams p) {
  extern __shared__ __align__(16) float sm[];
  __shared__ float red[2 * (kSincThreads / 32)];
  const int S = p.S, S4 = sinc_round4(S);
  float* gs = sm;                          // [gs_len]   G[pt0 + i]
  float* us = gs + sinc_gs_len(S);         // [S4 + 4]   u
  float* ups = us + S4 + 4;                // [S4 + 4]   u'
  float* pa = ups + S4 + 4;                // [kSincBwdTile]  partial A  [nMC][nPB * 4]
  float* pd = pa + kSincBwdTile;           // [kSincBwdTile]  partial A'
  const int tid = threadIdx.x;
  const int b = blockIdx.y, t = blockIdx.x;
  int j_lo, j_hi, pt0, pt1;                // frames [j_lo, j_hi), inputs [pt0, pt1)
  if (p.n_seg == 1) {
    j_lo = t * p.fpt; j_hi = min(p.F, j_lo + p.fpt);
    pt0 = j_lo * p.frame; pt1 = min(p.N, j_hi * p.frame);
  } else {
    j_lo = t / p.n_seg; j_hi = j_lo + 1;
    const int c = t - j_lo * p.n_seg;
    pt0 = j_lo * p.frame + c * p.seg;
    pt1 = min(min(pt0 + p.seg, (j_lo + 1) * p.frame), p.N);
    // the last frame may be shorter than its leading segments: a segment past N still
    // owns a partial sum, which sinc_dc_reduce reads
    if (pt0 >= pt1) {
      if (kDc && tid == 0) p.dc[((size_t)b * p.F + j_lo) * p.n_seg + c] = 0.f;
      return;
    }
  }
  const float* gb = p.g + (size_t)b * p.out_len;
  const int gs_len = sinc_gs_len(S);
  for (int i = tid; i < gs_len; i += kSincThreads) {
    const long long q = (long long)pt0 + i - p.start;
    gs[i] = (q >= 0 && q < p.out_len) ? gb[q] : 0.f;
  }
  for (int i = S + tid; i < S4 + 4; i += kSincThreads) {
    us[i] = 0.f;
    ups[i] = 0.f;
  }
  const float* cb = p.cutoff + (size_t)b * p.cutoff_stride;
  const float* xb = p.x + (size_t)b * p.N;
  const int half = S / 2;
  for (int j = j_lo; j < j_hi; ++j) {
    const int P0 = max(pt0, j * p.frame), P1 = min(pt1, (j + 1) * p.frame);
    if (P0 >= P1) break;
    const float c = __fmul_rn(cb[j], p.scale);
    __syncthreads();                       // the previous frame is done with us, pa, pd
    float su[2] = {0.f, 0.f};              // Sum u, Sum u'
    for (int m = tid; m < S; m += kSincThreads) {
      float du = 0.f;
      const float u = sinc_tap(c, m, S, kDc ? &du : nullptr);
      us[m] = u;
      su[0] += u;
      if (kDc) {
        ups[m] = du;
        su[1] += du;
      }
    }
    sinc_block_sum<2>(su, red);            // also publishes us, ups
    const float inv = 1.0f / fabsf(su[0]);
    // blocks of four inputs from Pa = P0 rounded down to pt0 (mod 4), times tap chunks
    const int Pa = P0 - ((P0 - pt0) & 3);
    const int nPB = (P1 - Pa + 3) / 4;
    const int chunk = sinc_round4((S4 + kSincThreads / nPB - 1) / (kSincThreads / nPB));
    const int nMC = (S4 + chunk - 1) / chunk;
    const int pbk = tid % nPB, mc = tid / nPB;
    if (mc < nMC) {
      const int pp = Pa + 4 * pbk - pt0;   // gs index of the block's first input
      const int m_lo = mc * chunk, m_hi = min(S4, m_lo + chunk);
      float A[4] = {0.f, 0.f, 0.f, 0.f}, D[4] = {0.f, 0.f, 0.f, 0.f};
      float4 lo = *reinterpret_cast<const float4*>(gs + pp + m_lo);
      for (int mb = m_lo; mb < m_hi; mb += 4) {
        const float4 hi = *reinterpret_cast<const float4*>(gs + pp + mb + 4);
        const float4 uv = *reinterpret_cast<const float4*>(us + mb);
        const float g8[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
        const float ui[4] = {uv.x, uv.y, uv.z, uv.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
#pragma unroll
          for (int r = 0; r < 4; ++r) A[r] = fmaf(ui[i], g8[r + i], A[r]);
        }
        if (kDc) {
          const float4 dv = *reinterpret_cast<const float4*>(ups + mb);
          const float di[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
#pragma unroll
            for (int r = 0; r < 4; ++r) D[r] = fmaf(di[i], g8[r + i], D[r]);
          }
        }
        lo = hi;
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        pa[mc * nPB * 4 + pbk * 4 + r] = A[r];
        if (kDc) pd[mc * nPB * 4 + pbk * 4 + r] = D[r];
      }
    }
    __syncthreads();
    float sx[2] = {0.f, 0.f};              // Sum x A, Sum x A'
    for (int e = tid; e < nPB * 4; e += kSincThreads) {
      const int q = Pa + e;
      if (q < P0 || q >= P1) continue;
      float A = 0.f, D = 0.f;
      for (int k = 0; k < nMC; ++k) {
        A += pa[k * nPB * 4 + e];
        if (kDc) D += pd[k * nPB * 4 + e];
      }
      if (p.dx) {
        const float v = inv * A;
        p.dx[(size_t)b * p.N + q] = p.high_pass ? gs[q - pt0 + half] - v : v;
      }
      if (kDc) {
        const float xv = xb[q];
        sx[0] = fmaf(xv, A, sx[0]);
        sx[1] = fmaf(xv, D, sx[1]);
      }
    }
    if (kDc) {
      sinc_block_sum<2>(sx, red);
      if (tid == 0) {
        const float s = su[0] < 0.f ? -1.f : 1.f;
        const float dc = inv * (sx[1] - s * su[1] * inv * sx[0]) * p.scale;
        const int c = p.n_seg == 1 ? 0 : t - j * p.n_seg;
        p.dc[((size_t)b * p.F + j) * p.n_seg + c] = p.high_pass ? -dc : dc;
      }
    }
  }
}

// d cutoff [cutoff_batch, F] from the partial sums [B, F, n_seg]: item ib sums its own
// segments, a shared cutoff every item's, in item then segment order.
__global__ void sinc_dc_reduce(const float* __restrict__ part, float* __restrict__ dc, int B,
                               int F, int n_seg, int shared, long long n_out) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n_out;
       e += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(e % F), ib = (int)(e / F);
    const int b_lo = shared ? 0 : ib, b_hi = shared ? B : ib + 1;
    float acc = 0.f;
    for (int bb = b_lo; bb < b_hi; ++bb) {
      const float* pp = part + ((size_t)bb * F + j) * n_seg;
      for (int c = 0; c < n_seg; ++c) acc += pp[c];
    }
    dc[e] = acc;
  }
}

}  // namespace ddsp
