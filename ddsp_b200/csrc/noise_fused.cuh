// Fused FilteredNoise.get_signal (synths.py:181-196): magnitudes -> windowed
// impulse responses (core.py:1534-1565, 1477-1531) -> time-varying FIR of
// uniform noise (core.py:1382-1473) [-> += harmonic audio, processors.py:174].
// IRs, noise and per-frame partial convolutions live only in shared memory.
//
// Formulation (SURVEY.md A.5/A.6).  The reference frames the input, convolves
// frame j with ITS impulse response h_j (FFT size >= frame + S - 1, i.e. a
// linear convolution) and overlap-adds:
//     y_j[n]  = sum_i x_j[i] h_j[n - i],  n in [0, frame + S - 1)
//     out[t]  = sum_j y_j[t + start - j * frame]
//
// Mapping.  A persistent CTA (12 warps) walks tiles of 32 input frames (29
// output frames + 3 halo for the decoder shape); ONE LANE OWNS ONE INPUT FRAME,
// so x_j, M_j, h_j are lane-private rows of shared memory with odd strides (no
// bank conflicts) and every warp-wide operand of the inner loops is either
// lane-private or a broadcast.
//   A. stage magnitudes (exp_sigmoid fused when they are raw network outputs)
//   B. warps 0..5: impulse-response synthesis as two half-size cosine sums
//        h0[n]      = E[n] + O[n],  h0[S0/2 - n] = E[n] - O[n],  n = 0..S0/4
//        E = even-k terms, O = odd-k terms of the irfft of a real spectrum
//      (half the MACs of a full cosine sum, a quarter of an irfft's outputs);
//      16 outputs per thread, table rows arrive as broadcast LDS.128;
//      warps 6..11 meanwhile generate the noise (Philox4x32-10) or copy it in
//      (the taps h_j[tap] = window[tap] * h0[|tap - shift|] are written by the
//      same warps straight from registers)
//   D. FIR: warp = block of 16 outputs of y_j held as 8 packed f32x2
//      accumulators; two register windows of 8 tap PAIRS slide over the lane's
//      IR row (one window of even-aligned pairs for even input samples, one of
//      odd-aligned pairs - from a copy of the row shifted by one tap - for odd
//      ones), so two input samples cost 3 LDS.64 + 32 lane-FMAs
//   E. overlap-add in shared memory (skewed layout, blocks that could collide
//      are serialised by frame-group), F. crop + (+= harmonic) + coalesced store
#pragma once
#include "noise.cuh"

namespace ddsp {

constexpr int kNfThreads = 384;          // 12 warps
constexpr int kNfWarps = kNfThreads / 32;
constexpr int kNfR = 16;                 // outputs per thread in the FIR
constexpr int kNfPad = 32;               // zero taps either side of h rows
constexpr int kNfMaxNb = 129;            // table / row sizes stay in smem

struct NoiseFusedParams {
  const float* __restrict__ mags;   // [B,F,nb]
  const float* __restrict__ noise;  // [B,N] or nullptr
  float* audio;                     // [B,N]
  uint64_t seed, offset;
  int B, F, nb, N, frame, start, accumulate;
  int item_base;                    // Philox item index of batch row 0
  int raw;                          // mags are raw network outputs:
  float bias;                       //   exp_sigmoid(x + bias) while staging
  int TFo, Hb, Ha;                  // output frames per tile, halo before/after
  int tiles_per_item, n_tiles;
  int Q, QP, ne, no;                // S0/4, padded column count, #even k, #odd k
  int mS, hS, xS;                   // smem row strides (floats); hS, xS = 2 mod 4
  int nq_shift;                     // log2(frame / 4) or -1
  int ylen, nblk, ngrp;             // frame + S - 1, FIR blocks, frame groups
  int outLen;                       // skewed OLA buffer length
  IrGeom g;
};

struct NfSmem {
  size_t off_te, off_to, off_win, off_m, off_raw, off_h, off_x, off_out, total;
};

__host__ __device__ inline NfSmem nf_smem_layout(const NoiseFusedParams& p) {
  NfSmem s;
  size_t o = 0;
  s.off_te = o;  o += sizeof(float) * (size_t)p.ne * p.QP;
  s.off_to = o;  o += sizeof(float) * (size_t)p.no * p.QP;
  s.off_win = o; o += sizeof(float) * (size_t)((p.g.S + 3) & ~3);
  s.off_m = o;   o += sizeof(float) * 32 * (size_t)p.mS;
  s.off_raw = o; o += sizeof(float) * 32 * (size_t)p.nb;
  s.off_h = o;   o += sizeof(float) * 64 * (size_t)p.hS;   // even + odd copies
  s.off_x = o;   o += sizeof(float) * 32 * (size_t)p.xS;
  s.off_out = o; o += sizeof(float) * (size_t)p.outLen;
  s.total = (o + 15) & ~(size_t)15;
  return s;
}

__device__ __forceinline__ float2 nf_ffma2(float x, float2 w, float2 acc) {
  return ffma2(make_float2(x, x), w, acc);
}

// cp.async (LDGSTS) of one float: global -> shared without register staging.
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(
                   (uint32_t)__cvta_generic_to_shared(smem_dst)),
               "l"(gsrc)
               : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.wait_all;" ::: "memory");
}

// One block of W = 4*W4 columns n0..n0+W-1 of BOTH half-size cosine sums
//   E[n] = sum_k' m[2k']   cos(2 pi 2k' n / S0),  O[n] = sum_k' m[2k'+1] cos(...)
// followed by the tap epilogue: h0[n] = E + O at zero-phase offsets +-n and
// h0[S0/2 - n] = E - O at offsets +-(S0/2 - n); h[tap] = win[tap] * h0[|tap-shift|].
template <int W4>
__device__ __forceinline__ void ir_block_eo(const float* __restrict__ mrow,
                                            const float* __restrict__ tE,
                                            const float* __restrict__ tO, int QP,
                                            int ne, int no, int n0, int Q,
                                            int shift, int S,
                                            const float* __restrict__ win,
                                            float* __restrict__ hrow,
                                            float* __restrict__ hrow_odd) {
  float aE[4 * W4], aO[4 * W4];
#pragma unroll
  for (int c = 0; c < 4 * W4; ++c) aE[c] = aO[c] = 0.f;
#pragma unroll 3
  for (int k = 0; k < ne; ++k) {
    const float m = mrow[2 * k];
    const float4* t4 = reinterpret_cast<const float4*>(tE + k * QP + n0);
#pragma unroll
    for (int q = 0; q < W4; ++q) {
      const float4 c = t4[q];
      aE[4 * q + 0] = fmaf(m, c.x, aE[4 * q + 0]);
      aE[4 * q + 1] = fmaf(m, c.y, aE[4 * q + 1]);
      aE[4 * q + 2] = fmaf(m, c.z, aE[4 * q + 2]);
      aE[4 * q + 3] = fmaf(m, c.w, aE[4 * q + 3]);
    }
  }
#pragma unroll 3
  for (int k = 0; k < no; ++k) {
    const float m = mrow[2 * k + 1];
    const float4* t4 = reinterpret_cast<const float4*>(tO + k * QP + n0);
#pragma unroll
    for (int q = 0; q < W4; ++q) {
      const float4 c = t4[q];
      aO[4 * q + 0] = fmaf(m, c.x, aO[4 * q + 0]);
      aO[4 * q + 1] = fmaf(m, c.y, aO[4 * q + 1]);
      aO[4 * q + 2] = fmaf(m, c.z, aO[4 * q + 2]);
      aO[4 * q + 3] = fmaf(m, c.w, aO[4 * q + 3]);
    }
  }
#pragma unroll
  for (int c = 0; c < 4 * W4; ++c) {
    const int n = n0 + c;
    if (n > Q) continue;
    const float hp = aE[c] + aO[c];       // h0 at |offset| = n
    const float hm = aE[c] - aO[c];       // h0 at |offset| = 2Q - n
    const int n2 = 2 * Q - n;
    int t;
    float v;
    t = shift + n;
    if (t >= 0 && t < S) { v = win[t] * hp; hrow[t] = v; hrow_odd[t + 1] = v; }
    t = shift - n;
    if (n != 0 && t >= 0 && t < S) { v = win[t] * hp; hrow[t] = v; hrow_odd[t + 1] = v; }
    if (n2 != n) {
      t = shift + n2;
      if (t >= 0 && t < S) { v = win[t] * hm; hrow[t] = v; hrow_odd[t + 1] = v; }
      t = shift - n2;
      if (t >= 0 && t < S) { v = win[t] * hm; hrow[t] = v; hrow_odd[t + 1] = v; }
    }
  }
}

__global__ void __launch_bounds__(kNfThreads, 2)
noise_fused_kernel(NoiseFusedParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const NfSmem L = nf_smem_layout(p);
  float* sTE = (float*)(smem_raw + L.off_te);
  float* sTO = (float*)(smem_raw + L.off_to);
  float* sWin = (float*)(smem_raw + L.off_win);
  float* sM = (float*)(smem_raw + L.off_m);
  float* sRaw = (float*)(smem_raw + L.off_raw);
  float* sH = (float*)(smem_raw + L.off_h);
  float* sX = (float*)(smem_raw + L.off_x);
  float* sOut = (float*)(smem_raw + L.off_out);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const IrGeom g = p.g;
  const int nb = p.nb, S = g.S, S0 = g.S0, frame = p.frame;
  const int Q = p.Q, QP = p.QP, ne = p.ne, no = p.no;
  const float invS0 = 1.0f / (float)S0;

  // ---- once per CTA: cosine tables, window, zero pads ----
  {
    for (int e = tid; e < ne * QP; e += kNfThreads) {
      const int k = e / QP, n = e - k * QP;          // even harmonic 2k
      const int ph = (int)(((long long)2 * k * n) % S0);
      const float ck = (k == 0 || 2 * k == nb - 1) ? invS0 : 2.0f * invS0;
      sTE[e] = (n <= Q) ? ck * cospif(2.0f * (float)ph * invS0) : 0.f;
    }
    for (int e = tid; e < no * QP; e += kNfThreads) {
      const int k = e / QP, n = e - k * QP;          // odd harmonic 2k+1
      const int ph = (int)(((long long)(2 * k + 1) * n) % S0);
      sTO[e] = (n < Q) ? 2.0f * invS0 * cospif(2.0f * (float)ph * invS0) : 0.f;
    }
    for (int j = tid; j < S; j += kNfThreads) {
      int idx; float w;
      ir_tap(g, j, &idx, &w);
      sWin[j] = w;
    }
    for (int e = tid; e < 64 * p.hS; e += kNfThreads) sH[e] = 0.f;
    for (int e = tid; e < 32 * p.xS; e += kNfThreads) sX[e] = 0.f;
  }
  __syncthreads();

  const int nblk8 = (Q + 1 + 7) >> 3;                // 8-column blocks of E/O
  const int nq = frame >> 2;                         // noise quads per frame
  const int n_ir_warps = min(nblk8, kNfWarps - 4);

  // raw magnitudes of a tile -> sRaw, asynchronously (consumed one tile later)
  auto prefetch_mags = [&](int tile) {
    const int b = tile / p.tiles_per_item;
    const int j0 = (tile - b * p.tiles_per_item) * p.TFo - p.Hb;
    const float* magb = p.mags + (size_t)b * p.F * nb;
    for (int e = tid; e < 32 * nb; e += kNfThreads) {
      const int jl = e / nb;
      const int j = j0 + jl;
      if (j >= 0 && j < p.F) cp_async4(sRaw + e, magb + ((long long)j0 * nb + e));
    }
  };
  if (blockIdx.x < p.n_tiles) prefetch_mags(blockIdx.x);

  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    const int b = tile / p.tiles_per_item;
    const int q0 = (tile - b * p.tiles_per_item) * p.TFo;   // first output frame
    const int j0 = q0 - p.Hb;                                // first input frame

    // ---- A. magnitudes: exp_sigmoid (if raw) and c_k / S0 while moving the
    //         prefetched slab into lane-private rows ----
    cp_async_wait_all();
    __syncthreads();
    for (int jl = warp; jl < 32; jl += kNfWarps) {
      const int j = j0 + jl;
      const float* src = sRaw + jl * nb;
      float* dst = sM + jl * p.mS;
      if (j < 0 || j >= p.F) {
        for (int k = lane; k < nb; k += 32) dst[k] = 0.f;
      } else if (p.raw) {
#pragma unroll 3
        for (int k = lane; k < nb; k += 32)
          dst[k] = exp_sigmoid_f(src[k] + p.bias);             // synths.py:176-177
      } else {
#pragma unroll 3
        for (int k = lane; k < nb; k += 32) dst[k] = src[k];
      }
    }
    for (int e = tid; e < p.outLen; e += kNfThreads) sOut[e] = 0.f;
    __syncthreads();
    {   // the staging buffer is free again: fetch the next tile's magnitudes
      const int nxt = tile + gridDim.x;
      if (nxt < p.n_tiles) prefetch_mags(nxt);
    }

    // ---- B. IR synthesis + taps (warps 0..) || noise staging (other warps) ----
    if (warp < n_ir_warps) {
      for (int blk = warp; blk < nblk8; blk += n_ir_warps) {
        const int n0 = blk << 3;
        const float* mrow = sM + lane * p.mS;
        float* hrow = sH + lane * p.hS + kNfPad;
        float* hrow_odd = sH + (32 + lane) * p.hS + kNfPad;
        if (Q + 1 - n0 > 4)
          ir_block_eo<2>(mrow, sTE, sTO, QP, ne, no, n0, Q, g.shift, S, sWin, hrow,
                         hrow_odd);
        else
          ir_block_eo<1>(mrow, sTE, sTO, QP, ne, no, n0, Q, g.shift, S, sWin, hrow,
                         hrow_odd);
      }
    } else {
      const int nw = kNfWarps - n_ir_warps;
      const float* nzb = p.noise ? p.noise + (size_t)b * p.N : nullptr;
      const int total = 32 * nq;                    // quads in the tile
      const long long p_lo = (long long)j0 * frame;
      const bool interior = (p_lo >= 0) && (p_lo + 32ll * frame <= p.N) && !nzb;
      if (interior) {
        // every sample exists: no bounds checks, 32-bit index math
        const uint32_t qbase = (uint32_t)(p_lo >> 2);
        for (int e = (warp - n_ir_warps) * 32 + lane; e < total; e += nw * 32) {
          int jl, qd;
          if (p.nq_shift >= 0) { jl = e >> p.nq_shift; qd = e & (nq - 1); }
          else { jl = e / nq; qd = e - jl * nq; }
          const float4 r = noise4(qbase + (uint32_t)e, (uint32_t)(b + p.item_base), p.seed, p.offset);
          float2* d = reinterpret_cast<float2*>(sX + jl * p.xS + 4 * qd);
          d[0] = make_float2(r.x, r.y);
          d[1] = make_float2(r.z, r.w);
        }
      } else {
        for (int e = (warp - n_ir_warps) * 32 + lane; e < total; e += nw * 32) {
          const int jl = e / nq, qd = e - jl * nq;
          const long long pp = (long long)(j0 + jl) * frame + 4 * qd;
          float v0 = 0.f, v1 = 0.f, v2 = 0.f, v3 = 0.f;
          if (pp >= 0 && pp < p.N) {
            if (nzb) {
              v0 = nzb[pp];
              if (pp + 1 < p.N) v1 = nzb[pp + 1];
              if (pp + 2 < p.N) v2 = nzb[pp + 2];
              if (pp + 3 < p.N) v3 = nzb[pp + 3];
            } else {
              const float4 r = noise4((uint32_t)(pp >> 2), (uint32_t)(b + p.item_base), p.seed,
                                      p.offset);
              v0 = r.x;
              if (pp + 1 < p.N) v1 = r.y;
              if (pp + 2 < p.N) v2 = r.z;
              if (pp + 3 < p.N) v3 = r.w;
            }
          }
          float* d = sX + jl * p.xS + 4 * qd;
          d[0] = v0; d[1] = v1; d[2] = v2; d[3] = v3;
        }
      }
    }
    __syncthreads();

    // The += operand (harmonic audio) is fetched now so its latency hides
    // behind the FIR; phase F consumes it.
    float* outb = p.audio + (size_t)b * p.N;
    const int nq_out = p.TFo * nq;
    const bool use_pre = p.accumulate && nq_out <= 2 * kNfThreads;
    float4 pre[2];
    pre[0] = pre[1] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (use_pre) {
#pragma unroll
      for (int it = 0; it < 2; ++it) {
        const int e = tid + it * kNfThreads;
        if (e < nq_out) {
          int ql, qd;
          if (p.nq_shift >= 0) { ql = e >> p.nq_shift; qd = e & (nq - 1); }
          else { ql = e / nq; qd = e - ql * nq; }
          const int t = (q0 + ql) * frame + 4 * qd;
          if (q0 + ql < p.F && t + 3 < p.N &&
              (reinterpret_cast<uintptr_t>(outb + t) & 15) == 0)
            pre[it] = *reinterpret_cast<const float4*>(outb + t);
        }
      }
    }

    // ---- D. FIR (lane = frame, warp = 16-output block), E. overlap-add ----
    {
      const float* xrow = sX + lane * p.xS;
      const float* hE = sH + lane * p.hS + kNfPad;          // h[t] at hE[t]
      const float* hO = sH + (32 + lane) * p.hS + kNfPad;   // h[t] at hO[t + 1]
      const int nchunk = (frame + 15) >> 4;
      for (int round = 0; round * kNfWarps < p.nblk; ++round) {
        const int blk = round * kNfWarps + warp;
        const int n0 = blk * kNfR;
        float2 acc2[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) acc2[c] = make_float2(0.f, 0.f);
        if (blk < p.nblk) {
          const int i_lo = max(0, n0 - (S - 1));
          const int i_hi = min(frame - 1, n0 + kNfR - 1);
          const int ch_lo = i_lo >> 4;
          const int ch_hi = min(i_hi >> 4, nchunk - 1);
          // windows for i = 16 * ch_lo: even-aligned pairs (h[b+2c], h[b+2c+1]),
          // odd-aligned pairs (h[b-1+2c], h[b+2c]) with b = n0 - i (even)
          int bse = n0 - (ch_lo << 4);
          float2 WE[8], WO[8];
#pragma unroll
          for (int r = 0; r < 8; ++r) {
            WE[r] = *reinterpret_cast<const float2*>(hE + bse + 2 * r);
            WO[r] = *reinterpret_cast<const float2*>(hO + bse + 2 * r);
          }
          for (int ch = ch_lo; ch <= ch_hi; ++ch) {
            const int ib = ch << 4;
#pragma unroll
            for (int e = 0; e < 8; ++e) {          // inputs ib + 2e, ib + 2e + 1
              const float2 xv = *reinterpret_cast<const float2*>(xrow + ib + 2 * e);
#pragma unroll
              for (int c = 0; c < 8; ++c)
                acc2[c] = nf_ffma2(xv.x, WE[(c - e) & 7], acc2[c]);
#pragma unroll
              for (int c = 0; c < 8; ++c)
                acc2[c] = nf_ffma2(xv.y, WO[(c - e) & 7], acc2[c]);
              // slide both windows by one pair (two taps)
              const int nb2 = n0 - ib - 2 * e - 2;
              WE[(-e - 1) & 7] = *reinterpret_cast<const float2*>(hE + nb2);
              WO[(-e - 1) & 7] = *reinterpret_cast<const float2*>(hO + nb2);
            }
          }
        }
        float acc[kNfR];
#pragma unroll
        for (int c = 0; c < 8; ++c) { acc[2 * c] = acc2[c].x; acc[2 * c + 1] = acc2[c].y; }
        // overlap-add: position o = frame * lane + n, stored skewed by o / frame
        // so lanes hit distinct banks.  Blocks of one frame-group cannot collide.
        const int grp = n0 / frame;
        const int nin = n0 - grp * frame;            // offset inside the group
        float* orow = sOut + (frame + 1) * (lane + grp) + nin;
        for (int gph = 0; gph < p.ngrp; ++gph) {
          if (blk < p.nblk && grp == gph) {
#pragma unroll
            for (int c = 0; c < kNfR; ++c) orow[c] += acc[c];
          }
          __syncthreads();
        }
      }
    }

    // ---- F. crop, (+= harmonic), store: 4 consecutive samples per thread ----
    {
      int it = 0;
      for (int e = tid; e < nq_out; e += kNfThreads, ++it) {
        int ql, qd;
        if (p.nq_shift >= 0) { ql = e >> p.nq_shift; qd = e & (nq - 1); }
        else { ql = e / nq; qd = e - ql * nq; }
        const int t = (q0 + ql) * frame + 4 * qd;
        if (t >= p.N || q0 + ql >= p.F) continue;
        const int r0 = 4 * qd + p.start;
        int f0 = 0, rem = r0;                        // r0 < frame + start
        while (rem >= frame) { rem -= frame; ++f0; }
        const int o = (ql + p.Hb) * frame + r0;     // unskewed OLA position
        const int sk = ql + p.Hb + f0;               // skew = position / frame
        float v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u)
          v[u] = sOut[o + u + sk + ((rem + u >= frame) ? 1 : 0)];
        if (t + 3 < p.N && ((reinterpret_cast<uintptr_t>(outb + t) & 15) == 0)) {
          float4* dst = reinterpret_cast<float4*>(outb + t);
          float4 r = make_float4(v[0], v[1], v[2], v[3]);
          if (p.accumulate) {
            const float4 a = use_pre ? (it == 0 ? pre[0] : pre[1]) : *dst;
            r.x += a.x; r.y += a.y; r.z += a.z; r.w += a.w;
          }
          *dst = r;
        } else {
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            if (t + u < p.N) {
              float r = v[u];
              if (p.accumulate) r += outb[t + u];
              outb[t + u] = r;
            }
          }
        }
      }
    }
    __syncthreads();
  }
}

inline int nf_odd(int v) { return v | 1; }

// Fills the derived fields; returns false if the shape is outside the fused path.
inline bool nf_configure(NoiseFusedParams& p, int F, int nb, int N,
                         int window_size) {
  if (nb < 3 || nb > kNfMaxNb || (nb & 1) == 0) return false;   // S0 % 4 == 0
  p.g = make_ir_geom(nb, window_size);
  p.F = F; p.nb = nb; p.N = N;
  p.frame = (N + F - 1) / F;
  const int S = p.g.S;
  p.start = (S - 1) / 2 - 1;
  if (p.start < 0) return false;
  if (p.frame < 16 || p.frame > 1024 || (p.frame & 15)) return false;
  p.ylen = p.frame + S - 1;
  p.Hb = (S - 1 - p.start + p.frame - 1) / p.frame;   // ceil((S-1-start)/frame)
  p.Ha = (p.frame - 1 + p.start) / p.frame;
  p.TFo = 32 - p.Hb - p.Ha;
  if (p.TFo < 16) return false;
  p.tiles_per_item = (F + p.TFo - 1) / p.TFo;
  p.Q = p.g.S0 / 4;
  p.QP = (p.Q + 1 + 3) & ~3;
  p.ne = (nb + 1) / 2;
  p.no = (nb - 1) / 2;
  p.mS = nf_odd(nb);
  p.hS = ((S + 2 * kNfPad + 2 + 3) & ~3) + 2;          // = 2 mod 4: conflict-free LDS.64
  p.xS = ((((p.frame + 15) & ~15) + 16 + 3) & ~3) + 2;
  p.nq_shift = -1;
  for (int sh = 0; sh < 12; ++sh)
    if ((p.frame >> 2) == (1 << sh)) p.nq_shift = sh;
  p.nblk = (p.ylen + kNfR - 1) / kNfR;
  p.ngrp = (p.nblk * kNfR + p.frame - 1) / p.frame;
  p.outLen = (p.frame + 1) * (32 + p.ngrp) + 16;
  return nf_smem_layout(p).total <= kMaxDynSmem;
}

inline bool noise_fused_supported(int F, int nb, int N, int window_size) {
  NoiseFusedParams p;
  return nf_configure(p, F, nb, N, window_size);
}

inline int launch_noise_fused(const float* mags, const float* noise,
                              uint64_t seed, uint64_t offset, float* audio,
                              int B, int F, int nb, int N, int window_size,
                              int accumulate, cudaStream_t st, int raw = 0,
                              float bias = 0.f, int item_base = 0) {
  NoiseFusedParams p;
  p.item_base = item_base;
  if (!nf_configure(p, F, nb, N, window_size)) {
    set_error("filtered_noise_forward: shape outside the fused path");
    return DDSP_B200_E_UNSUPPORTED;
  }
  p.mags = mags; p.noise = noise; p.audio = audio;
  p.seed = seed; p.offset = offset; p.B = B; p.accumulate = accumulate;
  p.raw = raw; p.bias = bias;
  const long long n_tiles = (long long)B * p.tiles_per_item;
  if (n_tiles >= (1ll << 31)) {
    set_error("filtered_noise_forward: too many tiles");
    return DDSP_B200_E_INVALID;
  }
  p.n_tiles = (int)n_tiles;
  const size_t smem = nf_smem_layout(p).total;
  const int ctas_per_sm = smem <= 110 * 1024 ? 2 : 1;
  const int grid = (int)std::min<long long>(n_tiles, (long long)num_sms() * ctas_per_sm);
  return launch("filtered_noise_forward(fused)", noise_fused_kernel, grid, kNfThreads, smem,
                st, p);
}

}  // namespace ddsp
