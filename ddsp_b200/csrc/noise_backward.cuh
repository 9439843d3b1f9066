// Backward of FilteredNoise (core.py:1534-1565, 1382-1473; C4, SURVEY.md 7.3-7).
// The output is linear in the magnitudes:
//   dL/dh_j[m] = sum_i x_j[i] gy_j[i + m],  gy_j[n] = g[frame j + n - start],
//   dL/dM_{j,k} = (c_k / S0) sum_m win[m] cos(2 pi k (m - shift) / S0) dL/dh_j[m].
// noise_backward_kernel writes d magnitudes; lane = frame, tile = 32 frames.
#pragma once
#include "noise.cuh"

namespace ddsp {

constexpr int kNbThreads = 256;

struct NoiseBwdParams {
  const float* __restrict__ grad;   // [B,N]
  const float* __restrict__ noise;  // [B,N] or nullptr (Philox(seed, offset))
  float* dmags;                     // [B,F,nb]
  uint64_t seed, offset;
  int B, F, nb, N, frame, start, S, ylen;
  int xS, gS, hS, nh;               // smem strides; nh = S0/2 + 1
  int tiles_per_item, n_tiles;
  int eo_tab;                       // 1: [nh][kEoStride] cosine table behind the rows (nb = 65)
  IrGeom g;
};
constexpr int kEoStride = 36;       // 33 columns k = 0..32, padded to float4s

// Offset in floats of the cosine table: behind the tables and rows, rounded up to a
// float4.
__host__ __device__ inline size_t noise_bwd_eo_offset(const NoiseBwdParams& p) {
  return ((size_t)p.g.S0 + p.S + 32 * (size_t)(p.xS + p.gS + p.hS) + 3) & ~(size_t)3;
}

__global__ void __launch_bounds__(kNbThreads)
noise_backward_kernel(NoiseBwdParams p) {
  extern __shared__ __align__(16) float sm[];
  float* sCos = sm;                              // [S0] cos(2 pi i / S0)
  float* sWin = sCos + p.g.S0;                   // [S]
  float* sX = sWin + p.S;                        // [32][xS]
  float* sG = sX + 32 * p.xS;                    // [32][gS]   gy rows
  float* sH = sG + 32 * p.gS;                    // [32][hS]   dh rows, then dh0
  // [nh][kEoStride] cos(2 pi k n / S0), k <= 32, read as float4: 16-byte aligned even
  // when S is odd (padded windows)
  float* sEo = sm + noise_bwd_eo_offset(p);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nb = p.nb, S = p.S, S0 = p.g.S0, frame = p.frame;
  for (int i = tid; i < S0; i += kNbThreads) sCos[i] = cospif(2.0f * (float)i / (float)S0);
  for (int j = tid; j < S; j += kNbThreads) {
    int idx; float w;
    ir_tap(p.g, j, &idx, &w);
    sWin[j] = w;
  }
  if (p.eo_tab) {
    for (int e = tid; e < p.nh * kEoStride; e += kNbThreads) {
      const int n = e / kEoStride, k = e - n * kEoStride;
      sEo[e] = (k <= 32) ? cospif(2.0f * (float)((k * n) % p.g.S0) / (float)p.g.S0) : 0.f;
    }
  }
  for (int e = tid; e < 32 * p.xS; e += kNbThreads) sX[e] = 0.f;   // pads stay zero
  for (int e = tid; e < 32 * p.gS; e += kNbThreads) sG[e] = 0.f;
  __syncthreads();
  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    const int b = tile / p.tiles_per_item;
    const int j0 = (tile - b * p.tiles_per_item) * 32;
    const float* gb = p.grad + (size_t)b * p.N;
    const float* nzb = p.noise ? p.noise + (size_t)b * p.N : nullptr;
    // stage x_j (noise) and gy_j rows
    for (int e = tid; e < 32 * frame; e += kNbThreads) {
      const int jl = e / frame, i = e - jl * frame;
      const long long pp = (long long)(j0 + jl) * frame + i;
      float v = 0.f;
      if (j0 + jl < p.F && pp < p.N) {
        if (nzb) v = nzb[pp];
        else {
          const float4 r = noise4((uint32_t)(pp >> 2), (uint32_t)b, p.seed, p.offset);
          const int u = (int)(pp & 3);
          v = u == 0 ? r.x : (u == 1 ? r.y : (u == 2 ? r.z : r.w));
        }
      }
      sX[jl * p.xS + i] = v;
    }
    for (int e = tid; e < 32 * p.ylen; e += kNbThreads) {
      const int jl = e / p.ylen, n = e - jl * p.ylen;
      const long long t = (long long)(j0 + jl) * frame + n - p.start;
      sG[jl * p.gS + n] = (j0 + jl < p.F && t >= 0 && t < p.N) ? gb[t] : 0.f;
    }
    __syncthreads();
    // dh[m] = sum_i x[i] gy[i + m]; lane = frame, warp loops over tap blocks of 8
    {
      const float* xrow = sX + lane * p.xS;
      const float* grow = sG + lane * p.gS;
      float* hrow = sH + lane * p.hS;
      // 16 taps per round; the 16-value window gy[i + m0 .. i + m0 + 15] slides
      // by one per input sample: 2 LDS feed 16 FFMA (rows are zero padded).
      const int nchunk = (frame + 15) >> 4;
      for (int m0 = warp * 16; m0 < S; m0 += (kNbThreads / 32) * 16) {
        float acc[16], W[16];
#pragma unroll
        for (int c = 0; c < 16; ++c) { acc[c] = 0.f; W[c] = grow[m0 + c]; }
        for (int ch = 0; ch < nchunk; ++ch) {
          const int ib = ch << 4;
#pragma unroll
          for (int u = 0; u < 16; ++u) {
            const float xv = xrow[ib + u];
#pragma unroll
            for (int c = 0; c < 16; ++c) acc[c] = fmaf(xv, W[(c + u) & 15], acc[c]);
            W[u & 15] = grow[ib + u + 1 + m0 + 15];
          }
        }
#pragma unroll
        for (int c = 0; c < 16; ++c)
          if (m0 + c < S) hrow[m0 + c] = acc[c] * sWin[m0 + c];
      }
    }
    __syncthreads();
    // fold taps onto |zero-phase offset| n: dh0[n] = sum_{m: |m - shift| = n (mod S0)} win dh
    // (stored after the S taps of each row), then dM_k = c_k/S0 sum_n cos(2 pi k n/S0) dh0[n]
    {
      float* hrow = sH + lane * p.hS;
      for (int n = warp; n < p.nh; n += kNbThreads / 32) {
        float v = 0.f;
        const int ta = p.g.shift + n, tb = p.g.shift - n;
        if (ta >= 0 && ta < S) v += hrow[ta];
        if (tb >= 0 && tb < S && tb != ta) v += hrow[tb];
        // offsets +-n + S0 alias only when S == S0 and n == S0/2 (tap 0): covered by tb
        hrow[S + n] = v;
      }
    }
    __syncthreads();
    if (p.eo_tab) {
      // nb = 65 (S0 = 128): cos(2 pi (64 - k) n / 128) = (-1)^n cos(2 pi k n / 128), so
      // with E[k] / O[k] the sums over even / odd n, dM_k = c (E + O) and dM_{64-k} =
      // c (E - O): half the multiplies, four columns per broadcast LDS.128.  Warp w
      // owns k = 4 w .. 4 w + 3; k = 32 rides with warp 0.
      const float* d0 = sH + lane * p.hS + S;
      const float invS0 = 1.0f / (float)S0;
      const int k0 = 4 * warp;
      float4 aE = make_float4(0.f, 0.f, 0.f, 0.f), aO = aE;
      float e32 = 0.f;                                  // k = 32: odd n contribute 0
      for (int n = 0; n < p.nh; n += 2) {
        const float de = d0[n];
        const float4 te = *reinterpret_cast<const float4*>(sEo + n * kEoStride + k0);
        aE.x = fmaf(de, te.x, aE.x); aE.y = fmaf(de, te.y, aE.y);
        aE.z = fmaf(de, te.z, aE.z); aE.w = fmaf(de, te.w, aE.w);
        if (warp == 0) e32 = fmaf(de, sEo[n * kEoStride + 32], e32);
        if (n + 1 < p.nh) {
          const float dd = d0[n + 1];
          const float4 to = *reinterpret_cast<const float4*>(sEo + (n + 1) * kEoStride + k0);
          aO.x = fmaf(dd, to.x, aO.x); aO.y = fmaf(dd, to.y, aO.y);
          aO.z = fmaf(dd, to.z, aO.z); aO.w = fmaf(dd, to.w, aO.w);
        }
      }
      if (j0 + lane < p.F) {
        float* dm = p.dmags + ((size_t)b * p.F + j0 + lane) * nb;
        const float E[4] = {aE.x, aE.y, aE.z, aE.w}, O[4] = {aO.x, aO.y, aO.z, aO.w};
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int k = k0 + c;                         // 0 .. 31
          const float ck = (k == 0) ? invS0 : 2.0f * invS0;
          dm[k] = ck * (E[c] + O[c]);
          dm[64 - k] = ck * (E[c] - O[c]);              // k = 0 -> 64 (same end weight)
        }
        if (warp == 0) dm[32] = 2.0f * invS0 * e32;
      }
    } else {
      const float* d0 = sH + lane * p.hS + S;
      const float invS0 = 1.0f / (float)S0;
      for (int k = warp; k < nb; k += kNbThreads / 32) {
        float acc = 0.f;
        int ph = 0;
        for (int n = 0; n < p.nh; ++n) {
          acc = fmaf(d0[n], sCos[ph], acc);
          ph += k; if (ph >= S0) ph -= S0;
        }
        const float ck = (k == 0 || k == nb - 1) ? invS0 : 2.0f * invS0;
        // transposed store through smem row reuse: write straight (32 lanes stride nb)
        if (j0 + lane < p.F)
          p.dmags[((size_t)b * p.F + j0 + lane) * nb + k] = ck * acc;
      }
    }
    __syncthreads();
  }
}

}  // namespace ddsp
