// Backward kernels of the two synthesizers (C4: decoder forward + backward
// through SpectralLoss; SURVEY.md 7.3-7, 8f-1).  The reference gets these from
// TF autodiff through every op of core.py; here they are the transposes of the
// fused forward kernels.
//
// Harmonic (core.py:1048-1111).  With ha = amplitudes * harmonic_distribution,
//   audio(t) = sum_k [w0(r) ha_{i,k} + w1(r) ha_{i+1,k}] m_k(t) sin(k phi(t)),
// so for upstream gradient g(t)
//   G0[i,k] = sum_{t in frame i} g(t) w0(r) m_k(t) sin(k phi(t))
//   G1[i,k] = sum_{t in frame i} g(t) w1(r) m_k(t) sin(k phi(t))
//   dL/dha[i,k] = G0[i,k] + G1[i-1,k]   (+ G1[F-1,k] for i = F-1: frame F := F-1)
// The kernel writes G0 and G1; the (cheap, frame-rate) recombination into
// d amplitudes / d harmonic_distribution happens in the host wrapper.
// d f0 (through the phase) is not built: in ae.gin f0 comes from the data
// (training/preprocessing.py:74-91).
//
// FilteredNoise (core.py:1534-1565, 1382-1473).  The output is linear in the
// magnitudes:  dL/dh_j[m] = sum_i x_j[i] gy_j[i + m],  gy_j[n] = g[frame j + n - start],
//   dL/dM_{j,k} = (c_k / S0) sum_m win[m] cos(2 pi k (m - shift) / S0) dL/dh_j[m].
#pragma once
#include "harmonic_common.cuh"
#include "noise_fused.cuh"

namespace ddsp {

// ---------------------------------------------------------------------------
// Harmonic backward.  Same tiling as the first fused forward kernel (grid (tiles, B), 256
// threads, one warp per frame pass, lane = samples r and r + 32).
// ---------------------------------------------------------------------------
constexpr int kHbThreads = 256;

// Sum 16 per-lane partials over the warp: afterwards lane l (even l) holds the
// total of value index ((l >> 1) & 15) in val[0].  31 shuffles for 16 values.
__device__ __forceinline__ float warp_reduce16(float (&val)[16], int lane) {
#pragma unroll
  for (int half = 8, bit = 16; half >= 1; half >>= 1, bit >>= 1) {
    const bool upper = (lane & bit) != 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (i < half) {
        const float send = upper ? val[i] : val[i + half];
        const float keep = upper ? val[i + half] : val[i];
        val[i] = keep + __shfl_xor_sync(0xffffffffu, send, bit);
      }
    }
  }
  // bits 16,8,4,2 selected the value; lanes l and l^1 hold two halves of it
  return val[0] + __shfl_xor_sync(0xffffffffu, val[0], 1);
}

template <bool WINDOW>
__global__ void __launch_bounds__(kHbThreads)
harmonic_backward_kernel(HarmonicParams p, const float* __restrict__ grad,
                         float* __restrict__ G0, float* __restrict__ G1) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int FT = p.FT, K = p.K, F = p.F, hop = p.hop;
  // smem: P, A, D (u64 x FT), red (double x 8), tab, f0, kc, w
  unsigned long long* sP = (unsigned long long*)smem_raw;
  unsigned long long* sA = sP + FT;
  unsigned long long* sD = sA + FT;
  double* sRedD = (double*)(sD + FT);
  float2* sTab = (float2*)(sRedD + 8);
  float* sF0 = (float*)(sTab + kSinTab);
  int* sKc = (int*)(sF0 + FT + 2);
  float* sW = (float*)(sKc + 2 * FT);

  const int b = blockIdx.y;
  const int i0 = blockIdx.x * FT;
  const int nfr = min(FT, F - i0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* f0b = p.f0 + (size_t)b * F;

  double part = 0.0;
  for (int j = tid; j < i0; j += kHbThreads) part += (double)f0b[j];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if (lane == 0) sRedD[warp] = part;
  for (int j = tid; j <= nfr; j += kHbThreads) sF0[j] = f0b[min(i0 + j, F - 1)];
  for (int j = tid; j < kSinTab; j += kHbThreads) {
    float s, c;
    sincospif(2.0f * (float)j / (float)kSinTab, &s, &c);
    sTab[j] = make_float2(s, c);
  }
  {
    const float inv_hop = 1.0f / (float)hop;
    for (int r = tid; r < hop; r += kHbThreads) {
      const float frac = (float)r * inv_hop;
      sW[r] = WINDOW ? (0.5f - 0.5f * cospif(frac)) : frac;
    }
  }
  __syncthreads();
  if (warp == 0) {
    double fsum = 0.0;
    for (int w = 0; w < kHbThreads / 32; ++w) fsum += sRedD[w];
    const double a_first = (double)f0b[0] * p.inv_sr;
    const double a_tile = (double)sF0[0] * p.inv_sr;
    unsigned long long P = turns_to_fix64(
        (double)hop * (fsum * p.inv_sr) + 0.5 * (hop - 1) * (a_tile - a_first));
    for (int base = 0; base < nfr; base += 32) {
      const int j = base + lane;
      unsigned long long tot = 0;
      if (j < nfr) {
        const double a0 = (double)sF0[j] * p.inv_sr;
        const double a1 = (double)sF0[j + 1] * p.inv_sr;
        sA[j] = turns_to_fix64(a0);
        sD[j] = turns_to_fix64((a1 - a0) / (double)hop);
        tot = turns_to_fix64((double)hop * a0 + (a1 - a0) * (0.5 * (hop - 1)));
      }
      unsigned long long incl = tot;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long up = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += up;
      }
      if (j < nfr) sP[j] = P + (incl - tot);
      P += __shfl_sync(0xffffffffu, incl, 31);
    }
  }
  for (int j = tid; j < nfr; j += kHbThreads) {
    const float f_lo = sF0[j], f_hi = sF0[j + 1];
    // any f0 < 1 Hz frame: treat all harmonics as live and mask per sample
    sKc[2 * j] = (f_lo >= 1.0f && f_hi >= 1.0f)
                     ? live_harmonics(f_lo, f_hi, 0.0f, K, p.nyquist) : -1;
    sKc[2 * j + 1] = (f_lo >= 1.0f && f_hi >= 1.0f)
                         ? live_harmonics(f_lo, f_hi, (float)(hop - 1) * (1.0f / (float)hop),
                                          K, p.nyquist) : -1;
  }
  __syncthreads();

  const float inv_hop = 1.0f / (float)hop;
  const float* gb = grad + (size_t)b * p.N + (size_t)i0 * hop;
  for (int li = warp; li < nfr; li += kHbThreads / 32) {
    const float f_lo = sF0[li], f_hi = sF0[li + 1];
    const int kc_a = sKc[2 * li], kc_b = sKc[2 * li + 1];
    float* g0row = G0 + ((size_t)b * F + i0 + li) * K;
    float* g1row = G1 + ((size_t)b * F + i0 + li) * K;
    const int kmax_frame = (kc_a < 0) ? K : max(kc_a, kc_b);
    for (int kb = 0; kb < kmax_frame; kb += 8) {     // 8 harmonics per round
      float tot0[8], tot1[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) tot0[c] = tot1[c] = 0.f;
      for (int r0 = 0; r0 < hop; r0 += 64) {
        const int ra = r0 + lane, rb = ra + 32;
        const unsigned long long pha = sP[li] + (unsigned long long)(ra + 1) * sA[li] +
            (unsigned long long)(((long long)ra * (ra + 1)) >> 1) * sD[li];
        const unsigned long long phb = sP[li] + (unsigned long long)(rb + 1) * sA[li] +
            (unsigned long long)(((long long)rb * (rb + 1)) >> 1) * sD[li];
        const uint32_t pa = (uint32_t)((pha + 0x80000000ull) >> 32);
        const uint32_t pb = (uint32_t)((phb + 0x80000000ull) >> 32);
        const float ga = gb[(size_t)li * hop + ra], gbv = gb[(size_t)li * hop + rb];
        const float w1a = sW[ra], w1b = sW[rb];
        int ka, kbb;
        if (kc_a >= 0 && kc_a == kc_b) {
          ka = kbb = kc_a;
        } else if (kc_a >= 0) {
          ka = live_harmonics(f_lo, f_hi, (float)ra * inv_hop, K, p.nyquist);
          kbb = live_harmonics(f_lo, f_hi, (float)rb * inv_hop, K, p.nyquist);
        } else {
          ka = kbb = K;       // exact per-oscillator mask below
        }
        // direct evaluation: one sinpif per oscillator (8 per round per sample)
        uint32_t qa = pa * (uint32_t)kb, qb = pb * (uint32_t)kb;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          qa += pa; qb += pb;
          const int k = kb + c + 1;
          float sa = sinpif((float)(int)qa * 4.656612873077393e-10f);
          float sb = sinpif((float)(int)qb * 4.656612873077393e-10f);
          bool la = k <= ka, lb = k <= kbb;
          if (kc_a < 0) {
            la = ref_harmonic_freq(f_lo, f_hi, (float)ra * inv_hop, k) < p.nyquist;
            lb = ref_harmonic_freq(f_lo, f_hi, (float)rb * inv_hop, k) < p.nyquist;
          }
          if (!la || k > K) sa = 0.f;
          if (!lb || k > K) sb = 0.f;
          const float pa_ = ga * sa, pb_ = gbv * sb;
          tot0[c] += pa_ * (1.0f - w1a) + pb_ * (1.0f - w1b);
          tot1[c] += pa_ * w1a + pb_ * w1b;
        }
      }
      float val[16];
#pragma unroll
      for (int c = 0; c < 8; ++c) { val[c] = tot0[c]; val[8 + c] = tot1[c]; }
      const float total = warp_reduce16(val, lane);
      if ((lane & 1) == 0) {
        // value index v = bits (lane>>1)&15 in halving order: bit 16 of lane picked
        // the upper half first, i.e. v's MSB = lane bit 4, ... LSB = lane bit 1.
        const int v = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 +
                      ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
        const int k = kb + (v & 7);
        if (k < K) {
          if (v < 8) g0row[k] = total; else g1row[k] = total;
        }
      }
    }
  }
}

inline size_t harmonic_backward_smem(int FT, int hop) {
  return sizeof(unsigned long long) * 3 * FT + sizeof(double) * 8 +
         sizeof(float2) * kSinTab + sizeof(float) * (FT + 2) + sizeof(int) * 2 * FT +
         sizeof(float) * hop + 16;
}

// ---------------------------------------------------------------------------
// Filtered-noise backward: d magnitudes.  Lane = frame, tile = 32 frames.
// ---------------------------------------------------------------------------
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
