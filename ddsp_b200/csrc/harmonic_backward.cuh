// Backward of the harmonic synthesizer (core.py:1048-1111; C4, SURVEY.md 7.3-7,
// 8f-1): the transposes of the fused forward.  With ha = amplitudes *
// harmonic_distribution,
//   audio(t) = sum_k [w0(r) ha_{i,k} + w1(r) ha_{i+1,k}] m_k(t) sin(k phi(t)),
// so for upstream gradient g(t)
//   G0[i,k] = sum_{t in frame i} g(t) w0(r) m_k(t) sin(k phi(t))
//   G1[i,k] = sum_{t in frame i} g(t) w1(r) m_k(t) sin(k phi(t))
//   dL/dha[i,k] = G0[i,k] + G1[i-1,k]   (+ G1[F-1,k] for i = F-1: frame F := F-1)
// harmonic_backward_kernel writes G0 and G1 at hops other than 64 (hop 64:
// harmonic_bwd2.cuh): grid (tiles, B), 256 threads, one warp per frame pass,
// lane = samples r and r + 32, one sinpif per oscillator.  controls_bwd.cuh
// recombines them.  The d f0 kernels run only when f0 requires grad.
#pragma once
#include "harmonic_common.cuh"

namespace ddsp {

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
    unsigned long long P = tile_phase_base(fsum, a_first, a_tile, hop, p.inv_sr);
    for (int base = 0; base < nfr; base += 32) {
      const int j = base + lane;
      unsigned long long tot = 0;
      if (j < nfr) {
        const double a0 = (double)sF0[j] * p.inv_sr;
        const double a1 = (double)sF0[j + 1] * p.inv_sr;
        sA[j] = turns_to_fix64(a0);
        sD[j] = frame_slope_fix64(a0, a1, hop);
        tot = frame_total_fix64(a0, a1, hop);
      }
      const unsigned long long incl = warp_scan_frame_totals(tot, lane);
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
// d f0 of core.harmonic_synthesis.  With phi in turns,
//   d audio(t) / d phi(t) = 2 pi sum_k k a_k(t) m_k(t) cos(2 pi k phi(t)),
//   c(t) = g(t) * that;  sr * phi(t) is a linear function of the frame values f0[j]
// (the transpose of resample('linear') followed by cumsum), which for a sample at
// offset r of frame i gives weights alpha = (hop+1)/2 and beta = (hop-1)/2 for the
// completed frames and p0(r) = (r+1) - r(r+1)/(2 hop), p1(r) = r(r+1)/(2 hop) for the
// current one.  Pass 1 (this kernel) reduces per frame
//   S_i = sum_r c,  Q0_i = sum_r c p0(r),  Q1_i = sum_r c p1(r);
// pass 2 (harmonic_df0_finalize) is the frame-rate suffix sum.
// Controls here are the synthesizer controls (amplitudes, normalised
// harmonic_distribution).  One thread per sample, one sincospif per oscillator.
// ---------------------------------------------------------------------------
constexpr int kDf0Threads = 256;
constexpr int kDf0Warps = kDf0Threads / 32;

template <bool WINDOW>
__global__ void __launch_bounds__(kDf0Threads)
harmonic_df0_kernel(HarmonicParams p, const float* __restrict__ grad,
                    float* __restrict__ sq /* [B, F, 3] */) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int FT = p.FT, Kp = p.Kp, K = p.K, F = p.F, hop = p.hop;
  unsigned long long* sP = reinterpret_cast<unsigned long long*>(smem_raw);
  unsigned long long* sA = sP + FT;
  unsigned long long* sD = sA + FT;
  unsigned long long* sRed = sD + FT;
  float* sF0 = reinterpret_cast<float*>(sRed + 8);
  float* sAmp = sF0 + (FT + 1);
  float* sAcc = sAmp + (FT + 1);                 // [kDf0Warps][FT][3]
  const int n_acc = kDf0Warps * 3 * FT;
  float* sX = sAcc + n_acc + (n_acc & 1);
  const int b = blockIdx.y;
  const int i0 = blockIdx.x * FT;
  const int nfr = min(FT, F - i0);
  const int tid = threadIdx.x;
  const float* f0b = p.f0 + (size_t)b * F;
  const float* ampb = p.amps + (size_t)b * F;

  unsigned long long part = 0;
  for (int j = tid; j < i0; j += kDf0Threads) {
    double a0 = (double)f0b[j] * p.inv_sr;
    double a1 = (double)f0b[min(j + 1, F - 1)] * p.inv_sr;
    part += frame_total_fix64(a0, a1, hop);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if ((tid & 31) == 0) sRed[tid >> 5] = part;
  for (int j = tid; j <= nfr; j += kDf0Threads) {
    int g = min(i0 + j, F - 1);
    sF0[j] = f0b[g];
    sAmp[j] = ampb[g];
  }
  for (int j = tid; j < n_acc; j += kDf0Threads) sAcc[j] = 0.f;
  if (p.hd != nullptr) {
    const float* hdb = p.hd + ((size_t)b * F + i0) * K;
    const int rows_in = min(nfr + 1, F - i0);
    for (int idx = tid; idx < rows_in * K; idx += kDf0Threads) {
      int r = idx / K, c = idx - r * K;
      sX[r * Kp + c] = hdb[idx];
    }
    if (rows_in < nfr + 1) {
      for (int c = tid; c < K; c += kDf0Threads)
        sX[nfr * Kp + c] = hdb[(size_t)(nfr - 1) * K + c];
    }
  } else {
    for (int j = tid; j <= nfr; j += kDf0Threads) sX[j * Kp] = 1.0f;
  }
  __syncthreads();
  if (tid == 0) {
    unsigned long long P = 0;
    for (int w = 0; w < kDf0Threads / 32; ++w) P += sRed[w];
    for (int j = 0; j < nfr; ++j) {
      double a0 = (double)sF0[j] * p.inv_sr;
      double a1 = (double)sF0[j + 1] * p.inv_sr;
      sP[j] = P;
      sA[j] = turns_to_fix64(a0);
      sD[j] = frame_slope_fix64(a0, a1, hop);
      P += frame_total_fix64(a0, a1, hop);
    }
  }
  __syncthreads();

  const int n_tile = nfr * hop;
  const float inv_hop = 1.0f / (float)hop;
  const float* gb = grad + (size_t)b * p.N + (size_t)i0 * hop;
  const int n_iter = (n_tile + kDf0Threads - 1) / kDf0Threads;
  const int lane = tid & 31;
  float* acc_w = sAcc + (tid >> 5) * 3 * FT;
  int cur = -1;                        // lane 0: the frame rc / rq0 / rq1 belong to
  float rc = 0.f, rq0 = 0.f, rq1 = 0.f;
  for (int it = 0; it < n_iter; ++it) {
    const int lt = it * kDf0Threads + tid;
    const bool ok = lt < n_tile;
    const int li = ok ? lt / hop : -1;
    float c = 0.f, q0 = 0.f, q1 = 0.f;
    if (ok) {
      const int r = lt - li * hop;
      const float frac = (float)r * inv_hop;
      const float f_lo = sF0[li], f_hi = sF0[li + 1];
      unsigned long long ph = sP[li] + (unsigned long long)(r + 1) * sA[li] +
          (unsigned long long)(((long long)r * (r + 1)) >> 1) * sD[li];
      const uint32_t p32 = (uint32_t)((ph + 0x80000000ull) >> 32);
      float w1 = WINDOW ? (0.5f - 0.5f * cospif(frac)) : frac;
      const float w0 = (1.0f - w1) * sAmp[li];
      w1 *= sAmp[li + 1];
      const float* x0 = sX + li * Kp;
      const float* x1 = x0 + Kp;
      const bool monotone = (f_lo >= 1.0f) && (f_hi >= 1.0f);
      const int klive = monotone ? live_harmonics(f_lo, f_hi, frac, K, p.nyquist) : K;
      float acc = 0.f;
      uint32_t pk = 0;
      for (int k = 1; k <= klive; ++k) {
        pk += p32;
        float a = x0[k - 1] * w0 + x1[k - 1] * w1;
        if (!monotone && !(ref_harmonic_freq(f_lo, f_hi, frac, k) < p.nyquist)) a = 0.f;
        acc = fmaf(a * (float)k, cospif((float)(int)pk * 4.656612873077393e-10f), acc);
      }
      c = gb[lt] * 6.283185307179586f * acc;
      const float tri = (float)r * (float)(r + 1) * (0.5f * inv_hop);
      q1 = c * tri;
      q0 = c * ((float)(r + 1) - tri);
    }
    // per-frame reduction in a fixed order, so d f0 is bit-reproducible: a warp's
    // samples are consecutive, so its frames ascend (one frame when hop is a multiple
    // of 32); each is reduced by shuffles and added to lane 0's running sums, which
    // go to the warp's own row of sAcc when the frame changes.  No atomics.
    const unsigned full = 0xffffffffu;
    const int first = __shfl_sync(full, li, 0);
    if (first >= 0) {
      const int last = __reduce_max_sync(full, li);
      for (int fr = first; fr <= last; ++fr) {
        float sc = li == fr ? c : 0.f, s0 = li == fr ? q0 : 0.f, s1 = li == fr ? q1 : 0.f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          sc += __shfl_xor_sync(full, sc, o);
          s0 += __shfl_xor_sync(full, s0, o);
          s1 += __shfl_xor_sync(full, s1, o);
        }
        if (lane == 0) {
          if (fr != cur) {
            if (cur >= 0) {
              acc_w[3 * cur + 0] = rc;
              acc_w[3 * cur + 1] = rq0;
              acc_w[3 * cur + 2] = rq1;
            }
            cur = fr;
            rc = rq0 = rq1 = 0.f;
          }
          rc += sc;
          rq0 += s0;
          rq1 += s1;
        }
      }
    }
  }
  if (lane == 0 && cur >= 0) {
    acc_w[3 * cur + 0] = rc;
    acc_w[3 * cur + 1] = rq0;
    acc_w[3 * cur + 2] = rq1;
  }
  __syncthreads();
  for (int j = tid; j < 3 * nfr; j += kDf0Threads) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kDf0Warps; ++w) s += sAcc[w * 3 * FT + j];
    sq[((size_t)b * F + i0) * 3 + j] = s;
  }
}

inline size_t harmonic_df0_smem(int FT, int Kp) {
  return sizeof(unsigned long long) * (3 * (size_t)FT + 8) +
         sizeof(float) * (2 * (size_t)(FT + 1) + kDf0Warps * 3 * (size_t)FT + 1 +
                          (size_t)(FT + 1) * Kp);
}

// pass 2: one thread per batch item walks the frames backwards.
//   d f0[j] = inv_sr [ (alpha + beta [j>=1]) Suf_j + beta [j>=1] S_j + Q0_j
//                      + Q1_{j-1} [j>=1] + Q1_{F-1} [j == F-1] ],  Suf_j = sum_{i>j} S_i
__global__ void __launch_bounds__(128)
harmonic_df0_finalize(const float* __restrict__ sq, float* __restrict__ d_f0, int B,
                      int F, int hop, float inv_sr) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float alpha = 0.5f * (float)(hop + 1), beta = 0.5f * (float)(hop - 1);
  const float* s = sq + (size_t)b * F * 3;
  float* out = d_f0 + (size_t)b * F;
  double suf = 0.0;
  for (int j = F - 1; j >= 0; --j) {
    const float S = s[3 * j], Q0 = s[3 * j + 1];
    double v = (double)(alpha + (j >= 1 ? beta : 0.f)) * suf + (double)Q0;
    if (j >= 1) v += (double)beta * S + (double)s[3 * (j - 1) + 2];
    if (j == F - 1) v += (double)s[3 * j + 2];
    out[j] = (float)(v * (double)inv_sr);
    suf += (double)S;
  }
}

}  // namespace ddsp
