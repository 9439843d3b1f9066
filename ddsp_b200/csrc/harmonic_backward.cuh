// Backward of the harmonic synthesizer (core.py:1048-1111; C4, SURVEY.md 7.3-7,
// 8f-1): the transposes of the fused forward.  With ha = amplitudes *
// harmonic_distribution,
//   audio(t) = sum_k [w0(r) ha_{i,k} + w1(r) ha_{i+1,k}] m_k(t) sin(k phi(t)),
// so for upstream gradient g(t)
//   G0[i,k] = sum_{t in frame i} g(t) w0(r) m_k(t) sin(k phi(t))
//   G1[i,k] = sum_{t in frame i} g(t) w1(r) m_k(t) sin(k phi(t))
//   dL/dha[i,k] = G0[i,k] + G1[i-1,k]   (+ G1[F-1,k] for i = F-1: frame F := F-1)
// harmonic_backward_kernel writes G0 and G1 at every hop that is a multiple of 64,
// with sin(k phi) from the same Reinsch chains as harmonic_v4_kernel instead of one
// sinpif per oscillator: 10 packed instructions per sample pair and harmonic pair,
// plus a 16-value transposing warp reduction per 8 harmonics and 64-sample block.
// The frame records and the phase (tile_phase_base, harmonic_common.cuh) are built
// as in harmonic_v4_kernel.  Every element of G0 / G1 is written (zeros above the
// live count), so the caller needs no memset.  controls_bwd.cuh recombines them.
// The d f0 kernels run only when f0 requires grad.
#pragma once
#include "harmonic_common.cuh"

namespace ddsp {

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

namespace hb {

constexpr int NW = 4;     // warps per CTA
constexpr int NT = NW * 32;

// Frame record of the third forward generation.
struct __align__(16) FrameRec {
  unsigned long long P, A;       // P carries the +2^31 rounding offset
  unsigned long long D;
  int kca, kcb;                  // live counts at r = 0 / r = hop-1; kca < 0: exact path
  float f_lo, f_hi, amp0, amp1;
};
static_assert(sizeof(FrameRec) == 48, "FrameRec must be three 16-byte words");

struct Smem {
  size_t off_tab, off_red, off_warp, warp_stride, total;
};
__host__ __device__ inline Smem smem_layout(int FW) {
  Smem s;
  size_t o = 0;
  s.off_tab = o; o += sizeof(float2) * kSinTab;
  s.off_red = o; o += 16 * NW;
  s.off_warp = o;
  s.warp_stride = sizeof(FrameRec) * FW;
  s.total = s.off_warp + NW * s.warp_stride;
  return s;
}

// Signed chain state of one sample: .x = odd-harmonic chain sin((1+2j) phi), .y =
// even-harmonic chain sin((2+2j) phi).  The forward kernel's chain (v, d) steps as
//   d' = d + na v,  v' = v + d'
// on the angle 2 phi reduced to [-pi/2, pi/2]; where the reduction shifted it by half
// a turn (sigma = -1) the true value is sin((1+2j) phi) = sigma^j v_j.  Here the sign
// rides along: S_j = sigma^j v_j, E_j = sigma^j d_j,
//   E' = sigma E + (sigma na) S,   S' = sigma S + E'.
struct Chain {
  float2 S, Dd;
  float2 sna;      // sigma * na
  float sigma;
};

__device__ __forceinline__ void chain_seed(Chain& c, uint32_t p,
                                           const float2* __restrict__ tab) {
  const uint32_t i = (p + (1u << (31 - kSinTabBits))) >> (32 - kSinTabBits);
  const int r = (int)(p - (i << (32 - kSinTabBits)));
  const float2 t = tab[i & (kSinTab - 1)];
  const float eps = (float)r * 1.4629180792671596e-9f;           // 2 pi / 2^32
  const float e2 = eps * eps;
  const float ce = fmaf(e2, -0.5f, 1.0f);
  const float se = eps * fmaf(e2, -0.16666667f, 1.0f);
  const float s1 = fmaf(t.y, se, t.x * ce);
  const float c1 = fmaf(-t.x, se, t.y * ce);
  const float ss = s1 * s1, cc = c1 * c1;
  const bool flip = ss > cc;                                     // cos(2 phi) < 0
  const float s2 = (s1 + s1) * c1;                               // sin(2 phi)
  const float na = -4.0f * fminf(ss, cc);
  c.S = make_float2(s1, s2);
  c.sigma = flip ? -1.0f : 1.0f;
  c.Dd = make_float2(flip ? 0.0f : s1 + s1, s2);
  c.sna = make_float2(c.sigma * na, c.sigma * na);
}
__device__ __forceinline__ void chain_step(Chain& c) {
  const float2 sg = make_float2(c.sigma, c.sigma);
  c.Dd = ffma2(c.sna, c.S, fmul2(sg, c.Dd));
  c.S = ffma2(sg, c.S, c.Dd);
}

// The first 64-sample block of a frame stores a total, the later ones add to it: the
// lane that stored an element is the only one that touches it again.
__device__ __forceinline__ void put(float* row, int k, float v, bool add) {
  if (add) v += row[k];
  row[k] = v;
}

}  // namespace hb

// Grid (tiles, B), NW warps of FW frames each.  Lane l takes samples r0 + l and
// r0 + l + 32 of each 64-sample block r0 of its warp's frames.  Six CTAs per SM hold
// it at 72 registers, no spills; bounded at four (80 and 88 registers) it ran 3 - 7 %
// slower on an H100 80GB HBM3 at a 700 W power limit.
template <bool WINDOW>
__global__ void __launch_bounds__(hb::NT, 6)
harmonic_backward_kernel(HarmonicParams p, const float* __restrict__ grad,
                         float* __restrict__ G0, float* __restrict__ G1, int FW) {
  using namespace hb;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int K = p.K, F = p.F, hop = p.hop;
  const int FT = FW * NW;
  const Smem L = smem_layout(FW);
  float2* sTab = (float2*)(smem_raw + L.off_tab);
  double* sRedD = (double*)(smem_raw + L.off_red);
  unsigned long long* sWarpTot = (unsigned long long*)(smem_raw + L.off_red) + NW;
  const int b = blockIdx.y;
  const int i0 = blockIdx.x * FT;
  const int nfr = min(FT, F - i0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* f0b = p.f0 + (size_t)b * F;
  FrameRec* sRec = (FrameRec*)(smem_raw + L.off_warp + warp * L.warp_stride);

  {
    double part = 0.0;
    for (int j = tid; j < i0; j += NT) part += (double)f0b[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (lane == 0) sRedD[warp] = part;
  }
  for (int j = tid; j < kSinTab; j += NT) sTab[j] = hcm::g_sincos256[j];
  const float inv_hop = 1.0f / (float)hop;
  const int w0f = warp * FW;
  const int nfw = max(0, min(FW, nfr - w0f));
  unsigned long long excl = 0;
  {
    const int g0 = i0 + w0f;
    const int g = min(g0 + lane, F - 1);
    float f = 0.f;
    if (lane <= nfw && nfw > 0) f = f0b[g];
    const float f_next = __shfl_down_sync(0xffffffffu, f, 1);
    unsigned long long tot = 0, Af = 0, Df = 0;
    if (lane < nfw) {
      const double a0 = (double)f * p.inv_sr;
      const double a1 = (double)f_next * p.inv_sr;
      Af = turns_to_fix64(a0);
      Df = frame_slope_fix64(a0, a1, hop);
      tot = frame_total_fix64(a0, a1, hop);
    }
    const unsigned long long incl = warp_scan_frame_totals(tot, lane);
    excl = incl - tot;
    if (lane == 31) sWarpTot[warp] = incl;
    int kca = -1, kcb = -1;
    if (lane < nfw && f >= 1.0f && f_next >= 1.0f) {
      kca = live_harmonics(f, f_next, 0.0f, K, p.nyquist);
      kcb = live_harmonics(f, f_next, (float)(hop - 1) * inv_hop, K, p.nyquist);
    }
    if (lane < nfw) {
      FrameRec r;
      r.P = 0; r.A = Af; r.D = Df; r.kca = kca; r.kcb = kcb;
      r.f_lo = f; r.f_hi = f_next; r.amp0 = 0.f; r.amp1 = 0.f;
      sRec[lane] = r;
    }
  }
  __syncthreads();
  if (nfw <= 0) return;
  {
    double base_sum = 0.0;
#pragma unroll
    for (int w = 0; w < NW; ++w) base_sum += sRedD[w];
    const double a_tile = (double)f0b[i0] * p.inv_sr;
    const double a_first = (double)f0b[0] * p.inv_sr;
    unsigned long long P0 = tile_phase_base(base_sum, a_first, a_tile, hop, p.inv_sr);
    for (int w = 0; w < warp; ++w) P0 += sWarpTot[w];
    if (lane < nfw) sRec[lane].P = P0 + excl + 0x80000000ull;
  }
  __syncwarp();

  // destination of this lane after warp_reduce16: value index v (bits 4..1 of the
  // lane, MSB first) = 8 * row + harmonic-in-round; odd lanes hold nothing
  const int vsel = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 +
                   ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
  const float* gb = grad + (size_t)b * p.N + (size_t)(i0 + w0f) * hop;
  for (int r0 = 0; r0 < hop; r0 += 64) {
    const bool add = r0 > 0;
    const uint32_t ra = r0 + lane, rb = ra + 32;
    const uint32_t c1a = ra + 1, c2a = (ra * (ra + 1)) >> 1;   // < 2^32 for r < 8192
    const uint32_t c1b = rb + 1, c2b = (rb * (rb + 1)) >> 1;
    const float fra = (float)ra * inv_hop, frb = (float)rb * inv_hop;
    const float w1a = WINDOW ? (0.5f - 0.5f * cospif(fra)) : fra;
    const float w1b = WINDOW ? (0.5f - 0.5f * cospif(frb)) : frb;
    for (int li = 0; li < nfw; ++li) {
      const FrameRec* rec = sRec + li;
      const ulonglong2 PA = *reinterpret_cast<const ulonglong2*>(&rec->P);
      const uint4 Dk = *reinterpret_cast<const uint4*>(&rec->D);
      const float4 fa = *reinterpret_cast<const float4*>(&rec->f_lo);
      const unsigned long long D = ((unsigned long long)Dk.y << 32) | Dk.x;
      const int kc_a = (int)Dk.z, kc_b = (int)Dk.w;
      const uint32_t pa = hcm::phase32(PA.x, PA.y, D, c1a, c2a);
      const uint32_t pb = hcm::phase32(PA.x, PA.y, D, c1b, c2b);
      const float ga = gb[(size_t)li * hop + ra], gv = gb[(size_t)li * hop + rb];
      const float u1a = ga * w1a, u0a = ga - u1a, u1b = gv * w1b, u0b = gv - u1b;
      float* g0row = G0 + ((size_t)b * F + i0 + w0f + li) * K;
      float* g1row = G1 + ((size_t)b * F + i0 + w0f + li) * K;
      if (kc_a < 0) {
        // f0 < 1 Hz: exact per-oscillator masks, one sinpif per oscillator
        for (int kb = 0; kb < K; kb += 8) {
          float val[16];
          uint32_t qa = pa * (uint32_t)kb, qb = pb * (uint32_t)kb;
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            qa += pa; qb += pb;
            const int k = kb + c + 1;
            float sa = sinpif((float)(int)qa * 4.656612873077393e-10f);
            float sb = sinpif((float)(int)qb * 4.656612873077393e-10f);
            if (k > K || !(ref_harmonic_freq(fa.x, fa.y, fra, k) < p.nyquist)) sa = 0.f;
            if (k > K || !(ref_harmonic_freq(fa.x, fa.y, frb, k) < p.nyquist)) sb = 0.f;
            val[c] = u0a * sa + u0b * sb;
            val[8 + c] = u1a * sa + u1b * sb;
          }
          const float total = warp_reduce16(val, lane);
          const int k = kb + (vsel & 7);
          if ((lane & 1) == 0 && k < K) {
            if (vsel < 8) put(g0row, k, total, add); else put(g1row, k, total, add);
          }
        }
        continue;
      }
      // The float32 live count is monotone in r within a frame, so the larger of its
      // values at r = 0 and r = hop - 1 bounds every sample's.
      const bool uniform = kc_a == kc_b;
      const int kmax = max(kc_a, kc_b);
      int ka = kc_a, kbl = kc_a;
      if (!uniform) {
        ka = live_harmonics(fa.x, fa.y, fra, K, p.nyquist);
        kbl = live_harmonics(fa.x, fa.y, frb, K, p.nyquist);
      }
      Chain ca, cb;
      chain_seed(ca, pa, sTab);
      chain_seed(cb, pb, sTab);
      for (int kb = 0; kb < kmax; kb += 8) {
        float val[16];
#pragma unroll
        for (int st = 0; st < 4; ++st) {
          // harmonics kb + 2 st + 1 (.x) and kb + 2 st + 2 (.y)
          float2 wa0 = make_float2(u0a, u0a), wa1 = make_float2(u1a, u1a);
          float2 wb0 = make_float2(u0b, u0b), wb1 = make_float2(u1b, u1b);
          if (!uniform) {
            const int k1 = kb + 2 * st + 1, k2 = k1 + 1;
            if (k1 > ka) { wa0.x = 0.f; wa1.x = 0.f; }
            if (k2 > ka) { wa0.y = 0.f; wa1.y = 0.f; }
            if (k1 > kbl) { wb0.x = 0.f; wb1.x = 0.f; }
            if (k2 > kbl) { wb0.y = 0.f; wb1.y = 0.f; }
          }
          const float2 t0 = ffma2(wb0, cb.S, fmul2(wa0, ca.S));
          const float2 t1 = ffma2(wb1, cb.S, fmul2(wa1, ca.S));
          val[2 * st] = t0.x; val[2 * st + 1] = t0.y;
          val[8 + 2 * st] = t1.x; val[8 + 2 * st + 1] = t1.y;
          chain_step(ca);
          chain_step(cb);
        }
        const float total = warp_reduce16(val, lane);
        const int k = kb + (vsel & 7);
        if ((lane & 1) == 0 && k < K) {
          const float out = (k < kmax) ? total : 0.f;     // harmonic numbers 1..kmax live
          if (vsel < 8) put(g0row, k, out, add); else put(g1row, k, out, add);
        }
      }
      if (!add) {
        for (int k = min(K, (kmax + 7) & ~7) + lane; k < K; k += 32) {
          g0row[k] = 0.f;
          g1row[k] = 0.f;
        }
      }
    }
  }
}

// Frames per warp: 16 64-sample blocks, halved while the batch has fewer than 8 CTAs
// per SM, down to 4 blocks or one frame (16 .. 4 frames at hop 64).
inline int launch_harmonic_backward(HarmonicParams p, const float* grad, float* g0,
                                    float* g1, cudaStream_t st) {
  using namespace hb;
  const int m = p.hop / 64;
  const long long want_ctas = 8ll * num_sms();
  int FW = std::max(1, 16 / m);
  while (FW > 1 && FW * m > 4 &&
         (long long)p.B * ((p.F + FW * NW - 1) / (FW * NW)) < want_ctas)
    FW >>= 1;
  FW = std::max(1, std::min(FW, (p.F + NW - 1) / NW));
  dim3 grid((p.F + FW * NW - 1) / (FW * NW), p.B);
  auto kern = p.amp_method == DDSP_B200_AMP_WINDOW ? harmonic_backward_kernel<true>
                                                   : harmonic_backward_kernel<false>;
  return launch("harmonic_backward", kern, grid, NT, smem_layout(FW).total, st, p, grad,
                g0, g1, FW);
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
