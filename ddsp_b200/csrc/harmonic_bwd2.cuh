// Harmonic backward for hop == 64: the transposes
//   G0[i,k] = sum_{t in frame i} g(t) w0(r) m_k(t) sin(k phi(t)),   G1 with w1
// (harmonic_backward.cuh) with sin(k phi) from the SAME Reinsch chains as
// harmonic_v4_kernel instead of one sinpif per oscillator: 10 packed instructions
// per sample pair and harmonic pair, plus a 16-value transposing warp reduction
// per 8 harmonics.  The frame records and the phase (tile_phase_base,
// harmonic_common.cuh) are built as in harmonic_v4_kernel.  Every element of
// G0 / G1 is written (zeros above the live count), so the caller needs no memset.
#pragma once
#include "harmonic_backward.cuh"

namespace ddsp {
namespace hb2 {

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

template <bool WINDOW>
__global__ void __launch_bounds__(NT, 4)
harmonic_backward2_kernel(HarmonicParams p, const float* __restrict__ grad,
                          float* __restrict__ G0, float* __restrict__ G1, int FW) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int hop = 64;
  const int K = p.K, F = p.F;
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

  const uint32_t ra = lane, rb = lane + 32;
  const uint32_t c1a = ra + 1, c2a = (ra * (ra + 1)) >> 1;
  const uint32_t c1b = rb + 1, c2b = (rb * (rb + 1)) >> 1;
  const float fra = (float)ra * inv_hop, frb = (float)rb * inv_hop;
  const float w1a = WINDOW ? (0.5f - 0.5f * cospif(fra)) : fra;
  const float w1b = WINDOW ? (0.5f - 0.5f * cospif(frb)) : frb;
  // destination of this lane after warp_reduce16: value index v (bits 4..1 of the
  // lane, MSB first) = 8 * row + harmonic-in-round; odd lanes hold nothing
  const int vsel = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 +
                   ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
  const float* gb = grad + (size_t)b * p.N + (size_t)(i0 + w0f) * hop;
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
    int k_done = 0;          // harmonics [0, k_done) of the rows are written
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
          if (vsel < 8) g0row[k] = total; else g1row[k] = total;
        }
      }
      k_done = K;
    } else {
      const bool uniform = kc_a == kc_b;
      int ka = kc_a, kbl = kc_a, kmax = kc_a;
      if (!uniform) {
        ka = live_harmonics(fa.x, fa.y, fra, K, p.nyquist);
        kbl = live_harmonics(fa.x, fa.y, frb, K, p.nyquist);
        kmax = __reduce_max_sync(0xffffffffu, max(ka, kbl));
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
          if (vsel < 8) g0row[k] = out; else g1row[k] = out;
        }
      }
      k_done = min(K, (kmax + 7) & ~7);
    }
    for (int k = k_done + lane; k < K; k += 32) {
      g0row[k] = 0.f;
      g1row[k] = 0.f;
    }
  }
}

}  // namespace hb2

inline bool harmonic_backward2_supported(const HarmonicParams& p) {
  return p.hop == 64 && p.B <= 65535;
}

inline int launch_harmonic_backward2(HarmonicParams p, const float* grad, float* g0,
                                     float* g1, cudaStream_t st) {
  using namespace hb2;
  int FW = 16;
  const long long want_ctas = 8ll * num_sms();
  while (FW > 4 && (long long)p.B * ((p.F + FW * NW - 1) / (FW * NW)) < want_ctas) FW >>= 1;
  FW = std::max(1, std::min(FW, (p.F + NW - 1) / NW));
  const size_t smem = smem_layout(FW).total;
  dim3 grid((p.F + FW * NW - 1) / (FW * NW), p.B);
  auto kern = p.amp_method == DDSP_B200_AMP_WINDOW ? harmonic_backward2_kernel<true>
                                                   : harmonic_backward2_kernel<false>;
  return launch("harmonic_backward(v2)", kern, grid, NT, smem, st, p, grad, g0, g1, FW);
}

}  // namespace ddsp
