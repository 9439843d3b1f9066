// Frame-rate oscillator bank with PER-SINUSOID frequencies - the fused form of
//   resample(frequencies, N) + resample(amplitudes, N, amp_method) +
//   core.oscillator_bank(...)                      (core.py:573-642, 911-962)
// for synths.Sinusoidal.get_signal (synths.py:305-323) and for
// core.harmonic_synthesis with harmonic_shifts (core.py:1084-1093, where
// f_k = f0 * k * (1 + shift_k) is no longer an integer multiple of one phase).
// The [B, N, K] envelopes the reference materialises never exist.
//
// Per sinusoid k the frequency is piecewise linear in time (v1 bilinear, frame
// F := frame F-1), so inside frame i the inclusive phase sum has the same closed
// form as the harmonic kernel, with per-k tables:
//   phi_k(i*hop + r) = P_ik + (r+1) a_ik + (a_{i+1,k} - a_ik)/hop * r(r+1)/2,
//   a = f/sr in turns, P_ik = sum_{j<i} [hop a_jk + (a_{j+1,k} - a_jk)(hop-1)/2]
// kept as 64-bit fixed-point turns (wrapping adds are exact).  Three passes:
//   1. per (b, tile, k) total of the frame sums         (grid n_tiles x B)
//   2. exclusive scan over the tiles per (b, k)         (oscbank_scan_chunks)
//   3. tables P/A/D for the tile in shared memory, then one thread per sample
//      loops over k: phase -> sinpif, Nyquist mask on the reference's float32
//      envelope (lo + (hi - lo) * frac, no FMA), two-row amplitude interpolation.
#pragma once
#include "harmonic_common.cuh"
#include "oscbank.cuh"

namespace ddsp {

constexpr int kSfThreads = 128;

// pass 1.  sums[b, tile, k] = sum of the frame totals of the tile's frames.
__global__ void __launch_bounds__(kSfThreads)
sinus_tile_sums(const float* __restrict__ f, unsigned long long* __restrict__ sums,
                int F, int K, int hop, int FT, int n_tiles, double inv_sr) {
  const int b = blockIdx.y, tile = blockIdx.x;
  const int i0 = tile * FT, i1 = min(F, i0 + FT);
  for (int k = threadIdx.x; k < K; k += kSfThreads) {
    const float* fp = f + ((size_t)b * F) * K + k;
    unsigned long long acc = 0;
    float cur = fp[(size_t)i0 * K];
    for (int i = i0; i < i1; ++i) {
      const float nxt = fp[(size_t)min(i + 1, F - 1) * K];
      acc += frame_total_fix64((double)cur * inv_sr, (double)nxt * inv_sr, hop);
      cur = nxt;
    }
    sums[((size_t)b * n_tiles + tile) * K + k] = acc;
  }
}

struct SfSmem {
  size_t off_P, off_A, off_D, off_f, off_a, total;
};
__host__ __device__ inline SfSmem sf_smem(int FT, int K) {
  SfSmem s;
  size_t o = 0;
  s.off_P = o; o += sizeof(unsigned long long) * (size_t)FT * K;
  s.off_A = o; o += sizeof(unsigned long long) * (size_t)FT * K;
  s.off_D = o; o += sizeof(unsigned long long) * (size_t)FT * K;
  s.off_f = o; o += sizeof(float) * (size_t)(FT + 1) * K;
  s.off_a = o; o += sizeof(float) * (size_t)(FT + 1) * K;
  s.total = o;
  return s;
}

// pass 3.
template <bool WINDOW>
__global__ void __launch_bounds__(kSfThreads)
sinus_apply(const float* __restrict__ f, const float* __restrict__ a,
            const unsigned long long* __restrict__ offs, float* __restrict__ out,
            int F, int K, int N, int hop, int FT, int n_tiles, double inv_sr,
            float nyquist, int accumulate) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const SfSmem L = sf_smem(FT, K);
  unsigned long long* sP = (unsigned long long*)(smem_raw + L.off_P);
  unsigned long long* sA = (unsigned long long*)(smem_raw + L.off_A);
  unsigned long long* sD = (unsigned long long*)(smem_raw + L.off_D);
  float* sF = (float*)(smem_raw + L.off_f);
  float* sAm = (float*)(smem_raw + L.off_a);
  const int b = blockIdx.y, tile = blockIdx.x;
  const int i0 = tile * FT, nfr = min(FT, F - i0);
  const int tid = threadIdx.x;

  // rows i0 .. i0 + nfr (frame F := frame F-1)
  for (int idx = tid; idx < (nfr + 1) * K; idx += kSfThreads) {
    const int r = idx / K, k = idx - r * K;
    const size_t g = ((size_t)b * F + min(i0 + r, F - 1)) * K + k;
    sF[idx] = f[g];
    sAm[idx] = a[g];
  }
  __syncthreads();
  // per-k tables: a running wrapping sum over the tile's frames
  for (int k = tid; k < K; k += kSfThreads) {
    unsigned long long P = offs[((size_t)b * n_tiles + tile) * K + k];
    for (int j = 0; j < nfr; ++j) {
      const float f_lo = sF[j * K + k], f_hi = sF[(j + 1) * K + k];
      const double a0 = (double)f_lo * inv_sr, a1 = (double)f_hi * inv_sr;
      sP[j * K + k] = P + 0x80000000ull;          // rounding offset for the top 32 bits
      sA[j * K + k] = turns_to_fix64(a0);
      sD[j * K + k] = frame_slope_fix64(a0, a1, hop);
      P += frame_total_fix64(a0, a1, hop);
    }
  }
  __syncthreads();

  const float inv_hop = 1.0f / (float)hop;
  float* outb = out + (size_t)b * N + (size_t)i0 * hop;
  const int n_tile = nfr * hop;
  for (int lt = tid; lt < n_tile; lt += kSfThreads) {
    const int li = lt / hop, r = lt - li * hop;
    const float frac = (float)r * inv_hop;
    const float w1 = WINDOW ? (0.5f - 0.5f * cospif(frac)) : frac;
    const float w0 = 1.0f - w1;
    const unsigned long long c1 = (unsigned long long)(r + 1);
    const unsigned long long c2 = (unsigned long long)(((long long)r * (r + 1)) >> 1);
    const unsigned long long* P = sP + li * K;
    const unsigned long long* A = sA + li * K;
    const unsigned long long* D = sD + li * K;
    const float* f0r = sF + li * K;
    const float* f1r = f0r + K;
    const float* a0r = sAm + li * K;
    const float* a1r = a0r + K;
    float acc = 0.f;
    for (int k = 0; k < K; ++k) {
      const unsigned long long ph = P[k] + c1 * A[k] + c2 * D[k];
      const float s = sinpif((float)(int)(uint32_t)(ph >> 32) * 4.656612873077393e-10f);
      const float lo = f0r[k], hi = f1r[k];
      const float fe = __fadd_rn(lo, __fmul_rn(__fsub_rn(hi, lo), frac));   // core.py:617-620
      float amp = fmaf(a1r[k], w1, a0r[k] * w0);
      if (fe >= nyquist) amp = 0.f;                                         // core.py:888-890
      acc = fmaf(amp, s, acc);
    }
    if (accumulate) acc += outb[lt];
    outb[lt] = acc;
  }
}

// ---------------------------------------------------------------------------
// Backward.  For one (b, k), upstream gradient g, s = sin 2 pi phi, m the
// forward's own float32 Nyquist decision and c = g m amp 2 pi cos 2 pi phi:
//   G0_i = sum_{t in i} g m s w0(r),  G1_i = sum_{t in i} g m s w1(r)
//   d A_i = G0_i + G1_{i-1}  (+ G1_{F-1} on the last frame, frame F := F-1)
// and with p1(r) = r(r+1)/(2 hop), p0(r) = (r+1) - p1(r), S_i = sum c,
// Q0_i = sum c p0, Q1_i = sum c p1 (sr phi is linear in the frame frequencies:
// alpha = (hop+1)/2, beta = (hop-1)/2 weigh the completed frames):
//   sr d f_j = (alpha + beta [j>=1]) sum_{i>j} S_i + beta [j>=1] S_j + Q0_j
//              + Q1_{j-1} [j>=1] + Q1_{F-1} [j == F-1].
// Two passes after the forward's passes 1-2 (the tile phase offsets):
//   4. sinus_bwd_frames: a CTA owns 32 consecutive (b, i, k) (one per lane) and
//      splits the frame's hop samples into kSbWarps contiguous segments, one per
//      warp.  A segment starts from the closed-form fixed-point phase and steps
//      it by exact wrapping adds, so every phase is bit-identical to the
//      forward's.  The warps' float partials are summed in warp order through
//      shared memory: G0, G1 (and S, Q0, Q1) per (b, i, k) are written once.
//   5. sinus_bwd_finalize: d A, and the frame-rate suffix sum of S and d f in
//      double, per (b, k) over frame chunks combined in a fixed order.
// No atomics, no memset: the gradients are bit-reproducible.  Without d f
// (PHASE false) there is no cos, no S/Q sum and no scan.
// ---------------------------------------------------------------------------
constexpr int kSbWarps = 4;
constexpr int kSbThreads = 32 * kSbWarps;

template <bool WINDOW, bool PHASE>
__global__ void __launch_bounds__(kSbThreads)
sinus_bwd_frames(const float* __restrict__ f, const float* __restrict__ a,
                 const float* __restrict__ g, const unsigned long long* __restrict__ offs,
                 float* __restrict__ part /* [5][B*F*K]: G0, G1, S, Q0, Q1 */,
                 int F, int K, int N, int hop, int FT, int n_tiles, int64_t BFK,
                 double inv_sr, float nyquist) {
  __shared__ float red[kSbWarps - 1][PHASE ? 5 : 2][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t p = (int64_t)blockIdx.x * 32 + lane;          // flat (b, i, k)
  const bool live = p < BFK;
  const int64_t pc = live ? p : BFK - 1;
  const int k = (int)(pc % K);
  const int64_t bi = pc / K;
  const int i = (int)(bi % F), b = (int)(bi / F);
  const int tile = i / FT, inx = min(i + 1, F - 1);
  const float* fb = f + (size_t)b * F * K + k;

  // the frame's phase: the tile offset plus the tile's frames before i
  unsigned long long P = offs[((size_t)b * n_tiles + tile) * K + k];
  for (int j = tile * FT; j < i; ++j)
    P += frame_total_fix64((double)fb[(size_t)j * K] * inv_sr,
                           (double)fb[(size_t)(j + 1) * K] * inv_sr, hop);
  const float lo = fb[(size_t)i * K], hi = fb[(size_t)inx * K];
  const double a0 = (double)lo * inv_sr, a1 = (double)hi * inv_sr;
  const unsigned long long A = turns_to_fix64(a0);
  const unsigned long long D = frame_slope_fix64(a0, a1, hop);
  const float am0 = PHASE ? a[(size_t)bi * K + k] : 0.f;
  const float am1 = PHASE ? a[((size_t)b * F + inx) * K + k] : 0.f;

  // this warp's segment [r0, r1) of the frame
  const int seg = (hop + kSbWarps - 1) / kSbWarps;
  const int r0 = min(hop, warp * seg), r1 = min(hop, r0 + seg);
  const unsigned long long ur0 = (unsigned long long)r0;
  unsigned long long ph = P + 0x80000000ull + (ur0 + 1) * A + ((ur0 * (ur0 + 1)) >> 1) * D;
  unsigned long long inc = A + (ur0 + 1) * D;                  // ph(r + 1) - ph(r)
  const float inv_hop = 1.0f / (float)hop;
  const float* gp = g + (size_t)b * N + (size_t)i * hop;
  float G0 = 0.f, G1 = 0.f, S = 0.f, Q0 = 0.f, Q1 = 0.f;
#pragma unroll 2
  for (int r = r0; r < r1; ++r) {
    const float frac = (float)r * inv_hop;
    const float w1 = WINDOW ? (0.5f - 0.5f * cospif(frac)) : frac;
    const float w0 = 1.0f - w1;
    const float fe = __fadd_rn(lo, __fmul_rn(__fsub_rn(hi, lo), frac));   // as the forward
    const float gm = (fe >= nyquist) ? 0.f : gp[r];
    const float x = (float)(int)(uint32_t)(ph >> 32) * 4.656612873077393e-10f;
    float s, c;
    sincospif(x, &s, &c);        // one call on both paths: d A does not depend on PHASE
    const float gs = gm * s;
    G0 = fmaf(gs, w0, G0);
    G1 = fmaf(gs, w1, G1);
    if (PHASE) {
      const float cc = gm * fmaf(am1, w1, am0 * w0) * c;
      const float tri = (float)r * (float)(r + 1) * (0.5f * inv_hop);
      S += cc;
      Q0 = fmaf(cc, (float)(r + 1) - tri, Q0);
      Q1 = fmaf(cc, tri, Q1);
    }
    ph += inc;
    inc += D;
  }

  // segment partials, summed in warp order
  if (warp > 0) {
    red[warp - 1][0][lane] = G0;
    red[warp - 1][1][lane] = G1;
    if (PHASE) {
      red[warp - 1][2][lane] = S;
      red[warp - 1][3][lane] = Q0;
      red[warp - 1][4][lane] = Q1;
    }
  }
  __syncthreads();
  if (warp == 0 && live) {
#pragma unroll
    for (int w = 0; w < kSbWarps - 1; ++w) {
      G0 += red[w][0][lane];
      G1 += red[w][1][lane];
      if (PHASE) {
        S += red[w][2][lane];
        Q0 += red[w][3][lane];
        Q1 += red[w][4][lane];
      }
    }
    part[p] = G0;
    part[BFK + p] = G1;
    if (PHASE) {
      part[2 * BFK + p] = S * 6.283185307179586f;
      part[3 * BFK + p] = Q0 * 6.283185307179586f;
      part[4 * BFK + p] = Q1 * 6.283185307179586f;
    }
  }
}

// pass 5.  A CTA owns one b and 32 sinusoids (one per lane); its warps own
// contiguous frame chunks.  The suffix sum of S is the later chunks' totals,
// added in warp order, then the running sum inside the chunk.  d_f may be NULL
// (then S/Q were not computed).
constexpr int kSfinWarps = 16;

__global__ void __launch_bounds__(32 * kSfinWarps)
sinus_bwd_finalize(const float* __restrict__ part, float* __restrict__ d_a,
                   float* __restrict__ d_f, int F, int K, int hop, int64_t BFK,
                   double inv_sr) {
  __shared__ double tot[kSfinWarps][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int k = blockIdx.x * 32 + lane, b = blockIdx.y;
  const bool live = k < K;
  const int chunk = (F + kSfinWarps - 1) / kSfinWarps;
  const int j0 = min(F, warp * chunk), j1 = min(F, j0 + chunk);
  const size_t base = (size_t)b * F * K + (live ? k : 0);
  const float* G0 = part + base;
  const float* G1 = G0 + BFK;
  float* da = d_a + base;
  if (live) {
#pragma unroll 4
    for (int j = j0; j < j1; ++j) {
      float v = G0[(size_t)j * K];
      if (j >= 1) v += G1[(size_t)(j - 1) * K];
      if (j == F - 1) v += G1[(size_t)j * K];
      da[(size_t)j * K] = v;
    }
  }
  if (d_f == nullptr) return;
  const float* S = G1 + BFK;
  const float* Q0 = S + BFK;
  const float* Q1 = Q0 + BFK;
  float* df = d_f + base;
  double t = 0.0;
  if (live) {
#pragma unroll 4
    for (int j = j0; j < j1; ++j) t += (double)S[(size_t)j * K];
  }
  tot[warp][lane] = t;
  __syncthreads();
  if (!live) return;
  const double alpha = 0.5 * (double)(hop + 1), beta = 0.5 * (double)(hop - 1);
  double suf = 0.0;                                            // sum_{i>j} S_i
  for (int w = kSfinWarps - 1; w > warp; --w) suf += tot[w][lane];
#pragma unroll 4
  for (int j = j1 - 1; j >= j0; --j) {
    const double s = (double)S[(size_t)j * K];
    double v = (double)Q0[(size_t)j * K];
    if (j >= 1) v += (alpha + beta) * suf + beta * s + (double)Q1[(size_t)(j - 1) * K];
    else v += alpha * suf;
    if (j == F - 1) v += (double)Q1[(size_t)j * K];
    df[(size_t)j * K] = (float)(v * inv_sr);
    suf += s;
  }
}

}  // namespace ddsp
