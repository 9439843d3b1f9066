// Fused harmonic synthesis: core.harmonic_synthesis (core.py:1048-1111) =
// get_harmonic_frequencies + resample('linear') + resample(amp_method) +
// oscillator_bank (core.py:911-962) in ONE kernel.  No [B,N,K] tensor exists.
//
// Maths (SURVEY.md Appendix A.1-A.3), per batch item, hop = N / F:
//   frame i = t / hop, r = t % hop, frac = r / hop, f_F := f_{F-1}
//   f0(t)   = f_i + (f_{i+1} - f_i) * frac                 (v1 bilinear)
//   phi(t)  = sum_{m<=t} f0(m)/sr  [turns]
//           = P_i + (r+1) a_i + (a_{i+1}-a_i)/hop * r(r+1)/2,  a = f/sr,
//             P_i = sum_{j<i} [hop a_j + (a_{j+1}-a_j)(hop-1)/2]
//   a_k(t)  = amp_i hd_{i,k} w0(r) + amp_{i+1} hd_{i+1,k} w1(r)
//             window: w1 = 0.5 - 0.5 cos(pi r / hop); linear: w1 = r/hop
//   audio(t)= sum_{k: f_k(t) < sr/2} a_k(t) sin(2 pi k phi(t))
// phi is 64-bit fixed point (wraps exactly); k*phi is a wrapping 32-bit multiply.
#pragma once
#include "harmonic_common.cuh"

namespace ddsp {

constexpr int kHarmThreads = 256;

// u64 P[FT], A[FT], D[FT]; u64 red[8]; float f0s[FT+1], amp[FT+1]; float xs[(FT+1)*Kp]
__host__ __device__ inline size_t harm_smem_bytes(int FT, int Kp) {
  return sizeof(unsigned long long) * (3 * (size_t)FT + 8) +
         sizeof(float) * (2 * (size_t)(FT + 1) + (size_t)(FT + 1) * Kp);
}

// ---------------------------------------------------------------------------
// Generic kernel: any integer hop, any K.  One thread = one sample at a time.
// MODE 0: Reinsch recurrence over harmonics; MODE 1: one sin per oscillator.
// ---------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(kHarmThreads)
harmonic_generic_kernel(HarmonicParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int FT = p.FT, Kp = p.Kp, K = p.K, F = p.F, hop = p.hop;
  unsigned long long* sP = reinterpret_cast<unsigned long long*>(smem_raw);
  unsigned long long* sA = sP + FT;
  unsigned long long* sD = sA + FT;
  unsigned long long* sRed = sD + FT;
  float* sF0 = reinterpret_cast<float*>(sRed + 8);
  float* sAmp = sF0 + (FT + 1);
  float* sX = sAmp + (FT + 1);

  const int b = blockIdx.y;
  const int i0 = blockIdx.x * FT;            // first frame of the tile
  const int nfr = min(FT, F - i0);           // frames in this tile
  const int tid = threadIdx.x;
  const float* f0b = p.f0 + (size_t)b * F;
  const float* ampb = p.amps + (size_t)b * F;

  // ---- 1. phase at the start of the tile: wrapping sum of frame totals ----
  unsigned long long part = 0;
  for (int j = tid; j < i0; j += kHarmThreads) {
    double a0 = (double)f0b[j] * p.inv_sr;
    double a1 = (double)f0b[min(j + 1, F - 1)] * p.inv_sr;
    part += frame_total_fix64(a0, a1, hop);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if ((tid & 31) == 0) sRed[tid >> 5] = part;

  // ---- 2. stage the tile's frame data ----
  for (int j = tid; j <= nfr; j += kHarmThreads) {
    int g = min(i0 + j, F - 1);              // frame F is a copy of F-1
    sF0[j] = f0b[g];
    sAmp[j] = ampb[g];
  }
  if (p.hd != nullptr) {
    const float* hdb = p.hd + ((size_t)b * F + i0) * K;
    const int rows_in = min(nfr + 1, F - i0);   // rows that exist in memory
    for (int idx = tid; idx < rows_in * K; idx += kHarmThreads) {
      int r = idx / K, c = idx - r * K;
      sX[r * Kp + c] = hdb[idx];
    }
    if (rows_in < nfr + 1) {                    // frame F := frame F-1 (from HBM:
      for (int c = tid; c < K; c += kHarmThreads)  // the smem row is not synced yet)
        sX[nfr * Kp + c] = hdb[(size_t)(nfr - 1) * K + c];
    }
  } else {
    for (int j = tid; j <= nfr; j += kHarmThreads) sX[j * Kp] = 1.0f;
  }
  __syncthreads();

  // ---- 3. per-frame phase tables (one thread; FT is small) ----
  if (tid == 0) {
    unsigned long long P = 0;
    for (int w = 0; w < kHarmThreads / 32; ++w) P += sRed[w];
    const double init_rad = p.init_phase ? (double)p.init_phase[b] : 0.0;
    const unsigned long long Pinit = turns_to_fix64(init_rad * 0.15915494309189535);
    P += Pinit;
    for (int j = 0; j < nfr; ++j) {
      double a0 = (double)sF0[j] * p.inv_sr;
      double a1 = (double)sF0[j + 1] * p.inv_sr;
      sP[j] = P;
      sA[j] = turns_to_fix64(a0);
      sD[j] = frame_slope_fix64(a0, a1, hop);
      P += frame_total_fix64(a0, a1, hop);
    }
    if (p.final_phase != nullptr && i0 + nfr == F) {
      // angular_cumsum's last value in [0, 2 pi) plus the initial phase
      // (core.py:1004-1012): final_phase = phases[:, -1]
      const double turns = (double)(P - Pinit) * 5.421010862427522e-20;   // 2^-64
      p.final_phase[b] = (float)(turns * 6.283185307179586 + init_rad);
    }
  }
  __syncthreads();

  // ---- 4. samples ----
  const int t_begin = i0 * hop;
  const int n_tile = nfr * hop;
  const float inv_hop = 1.0f / (float)hop;
  float* outb = p.audio + (size_t)b * p.N;
  for (int lt = tid; lt < n_tile; lt += kHarmThreads) {
    const int li = lt / hop;
    const int r = lt - li * hop;
    const float frac = (float)r * inv_hop;
    const float f_lo = sF0[li], f_hi = sF0[li + 1];

    // phase of the fundamental, 64-bit fixed point turns (inclusive cumsum)
    unsigned long long ph = sP[li] + (unsigned long long)(r + 1) * sA[li] +
        (unsigned long long)(((long long)r * (r + 1)) >> 1) * sD[li];
    const uint32_t p32 = (uint32_t)((ph + 0x80000000ull) >> 32);

    // amplitude interpolation weights (amp folded in)
    float w1;
    if (p.amp_method == DDSP_B200_AMP_WINDOW) {
      w1 = 0.5f - 0.5f * cospif(frac);
    } else {
      w1 = frac;
    }
    const float w0 = (1.0f - w1) * sAmp[li];
    w1 *= sAmp[li + 1];
    const float* x0 = sX + li * Kp;
    const float* x1 = x0 + Kp;

    // live harmonic count (Nyquist mask of oscillator_bank, core.py:942)
    const bool monotone = !p.mask_nyquist || ((f_lo >= 1.0f) && (f_hi >= 1.0f));
    int klive = (p.mask_nyquist && monotone)
                    ? live_harmonics(f_lo, f_hi, frac, K, p.nyquist) : K;

    float acc = 0.f;
    if (MODE == 1 || !monotone) {
      // one sin per oscillator; exact per-oscillator mask
      uint32_t pk = 0;
      for (int k = 1; k <= klive; ++k) {
        pk += p32;
        float a = x0[k - 1] * w0 + x1[k - 1] * w1;
        if (!monotone &&
            !(ref_harmonic_freq(f_lo, f_hi, frac, k) < p.nyquist)) a = 0.f;
        float s = sinpif((float)(int)pk * 4.656612873077393e-10f);  // 2^-31
        acc = fmaf(a, s, acc);
      }
    } else {
      // Reinsch recurrence over k on the reduced angle psi in [-pi/2, pi/2];
      // if phi was shifted by half a turn, sin(k phi) = (-1)^k sin(k psi).
      int ps = (int)p32;
      const bool flip = (ps >= (1 << 30)) || (ps < -(1 << 30));
      if (flip) ps ^= 0x80000000;
      const float u = (float)ps * 2.3283064365386963e-10f;   // turns, |u|<=.25
      float sh, ch;
      sincospif(u, &sh, &ch);                 // half angle: sin/cos(psi/2)
      const float alpha = 4.0f * sh * sh;     // 4 sin^2(psi/2)
      float s = 2.0f * sh * ch;               // sin(psi)
      float d = s;                            // s_1 - s_0
      float acc_o0 = 0.f, acc_o1 = 0.f, acc_e0 = 0.f, acc_e1 = 0.f;
      int k = 1;
      for (; k + 1 <= klive; k += 2) {
        acc_o0 = fmaf(x0[k - 1], s, acc_o0);
        acc_o1 = fmaf(x1[k - 1], s, acc_o1);
        d = fmaf(-alpha, s, d);
        s += d;
        acc_e0 = fmaf(x0[k], s, acc_e0);
        acc_e1 = fmaf(x1[k], s, acc_e1);
        d = fmaf(-alpha, s, d);
        s += d;
      }
      if (k <= klive) {
        acc_o0 = fmaf(x0[k - 1], s, acc_o0);
        acc_o1 = fmaf(x1[k - 1], s, acc_o1);
      }
      const float odd = acc_o0 * w0 + acc_o1 * w1;
      const float even = acc_e0 * w0 + acc_e1 * w1;
      acc = flip ? (even - odd) : (even + odd);
    }
    const int t = t_begin + lt;
    if (p.accumulate) acc += outb[t];
    outb[t] = acc;
  }
}

}  // namespace ddsp
