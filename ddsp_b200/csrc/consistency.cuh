// Gaussian-mixture negative log-likelihoods of the consistency losses
// (losses.KDEConsistencyLoss and losses.TWMLoss, losses.py:689-1061), evaluated per
// frame on-chip: the reference's pairwise [.., Ka, Kb] / [.., C, P, G] log-prob
// tensors are never written to memory, in the forward or the backward.
//
// Mode A, mixture_nll_kernel: for frame r = (b, t), queries x[r, q], components
// mu[r, j] and log-weights lw[r, j] (log_softmax'd by the caller) and one scale s,
//   nll[r, q] = -logsumexp_j(lw_j - z_qj^2 / 2) + log s + log(2 pi) / 2,
//   z_qj = (x_q - mu_j) / s.
// One CTA per frame stages M_j = mu_j / s and lw_j in shared memory; a thread takes a
// query.  The logsumexp is shifted by its largest term j*, found in a first pass.  The
// second pass forms each exponent relative to j* as a product of differences,
//   (lw_j - z_j^2/2) - (lw_j* - z_j*^2/2) = (lw_j - lw_j*) - (M_j* - M_j)(z_j + z_j*)/2,
// so it carries the relative rounding of its own (small) value, not that of the
// 1e6-sized terms of a far query; the largest term is exactly exp(0) = 1.
//
// Mode A backward, mixture_nll_backward_kernel: with responsibilities r_qj,
//   dx_q = g_q / s sum_j r_qj z_qj,  dmu_j = -1/s sum_q g_q r_qj z_qj,
//   dlw_j = -sum_q g_q r_qj.
// Queries are taken in chunks of kChunk: a thread per query computes dx and stashes
// its shift (X_q, z_q*, M_j*, lw_j* + log sum) and g_q in shared memory; then a thread
// per component adds the chunk's terms to its own running sums in ascending q.  Every
// sum runs in a fixed order in one thread: no atomics, bit-reproducible.
//
// Mode B, comb_nll_kernel (TWM's p(sinusoids | harmonics)): for candidates f0[r, c] and
// points f[r, p] with amplitudes a[r, p],
//   out[r, c] = sum_p a_p nu(f_p / f0_c) / D,  D = sum_p a_p (safe_divide: 0 -> 1e-7,
//   and 1e-7 for f0_c = 0 too),
//   nu(q) = -logsumexp_{k=1..G}(-log G - ((q - k)/s)^2 / 2) + log s + log(2 pi) / 2.
// The comb's largest term is its nearest k0 = clamp(rint(q), 1, G); only the terms
// k0 - W .. k0 + W are summed, W chosen on the host so that the omitted terms are below
// 2^-25 of the sum (DESIGN §3.17).  One CTA per frame, a thread per candidate.
//
// Mode B backward, comb_nll_backward_kernel: a thread per candidate recomputes its row
// (out_c and d f0_c = -g_c / (D f0_c) sum_p a_p nu'(q) q, 0 at f0_c = 0), then a thread
// per point sums over the candidates in ascending c:
//   d a_p = sum_c g_c (nu_pc - out_c [D != 0]) / D,  d f_p = sum_c g_c a_p nu'_pc / (D f0_c).
//
// Mode C, sin_to_harm_kernel (core.sinusoidal_to_harmonic, core.py:733-781): for
// sinusoids a[r, s], f[r, s] and one f0[r], with den = f0 (1e-7 where f0 = 0),
//   q_ks = (f_s - f0 k) / den,  w_ks = exp(-(|q_ks| / width)^2),  k = 1..K,
//   W_ks = w_ks / sw_k where normalize and sw_k = sum_s w_ks > 1, else w_ks,
//   HA_k = sum_s W_ks a_s (0 where f0 k >= nyquist),  D = sum_k HA_k,
//   harm_amp[r] = D,  harm_dist[r, k] = HA_k / Ds  (Ds = D, 1e-7 where D = 0).
// One CTA per frame stages a and f; a thread per harmonic sums over the sinusoids (q
// and w in the reference's float32 op order; the normalised sum as sum_s w a / sw).
// D is the sum of the threads' partial sums, added by thread 0 in thread order.
//
// Mode C backward, sin_to_harm_backward_kernel: with upstream g_A and g_k,
//   dHA_k = g_A + (g_k - [D != 0] sum_j g_j HA_j / Ds) / Ds  (0 where masked),
//   the same as TensorFlow's g_k / Ds + g_A - sum_j g_j HA_j / Ds^2 without its inf - inf
//   at a tiny D,
//   alpha_k = dHA_k / sw_k, beta_k = HA_k before the mask where normalised, else
//   alpha_k = dHA_k, beta_k = 0;  e_ks = alpha_k (a_s - beta_k) w_ks q_ks,
//   d a_s = sum_k alpha_k w_ks,  d f_s = -2 / (width^2 den) sum_k e_ks,
//   d f0 = 2 / (width^2 den) sum_ks e_ks (k + [f0 != 0] q_ks)
// (the f0 k path, and the denominator's unless safe_divide took its constant).  A first
// pass recomputes D, a second sum_j g_j HA_j / Ds (from the first kHarmChunk rows kept in
// shared memory, later rows recomputed).  Then harmonics are taken in chunks of
// kHarmChunk: a thread per harmonic writes alpha and beta to shared memory, then a
// thread per sinusoid adds the chunk's terms to its running sums in ascending k.
// Harmonics with alpha_k = 0 (every masked one) and pairs whose float32 weight is 0
// add exactly 0 and are skipped.  No atomics: bit-reproducible.
#pragma once
#include "common.cuh"

namespace ddsp {
namespace cons_ {

constexpr int kThreads = 128;
// components (mode A), candidates and points (mode B) staged per frame
constexpr int kMaxStaged = DDSP_B200_CONSISTENCY_MAX_STAGED;
constexpr int kChunk = 512;        // queries per shared-memory chunk of the mode A backward
constexpr int kHarmChunk = 256;    // harmonics per shared-memory chunk of the mode C backward

struct MixParams {
  const float* x;      // [R, Q]
  const float* mu;     // [R, J]
  const float* lw;     // [R, J]
  int Q, J;
  float inv_scale;     // 1 / s
  float log_norm;      // log s + log(2 pi) / 2
};

struct CombParams {
  const float* f0;     // [R, C]
  const float* f;      // [R, P]
  const float* a;      // [R, P]
  int C, P, G, W;
  float inv_scale;     // 1 / s
  float log_norm;      // log G + log s + log(2 pi) / 2
};

struct S2HParams {
  const float* a;      // [R, S]
  const float* f;      // [R, S]
  const float* f0;     // [R]
  int S, K;
  float width;         // harmonic_width, nonzero
  float nyquist;       // sample_rate / 2
  int normalize;
};

// One query against the staged components: the shift j* and the sums
// s = sum_j exp(d_j) and t = sum_j exp(d_j) z_j (d relative to j*).
struct MixRow {
  float zs, ms, ls, s, t;
};

__device__ __forceinline__ MixRow mix_row(float X, const float* M, const float* LW, int J) {
  float best = -INFINITY;
  int js = 0;
  for (int j = 0; j < J; ++j) {
    const float z = X - M[j];
    const float v = fmaf(-0.5f * z, z, LW[j]);
    if (v > best) {
      best = v;
      js = j;
    }
  }
  MixRow o;
  o.ms = M[js];
  o.ls = LW[js];
  o.zs = X - o.ms;
  o.s = 0.f;
  o.t = 0.f;
  for (int j = 0; j < J; ++j) {
    const float z = X - M[j];
    const float e = __expf(fmaf(-0.5f * (o.ms - M[j]), z + o.zs, LW[j] - o.ls));
    o.s += e;
    o.t = fmaf(e, z, o.t);
  }
  return o;
}

__device__ __forceinline__ void stage_components(const MixParams& p, int64_t r, float* M,
                                                 float* LW) {
  const float* mu = p.mu + r * p.J;
  const float* lw = p.lw + r * p.J;
  for (int j = threadIdx.x; j < p.J; j += blockDim.x) {
    M[j] = mu[j] * p.inv_scale;
    LW[j] = lw[j];
  }
}

// grid: one CTA per frame; smem: 2 J floats
__global__ void __launch_bounds__(kThreads) mixture_nll_kernel(MixParams p, float* nll) {
  extern __shared__ float sm[];
  float* M = sm;
  float* LW = sm + p.J;
  const int64_t r = blockIdx.x;
  stage_components(p, r, M, LW);
  __syncthreads();
  const float* x = p.x + r * p.Q;
  float* out = nll + r * p.Q;
  for (int q = threadIdx.x; q < p.Q; q += blockDim.x) {
    const MixRow o = mix_row(x[q] * p.inv_scale, M, LW, p.J);
    // L = lw_j* - z*^2 / 2 + log s
    out[q] = -(fmaf(-0.5f * o.zs, o.zs, o.ls) + __logf(o.s)) + p.log_norm;
  }
}

// grid: one CTA per frame; smem: 4 J + 5 kChunk floats
__global__ void __launch_bounds__(kThreads) mixture_nll_backward_kernel(
    MixParams p, const float* grad, float* dx, float* dmu, float* dlw) {
  extern __shared__ float sm[];
  float* M = sm;
  float* LW = M + p.J;
  float* accz = LW + p.J;          // sum_q g r z, per component
  float* accw = accz + p.J;        // sum_q g r
  float* cX = accw + p.J;          // per query of the chunk: X_q
  float* cZ = cX + kChunk;         //   z_q*
  float* cM = cZ + kChunk;         //   M_j*
  float* cK = cM + kChunk;         //   lw_j* + log s_q
  float* cG = cK + kChunk;         //   g_q
  const int64_t r = blockIdx.x;
  stage_components(p, r, M, LW);
  for (int j = threadIdx.x; j < p.J; j += blockDim.x) {
    accz[j] = 0.f;
    accw[j] = 0.f;
  }
  __syncthreads();
  const float* x = p.x + r * p.Q;
  const float* g = grad + r * p.Q;
  float* dxr = dx + r * p.Q;
  for (int q0 = 0; q0 < p.Q; q0 += kChunk) {
    const int n = min(kChunk, p.Q - q0);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const float X = x[q0 + i] * p.inv_scale;
      const MixRow o = mix_row(X, M, LW, p.J);
      const float gq = g[q0 + i];
      dxr[q0 + i] = gq * p.inv_scale * (o.t / o.s);
      cX[i] = X;
      cZ[i] = o.zs;
      cM[i] = o.ms;
      cK[i] = o.ls + __logf(o.s);
      cG[i] = gq;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < p.J; j += blockDim.x) {
      const float Mj = M[j], LWj = LW[j];
      float az = accz[j], aw = accw[j];
      for (int i = 0; i < n; ++i) {
        const float z = cX[i] - Mj;
        const float gr = cG[i] * __expf(fmaf(-0.5f * (cM[i] - Mj), z + cZ[i], LWj - cK[i]));
        az = fmaf(gr, z, az);
        aw += gr;
      }
      accz[j] = az;
      accw[j] = aw;
    }
    __syncthreads();
  }
  float* dmur = dmu + r * p.J;
  float* dlwr = dlw + r * p.J;
  for (int j = threadIdx.x; j < p.J; j += blockDim.x) {
    dmur[j] = -accz[j] * p.inv_scale;
    dlwr[j] = -accw[j];
  }
}

// nu(q) of the comb and d nu / dq.  NaN q stays NaN (fmaxf picks k0 = 1).
__device__ __forceinline__ float comb_nu(float q, const CombParams& p, float* dnu) {
  const float k0 = fminf(fmaxf(rintf(q), 1.f), (float)p.G);
  const float z0 = (q - k0) * p.inv_scale;
  float s = 1.f, t = z0;
  for (int n = 1; n <= p.W; ++n) {
#pragma unroll
    for (int side = -1; side <= 1; side += 2) {
      const float k = k0 + (float)(side * n);
      if (k >= 1.f && k <= (float)p.G) {
        const float z = (q - k) * p.inv_scale;
        // -(z^2 - z0^2) / 2 = -(k0 - k) / s (z + z0) / 2
        const float e = __expf(-0.5f * (k0 - k) * p.inv_scale * (z + z0));
        s += e;
        t = fmaf(e, z, t);
      }
    }
  }
  *dnu = (t / s) * p.inv_scale;
  return fmaf(0.5f * z0, z0, p.log_norm) - __logf(s);
}

// D = sum_p a_p in a fixed order by warp 0 (lane-strided, then a shuffle tree)
__device__ __forceinline__ float stage_points(const CombParams& p, int64_t r, float* F,
                                              float* A, float* F0, float* red) {
  const float* f = p.f + r * p.P;
  const float* a = p.a + r * p.P;
  const float* f0 = p.f0 + r * p.C;
  for (int i = threadIdx.x; i < p.P; i += blockDim.x) {
    F[i] = f[i];
    A[i] = a[i];
  }
  for (int c = threadIdx.x; c < p.C; c += blockDim.x) {
    const float v = f0[c];
    F0[c] = v == 0.f ? 1e-7f : v;
  }
  if (threadIdx.x < 32) {
    float d = 0.f;
    for (int i = threadIdx.x; i < p.P; i += 32) d += a[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    if (threadIdx.x == 0) red[0] = d;
  }
  __syncthreads();
  return red[0];
}

// grid: one CTA per frame; smem: 2 P + C + 1 floats
__global__ void __launch_bounds__(kThreads) comb_nll_kernel(CombParams p, float* out) {
  extern __shared__ float sm[];
  float* F = sm;
  float* A = F + p.P;
  float* F0 = A + p.P;
  float* red = F0 + p.C;
  const int64_t r = blockIdx.x;
  const float D = stage_points(p, r, F, A, F0, red);
  const float Ds = D == 0.f ? 1e-7f : D;
  float* o = out + r * p.C;
  for (int c = threadIdx.x; c < p.C; c += blockDim.x) {
    const float f0 = F0[c];
    float acc = 0.f, dnu;
    for (int i = 0; i < p.P; ++i) acc = fmaf(A[i], comb_nu(F[i] / f0, p, &dnu), acc);
    o[c] = acc / Ds;
  }
}

// grid: one CTA per frame; smem: 2 P + 3 C + 1 floats
__global__ void __launch_bounds__(kThreads) comb_nll_backward_kernel(
    CombParams p, const float* grad, float* d_f0, float* d_f, float* d_a) {
  extern __shared__ float sm[];
  float* F = sm;
  float* A = F + p.P;
  float* F0 = A + p.P;
  float* H = F0 + p.C;             // g_c / D
  float* S = H + p.C;              // out_c where D != 0, else 0
  float* red = S + p.C;
  const int64_t r = blockIdx.x;
  const float D = stage_points(p, r, F, A, F0, red);
  const float Ds = D == 0.f ? 1e-7f : D;
  const float* g = grad + r * p.C;
  const float* f0r = p.f0 + r * p.C;
  float* df0 = d_f0 + r * p.C;
  for (int c = threadIdx.x; c < p.C; c += blockDim.x) {
    const float f0 = F0[c];
    float an = 0.f, ad = 0.f, dnu;
    for (int i = 0; i < p.P; ++i) {
      const float q = F[i] / f0;
      an = fmaf(A[i], comb_nu(q, p, &dnu), an);
      ad = fmaf(A[i] * dnu, q, ad);
    }
    const float h = g[c] / Ds;
    H[c] = h;
    S[c] = D != 0.f ? an / Ds : 0.f;
    df0[c] = f0r[c] != 0.f ? -h * ad / f0 : 0.f;
  }
  __syncthreads();
  float* dfr = d_f + r * p.P;
  float* dar = d_a + r * p.P;
  for (int i = threadIdx.x; i < p.P; i += blockDim.x) {
    const float fi = F[i];
    float da = 0.f, dfs = 0.f, dnu;
    for (int c = 0; c < p.C; ++c) {
      const float f0 = F0[c];
      const float nu = comb_nu(fi / f0, p, &dnu);
      da = fmaf(H[c], nu - S[c], da);
      dfs = fmaf(H[c], dnu / f0, dfs);
    }
    dar[i] = da;
    dfr[i] = dfs * A[i];
  }
}

// The sum of one value per thread, added by thread 0 in thread order; every thread gets
// it.  red: kThreads + 1 floats.
__device__ __forceinline__ float ordered_block_sum(float v, float* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < kThreads; ++i) s += red[i];
    red[kThreads] = s;
  }
  __syncthreads();
  return red[kThreads];
}

__device__ __forceinline__ void stage_sinusoids(const S2HParams& p, int64_t r, float* A,
                                                float* F) {
  const float* a = p.a + r * p.S;
  const float* f = p.f + r * p.S;
  for (int s = threadIdx.x; s < p.S; s += blockDim.x) {
    A[s] = a[s];
    F[s] = f[s];
  }
}

// w_ks as the reference forms it: freqs_ratio = |(f - hf) / den|, exp(-(ratio / width)^2)
__device__ __forceinline__ float s2h_weight(float f, float hf, float den, float width,
                                            float* q) {
  *q = (f - hf) / den;
  const float u = fabsf(*q) / width;
  return expf(-(u * u));
}

// Harmonic k's sum of weights sw and its amplitude before the Nyquist mask,
// hp = sum_s W_ks a_s.
struct S2HRow {
  float sw, hp;
};

__device__ __forceinline__ S2HRow s2h_row(const S2HParams& p, float hf, float den,
                                          const float* A, const float* F) {
  float sw = 0.f, swa = 0.f, q;
  for (int s = 0; s < p.S; ++s) {
    const float w = s2h_weight(F[s], hf, den, p.width, &q);
    sw += w;
    swa = fmaf(w, A[s], swa);
  }
  return {sw, p.normalize && sw > 1.f ? swa / sw : swa};
}

// grid: one CTA per frame; smem: 2 S + kThreads + 1 floats
__global__ void __launch_bounds__(kThreads) sin_to_harm_kernel(S2HParams p, float* harm_amp,
                                                               float* harm_dist) {
  extern __shared__ float sm[];
  float* A = sm;
  float* F = A + p.S;
  float* red = F + p.S;
  const int64_t r = blockIdx.x;
  stage_sinusoids(p, r, A, F);
  const float f0 = p.f0[r];
  const float den = f0 == 0.f ? 1e-7f : f0;
  __syncthreads();
  float* dist = harm_dist + r * p.K;
  float part = 0.f;
  for (int k = threadIdx.x; k < p.K; k += blockDim.x) {
    const float hf = f0 * (float)(k + 1);
    const float ha = hf >= p.nyquist ? 0.f : s2h_row(p, hf, den, A, F).hp;
    dist[k] = ha;     // HA_k until D is known; read back by this thread only
    part += ha;
  }
  const float D = ordered_block_sum(part, red);
  const float Ds = D == 0.f ? 1e-7f : D;
  for (int k = threadIdx.x; k < p.K; k += blockDim.x) dist[k] = dist[k] / Ds;
  if (threadIdx.x == 0) harm_amp[r] = D;
}

// grid: one CTA per frame; smem: 4 S + 4 kHarmChunk + kThreads + 1 floats
__global__ void __launch_bounds__(kThreads) sin_to_harm_backward_kernel(
    S2HParams p, const float* g_amp, const float* g_dist, float* d_a, float* d_f,
    float* d_f0) {
  extern __shared__ float sm[];
  float* A = sm;
  float* F = A + p.S;
  float* ES = F + p.S;             // sum_k e_ks, per sinusoid
  float* AS = ES + p.S;            // sum_k alpha_k w_ks
  float* cSW = AS + p.S;           // first chunk's sw_k, kept from the first pass
  float* cHP = cSW + kHarmChunk;   //   and hp_k
  float* cAl = cHP + kHarmChunk;   // per harmonic of the chunk: alpha_k
  float* cBe = cAl + kHarmChunk;   //   beta_k
  float* red = cBe + kHarmChunk;
  const int64_t r = blockIdx.x;
  stage_sinusoids(p, r, A, F);
  for (int s = threadIdx.x; s < p.S; s += blockDim.x) {
    ES[s] = 0.f;
    AS[s] = 0.f;
  }
  const float f0 = p.f0[r];
  const float den = f0 == 0.f ? 1e-7f : f0;
  __syncthreads();
  const float* gd = g_dist + r * p.K;
  float pd = 0.f;
  for (int k = threadIdx.x; k < p.K; k += blockDim.x) {
    const float hf = f0 * (float)(k + 1);
    S2HRow h = {0.f, 0.f};
    if (!(hf >= p.nyquist)) h = s2h_row(p, hf, den, A, F);
    pd += h.hp;
    if (k < kHarmChunk) {
      cSW[k] = h.sw;
      cHP[k] = h.hp;
    }
  }
  const float D = ordered_block_sum(pd, red);
  const float Ds = D == 0.f ? 1e-7f : D;
  // dHA_k = g_A + (g_k - Gd) / Ds with Gd = sum_j g_j dist_j (0 where D = 0): the two
  // 1 / Ds terms are combined before the division, and dist_j = HA_j / Ds keeps its
  // precision when HA and D are tiny, so a small D cancels instead of giving inf - inf
  float pg = 0.f;
  if (D != 0.f) {
    for (int k = threadIdx.x; k < p.K; k += blockDim.x) {
      const float hf = f0 * (float)(k + 1);
      if (hf >= p.nyquist) continue;
      const float hp = k < kHarmChunk ? cHP[k] : s2h_row(p, hf, den, A, F).hp;
      pg = fmaf(gd[k], hp / Ds, pg);
    }
  }
  const float Gd = ordered_block_sum(pg, red);
  const float ga = g_amp[r];
  float pf = 0.f;
  for (int k0 = 0; k0 < p.K; k0 += kHarmChunk) {
    const int n = min(kHarmChunk, p.K - k0);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const float hf = f0 * (float)(k0 + i + 1);
      float al = 0.f, be = 0.f;
      if (!(hf >= p.nyquist)) {
        const S2HRow h = k0 == 0 ? S2HRow{cSW[i], cHP[i]} : s2h_row(p, hf, den, A, F);
        const float dha = ga + (gd[k0 + i] - Gd) / Ds;
        const bool sel = p.normalize && h.sw > 1.f;
        al = sel ? dha / h.sw : dha;
        be = sel ? h.hp : 0.f;
      }
      cAl[i] = al;
      cBe[i] = be;
    }
    __syncthreads();
    for (int s = threadIdx.x; s < p.S; s += blockDim.x) {
      const float a = A[s], fs = F[s];
      float es = ES[s], as = AS[s];
      for (int i = 0; i < n; ++i) {
        const float al = cAl[i];
        if (al == 0.f) continue;
        const float kf = (float)(k0 + i + 1);
        float q;
        const float w = s2h_weight(fs, f0 * kf, den, p.width, &q);
        if (w == 0.f) continue;     // adds exactly 0 (alpha may be inf where D is tiny)
        const float e = al * (a - cBe[i]) * w * q;
        es += e;
        as = fmaf(al, w, as);
        pf = fmaf(e, f0 != 0.f ? kf + q : kf, pf);
      }
      ES[s] = es;
      AS[s] = as;
    }
    __syncthreads();
  }
  const float F0 = ordered_block_sum(pf, red);
  const float k2 = 2.f / (p.width * p.width);
  float* dfr = d_f + r * p.S;
  float* dar = d_a + r * p.S;
  for (int s = threadIdx.x; s < p.S; s += blockDim.x) {
    dfr[s] = -k2 * ES[s] / den;
    dar[s] = AS[s];
  }
  if (threadIdx.x == 0) d_f0[r] = k2 * F0 / den;
}

}  // namespace cons_
}  // namespace ddsp
