// Backward of the direct-form time-varying FIR (fir_kernel) and of the impulse-response
// synthesis (ir_kernel), both in noise.cuh.  With frame = ceil(N / F), fr(p) = p / frame,
// the crop `start` and the upstream gradient g, let G[q] = g[q - start] for
// 0 <= q - start < out_len (0 otherwise).  Then
//   d audio:  dx[p]   = sum_{m<S} h_{fr(p)}[m] G[p + m]          fir_adjoint_kernel
//   d IR:     dh_j[m] = sum_{p in frame j, p<N} x[p] G[p + m]     fir_dir_kernel (+ fir_dir_reduce)
//   d mags:   dM_k    = (c_k / S0) sum_j w_j cos(2 pi k idx_j / S0) dh_j[j]
//                                                                 ir_backward_kernel
// with c_0 = c_{nb-1} = 1 and c_k = 2 otherwise; idx_j, w_j are ir_tap's.  The IR of a
// sample is chosen by its own frame, so within a frame d audio is a plain correlation.
// No float atomics: every output is written once, and split sums are added in a fixed
// order, so the gradients are bit-reproducible.
#pragma once
#include "noise.cuh"

namespace ddsp {

constexpr int kFadjThreads = 256;

// d audio: one thread per INPUT sample.  The CTA's window of G (kFadjThreads + S - 1
// values, the crop offset applied) is staged in shared memory; the taps come through
// L1, as in fir_kernel.
__global__ void __launch_bounds__(kFadjThreads)
fir_adjoint_kernel(const float* __restrict__ g, const float* __restrict__ ir,
                   float* __restrict__ dx, int N, int S, int frame, int ir_batch_stride,
                   int start, int out_len) {
  extern __shared__ __align__(16) float sg[];   // [kFadjThreads + S - 1]
  const int b = blockIdx.y;
  const int p0 = blockIdx.x * kFadjThreads;
  const int tid = threadIdx.x;
  const float* gb = g + (size_t)b * out_len;
  const float* irb = ir + (size_t)b * ir_batch_stride;
  const long long t0 = (long long)p0 - start;   // g index of G[p0]
  const int win = kFadjThreads + S - 1;
  for (int i = tid; i < win; i += kFadjThreads) {
    const long long t = t0 + i;
    sg[i] = (t >= 0 && t < out_len) ? gb[t] : 0.f;
  }
  __syncthreads();
  const int p = p0 + tid;
  if (p >= N) return;
  const float* h = irb + (size_t)(p / frame) * S;
  // taps whose output lies inside the crop: 0 <= p + m - start < out_len
  const int m_lo = max(0, start - p);
  const int m_hi = (int)min((long long)S - 1, (long long)start + out_len - 1 - p);
  float acc = 0.f;
  for (int m = m_lo; m <= m_hi; ++m) acc = fmaf(h[m], sg[tid + m], acc);
  dx[(size_t)b * N + p] = acc;
}

// d IR: rows are segments of one frame of one item; frames longer than kDirChunk
// samples are split into n_chunk segments of `seg` samples, whose partial sums
// fir_dir_reduce adds in segment order.  A CTA owns kDirRows rows (lane = row) and
// kDirTaps taps (16 per warp), and stages the rows' x and G windows in shared memory.
constexpr int kDirThreads = 256;
constexpr int kDirRows = 32;
constexpr int kDirTaps = 16 * (kDirThreads / 32);   // 128
constexpr int kDirChunk = 256;

struct FirDirParams {
  const float* __restrict__ x;   // [B, N]
  const float* __restrict__ g;   // [B, out_len]
  float* out;                    // [n_rows, S]
  int N, S, F, frame, start, out_len;
  int n_chunk, seg, segp;        // segments per frame, their length, rounded up to 16
  int xS, gS;                    // shared-memory row strides (odd: conflict-free)
  long long n_rows;              // B * F * n_chunk
};

// Segments of a frame: at most kDirChunk samples each, as even as the frame allows.
__host__ __device__ inline void fir_dir_segments(int frame, int* n_chunk, int* seg) {
  *n_chunk = (frame + kDirChunk - 1) / kDirChunk;
  *seg = (frame + *n_chunk - 1) / *n_chunk;
}

__host__ __device__ inline size_t fir_dir_smem(const FirDirParams& p) {
  return sizeof(float) * kDirRows * ((size_t)p.xS + p.gS);
}

__global__ void __launch_bounds__(kDirThreads)
fir_dir_kernel(FirDirParams p) {
  extern __shared__ __align__(16) float sm[];
  float* sX = sm;                       // [kDirRows][xS]  x of the row, zero padded
  float* sG = sm + kDirRows * p.xS;     // [kDirRows][gS]  G[row start + t0 + i]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long r0 = (long long)blockIdx.x * kDirRows;
  const int t0 = blockIdx.y * kDirTaps;
  const int per_item = p.F * p.n_chunk;
  for (int e = tid; e < kDirRows * p.segp; e += kDirThreads) {
    const int rl = e / p.segp, i = e - rl * p.segp;
    const long long r = r0 + rl;
    float v = 0.f;
    if (r < p.n_rows) {
      const int b = (int)(r / per_item), rem = (int)(r - (long long)b * per_item);
      const int j = rem / p.n_chunk, c = rem - j * p.n_chunk;
      const int ps = j * p.frame + c * p.seg;
      const int pe = min(min(ps + p.seg, (j + 1) * p.frame), p.N);
      if (ps + i < pe) v = p.x[(size_t)b * p.N + ps + i];
    }
    sX[rl * p.xS + i] = v;
  }
  const int glen = p.segp + kDirTaps;
  for (int e = tid; e < kDirRows * glen; e += kDirThreads) {
    const int rl = e / glen, i = e - rl * glen;
    const long long r = r0 + rl;
    float v = 0.f;
    if (r < p.n_rows) {
      const int b = (int)(r / per_item), rem = (int)(r - (long long)b * per_item);
      const int j = rem / p.n_chunk, c = rem - j * p.n_chunk;
      const long long t = (long long)j * p.frame + c * p.seg + t0 + i - p.start;
      if (t >= 0 && t < p.out_len) v = p.g[(size_t)b * p.out_len + t];
    }
    sG[rl * p.gS + i] = v;
  }
  __syncthreads();
  // dh[m] = sum_i x[i] G[i + m] for the warp's 16 taps: the window G[i + m0 .. i + m0 + 15]
  // slides by one per input sample, so 2 LDS feed 16 FFMA
  const int m0 = warp * 16;
  float acc[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) acc[c] = 0.f;
  if (t0 + m0 < p.S) {
    const float* xrow = sX + lane * p.xS;
    const float* grow = sG + lane * p.gS;
    float W[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) W[c] = grow[m0 + c];
    for (int ib = 0; ib < p.segp; ib += 16) {
#pragma unroll
      for (int u = 0; u < 16; ++u) {
        const float xv = xrow[ib + u];
#pragma unroll
        for (int c = 0; c < 16; ++c) acc[c] = fmaf(xv, W[(c + u) & 15], acc[c]);
        W[u & 15] = grow[ib + u + 1 + m0 + 15];
      }
    }
  }
  __syncthreads();
  // transpose through shared memory so that the rows are stored coalesced
  float* sO = sG;                       // [kDirRows][kDirTaps + 1]
#pragma unroll
  for (int c = 0; c < 16; ++c) sO[lane * (kDirTaps + 1) + m0 + c] = acc[c];
  __syncthreads();
  for (int e = tid; e < kDirRows * kDirTaps; e += kDirThreads) {
    const int rl = e / kDirTaps, t = e - rl * kDirTaps;
    const long long r = r0 + rl;
    if (r < p.n_rows && t0 + t < p.S)
      p.out[(size_t)r * p.S + t0 + t] = sO[rl * (kDirTaps + 1) + t];
  }
}

// d IR [ir_batch, F, S] from the partial sums [B, F, n_chunk, S]: item ib sums its own
// segments, a shared IR (ir_batch 1) every item's, in item then segment order.
__global__ void fir_dir_reduce(const float* __restrict__ part, float* __restrict__ d_ir,
                               int B, int F, int S, int n_chunk, int shared,
                               long long n_out) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n_out;
       e += (long long)gridDim.x * blockDim.x) {
    const long long rest = e / S;
    const int m = (int)(e - rest * S);
    const int j = (int)(rest % F), ib = (int)(rest / F);
    const int b_lo = shared ? 0 : ib, b_hi = shared ? B : ib + 1;
    float acc = 0.f;
    for (int b = b_lo; b < b_hi; ++b) {
      const float* pp = part + ((size_t)b * F + j) * n_chunk * S + m;
      for (int c = 0; c < n_chunk; ++c) acc += pp[(size_t)c * S];
    }
    d_ir[e] = acc;
  }
}

// d magnitudes from d IR: the transpose of ir_kernel.  Frames are staged kIrFrames per
// CTA, with the window applied and the taps folded onto their |zero-phase offset| n
// (cos(2 pi k idx / S0) depends on idx only through it), as [n][kIrFrames] so that one
// broadcast LDS.128 pair serves every frame; one thread per bin steps (k n) mod S0 through
// the cosine table and accumulates in double, as the forward does.
// smem: cos table S0 + kIrFrames * nb folded taps (nb = S0 / 2 + 1 offsets).
__global__ void __launch_bounds__(kIrThreads)
ir_backward_kernel(const float* __restrict__ d_ir, float* __restrict__ d_mags,
                   int64_t BF, IrGeom g) {
  extern __shared__ __align__(16) float sm[];
  float* sCos = sm;                     // [S0]
  float* sD = sm + ((g.S0 + 3) & ~3);   // [nb][kIrFrames]
  const int tid = threadIdx.x;
  const int64_t f0 = (int64_t)blockIdx.x * kIrFrames;
  const int nf = (int)min((int64_t)kIrFrames, BF - f0);
  // offsets the taps reach: |j - shift| <= half for a padded window, S0 / 2 otherwise
  const int nh = g.padded ? min(g.half, g.S0 / 2) + 1 : g.nb;
  for (int i = tid; i < g.S0; i += kIrThreads)
    sCos[i] = cospif(2.0f * (float)i / (float)g.S0);
  for (int e = tid; e < kIrFrames * nh; e += kIrThreads) {
    const int n = e / kIrFrames, fr = e - n * kIrFrames;
    float v = 0.f;
    if (fr < nf) {
      const float* d = d_ir + (f0 + fr) * g.S;
      // taps shift +- n; offsets +-n + S0 alias only when S == S0 and n == S0 / 2
      // (tap 0), which tb covers
      const int ta = g.shift + n, tb = g.shift - n;
      int idx; float w;
      if (ta >= 0 && ta < g.S) { ir_tap(g, ta, &idx, &w); v = fmaf(w, d[ta], v); }
      if (tb >= 0 && tb < g.S && tb != ta) { ir_tap(g, tb, &idx, &w); v = fmaf(w, d[tb], v); }
    }
    sD[e] = v;
  }
  __syncthreads();
  const float inv = 1.0f / (float)g.S0;
  for (int k = tid; k < g.nb; k += kIrThreads) {
    double acc[kIrFrames];
#pragma unroll
    for (int fr = 0; fr < kIrFrames; ++fr) acc[fr] = 0.0;
    int ph = 0;                                  // (k * n) mod S0
    for (int n = 0; n < nh; ++n) {
      const double c = (double)sCos[ph];
      const float4 a = *reinterpret_cast<const float4*>(sD + n * kIrFrames);
      const float4 bq = *reinterpret_cast<const float4*>(sD + n * kIrFrames + 4);
      acc[0] = fma((double)a.x, c, acc[0]);  acc[1] = fma((double)a.y, c, acc[1]);
      acc[2] = fma((double)a.z, c, acc[2]);  acc[3] = fma((double)a.w, c, acc[3]);
      acc[4] = fma((double)bq.x, c, acc[4]); acc[5] = fma((double)bq.y, c, acc[5]);
      acc[6] = fma((double)bq.z, c, acc[6]); acc[7] = fma((double)bq.w, c, acc[7]);
      ph += k;
      if (ph >= g.S0) ph -= g.S0;
    }
    const float ck = (k == 0 || k == g.nb - 1) ? inv : 2.0f * inv;
#pragma unroll
    for (int fr = 0; fr < kIrFrames; ++fr)
      if (fr < nf) d_mags[(f0 + fr) * g.nb + k] = ck * (float)acc[fr];
  }
}
static_assert(kIrFrames == 8, "ir_backward_kernel reads the folded taps as two float4s");

}  // namespace ddsp
