// Wavetable synthesis: core.wavetable_synthesis (core.py:1238-1282, on
// core.linear_lookup, 1168-1214) and synths.Wavetable.get_signal
// (synths.py:241-257), forward and backward.  The reference resamples the tables
// to audio rate and builds [B, N, W + 1] distance, weight and product tensors of
// which two columns per row carry weight; here the tables stay at frame rate.
//
// f0 and amplitudes have F frames, hop = N / F.  a = f0 / sr in turns, piecewise
// linear in time (frame F := frame F-1).  The phase is the EXCLUSIVE sum
//   phi(i hop + r) = P_i + r a_i + D_i r (r - 1) / 2,   D_i = (a_{i+1} - a_i) / hop,
// with P_i the frame totals of the sinusoidal kernels, all in 64-bit fixed-point
// turns (wrapping adds are exact; wt_fix64 is exact at half turns).  pos = phi * W is then exact: j0 is
// the high word of the 128-bit product phi * W and the low word is frac * 2^64.
//   out(t) = amp(t) [(1 - frac) T_t[j0] + frac T_t[j1]],   j1 = (j0 + 1) mod W
// (the reference's wrap column).  T_t interpolates the [B, Fw, W] tables in time
// with resample_kernel's 'linear' taps (add_endpoint); Fw == 1 is a static table.
//
// Passes:
//   1-2. wt_tile_sums + oscbank_scan_chunks (K = 1): phase offset per tile of kFT
//        frames (sinusoidal.cuh's tile sums form a = f0 * (1 / sr), which is not
//        exact at f0 = m sr / W; here a = f0 / sr, as the reference divides)
//   3.   wt_frame_phase: P, A = a_i, D per frame (a block scan inside the tile)
//   4.   wt_forward: one thread per sample, tables read through L1 / L2 (every
//        Fw, including tiles that span more table frames than a cache holds)
// Backward, after passes 1-3:
//   5.   wt_bwd_frames: per frame the sums G0, G1 (d amplitudes) and S, Q0, Q1
//        (d f0) of sinusoidal.cuh with the exclusive coefficients
//        p1 = r (r - 1) / (2 hop), p0 = r - p1, then sinus_bwd_finalize (K = 1)
//   6.   wt_bwd_table: d wavetables.  A CTA owns one table frame, one segment of
//        the samples that read it and one range of columns; each warp scatters
//        into its own shared buffer with taps.cuh's scatter_tap (strictly
//        increasing targets, else lanes with one target summed in lane order),
//        and the warp buffers are added in warp order.  Several segments
//        (static tables, few table frames) leave partial tables that
//        wt_table_reduce adds in segment order.
// Gradients are TensorFlow's subgradients: d phase = W (T_t[j1] - T_t[j0]) off the
// knots and 0 where pos is an integer.  No atomics, no memset: every gradient is
// bit-reproducible.
#pragma once
#include "harmonic_common.cuh"
#include "sinusoidal.cuh"
#include "taps.cuh"

namespace ddsp {
namespace wt_ {

constexpr int kFT = 256;          // frames per phase tile (threads of wt_frame_phase)
constexpr int kThreads = 256;     // forward: one thread per sample
constexpr int kMaxW = 1 << 20;    // columns (2-D processor tables are N long)
constexpr int kTabWarps = 4;      // d wavetables: per-warp column buffers
constexpr int kTabCols = 4096;    // columns per d-wavetable CTA (64 KB of buffers)
constexpr int kTabSeg = 4096;     // at most ~this many samples per d-wavetable CTA

__host__ __device__ inline int table_col_tiles(int W) {
  return (W + kTabCols - 1) / kTabCols;
}
__host__ __device__ inline size_t table_smem_bytes(int W) {
  return sizeof(float) * (size_t)kTabWarps * (size_t)(W < kTabCols ? W : kTabCols);
}
// Sample segments per table frame: a frame of a 'linear' Fw -> N resample is read
// by fewer than 2 N / Fw + 2 samples; a static table by all N.
__host__ __device__ inline int table_segments(int N, int Fw) {
  const long long per = Fw == 1 ? (long long)N : (2ll * N + Fw - 1) / Fw + 2;
  return (int)((per + kTabSeg - 1) / kTabSeg);
}

// Turns as 64-bit fixed point (2^64 = one turn), exact for every multiple of 2^-52
// turn: frac(turns) in [0, 1) scaled by 2^64 is an exact unsigned conversion, and a
// half turn becomes exactly 2^63.  (common.cuh's turns_to_fix64 goes through a signed
// conversion of [-0.5, 0.5] turn, which clamps a half turn to 2^63 - 1: harmless for
// an oscillator, but here the knot test needs the exact low word.)
__device__ __forceinline__ unsigned long long wt_fix64(double turns) {
  const double x = (turns - floor(turns)) * 18446744073709551616.0;   // [0, 2^64]
  return x >= 18446744073709551616.0 ? 0ull : __double2ull_rn(x);
}

// Fixed-point phase coefficients of frame i: its total, a_i and D_i.  a = f0 / sr is
// a division, as the reference's phase velocity: f0 = m sr / W then puts every
// sample exactly on a knot.
struct FrameCoef {
  unsigned long long tot, a, d;
};
__device__ __forceinline__ FrameCoef frame_coef(const float* __restrict__ f0row, int i,
                                                int F, int hop, double sr) {
  const double a0 = (double)f0row[i] / sr;
  const double a1 = (double)f0row[min(i + 1, F - 1)] / sr;
  FrameCoef c;
  c.tot = wt_fix64((double)hop * a0 + (a1 - a0) * (0.5 * (hop - 1)));
  c.a = wt_fix64(a0);
  c.d = wt_fix64((a1 - a0) / (double)hop);
  return c;
}

// pass 1.  sums[b, tile] = the tile's frame totals (wrapping adds: exact in any
// order).  One thread per frame.
__global__ void __launch_bounds__(kFT)
wt_tile_sums(const float* __restrict__ f0, unsigned long long* __restrict__ sums, int F,
             int hop, int n_tiles, double sr) {
  __shared__ unsigned long long wsum[kFT / 32];
  const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i = blockIdx.x * kFT + threadIdx.x;
  const unsigned long long tot =
      i < F ? frame_coef(f0 + (size_t)b * F, i, F, hop, sr).tot : 0ull;
  const unsigned long long incl = warp_scan_frame_totals(tot, lane);
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  if (threadIdx.x != 0) return;
  unsigned long long s = 0;
  for (int w = 0; w < kFT / 32; ++w) s += wsum[w];
  sums[(size_t)b * n_tiles + blockIdx.x] = s;
}

// pass 3.  P_i = tile offset + the tile's earlier frame totals.
__global__ void __launch_bounds__(kFT)
wt_frame_phase(const float* __restrict__ f0, const unsigned long long* __restrict__ offs,
               unsigned long long* __restrict__ P, unsigned long long* __restrict__ A,
               unsigned long long* __restrict__ D, int F, int hop, int n_tiles, double sr) {
  __shared__ unsigned long long wsum[kFT / 32];
  const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i = blockIdx.x * kFT + threadIdx.x;
  const bool live = i < F;
  const size_t row = (size_t)b * F;
  FrameCoef c;
  c.tot = c.a = c.d = 0ull;
  if (live) c = frame_coef(f0 + row, i, F, hop, sr);
  const unsigned long long incl = warp_scan_frame_totals(c.tot, lane);
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  if (!live) return;
  unsigned long long base = offs[(size_t)b * n_tiles + blockIdx.x];
  for (int w = 0; w < warp; ++w) base += wsum[w];
  P[row + i] = base + incl - c.tot;
  A[row + i] = c.a;
  D[row + i] = c.d;
}

// phase of sample r of a frame (wrapping: exact)
__device__ __forceinline__ unsigned long long sample_phase(unsigned long long P,
                                                           unsigned long long A,
                                                           unsigned long long D, int r) {
  const unsigned long long ur = (unsigned long long)r;
  const unsigned long long tri = r > 0 ? (ur * (ur - 1)) >> 1 : 0ull;
  return P + ur * A + tri * D;
}

struct Pos {
  int j0, j1;     // columns; j1 = (j0 + 1) mod W, the wrap column
  float w0, w1;   // 1 - frac, frac
  bool knot;      // pos is an integer: d phase is 0
};

__device__ __forceinline__ Pos lookup_pos(unsigned long long phi, int W) {
  const unsigned long long uw = (unsigned long long)W;
  const unsigned long long lo = phi * uw;
  Pos p;
  p.j0 = (int)__umul64hi(phi, uw);
  p.j1 = p.j0 + 1 == W ? 0 : p.j0 + 1;
  const double fr = (double)lo * 5.421010862427522e-20;   // 2^-64
  p.w0 = (float)(1.0 - fr);
  p.w1 = (float)fr;
  p.knot = lo == 0ull;
  return p;
}

struct TabTaps {
  int k0, k1;     // table frames
  float v0, v1;   // their weights
};

// resample_kernel's 'linear' taps from Fw frames to N samples; Fw == 1 is static.
__device__ __forceinline__ TabTaps table_taps(const rt_::ResampleGeom& g, int t) {
  TabTaps q;
  if (g.F == 1) {
    q.k0 = q.k1 = 0; q.v0 = 1.f; q.v1 = 0.f;
    return q;
  }
  int idx[2];
  float w[2];
  rt_::resample_taps(g, t, idx, w);
  q.k0 = idx[0]; q.k1 = idx[1]; q.v0 = w[0]; q.v1 = w[1];
  return q;
}

// weight of the later amplitude frame at offset r ('window' as resample_kernel)
template <bool WINDOW>
__device__ __forceinline__ float amp_w1(int r, int hop) {
  const float x = (float)r / (float)hop;
  return WINDOW ? 0.5f - 0.5f * cospif(x) : x;
}

__device__ __forceinline__ float table_value(const float* __restrict__ t0,
                                             const float* __restrict__ t1,
                                             const TabTaps& q, int j) {
  return fmaf(q.v1, __ldg(t1 + j), q.v0 * __ldg(t0 + j));
}

// pass 4.  out[b, t]; tab is [B, Fw, W].
template <bool WINDOW>
__global__ void __launch_bounds__(kThreads)
wt_forward(const float* __restrict__ amps, const float* __restrict__ tab,
           const unsigned long long* __restrict__ P, const unsigned long long* __restrict__ A,
           const unsigned long long* __restrict__ D, float* __restrict__ out, int F, int N,
           int hop, int Fw, int W) {
  const int b = blockIdx.y;
  const int t = blockIdx.x * kThreads + threadIdx.x;
  if (t >= N) return;
  const int i = t / hop, r = t - i * hop;
  const size_t fi = (size_t)b * F + i, fn = (size_t)b * F + min(i + 1, F - 1);
  const Pos p = lookup_pos(sample_phase(P[fi], A[fi], D[fi], r), W);
  const float w1 = amp_w1<WINDOW>(r, hop);
  const float amp = fmaf(__ldg(amps + fn), w1, __ldg(amps + fi) * (1.0f - w1));
  const TabTaps q = table_taps(rt_::resample_geom(Fw, N, 1, 1), t);
  const float* t0 = tab + ((size_t)b * Fw + q.k0) * W;
  const float* t1 = tab + ((size_t)b * Fw + q.k1) * W;
  const float v0 = table_value(t0, t1, q, p.j0), v1 = table_value(t0, t1, q, p.j1);
  out[(size_t)b * N + t] = amp * fmaf(p.w1, v1, p.w0 * v0);
}

// pass 5.  A CTA owns 32 consecutive (b, i) (one per lane); its warps split the
// frame's hop samples into contiguous segments whose partials are added in warp
// order.  part is [5][B F]: G0, G1, S, Q0, Q1 (S, Q in turns).
template <bool WINDOW, bool PHASE>
__global__ void __launch_bounds__(kSbThreads)
wt_bwd_frames(const float* __restrict__ amps, const float* __restrict__ tab,
              const float* __restrict__ g, const unsigned long long* __restrict__ Pf,
              const unsigned long long* __restrict__ Af,
              const unsigned long long* __restrict__ Df, float* __restrict__ part, int F,
              int N, int hop, int Fw, int W, int64_t BF) {
  __shared__ float red[kSbWarps - 1][PHASE ? 5 : 2][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t p = (int64_t)blockIdx.x * 32 + lane;          // flat (b, i)
  const bool live = p < BF;
  const int64_t pc = live ? p : BF - 1;
  const int i = (int)(pc % F), b = (int)(pc / F);
  const size_t fn = (size_t)b * F + min(i + 1, F - 1);
  const unsigned long long P = Pf[pc], A = Af[pc], D = Df[pc];
  const float am0 = PHASE ? amps[pc] : 0.f, am1 = PHASE ? amps[fn] : 0.f;
  const rt_::ResampleGeom geom = rt_::resample_geom(Fw, N, 1, 1);
  const float* tb = tab + (size_t)b * Fw * W;
  const float* gp = g + (size_t)b * N + (size_t)i * hop;
  const float half_inv_hop = 0.5f / (float)hop;

  const int seg = (hop + kSbWarps - 1) / kSbWarps;
  const int r0 = min(hop, warp * seg), r1 = min(hop, r0 + seg);
  float G0 = 0.f, G1 = 0.f, S = 0.f, Q0 = 0.f, Q1 = 0.f;
  for (int r = r0; r < r1; ++r) {
    const Pos ps = lookup_pos(sample_phase(P, A, D, r), W);
    const TabTaps q = table_taps(geom, i * hop + r);
    const float* t0 = tb + (size_t)q.k0 * W;
    const float* t1 = tb + (size_t)q.k1 * W;
    const float v0 = table_value(t0, t1, q, ps.j0), v1 = table_value(t0, t1, q, ps.j1);
    const float gt = gp[r];
    const float w1 = amp_w1<WINDOW>(r, hop), w0 = 1.0f - w1;
    const float gl = gt * fmaf(ps.w1, v1, ps.w0 * v0);
    G0 = fmaf(gl, w0, G0);
    G1 = fmaf(gl, w1, G1);
    if (PHASE) {
      const float amp = fmaf(am1, w1, am0 * w0);
      const float cc = ps.knot ? 0.f : gt * amp * ((float)W * (v1 - v0));
      const float p1 = (float)r * (float)(r > 0 ? r - 1 : 0) * half_inv_hop;
      S += cc;
      Q0 = fmaf(cc, (float)r - p1, Q0);
      Q1 = fmaf(cc, p1, Q1);
    }
  }

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
    part[BF + p] = G1;
    if (PHASE) {
      part[2 * BF + p] = S;
      part[3 * BF + p] = Q0;
      part[4 * BF + p] = Q1;
    }
  }
}

// pass 6.  grid (Fw * n_seg * n_ct, B): table frame k, sample segment s, column
// tile c.  dst is d wavetables [B, Fw, W] (n_seg == 1) or the partial tables
// [B, Fw, n_seg, W].
template <bool WINDOW>
__global__ void __launch_bounds__(kTabWarps * 32)
wt_bwd_table(const float* __restrict__ amps, const float* __restrict__ g,
             const unsigned long long* __restrict__ Pf,
             const unsigned long long* __restrict__ Af,
             const unsigned long long* __restrict__ Df, float* __restrict__ dst, int F,
             int N, int hop, int Fw, int W, int n_seg) {
  extern __shared__ float wt_buf[];                    // [kTabWarps][cols]
  __shared__ float stage[kTabWarps][32];
  const int n_ct = table_col_tiles(W);
  const int c = blockIdx.x % n_ct;
  const int ks = blockIdx.x / n_ct;
  const int k = ks / n_seg, s = ks - k * n_seg;
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = c * kTabCols, cols = min(kTabCols, W - c0);
  float* buf = wt_buf + warp * cols;
  for (int j = lane; j < cols; j += 32) buf[j] = 0.f;
  __syncwarp();

  // the samples that read table frame k: lo(t) <= k <= hi(t), one range
  const rt_::ResampleGeom geom = rt_::resample_geom(Fw, N, 1, 1);
  int t0 = 0, t1 = N;
  if (Fw > 1) {
    t0 = rt_::resample_bound(geom, k, true);
    t1 = rt_::resample_bound(geom, k, false);
  }
  const long long len = t1 - t0;
  const int a = t0 + (int)(len * s / n_seg), e = t0 + (int)(len * (s + 1) / n_seg);
  const size_t row = (size_t)b * F;
  const float* gb = g + (size_t)b * N;
  for (int base = a + warp * 32; base < e; base += kTabWarps * 32) {   // warp-uniform
    const int t = base + lane;
    const bool live = t < e;
    Pos ps;
    ps.j0 = ps.j1 = 0; ps.w0 = ps.w1 = 0.f;
    float cv = 0.f;
    if (live) {
      const int i = t / hop, r = t - i * hop;
      const size_t fi = row + i, fn = row + min(i + 1, F - 1);
      ps = lookup_pos(sample_phase(Pf[fi], Af[fi], Df[fi], r), W);
      const float w1 = amp_w1<WINDOW>(r, hop);
      const float amp = fmaf(__ldg(amps + fn), w1, __ldg(amps + fi) * (1.0f - w1));
      const TabTaps q = table_taps(geom, t);
      const float wk = (q.k0 == k ? q.v0 : 0.f) + (q.k1 == k ? q.v1 : 0.f);
      cv = __ldg(gb + t) * amp * wk;
    }
    md_::scatter_tap(buf, stage[warp], ps.j0, cv * ps.w0,
                     live && ps.j0 >= c0 && ps.j0 < c0 + cols, c0, lane);
    md_::scatter_tap(buf, stage[warp], ps.j1, cv * ps.w1,
                     live && ps.j1 >= c0 && ps.j1 < c0 + cols, c0, lane);
  }
  __syncthreads();
  float* out = dst + (((size_t)b * Fw + k) * n_seg + s) * W + c0;
  for (int j = threadIdx.x; j < cols; j += kTabWarps * 32) {
    float acc = 0.f;
#pragma unroll
    for (int w = 0; w < kTabWarps; ++w) acc += wt_buf[w * cols + j];
    out[j] = acc;
  }
}

// d wavetables [R, W] = partial tables [R, n_seg, W] added in segment order.
__global__ void __launch_bounds__(256)
wt_table_reduce(const float* __restrict__ part, float* __restrict__ d_tab, int64_t RW,
                int W, int n_seg) {
  for (int64_t x = (int64_t)blockIdx.x * 256 + threadIdx.x; x < RW;
       x += (int64_t)gridDim.x * 256) {
    const int64_t rr = x / W;
    const int j = (int)(x - rr * W);
    const float* p = part + (size_t)rr * n_seg * W + j;
    float acc = 0.f;
    for (int s = 0; s < n_seg; ++s) acc += p[(size_t)s * W];
    d_tab[x] = acc;
  }
}

}  // namespace wt_
}  // namespace ddsp
