// noise_ring: FilteredNoise.get_signal for the decoder shape (n_frequencies = 65,
// frame = 64 samples, 128-tap IR; ae.gin:60-68), third generation.  Same maths as
// noise_fused.cuh (windowed zero-phase IR per frame by E/O cosine
// sums, Philox noise, time-varying FIR == the reference's framed FFT convolution
// + overlap-add + crop, core.py:1382-1473); the second generation was bound by
// shared-memory bandwidth and by consumer warps marching in lock step through an
// overlap-add buffer.  What changed:
//
//   * GATHER FORM, NO OVERLAP-ADD.  out[64 q + n] = sum_i x_q[i] h_q[n + 62 - i]
//     + sum_i x_{q+1}[i] h_{q+1}[n - 2 - i] + sum_i x_{q-1}[i] h_{q-1}[n + 126 - i]
//     (+ x_{q-2}[63] h_{q-2}[127] for n = 0), taps outside [0, 128) being zero:
//     exactly 128 MACs per output.  A lane owns output frame q and reads the rows
//     of frames q-2 .. q+1; a warp finishes its 32 x R output block in registers
//     and writes it straight to HBM (st / red.add for the fused Add) - consumer
//     warps never talk to each other.
//   * ROW RING, NO HALO.  A persistent CTA walks a contiguous range of frames; the
//     impulse responses and noise rows live in a ring of seven 32-row slots in shared
//     memory (lane-private rows, strides = 2 mod 4 floats: conflict-free LDS.64),
//     so neighbouring tiles share their edge rows instead of recomputing them.
//   * ONE ACCUMULATOR PER OUTPUT, TAP-STATIONARY ORDER.  A consumer warp owns a
//     unit of R consecutive outputs of its lane's frame, one register each.  A body
//     holds R inputs of one row in registers and streams the taps through: tap
//     h[m] serves every (output, input) pair on its diagonal, so up to R scalar
//     FFMAs share one tap, and a body of R x R MACs loads R inputs and 2 R taps
//     (LDS.64 pairs).
//   * TRIANGULAR TRIMMING at compile time: the rows of frames q+1 and q-1 cover
//     complementary triangles of the (n, i) square; fully unrolled bodies skip the
//     (n, i) pairs whose taps are out of range.
//   * producers: groups of 4 warps take turns on tiles; a group takes its tile from
//     raw magnitudes (TMA) through exp_sigmoid, the cosine sums and the windowed taps
//     to the Philox rows, and asks for its ring slot only when the sums are done.
//     The cosine sums are a matrix product with a constant operand, [32 frames x 65
//     magnitudes] x [65 x 65 cosines], split into its even-k and odd-k halves
//     (h0[n] = E[n] + O[n], h0[64 - n] = E[n] - O[n]) and run on the FP64 tensor
//     cores (mma.m16n8k4.f64, 154 per tile); each tap is rounded to float once.
#pragma once
#include "noise_fused.cuh"

namespace ddsp {

namespace nr_ {
constexpr int NB = 65, FRAME = 64, S = 128, S0 = 128, Q = 32, SHIFT = 64;
// A consumer warp owns a UNIT of R outputs of 32 frames: R accumulators and the R
// inputs of a body in registers.  R = 16: four units per frame, 9 KB of FIR bodies
// (a 32-output unit was timed slower on the H100, DESIGN.md 3.2).
constexpr int R = 16;
constexpr int UPT = FRAME / R;                     // units per 64-sample frame
// Consumer warps, producer groups and ring slots.  The consumer tile groups hold
// NTG + 1 slots between them; what is left decouples producers from consumers.
// 227 KB of shared memory hold 7 slots next to the cosine table and the three
// raw-magnitude staging buffers.  Other warp shapes were timed slower (DESIGN.md 3.2).
constexpr int CONS_WARPS = 8, PROD_GROUPS = 3;
constexpr int GROUP_WARPS = 4, PROD_WARPS = GROUP_WARPS * PROD_GROUPS;
constexpr int NTG = CONS_WARPS / UPT;              // consumption tiles in flight
static_assert((NTG & (NTG - 1)) == 0, "tile groups: a power of two");
constexpr int SLOTS = 7;
static_assert(SLOTS > NTG + 1, "the ring must leave slots to the producers");
constexpr int RING = 32 * SLOTS;
// Every warp runs under the launch budget (65536 / THREADS registers: 96 for 640
// threads); the scalar FIR needs no more, so there is no register split, and a
// shape with more warps than that would starve the consumers of registers.
constexpr int THREADS = 32 * (CONS_WARPS + PROD_WARPS);
static_assert(THREADS <= 640, "noise_ring: the FIR needs 96 registers per thread");
constexpr int HPAD = 2, HS = 134, XS = 66, MS = 65;   // row strides (floats)
constexpr int NQ = FRAME / 4;

// IR synthesis on the FP64 tensor cores: per tile, H[f][n] = sum_k M[f][k] C[k][n]
// as mma.m16n8k4 (A = 16 frames x 4 k, B = 4 k x 8 n), once over the even k (E)
// and once over the odd k (O), for n = 0 .. 31 (four n-tiles) plus E at n = 32
// (a fifth n-tile, one live column: O[32] = 0).  Within k-step s, lane (g, t) =
// (lane / 4, lane % 4) takes index kk = 16 (s / 4) + 4 t + s % 4 of its half (k = 2 kk
// or 2 kk + 1): frames g and g + 8 then read the magnitude rows (stride 65 floats)
// on 32 distinct banks.  The table C[k][n] c_k / S0 (c_k = 1 at k = 0, 64, else 2)
// is stored as B fragments, one double per lane, in that k order.
constexpr int E_STEPS = 9, O_STEPS = 8;            // 33 even k (padded to 36), 32 odd k
constexpr int E_NT = 5, O_NT = 4;                  // n-tiles of 8 columns
constexpr int TAB_E = E_STEPS * E_NT * 32, TAB = TAB_E + O_STEPS * O_NT * 32;   // doubles
__host__ __device__ constexpr int ir_kk(int s, int t) { return 16 * (s >> 2) + 4 * t + (s & 3); }

// -DDDSP_NR_TIMING: per-warp cycle counters by phase (tools/noise_timing.py reads
// them back through ddsp_b200_debug_noise_timing); measurement builds only.
#ifdef DDSP_NR_TIMING
#define NR_TIMING_DECL unsigned tprev__ = (unsigned)clock()
__device__ unsigned g_nr_timing[kMaxSMs * 32 * 8];
#define NR_LAP(i)                                                                       \
  do {                                                                                  \
    const unsigned n__ = (unsigned)clock();                                             \
    if (lane == 0) atomicAdd(&g_nr_timing[(blockIdx.x * 32 + warp) * 8 + (i)], n__ - tprev__); \
    tprev__ = n__;                                                                      \
  } while (0)
#else
#define NR_TIMING_DECL
#define NR_LAP(i)
#endif

struct Smem {
  double ctab[TAB];
  float win[S];
  alignas(16) float raw[PROD_GROUPS][32 * NB + 8];
  alignas(16) float h[RING * HS];
  alignas(16) float x[RING * XS];
  alignas(8) unsigned long long full[SLOTS], empty[SLOTS], rawbar[PROD_GROUPS];
};

struct Params {
  const float* __restrict__ mags;
  const float* __restrict__ noise;
  float* audio;
  uint64_t seed, offset;
  int B, F, N, accumulate, raw, item_base;
  float bias;
};

// A contiguous run of output frames [s0, s0 + len) of batch item b.
struct Seg {
  int b, s0, len, nP, nC;
};

__device__ __forceinline__ bool next_seg(long long& g, long long g1, int F, Seg& sg) {
  if (g >= g1) return false;
  sg.b = (int)(g / F);
  sg.s0 = (int)(g - (long long)sg.b * F);
  sg.len = (int)min((long long)(F - sg.s0), g1 - g);
  sg.nP = (sg.len + 3 + 31) >> 5;       // production tiles: rows s0-2 .. s0+len
  sg.nC = (sg.len + 31) >> 5;           // consumption tiles
  g += sg.len;
  return true;
}

__device__ __forceinline__ void mbar_arrive_n(void* bar, int n) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(n)
               : "memory");
}

// Shared-memory loads the scheduler may neither merge nor reorder (software
// pipelines that need several loads in flight with distinct destinations).
__device__ __forceinline__ float4 lds128v(const float* p) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "r"(smem_u32(p)));
  return v;
}
__device__ __forceinline__ float lds32v(const float* p) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(smem_u32(p)));
  return v;
}

// d += a b on the FP64 tensor cores: A 16 x 4 (a0: row lane / 4, a1: row lane / 4 + 8,
// column lane % 4), B 4 x 8 (row lane % 4, column lane / 4), D 16 x 8 (d[0..1]: row
// lane / 4, d[2..3]: row lane / 4 + 8, columns 2 (lane % 4) + {0, 1}).
__device__ __forceinline__ void dmma_16x8x4(double (&d)[4], double a0, double a1, double b) {
  asm("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5}, {%6}, "
      "{%0, %1, %2, %3};"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a0), "d"(a1), "d"(b));
}

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c,
                                           float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a),
               "f"(b), "f"(c), "f"(d)
               : "memory");
}

// ---- consumer: FIR bodies ---------------------------------------------------
// The dynamic shared memory, addressed by float offsets from its base: indexing
// the __shared__ symbol itself keeps every access an LDS / STS (pointers carried
// through the op program lose the address space and become generic loads).
extern __shared__ __align__(16) unsigned char nr_smem[];
constexpr int X_OFF = (int)(offsetof(Smem, x) / 4), H_OFF = (int)(offsetof(Smem, h) / 4);
__device__ __forceinline__ float lds1(int off) {
  return reinterpret_cast<const float*>(nr_smem)[off];
}
__device__ __forceinline__ float2 lds2(int off) {   // off even
  return *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(nr_smem) + off);
}

// One body: y[k + d] += x[xo + k] * h[ho + d] for 0 <= k, k + d < R and
// DLO <= d <= DHI.  The R inputs sit in registers and the taps stream through as
// pairs (h[ho + 2j], h[ho + 2j + 1]) - xo and ho are even - each tap serving the
// whole diagonal d (up to R FFMAs on one multiplicand).  Templates rather than
// loops: every index is a constant, so y and X stay in registers.
template <int D, int DLO, int DHI>
__device__ __forceinline__ void fir_diag(float (&y)[R], const float (&X)[R], float t) {
  if constexpr (D >= DLO && D <= DHI) {
#pragma unroll
    for (int k = (D < 0 ? -D : 0); k < (D > 0 ? R - D : R); ++k)
      y[k + D] = fmaf(X[k], t, y[k + D]);
  }
}
template <int J, int DLO, int DHI>
__device__ __forceinline__ void fir_pairs(float (&y)[R], const float (&X)[R], int ho) {
  if constexpr (2 * J + 1 >= DLO) {
    const float2 P = lds2(ho + 2 * J);
    fir_diag<2 * J + 1, DLO, DHI>(y, X, P.y);
    fir_diag<2 * J, DLO, DHI>(y, X, P.x);
    fir_pairs<J - 1, DLO, DHI>(y, X, ho);
  }
}
template <int DLO, int DHI>
__device__ __forceinline__ void fir_body(float (&y)[R], int xo, int ho) {
  float X[R];
#pragma unroll
  for (int k = 0; k < R; k += 2) {
    const float2 v = lds2(xo + k);
    X[k] = v.x;
    X[k + 1] = v.y;
  }
  fir_pairs<DHI / 2, DLO, DHI>(y, X, ho);
}

// The FIR of one unit runs as a short PROGRAM of R x R bodies, executed by a
// loop with a switch so that each body exists once in the instruction stream
// (fully inlined, the consumer code stalls on instruction fetch).
// Unit u has outputs N0 = R u .. N0 + R - 1; body j of a row covers its inputs
// R j .. R j + R - 1.  Input i of the row of frame q + s reaches output n through
// tap m = n - i + C with C = 62 (s = 0), -2 (s = 1), 126 (s = -1):
//   frame q  : UPT FULL bodies (the one tap below 0, m = -1, is padding).
//   frame q+1: reaches n >= i + 2: u FULL bodies, then body u as the LOWER
//              triangle d = n - i >= 2 (taps 0 .. R - 3).
//   frame q-1: reaches n <= i + 1: body u as the UPPER triangle d <= 1 (taps up
//              to 127), then FULL bodies to the end of the row.
// What is left is one MAC: the input before N0 through tap 127 into output N0 -
// x[N0 - 1] of frame q-1, or for u = 0 x[63] of frame q-2.
enum { OP_FULL = 0, OP_LOWER = 1, OP_UPPER = 2 };
constexpr int N_OPS = 2 * UPT + 1;

// xr / hr: row offsets (x, and h at tap 0) of frames q+1, q, q-1, q-2.
__device__ __forceinline__ void consume_unit(float (&y)[R], int u, const int (&xr)[4],
                                             const int (&hr)[4]) {
  const int N0 = R * u;
  const int xm1 = xr[0], hm1 = hr[0], x0 = xr[1], h0 = hr[1], xp1 = xr[2], hp1 = hr[2];
#pragma unroll 1
  for (int i = 0; i < N_OPS; ++i) {
    int kind = OP_FULL, xo, ho;
    if (i < UPT) {
      xo = x0 + R * i;
      ho = h0 + N0 + 62 - R * i;
    } else if (i < UPT + u) {
      const int j = i - UPT;
      xo = xm1 + R * j;
      ho = hm1 + N0 - 2 - R * j;
    } else if (i == UPT + u) {
      kind = OP_LOWER;
      xo = xm1 + N0;
      ho = hm1 - 2;
    } else if (i == UPT + u + 1) {
      kind = OP_UPPER;
      xo = xp1 + N0;
      ho = hp1 + 126;
    } else {
      const int j = i - UPT - 1;
      xo = xp1 + R * j;
      ho = hp1 + N0 + 126 - R * j;
    }
    switch (kind) {
      case OP_FULL: fir_body<-(R - 1), R - 1>(y, xo, ho); break;
      case OP_LOWER: fir_body<2, R - 1>(y, xo, ho); break;
      default: fir_body<-(R - 1), 1>(y, xo, ho); break;
    }
  }
  const int xe = u ? xp1 + N0 - 1 : xr[3] + 63, he = u ? hp1 + 127 : hr[3] + 127;
  y[0] = fmaf(lds1(xe), lds1(he), y[0]);
}
__global__ void __launch_bounds__(nr_::THREADS, 1)
noise_ring_kernel(Params p) {
  Smem& sm = *reinterpret_cast<Smem*>(nr_smem);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // ---- once: tables, window, zeroed ring (pads stay zero), barriers ----
  for (int e = tid; e < TAB; e += THREADS) {
    // B fragment (half, k-step s, n-tile nt), lane l: C[k][8 nt + l / 4] c_k / S0
    const bool even = e < TAB_E;
    const int ee = even ? e : e - TAB_E, nts = even ? E_NT : O_NT;
    const int l = ee & 31, s = (ee >> 5) / nts, nt = (ee >> 5) - s * nts;
    const int kk = ir_kk(s, l & 3), k = even ? 2 * kk : 2 * kk + 1, n = 8 * nt + (l >> 2);
    double v = 0.0;
    if (k < NB && n <= Q) {
      const double ck = (k == 0 || k == NB - 1) ? 1.0 : 2.0;
      v = ck / S0 * cospi(2.0 * (double)((k * n) % S0) / S0);
    }
    sm.ctab[e] = v;
  }
  for (int j = tid; j < S; j += THREADS)
    sm.win[j] = 0.5f - 0.5f * cospif(2.0f * (float)j / (float)S0);   // core.py:1498,1515
  for (int e = tid; e < RING * HS; e += THREADS) sm.h[e] = 0.f;
  for (int e = tid; e < RING * XS; e += THREADS) sm.x[e] = 0.f;
#ifdef DDSP_NR_TIMING
  for (int e = tid; e < 32 * 8; e += THREADS) g_nr_timing[blockIdx.x * 32 * 8 + e] = 0;
#endif
  if (tid == 0) {
    for (int i = 0; i < SLOTS; ++i) {
      mbar_init(&sm.full[i], GROUP_WARPS);          // one arrive per producer warp
      mbar_init(&sm.empty[i], 2 * UPT);
    }
    for (int i = 0; i < PROD_GROUPS; ++i) mbar_init(&sm.rawbar[i], 1);
  }
  __syncthreads();

  // this CTA's frames: an even share of the B * F frames, cut at item boundaries
  const long long T = (long long)p.B * p.F;
  const long long g_lo = T * blockIdx.x / gridDim.x;
  const long long g_hi = T * (blockIdx.x + 1) / gridDim.x;

  if (warp < CONS_WARPS) {
    // =========================== CONSUMERS ===================================
    const int tg = warp / UPT, unit = warp % UPT;      // tile group, unit of the tile
    long long g = g_lo;
    Seg sg;
    int pbase = 0, ct = 0;                   // ct: consumption tiles before this segment
    bool dep_done = false;
    NR_TIMING_DECL;
    while (next_seg(g, g_hi, p.F, sg)) {
      // tiles ct + t of the CTA go round-robin over the tile groups
      for (int t = (tg - ct) & (NTG - 1); t < sg.nC; t += NTG) {
        NR_LAP(3);
        // rows of this tile live in production tiles t and t+1 of the segment
        // (two producer groups finish tiles out of order: wait for both)
        {
          const int P0 = pbase + t, P1 = pbase + min(t + 1, sg.nP - 1);
          mbar_wait(&sm.full[P0 % SLOTS], (P0 / SLOTS) & 1);
          mbar_wait(&sm.full[P1 % SLOTS], (P1 / SLOTS) & 1);
        }
        NR_LAP(0);
        const int q_rel = 32 * t + lane;                // output frame, relative
        // lanes past the end of the segment redo its last frame (and store
        // nothing): they must not wander into rows nobody produced
        const int rho = min(q_rel, sg.len - 1) + 2;     // its production row
        const int rbase = pbase * 32;
        int xr[4], hr[4];
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          const int row = (rbase + rho + 1 - s) % RING;
          xr[s] = X_OFF + row * XS;
          hr[s] = H_OFF + row * HS + HPAD;
        }
        float y[R];
#pragma unroll
        for (int c = 0; c < R; ++c) y[c] = 0.f;
        consume_unit(y, unit, xr, hr);
        __syncwarp();
        NR_LAP(1);
        if (lane == 0) {
          // release the slots: a production tile is read by consumption tiles
          // tau-1 and tau (UPT warps each); a lone reader arrives twice.
#pragma unroll
          for (int d = 0; d < 2; ++d) {
            const int tau = t + d;
            if (tau < sg.nP) {
              const int readers = (tau >= 1 ? 1 : 0) + (tau < sg.nC ? 1 : 0);
              mbar_arrive_n(&sm.empty[(pbase + tau) % SLOTS], 2 / readers);
            }
          }
        }
        // ---- store / accumulate this lane's R outputs ----
        if (!dep_done) {
          // programmatic dependent launch: this grid may have started while the
          // harmonic kernel was still draining; its audio must be complete (and
          // visible) before the first add lands.  No-op for a plain launch.
          asm volatile("griddepcontrol.wait;" ::: "memory");
          dep_done = true;
        }
        if (q_rel < sg.len) {
          constexpr int NOUT = R;
          const long long t0 = (long long)(sg.s0 + q_rel) * FRAME + NOUT * unit;
          float* o = p.audio + (size_t)sg.b * p.N + t0;
          if (t0 + NOUT <= p.N && (reinterpret_cast<uintptr_t>(o) & 15) == 0) {
#pragma unroll
            for (int w4 = 0; w4 < NOUT / 4; ++w4) {
              if (p.accumulate)
                red_add_v4(o + 4 * w4, y[4 * w4], y[4 * w4 + 1], y[4 * w4 + 2],
                           y[4 * w4 + 3]);
              else
                *reinterpret_cast<float4*>(o + 4 * w4) =
                    make_float4(y[4 * w4], y[4 * w4 + 1], y[4 * w4 + 2], y[4 * w4 + 3]);
            }
          } else {
#pragma unroll
            for (int w1 = 0; w1 < NOUT; ++w1) {
              if (t0 + w1 < p.N) {
                if (p.accumulate) o[w1] += y[w1]; else o[w1] = y[w1];
              }
            }
          }
        }
        NR_LAP(2);
      }
      ct += sg.nC;
      pbase += sg.nP;
    }
  } else {
    // =============================== PRODUCERS ===============================
    // PROD_GROUPS groups of four warps; group g builds the production tiles P = g
    // (mod PROD_GROUPS) end to end: magnitudes (TMA) -> exp_sigmoid (in place) ->
    // both cosine half-sums -> windowed taps, then the tile's noise rows.  A group
    // has PROD_GROUPS tile periods for one tile, so its latency chains (TMA, MUFU,
    // LDS) stay off the consumers' critical path.
    const int grp = (warp - CONS_WARPS) / GROUP_WARPS;
    const int iw = (warp - CONS_WARPS) % GROUP_WARPS;   // column block / slice
    const int ptid = tid - (CONS_WARPS + GROUP_WARPS * grp) * 32;   // 0..127 within the group
    constexpr int PT = 32 * GROUP_WARPS;
    const int bar_id = 1 + grp;
    float* s_raw = sm.raw[grp];
    void* rawbar = &sm.rawbar[grp];
    const float* mags_end = p.mags + (size_t)p.B * p.F * NB;
    // Raw magnitudes of a production tile -> s_raw (asynchronously; consumed one
    // of the group's tiles later).  The valid rows are contiguous in HBM: ONE TMA
    // bulk copy of the enclosing 16-byte aligned span (rows are only 4-byte
    // aligned: 65 floats); row r lands at s_raw[roff + 65 r].  Spans that would
    // leave the tensor fall back to per-element cp.async.
    auto prefetch = [&](const Seg& s, int tau) -> int {
      const int jb = s.s0 - 2 + 32 * tau;
      const int r_lo = max(0, -jb), r_hi = min(32, p.F - jb);
      if (r_hi <= r_lo) {
        if (ptid == 0) mbar_arrive(rawbar);
        return 0;
      }
      const float* src = p.mags + ((size_t)s.b * p.F + jb + r_lo) * NB;
      const uintptr_t a = reinterpret_cast<uintptr_t>(src);
      const int off = (int)((a & 15) >> 2);
      const uint32_t bytes = (uint32_t)(((off + (r_hi - r_lo) * NB) * 4 + 15) & ~15);
      const uintptr_t a_al = a & ~(uintptr_t)15;
      if (a_al >= reinterpret_cast<uintptr_t>(p.mags) &&
          a_al + bytes <= reinterpret_cast<uintptr_t>(mags_end)) {
        if (ptid == 0) {
          mbar_expect_tx(rawbar, bytes);
          tma_bulk_g2s(s_raw, reinterpret_cast<const void*>(a_al), bytes, rawbar);
        }
        return off - r_lo * NB;
      }
      for (int e = ptid; e < (r_hi - r_lo) * NB; e += PT) cp_async4(s_raw + e, src + e);
      cp_async_wait_all();
      named_bar(bar_id, PT);
      if (ptid == 0) mbar_arrive(rawbar);
      return -r_lo * NB;
    };
    // iterator over the CTA's production tiles: (segment, tau), global index P
    struct It {
      long long g;     // frames consumed by next_seg so far
      Seg sg;
      int tau, P;
      bool ok;
    };
    auto it_begin = [&]() {
      It it;
      it.g = g_lo; it.tau = 0; it.P = 0;
      it.ok = next_seg(it.g, g_hi, p.F, it.sg);
      return it;
    };
    auto it_next = [&](It& it) {
      ++it.P;
      if (++it.tau >= it.sg.nP) {
        it.tau = 0;
        it.ok = next_seg(it.g, g_hi, p.F, it.sg);
      }
    };
    It cur = it_begin();
    for (int i = 0; i < grp && cur.ok; ++i) it_next(cur);
    int roff = 0;
    if (cur.ok) roff = prefetch(cur.sg, cur.tau);
    int n_mine = 0;                                   // tiles this group has staged
    NR_TIMING_DECL;
    while (cur.ok) {
      NR_LAP(7);
      It nxt = cur;
      for (int i = 0; i < PROD_GROUPS && nxt.ok; ++i) it_next(nxt);
      const Seg& sg = cur.sg;
      const int P = cur.P, slot = P % SLOTS;
      const int jb = sg.s0 - 2 + 32 * cur.tau;
      // A. exp_sigmoid in place on the raw rows (synths.py:176-177); rows of frames
      //    outside [0, F) hold nothing and are forced to zero taps below
      mbar_wait(rawbar, n_mine & 1);
      NR_LAP(0);
      const bool row_ok = (jb + lane >= 0) && (jb + lane < p.F);
      if (p.raw && row_ok) {
        float* src = s_raw + roff + lane * NB + iw * 17;
        float v[17];
#pragma unroll
        for (int k = 0; k < 17; ++k) v[k] = (iw * 17 + k < NB) ? src[k] : 0.f;
#pragma unroll
        for (int k = 0; k < 17; ++k) v[k] = exp_sigmoid_f(v[k] + p.bias);
#pragma unroll
        for (int k = 0; k < 17; ++k)
          if (iw * 17 + k < NB) src[k] = v[k];
      }
      named_bar(bar_id, PT);       // rows complete
      ++n_mine;
      NR_LAP(1);
      // the tile's noise rows (C. below): 512 quads, 128 per warp
      const float* nzb = p.noise ? p.noise + (size_t)sg.b * p.N : nullptr;
      const uint32_t item = (uint32_t)(sg.b + p.item_base);
      const long long p_lo = (long long)jb * FRAME;
      const bool interior = (jb >= 0) && (jb + 32 <= p.F) &&
                            (p_lo + 32ll * FRAME <= p.N) && !nzb;
      constexpr int PER = 32 * NQ / 4;                 // 128 quads per warp
      // B. the cosine sums as FP64 tensor-core products (see ir_kk): warp iw takes the
      //    frames of m-tile iw / 2 and the n-tiles 2 (iw % 2), 2 (iw % 2) + 1 of both
      //    halves; warps 1 and 3 also the n = 32 column of E.  Magnitude rows of
      //    frames outside [0, F) are read from the buffer's start and their taps
      //    forced to zero below; k past 64 (the even half's padding) reads zero.
      {
        const int g = lane >> 2, t = lane & 3;
        const int ntb = 2 * (iw & 1);
        const bool mid = iw & 1;
        const int f0 = 16 * (iw >> 1) + g, f1 = f0 + 8;
        const bool ok0 = (jb + f0 >= 0) && (jb + f0 < p.F);
        const bool ok1 = (jb + f1 >= 0) && (jb + f1 < p.F);
        const float* m0 = ok0 ? s_raw + roff + f0 * NB : s_raw;
        const float* m1 = ok1 ? s_raw + roff + f1 * NB : s_raw;
        const double* tb = sm.ctab + lane;
        double aE[3][4], aO[2][4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          aE[0][c] = aE[1][c] = aE[2][c] = 0.0;
          aO[0][c] = aO[1][c] = 0.0;
        }
#pragma unroll
        for (int s = 0; s < E_STEPS; ++s) {
          const int k = 2 * ir_kk(s, t);
          const bool kin = s < E_STEPS - 1 || k < NB;
          const double e0 = kin ? (double)m0[k] : 0.0, e1 = kin ? (double)m1[k] : 0.0;
          dmma_16x8x4(aE[0], e0, e1, tb[(s * E_NT + ntb) * 32]);
          dmma_16x8x4(aE[1], e0, e1, tb[(s * E_NT + ntb + 1) * 32]);
          if (mid) dmma_16x8x4(aE[2], e0, e1, tb[(s * E_NT + 4) * 32]);
          if (s < O_STEPS) {
            const double o0 = m0[k + 1], o1 = m1[k + 1];
            dmma_16x8x4(aO[0], o0, o1, tb[TAB_E + (s * O_NT + ntb) * 32]);
            dmma_16x8x4(aO[1], o0, o1, tb[TAB_E + (s * O_NT + ntb + 1) * 32]);
          }
        }
        NR_LAP(3);
        named_bar(bar_id, PT);     // the group is done reading the rows
        if (nxt.ok) roff = prefetch(nxt.sg, nxt.tau);
        NR_LAP(4);
        // Only now does the group need its ring slot: the sums above live in registers.
        if (P >= SLOTS) mbar_wait(&sm.empty[slot], ((P / SLOTS) - 1) & 1);
        NR_LAP(2);
        // h0[n] = E + O and h0[64 - n] = E - O, each rounded to float once, times the
        // periodic Hann window (win[128 - i] == win[i]): taps 64 +- n and n, 128 - n
        float* hs = sm.h + slot * 32 * HS + HPAD;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int n = 8 * (ntb + j) + 2 * t;          // this lane's columns n, n + 1
          const float2 wp = *reinterpret_cast<const float2*>(sm.win + SHIFT + n);
          const float2 wm = *reinterpret_cast<const float2*>(sm.win + n);
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const bool ok = r ? ok1 : ok0;
            float* hr = hs + (r ? f1 : f0) * HS;
            const double E0 = aE[j][2 * r], E1 = aE[j][2 * r + 1];
            const double O0 = aO[j][2 * r], O1 = aO[j][2 * r + 1];
            const float p0 = ok ? wp.x * (float)(E0 + O0) : 0.f;
            const float p1 = ok ? wp.y * (float)(E1 + O1) : 0.f;
            const float q0 = ok ? wm.x * (float)(E0 - O0) : 0.f;
            const float q1 = ok ? wm.y * (float)(E1 - O1) : 0.f;
            *reinterpret_cast<float2*>(hr + SHIFT + n) = make_float2(p0, p1);
            hr[SHIFT - n] = p0;
            hr[SHIFT - n - 1] = p1;
            *reinterpret_cast<float2*>(hr + n) = make_float2(q0, q1);
            if (n != 0) hr[S - n] = q0;                  // tap 128 does not exist
            hr[S - n - 1] = q1;
          }
        }
        if (mid && t == 0) {                             // n = 32: taps 32 and 96
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const float v = (r ? ok1 : ok0) ? sm.win[Q] * (float)aE[2][2 * r] : 0.f;
            float* hr = hs + (r ? f1 : f0) * HS;
            hr[Q] = v;
            hr[S - Q] = v;
          }
        }
      }
      NR_LAP(5);
      // C. the tile's noise rows
      {
        float* xs = sm.x + slot * 32 * XS;
        if (interior) {
          const uint32_t qbase = (uint32_t)(p_lo >> 2);
#pragma unroll
          for (int it = 0; it < PER / 32; ++it) {
            const int e = iw * PER + it * 32 + lane;
            const int r = e >> 4, qd = e & 15;
            const float4 v = noise4(qbase + (uint32_t)e, item, p.seed, p.offset);
            float2* d = reinterpret_cast<float2*>(xs + r * XS + 4 * qd);
            d[0] = make_float2(v.x, v.y);
            d[1] = make_float2(v.z, v.w);
          }
        } else {
          for (int it = 0; it < PER / 32; ++it) {
            const int e = iw * PER + it * 32 + lane;
            const int r = e >> 4, qd = e & 15;
            const int j = jb + r;
            const long long pp = (long long)j * FRAME + 4 * qd;
            float v[4] = {0.f, 0.f, 0.f, 0.f};
            if (j >= 0 && j < p.F && pp < p.N) {
              if (nzb) {
#pragma unroll
                for (int u = 0; u < 4; ++u) if (pp + u < p.N) v[u] = nzb[pp + u];
              } else {
                const float4 r4 = noise4((uint32_t)(pp >> 2), item, p.seed, p.offset);
                v[0] = r4.x;
                if (pp + 1 < p.N) v[1] = r4.y;
                if (pp + 2 < p.N) v[2] = r4.z;
                if (pp + 3 < p.N) v[3] = r4.w;
              }
            }
            float2* d = reinterpret_cast<float2*>(xs + r * XS + 4 * qd);
            d[0] = make_float2(v[0], v[1]);
            d[1] = make_float2(v[2], v[3]);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.full[slot]);
      NR_LAP(6);
      cur = nxt;
    }
  }
}

}  // namespace nr_

inline bool noise_ring_supported(int F, int nb, int N, int window_size) {
  if (nb != nr_::NB) return false;
  if (N % F != 0 || N / F != nr_::FRAME) return false;
  IrGeom g = make_ir_geom(nb, window_size);
  return !g.padded && g.S == nr_::S;
}

inline int launch_noise_ring(const float* mags, const float* noise, uint64_t seed,
                             uint64_t offset, float* audio, int B, int F, int N,
                             int accumulate, cudaStream_t st, int raw, float bias,
                             int item_base, int overlap_previous = 0) {
  nr_::Params p;
  p.mags = mags; p.noise = noise; p.audio = audio; p.seed = seed; p.offset = offset;
  p.B = B; p.F = F; p.N = N; p.accumulate = accumulate; p.raw = raw; p.bias = bias;
  p.item_base = item_base;
  const long long T = (long long)B * F;
  const size_t smem = sizeof(nr_::Smem);
  static_assert(sizeof(nr_::Smem) <= 227 * 1024, "noise_ring shared memory");
  int rc = set_smem(nr_::noise_ring_kernel, smem, "filtered_noise_forward");
  if (rc) return rc;
  // one persistent CTA per SM; tiny workloads get one CTA per 32-frame tile
  const int grid = (int)std::max<long long>(
      1, std::min<long long>((long long)num_sms(), (T + 31) / 32));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(nr_::THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  // Programmatic dependent launch (decoder path): let this grid's CTAs start on
  // SMs the harmonic kernel has already vacated - tables, TMA, the first impulse
  // responses and noise rows do not depend on it; the consumers wait
  // (griddepcontrol.wait) before their first add into the audio buffer.
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = overlap_previous ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, nr_::noise_ring_kernel, p);
  if (e != cudaSuccess) {
    set_error("filtered_noise_forward(ring): launch failed: %s", cudaGetErrorString(e));
    return DDSP_B200_E_CUDA;
  }
  DDSP_CHECK_LAUNCH("filtered_noise_forward(ring)");
  return 0;
}

// noise_ring for the decoder shape (65 bands, 64-sample frames, 128 taps), the
// generic fused kernel (noise_fused.cuh) for every other shape it supports.
inline int launch_noise_best(const float* mags, const float* noise, uint64_t seed,
                             uint64_t offset, float* audio, int B, int F, int nb,
                             int N, int window_size, int accumulate,
                             cudaStream_t st, int raw = 0, float bias = 0.f,
                             int item_base = 0, int overlap_previous = 0) {
  if (noise_ring_supported(F, nb, N, window_size))
    return launch_noise_ring(mags, noise, seed, offset, audio, B, F, N, accumulate,
                             st, raw, bias, item_base, overlap_previous);
  return launch_noise_fused(mags, noise, seed, offset, audio, B, F, nb, N,
                            window_size, accumulate, st, raw, bias, item_base);
}

}  // namespace ddsp
