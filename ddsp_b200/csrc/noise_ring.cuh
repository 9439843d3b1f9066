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
//     of frames q-2 .. q+1; a warp finishes its 32 x 32 output block in registers
//     and writes it straight to HBM (st / red.add for the fused Add) - consumer
//     warps never talk to each other.
//   * ROW RING, NO HALO.  A persistent CTA walks a contiguous range of frames; the
//     impulse responses and noise rows live in a ring of eight 32-row slots in shared
//     memory (lane-private rows, strides = 2 mod 4 floats: conflict-free LDS.64),
//     so neighbouring tiles share their edge rows instead of recomputing them.
//   * TWO ACCUMULATOR SETS ON ONE TAP PAIR.  For an even input x[i] the tap pair
//     (h[m], h[m+1]) feeds the output pair (n, n+1); for the odd input x[i+1] the
//     SAME pair feeds (n+1, n+2).  Set A holds pairs (n, n+1), set B pairs
//     (n+1, n+2): every MAC is an f32x2 FMA with a broadcast scalar input and ONE
//     copy of the impulse response in shared memory.
//   * TAP-STATIONARY ORDER.  The 16 input pairs of a body sit in registers and the
//     tap pairs stream through: a pair serves every (output, input) combination on
//     its diagonal, so up to 32 consecutive f32x2 FMAs share their multiplicand
//     (the earlier sliding 16-pair tap window changed it every other instruction).
//   * TRIANGULAR TRIMMING at compile time: the rows of frames q+1 and q-1 cover
//     complementary triangles of the (n, i) square; fully unrolled bodies skip the
//     pairs whose taps are all out of range.
//   * producers: two groups of 4 warps alternate tiles; a group takes its tile
//     from raw magnitudes (TMA) through exp_sigmoid, the cosine sums (odd k, and the
//     even k split once more by quarter-wave symmetry: 1601 MACs per frame instead
//     of 4225; in registers as f32x2, no exchange) and the windowed taps to the
//     Philox rows, and asks for its ring slot only when the sums are done.
#pragma once
#include "noise_fused.cuh"

namespace ddsp {

namespace nr_ {
constexpr int NB = 65, FRAME = 64, S = 128, S0 = 128, Q = 32, QP = 36;
constexpr int NE = 33, NO = 32, SHIFT = 64;
// A consumer warp owns a UNIT of 2 NW outputs of 32 frames: NW input pairs in
// registers, NW + NW + 1 packed accumulators.  NW = 16 (two units per frame, ~150
// registers, 9 KB FIR bodies) is the product; NW = 8 (four units, 96 registers,
// twice the shared-memory loads per FMA) compiles (-DDDSP_NR_NW=8) as an
// alternative for A/B timing.
#ifndef DDSP_NR_NW
#define DDSP_NR_NW 16
#endif
constexpr int NW = DDSP_NR_NW;
constexpr int UPT = FRAME / (2 * NW);              // units per 64-sample frame
// Producer groups and ring slots.  The four consumer tile groups hold NTG + 1 = 5
// slots between them; what is left decouples producers from consumers.  227 KB of
// shared memory hold 7 slots next to three raw-magnitude staging buffers or 8 next
// to two; the default is 2 groups / 8 slots.
#ifndef DDSP_NR_PROD_GROUPS
#define DDSP_NR_PROD_GROUPS 2
#endif
#ifndef DDSP_NR_MAX_SLOTS
#define DDSP_NR_MAX_SLOTS 8
#endif
constexpr int CONS_WARPS = 8, PROD_GROUPS = DDSP_NR_PROD_GROUPS, PROD_WARPS = 4 * PROD_GROUPS;
constexpr int NTG = CONS_WARPS / UPT;              // consumption tiles in flight
static_assert((NTG & (NTG - 1)) == 0, "tile groups: a power of two");
constexpr int SLOTS = DDSP_NR_MAX_SLOTS;
constexpr int RING = 32 * SLOTS;
constexpr int THREADS = 32 * (CONS_WARPS + PROD_WARPS);
// NW = 16 only: 512 threads launch with 128 registers each (the whole file); the
// consumers (256 threads) grow to CONS_REGS out of what the producers (256 threads)
// give back: CONS_REGS + PROD_REGS <= 256.  On sm_90a the producers spill a little
// at 88 (fewer bytes at 96 or 104); the three splits time the same on H100
// (DESIGN.md 3.2).  (Three groups: 640 threads at 96,
// 144 / 64.  A split that leaves setmaxnreg.inc short of registers hangs the CTA.)
#ifndef DDSP_NR_PROD_REGS
#define DDSP_NR_PROD_REGS 88
#endif
#ifndef DDSP_NR_CONS_REGS
#define DDSP_NR_CONS_REGS 168
#endif
static_assert(DDSP_NR_NW != 16 ||
                  8 * DDSP_NR_CONS_REGS + 4 * DDSP_NR_PROD_GROUPS * DDSP_NR_PROD_REGS <= 2048,
              "noise_ring register split exceeds the SM's 64 K registers");
constexpr int CONS_REGS = (NW == 16) ? DDSP_NR_CONS_REGS : 0, PROD_REGS = DDSP_NR_PROD_REGS;
constexpr int HPAD = 2, HS = 134, XS = 66, MS = 65;   // row strides (floats)
constexpr int NQ = FRAME / 4;

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
  float te[NE * QP];
  float to[NO * QP];
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

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c,
                                           float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a),
               "f"(b), "f"(c), "f"(d)
               : "memory");
}

// ---- consumer: FIR bodies ---------------------------------------------------
// Set A's pair c holds outputs (N0 + 2c, N0 + 2c + 1), set B's pair c outputs
// (N0 + 2c + 1, N0 + 2c + 2); Bm1 is set B's pair c = -1 (outputs N0 - 1, N0).
struct Acc {
  float2 A[NW], B[NW], Bm1;
};

// The FIR of one unit runs as a short PROGRAM of NW-step bodies, executed by a
// loop with a switch so that each body exists once in the instruction stream
// (fully inlined, 80 KB of consumer code stalled on instruction fetch).
// A body covers NW steps k of one row: inputs xp[2k], xp[2k+1]; the tap pair that
// takes them to accumulator pair c is P(c - k) = (h[m], h[m+1]) at hp + 2 (c - k).
//   FULL : every pair (c, k) matters.
//   LOWER: only c >= k + 1 (taps left of the row start are zero), NW - 1 steps.
//   UPPER: only c <= k (taps right of the row end are zero).
enum { OP_FULL = 0, OP_LOWER = 1, OP_UPPER = 2 };
struct Op {
  const float* xp;
  const float* hp;
  int kind;
  int set_xo;       // xo_prev := xo before the body
  float xo;
  int final_op;     // afterwards: Bm1 += xo_prev * P(-NW)  (the last odd input)
};
constexpr int N_OPS = 2 * UPT + 1;

// Op i of unit u (outputs N0 = 2 NW u ..).  x_m1 / h_m1: rows of frame q+1 (tap
// offset C = -2); x_0 / h_0: frame q (C = 62); x_p1 / h_p1: frame q-1 (C = 126).
// h_* point at tap 0.  Body j of a row covers inputs 2 NW j .. 2 NW (j+1) - 1.
//   frame q  : UPT FULL bodies (every (n, i) pair is in range); the closing op
//              (x[63] with taps (N0-2, N0-1)) is all padding for N0 = 0.
//   frame q+1: reaches outputs n >= i + 2: u FULL bodies, then the shrinking
//              triangle.
//   frame q-1: covers i >= n - 1: the growing triangle in body u (entered with
//              x[N0-1] -> output N0), then FULL bodies to the end of the row.
__device__ __forceinline__ Op block_op(int i, int u, const float* x_m1,
                                       const float* h_m1, const float* x_0,
                                       const float* h_0, const float* x_p1,
                                       const float* h_p1) {
  const int N0 = 2 * NW * u;
  if (i < UPT)
    return Op{x_0 + 2 * NW * i, h_0 + N0 + 62 - 2 * NW * i, OP_FULL, i == 0, 0.f,
              (i == UPT - 1) && (N0 != 0)};
  i -= UPT;
  if (i < u)
    return Op{x_m1 + 2 * NW * i, h_m1 + N0 - 2 - 2 * NW * i, OP_FULL, i == 0, 0.f, 0};
  if (i == u) return Op{x_m1 + N0, h_m1 - 2, OP_LOWER, u == 0, 0.f, 0};
  i -= 1;                                              // body index in frame q-1
  if (i == u)
    return Op{x_p1 + N0, h_p1 + 126, OP_UPPER, 1, (u > 0) ? x_p1[N0 - 1] : 0.f,
              u == UPT - 1};
  return Op{x_p1 + 2 * NW * i, h_p1 + N0 + 126 - 2 * NW * i, OP_FULL, 0, 0.f,
            i == UPT - 1};
}

// TAP-STATIONARY ORDER: the NW input pairs of a body sit in registers and the tap
// pairs stream through - a pair P(d) at hp + 2 d serves every (c, k) with c - k = d,
// so up to 2 NW consecutive f32x2 FMAs share their multiplicand (the operand
// collector keeps it).  Bm1 (= B[-1]) takes x[2k - 1] through P(-k).
__device__ __forceinline__ void consume_block(Acc& a, int u, const float* x_m1,
                                                 const float* h_m1, const float* x_0,
                                                 const float* h_0, const float* x_p1,
                                                 const float* h_p1) {
  float xo_prev = 0.f;
  constexpr int M = NW - 1;
#pragma unroll 1
  for (int i = 0; i < N_OPS; ++i) {
    const Op op = block_op(i, u, x_m1, h_m1, x_0, h_0, x_p1, h_p1);
    const float* __restrict__ xp = op.xp;
    const float* __restrict__ hp = op.hp;
    float2 X[NW];
#pragma unroll
    for (int k = 0; k < NW; ++k) X[k] = *reinterpret_cast<const float2*>(xp + 2 * k);
    if (op.set_xo) xo_prev = op.xo;
    switch (op.kind) {
      case OP_FULL:
#pragma unroll
        for (int d = M; d >= -M; --d) {
          const float2 P = *reinterpret_cast<const float2*>(hp + 2 * d);
#pragma unroll
          for (int k = (d < 0 ? -d : 0); k <= (d > 0 ? M - d : M); ++k) {
            a.A[k + d] = nf_ffma2(X[k].x, P, a.A[k + d]);
            a.B[k + d] = nf_ffma2(X[k].y, P, a.B[k + d]);
          }
          if (d <= 0) a.Bm1 = nf_ffma2(d == 0 ? xo_prev : X[d < 0 ? -d - 1 : 0].y, P, a.Bm1);
        }
        xo_prev = X[M].y;
        break;
      case OP_LOWER:
#pragma unroll
        for (int d = M; d >= 1; --d) {
          const float2 P = *reinterpret_cast<const float2*>(hp + 2 * d);
#pragma unroll
          for (int k = 0; k <= M - d; ++k) {
            a.A[k + d] = nf_ffma2(X[k].x, P, a.A[k + d]);
            a.B[k + d] = nf_ffma2(X[k].y, P, a.B[k + d]);
          }
        }
        xo_prev = X[M - 1].y;
        break;
      default:
#pragma unroll
        for (int d = 0; d >= -M; --d) {
          const float2 P = *reinterpret_cast<const float2*>(hp + 2 * d);
#pragma unroll
          for (int k = -d; k <= M; ++k) {
            a.A[k + d] = nf_ffma2(X[k].x, P, a.A[k + d]);
            a.B[k + d] = nf_ffma2(X[k].y, P, a.B[k + d]);
          }
          a.Bm1 = nf_ffma2(d == 0 ? xo_prev : X[d < 0 ? -d - 1 : 0].y, P, a.Bm1);
        }
        xo_prev = X[M].y;
        break;
    }
    if (op.final_op)
      a.Bm1 = nf_ffma2(xo_prev, *reinterpret_cast<const float2*>(hp - 2 * NW), a.Bm1);
  }
}
__global__ void __launch_bounds__(nr_::THREADS, 1)
noise_ring_kernel(Params p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float invS0 = 1.0f / (float)S0;

  // ---- once: tables, window, zeroed ring (pads stay zero), barriers ----
  for (int e = tid; e < NE * QP; e += THREADS) {
    const int k = e / QP, n = e - k * QP;
    const int ph = (2 * k * n) % S0;
    const float ck = (k == 0 || 2 * k == NB - 1) ? invS0 : 2.0f * invS0;
    sm.te[e] = (n <= Q) ? ck * cospif(2.0f * (float)ph * invS0) : 0.f;
  }
  for (int e = tid; e < NO * QP; e += THREADS) {
    // odd-k table, laid out by producer warp: columns 8 w + c hold n = 4 w + c
    // (c < 4) and its mirror n = 32 - 4 w - (c - 4) (c >= 4); column 32 holds n = 16
    const int k = e / QP, col = e - k * QP;
    int n = -1;
    if (col < 32) {
      const int w = col >> 3, c = col & 7;
      n = (c < 4) ? 4 * w + c : 32 - 4 * w - (c - 4);
    } else if (col == 32) {
      n = 16;
    }
    const int ph = ((2 * k + 1) * max(n, 0)) % S0;
    sm.to[e] = (n >= 0) ? 2.0f * invS0 * cospif(2.0f * (float)ph * invS0) : 0.f;
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
      mbar_init(&sm.full[i], 4);
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
    if (CONS_REGS != 0)   // NW = 16: the FIR wants ~150 registers, from the producers
      asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONS_REGS ? CONS_REGS : 96));
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
        auto xrow = [&](int r) { return sm.x + ((rbase + r) % RING) * XS; };
        auto hrow = [&](int r) { return sm.h + ((rbase + r) % RING) * HS + HPAD; };
        Acc a;
#pragma unroll
        for (int c = 0; c < NW; ++c) a.A[c] = a.B[c] = make_float2(0.f, 0.f);
        a.Bm1 = make_float2(0.f, 0.f);
        consume_block(a, unit, xrow(rho + 1), hrow(rho + 1), xrow(rho), hrow(rho),
                      xrow(rho - 1), hrow(rho - 1));
        // frame q-2 reaches output 0 only: input 63 through tap 127
        if (unit == 0)
          a.A[0].x = fmaf(xrow(rho - 2)[63], hrow(rho - 2)[127], a.A[0].x);
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
        // ---- store / accumulate this lane's 2 NW outputs ----
        if (!dep_done) {
          // programmatic dependent launch: this grid may have started while the
          // harmonic kernel was still draining; its audio must be complete (and
          // visible) before the first add lands.  No-op for a plain launch.
          asm volatile("griddepcontrol.wait;" ::: "memory");
          dep_done = true;
        }
        if (q_rel < sg.len) {
          constexpr int NOUT = 2 * NW;
          const long long t0 = (long long)(sg.s0 + q_rel) * FRAME + NOUT * unit;
          float* o = p.audio + (size_t)sg.b * p.N + t0;
          float v[NOUT];
#pragma unroll
          for (int c = 0; c < NW; ++c) {
            const float2 bp = (c == 0) ? a.Bm1 : a.B[c - 1];
            v[2 * c] = a.A[c].x + bp.y;
            v[2 * c + 1] = a.A[c].y + a.B[c].x;
          }
          if (t0 + NOUT <= p.N && (reinterpret_cast<uintptr_t>(o) & 15) == 0) {
#pragma unroll
            for (int w4 = 0; w4 < NOUT / 4; ++w4) {
              if (p.accumulate)
                red_add_v4(o + 4 * w4, v[4 * w4], v[4 * w4 + 1], v[4 * w4 + 2],
                           v[4 * w4 + 3]);
              else
                *reinterpret_cast<float4*>(o + 4 * w4) =
                    make_float4(v[4 * w4], v[4 * w4 + 1], v[4 * w4 + 2], v[4 * w4 + 3]);
            }
          } else {
#pragma unroll
            for (int w1 = 0; w1 < NOUT; ++w1) {
              if (t0 + w1 < p.N) {
                if (p.accumulate) o[w1] += v[w1]; else o[w1] = v[w1];
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
    if (CONS_REGS != 0)
      asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PROD_REGS));
    // PROD_GROUPS groups of four warps; group g builds the production tiles P = g
    // (mod PROD_GROUPS) end to end: magnitudes (TMA) -> exp_sigmoid (in place) ->
    // both cosine half-sums -> windowed taps, then the tile's noise rows.  A group
    // has PROD_GROUPS tile periods for one tile, so its latency chains (TMA, MUFU,
    // LDS) stay off the consumers' critical path.
    const int grp = (warp - CONS_WARPS) >> 2;
    const int iw = (warp - CONS_WARPS) & 3;           // column block / slice
    const int ptid = tid - (CONS_WARPS + 4 * grp) * 32;   // 0..127 within the group
    constexpr int PT = 128;
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
      const float* mrow = row_ok ? s_raw + roff + lane * NB : s_raw;
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
      // B. the cosine sums, with the quarter-wave symmetry of the even-k half:
      //    h0[n] = E[n] + O[n], h0[64 - n] = E[n] - O[n] (SURVEY A.5), and, splitting
      //    the even k = 2 j by the parity of j, E[n] = EE[n] + EO[n], E[32 - n] =
      //    EE[n] - EO[n]: 289 + 256 + 1056 MACs per frame instead of 1089 + 1024.
      //    Warp w owns n = 4 w .. 4 w + 3 and their mirrors 32 - n (warp 3 also the
      //    self-mirrored n = 16, where EO vanishes).
      {
        const int c0 = 4 * iw;
        float2 aEE[2], aEO[2], aOa[2], aOb[2];
        float ee16 = 0.f, o16 = 0.f;
#pragma unroll
        for (int c = 0; c < 2; ++c) aEE[c] = aEO[c] = aOa[c] = aOb[c] = make_float2(0.f, 0.f);
        // Software-pipelined over groups of four k (two register sets: the loads of
        // group j2 + 1 are in flight while group j2 is multiplied); volatile loads so
        // that their order and their distinct destinations stay.
        struct Term { float m0, m1, m2, m3; float4 e0, e1, oa0, ob0, oa1, ob1; };
        auto load_term = [&](Term& t, int j2) {
          const float* pm = mrow + 4 * j2;               // k = 4 j2 .. 4 j2 + 3
          const float* pe = sm.te + (2 * j2) * QP + c0;
          const float* po = sm.to + (2 * j2) * QP + 8 * iw;
          t.m0 = lds32v(pm); t.m1 = lds32v(pm + 1);
          t.m2 = lds32v(pm + 2); t.m3 = lds32v(pm + 3);
          t.e0 = lds128v(pe); t.e1 = lds128v(pe + QP);
          t.oa0 = lds128v(po); t.ob0 = lds128v(po + 4);
          t.oa1 = lds128v(po + QP); t.ob1 = lds128v(po + QP + 4);
        };
        auto mac_term = [&](const Term& t, int j2) {
          aEE[0] = nf_ffma2(t.m0, make_float2(t.e0.x, t.e0.y), aEE[0]);
          aEE[1] = nf_ffma2(t.m0, make_float2(t.e0.z, t.e0.w), aEE[1]);
          aOa[0] = nf_ffma2(t.m1, make_float2(t.oa0.x, t.oa0.y), aOa[0]);
          aOa[1] = nf_ffma2(t.m1, make_float2(t.oa0.z, t.oa0.w), aOa[1]);
          aOb[0] = nf_ffma2(t.m1, make_float2(t.ob0.x, t.ob0.y), aOb[0]);
          aOb[1] = nf_ffma2(t.m1, make_float2(t.ob0.z, t.ob0.w), aOb[1]);
          aEO[0] = nf_ffma2(t.m2, make_float2(t.e1.x, t.e1.y), aEO[0]);
          aEO[1] = nf_ffma2(t.m2, make_float2(t.e1.z, t.e1.w), aEO[1]);
          aOa[0] = nf_ffma2(t.m3, make_float2(t.oa1.x, t.oa1.y), aOa[0]);
          aOa[1] = nf_ffma2(t.m3, make_float2(t.oa1.z, t.oa1.w), aOa[1]);
          aOb[0] = nf_ffma2(t.m3, make_float2(t.ob1.x, t.ob1.y), aOb[0]);
          aOb[1] = nf_ffma2(t.m3, make_float2(t.ob1.z, t.ob1.w), aOb[1]);
          if (iw == 3) {
            ee16 = fmaf(t.m0, sm.te[(2 * j2) * QP + 16], ee16);
            o16 = fmaf(t.m1, sm.to[(2 * j2) * QP + 32], o16);
            o16 = fmaf(t.m3, sm.to[(2 * j2 + 1) * QP + 32], o16);
          }
        };
        Term tA, tB;
        load_term(tA, 0);
#pragma unroll 1
        for (int j2 = 0; j2 < NO / 2; j2 += 2) {
          load_term(tB, j2 + 1);
          mac_term(tA, j2);
          // j2 + 2 = 16 is k = 64, the last even-even term: the rest of that group is
          // read (table rows past the end run into the next array, mrow[65 .. 67] into
          // the next row / the pad) and never used
          load_term(tA, j2 + 2);
          mac_term(tB, j2 + 1);
        }
        aEE[0] = nf_ffma2(tA.m0, make_float2(tA.e0.x, tA.e0.y), aEE[0]);
        aEE[1] = nf_ffma2(tA.m0, make_float2(tA.e0.z, tA.e0.w), aEE[1]);
        if (iw == 3) ee16 = fmaf(tA.m0, sm.te[NO * QP + 16], ee16);
        NR_LAP(3);
        named_bar(bar_id, PT);     // the group is done reading the rows
        if (nxt.ok) roff = prefetch(nxt.sg, nxt.tau);
        NR_LAP(4);
        // Only now does the group need its ring slot: the sums above live in registers.
        if (P >= SLOTS) mbar_wait(&sm.empty[slot], ((P / SLOTS) - 1) & 1);
        NR_LAP(2);
        float* hr = sm.h + (slot * 32 + lane) * HS + HPAD;
        const float EEv[4] = {aEE[0].x, aEE[0].y, aEE[1].x, aEE[1].y};
        const float EOv[4] = {aEO[0].x, aEO[0].y, aEO[1].x, aEO[1].y};
        const float OA[4] = {aOa[0].x, aOa[0].y, aOa[1].x, aOa[1].y};
        const float OB[4] = {aOb[0].x, aOb[0].y, aOb[1].x, aOb[1].y};
        // window values as 16-byte loads: the periodic Hann window has win[128 - i] ==
        // win[i], so the mirrors' win[64 + (32 - n)] = win[32 + n], win[32 - n] = win[96 + n]
        const float4 wpa4 = *reinterpret_cast<const float4*>(sm.win + SHIFT + c0);
        const float4 wma4 = *reinterpret_cast<const float4*>(sm.win + c0);
        const float4 wpb4 = *reinterpret_cast<const float4*>(sm.win + Q + c0);
        const float4 wmb4 = *reinterpret_cast<const float4*>(sm.win + SHIFT + Q + c0);
        const float WPA[4] = {wpa4.x, wpa4.y, wpa4.z, wpa4.w}, WMA[4] = {wma4.x, wma4.y, wma4.z, wma4.w};
        const float WPB[4] = {wpb4.x, wpb4.y, wpb4.z, wpb4.w}, WMB[4] = {wmb4.x, wmb4.y, wmb4.z, wmb4.w};
        float vpa[4], vma[4], vpb[4], vmb[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float Ea = EEv[c] + EOv[c], Eb = EEv[c] - EOv[c];     // E[n], E[32 - n]
          vpa[c] = row_ok ? WPA[c] * (Ea + OA[c]) : 0.f;   // n:      taps 64 +- n
          vma[c] = row_ok ? WMA[c] * (Ea - OA[c]) : 0.f;   //         taps n, 128 - n
          vpb[c] = row_ok ? WPB[c] * (Eb + OB[c]) : 0.f;   // 32 - n: taps 96 - n, 32 + n
          vmb[c] = row_ok ? WMB[c] * (Eb - OB[c]) : 0.f;   //         taps 32 - n, 96 + n
        }
        // v[c] to hr[base + c] / hr[base - c]; 8-byte stores where the pair starts even
        auto st_up = [&](int base, const float* v) {
          *reinterpret_cast<float2*>(hr + base) = make_float2(v[0], v[1]);
          *reinterpret_cast<float2*>(hr + base + 2) = make_float2(v[2], v[3]);
        };
        auto st_down = [&](int base, const float* v, bool first) {
          if (first) hr[base] = v[0];
          *reinterpret_cast<float2*>(hr + base - 2) = make_float2(v[2], v[1]);
          hr[base - 3] = v[3];
        };
        st_up(SHIFT + c0, vpa);                          // 64 + n
        st_down(SHIFT - c0, vpa, true);                  // 64 - n
        st_up(c0, vma);                                  // n
        st_down(S - c0, vma, c0 != 0);                   // 128 - n (tap 128 does not exist)
        st_down(SHIFT + Q - c0, vpb, true);              // 64 + (32 - n)
        st_up(Q + c0, vpb);                              // 64 - (32 - n)
        st_down(Q - c0, vmb, true);                      // 32 - n
        st_up(SHIFT + Q + c0, vmb);                      // 128 - (32 - n)
        if (iw == 3) {                                   // n = 16
          const float vp16 = row_ok ? sm.win[SHIFT + 16] * (ee16 + o16) : 0.f;
          const float vm16 = row_ok ? sm.win[16] * (ee16 - o16) : 0.f;
          hr[SHIFT + 16] = vp16;
          hr[SHIFT - 16] = vp16;
          hr[16] = vm16;
          hr[S - 16] = vm16;
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
  cudaError_t e = cudaFuncSetAttribute(
      nr_::noise_ring_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) {
    set_error("filtered_noise_forward: cannot reserve %zu B smem: %s", smem,
              cudaGetErrorString(e));
    return DDSP_B200_E_CUDA;
  }
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
  e = cudaLaunchKernelEx(&cfg, nr_::noise_ring_kernel, p);
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
