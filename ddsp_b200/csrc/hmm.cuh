// losses.HmmTranscriber (losses.py:247-345): tfp's HiddenMarkovModel with K states
// (state 0 "off", state j >= 1 MIDI pitch j), observations x_t = (pitch_t, amps_t)
// under MultivariateNormalDiag(loc_j, scale_j), a uniform initial distribution and the
// transition matrix A = hold on the diagonal and other everywhere else.
//
// Structure.  Because A = other * 11^T + (hold - other) I, one step of the forward
// algorithm on a vector w is
//     (A^T w)_j = hold * w_j + other * sum_{i != j} w_i,
// O(K) instead of O(K^2).  Both terms are non-negative, so the step never cancels, even
// for hold < other or hold = 0; sum_{i != j} w_i is S - w_j except at j = argmax w,
// where S - w_j could cancel and the sum is formed without w_j instead.  One CTA runs
// one sequence with a thread per state (blockDim = K rounded up to a warp).
//
// Forward (hmm_log_prob_kernel).  q_t = A^T e_{t-1} (q_0 = 1), a_t = l_t + log q_t,
// M_t = max a_t, e_t = exp(a_t - M_t) (max 1), S_t = sum e_t; log_prob =
// -log K + sum_t M_t + log S_{T-1}, accumulated in FP64 so that T = 1000 costs no
// float32 digits.  Two block reductions per step.
//
// Backward (hmm_backward_kernel).  d x_td = g * sum_j gamma_t(j) * dl_t(j)/dx_td with
// gamma_t proportional to e_t * b_t and b_{t-1} = A (exp(l_t) b_t) (the same structured
// step).  Nothing is stored between the forward and the backward: the kernel re-runs the
// forward, writing q at the start of every `seg` steps to `ckpt` (the caller's
// [B, ceil(T / seg), K] floats, each thread reading back only what it wrote), then walks
// the segments last to first: it recomputes a segment's e_t into shared memory
// (seg x K floats) and scans b back through it.  No atomics: the gradients are
// bit-reproducible.
//
// Viterbi (hmm_viterbi_kernel).  d_t(j) = l_t(j) + max(d_{t-1}(j) + log hold,
// max_{i != j} d_{t-1}(i) + log other), kept relative to max d_{t-1}.  The best other
// state is the argmax i1 of d_{t-1}, or its second best i2 for j = i1, so a back
// pointer is one bit ("stayed") per (t, j) plus (i1, i2) per step, all in shared memory:
// T * (ceil(K / 32) + 1) 32-bit words.  Ties go to the lowest index, in the choice
// between staying and moving and in the final argmax, as np.argmax's do.  Thread 0
// backtracks and writes the int64 path.
#pragma once
#include <math.h>
#include <stdint.h>

#include "common.cuh"

namespace ddsp {
namespace hmm_ {

constexpr int kMaxStates = DDSP_B200_HMM_MAX_STATES;
// Shared floats of the backward's segment buffer: seg * K <= kSegFloats (192 KB).
constexpr int kSegFloats = DDSP_B200_HMM_SEGMENT_FLOATS;
// Shared bytes of the Viterbi back pointers: 4 T (ceil(K / 32) + 1) <= kViterbiBytes.
constexpr size_t kViterbiBytes = DDSP_B200_HMM_VITERBI_BYTES;
constexpr float kLog2Pi = 1.8378770664093453f;

struct Params {
  const float2* obs;    // [B, T] (pitch, amps)
  const float2* loc;    // [K]
  const float2* scale;  // [K]
  int T, K;
  float hold, other;          // transition probabilities
  float log_hold, log_other;  // their logs (-inf for 0)
  double log_init;            // -log K
};

// ---- block reductions -----------------------------------------------------------
// Every reduction combines the warp's values by an xor butterfly (each combine is
// symmetric, so all lanes hold the same bits), then the warps' values in warp order
// from shared memory: one __syncthreads, the same result in every thread, and the
// same order on every run.  Callers alternate two slot arrays, so a slot is rewritten
// only after every thread has passed the barrier that follows its last read.
struct MaxArg { float v; int i; };       // maximum, lowest index on ties
struct Sum2 { float s, sx; };            // sum, and sum without the argmax
struct Top2 { float v1; int i1; float v2; int i2; };   // best and second best
struct Post { float w, wp, wa; MaxArg m; };            // backward: gamma sums + max

__device__ __forceinline__ bool better(float va, int ia, float vb, int ib) {
  return va > vb || (va == vb && ia < ib);
}
__device__ __forceinline__ MaxArg combine(MaxArg a, MaxArg b) {
  return better(a.v, a.i, b.v, b.i) ? a : b;
}
__device__ __forceinline__ Sum2 combine(Sum2 a, Sum2 b) { return {a.s + b.s, a.sx + b.sx}; }
__device__ __forceinline__ Post combine(Post a, Post b) {
  return {a.w + b.w, a.wp + b.wp, a.wa + b.wa, combine(a.m, b.m)};
}
__device__ __forceinline__ Top2 combine(Top2 a, Top2 b) {
  if (better(a.v1, a.i1, b.v1, b.i1))
    return better(a.v2, a.i2, b.v1, b.i1) ? a : Top2{a.v1, a.i1, b.v1, b.i1};
  return better(b.v2, b.i2, a.v1, a.i1) ? b : Top2{b.v1, b.i1, a.v1, a.i1};
}

__device__ __forceinline__ MaxArg shfl(MaxArg x, int o) {
  return {__shfl_xor_sync(~0u, x.v, o), __shfl_xor_sync(~0u, x.i, o)};
}
__device__ __forceinline__ Sum2 shfl(Sum2 x, int o) {
  return {__shfl_xor_sync(~0u, x.s, o), __shfl_xor_sync(~0u, x.sx, o)};
}
__device__ __forceinline__ Post shfl(Post x, int o) {
  return {__shfl_xor_sync(~0u, x.w, o), __shfl_xor_sync(~0u, x.wp, o),
          __shfl_xor_sync(~0u, x.wa, o), shfl(x.m, o)};
}
__device__ __forceinline__ Top2 shfl(Top2 x, int o) {
  return {__shfl_xor_sync(~0u, x.v1, o), __shfl_xor_sync(~0u, x.i1, o),
          __shfl_xor_sync(~0u, x.v2, o), __shfl_xor_sync(~0u, x.i2, o)};
}

template <class V>
__device__ __forceinline__ V block_reduce(V v, V* slots, int& parity) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = combine(v, shfl(v, o));
  V* s = slots + 32 * parity;
  parity ^= 1;
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
  __syncthreads();
  V r = s[0];
  const int nw = blockDim.x >> 5;
  for (int w = 1; w < nw; ++w) r = combine(r, s[w]);
  return r;
}

// ---- one state's observation model ---------------------------------------------------
struct State {
  float lp, la;   // loc
  float ip, ia;   // 1 / scale
  float c;        // -log scale_p - log scale_a - log 2 pi
};

__device__ __forceinline__ State load_state(const Params& p, int j) {
  State s{0.f, 0.f, 0.f, 0.f, 0.f};
  if (j < p.K) {
    const float2 l = p.loc[j], sc = p.scale[j];
    s.lp = l.x; s.la = l.y;
    s.ip = 1.0f / sc.x; s.ia = 1.0f / sc.y;
    s.c = -(logf(sc.x) + logf(sc.y)) - kLog2Pi;
  }
  return s;
}

// MultivariateNormalDiag.log_prob of x under the state
__device__ __forceinline__ float log_lik(const State& s, float2 x) {
  const float zp = (x.x - s.lp) * s.ip, za = (x.y - s.la) * s.ia;
  return s.c - 0.5f * fmaf(zp, zp, za * za);
}

// hold * w + other * (sum of the other states' w), from the step's sums
__device__ __forceinline__ float transit(const Params& p, float w, bool is_max, Sum2 s) {
  return fmaf(p.hold, w, p.other * (is_max ? s.sx : s.s - w));
}

// One forward step: q -> e (returned), its argmax and sums; M is added to `c`.
__device__ __forceinline__ float forward_step(const Params& p, const State& st, float q,
                                              float2 x, MaxArg* mslots, Sum2* sslots,
                                              int& parity, MaxArg& m, Sum2& s, double& c) {
  const int j = threadIdx.x;
  const float a = j < p.K ? log_lik(st, x) + logf(q) : -INFINITY;
  m = block_reduce(MaxArg{a, j}, mslots, parity);
  const float e = j < p.K ? expf(a - m.v) : 0.f;
  s = block_reduce(Sum2{e, j == m.i ? 0.f : e}, sslots, parity);
  c += (double)m.v;
  return e;
}

__global__ void __launch_bounds__(kMaxStates)
hmm_log_prob_kernel(Params p, float* __restrict__ log_prob) {
  __shared__ MaxArg mslots[64];
  __shared__ Sum2 sslots[64];
  int parity = 0;
  const int b = blockIdx.x;
  const float2* obs = p.obs + (size_t)b * p.T;
  const State st = load_state(p, threadIdx.x);
  double c = p.log_init;
  float q = 1.0f;
  float2 x = obs[0];
  MaxArg m;
  Sum2 s;
  for (int t = 0; t < p.T; ++t) {
    const float2 xn = obs[t + 1 < p.T ? t + 1 : t];
    const float e = forward_step(p, st, q, x, mslots, sslots, parity, m, s, c);
    q = transit(p, e, threadIdx.x == m.i, s);
    x = xn;
  }
  if (threadIdx.x == 0) log_prob[b] = (float)(c + log((double)s.s));
}

// dyn smem: seg * K floats (e_t of one segment, [t - t0][j])
__global__ void __launch_bounds__(kMaxStates)
hmm_backward_kernel(Params p, int seg, const float* __restrict__ grad,
                    float2* __restrict__ d_obs, float* __restrict__ ckpt) {
  extern __shared__ float ebuf[];
  __shared__ MaxArg mslots[64];
  __shared__ Sum2 sslots[64];
  __shared__ Post pslots[64];
  int parity = 0;
  const int b = blockIdx.x, j = threadIdx.x;
  const int nseg = (p.T + seg - 1) / seg;
  const float2* obs = p.obs + (size_t)b * p.T;
  float2* dx = d_obs + (size_t)b * p.T;
  float* ck = ckpt + (size_t)b * nseg * p.K + j;
  const State st = load_state(p, j);
  const float g = grad[b];
  double c = 0.0;   // the normaliser is not needed here
  MaxArg m;
  Sum2 s;

  // forward, keeping q at every segment start
  float q = 1.0f;
  float2 x = obs[0];
  for (int t = 0; t < p.T; ++t) {
    const float2 xn = obs[t + 1 < p.T ? t + 1 : t];
    if (t % seg == 0 && j < p.K) ck[(size_t)(t / seg) * p.K] = q;
    const float e = forward_step(p, st, q, x, mslots, sslots, parity, m, s, c);
    q = transit(p, e, j == m.i, s);
    x = xn;
  }

  // segments last to first: recompute e_t, then scan b back through them
  float bt = 1.0f;   // b_t(j), t = T - 1
  for (int sg = nseg - 1; sg >= 0; --sg) {
    const int t0 = sg * seg, t1 = min(t0 + seg, p.T);
    q = j < p.K ? ck[(size_t)sg * p.K] : 1.0f;
    x = obs[t0];
    for (int t = t0; t < t1; ++t) {
      const float2 xn = obs[t + 1 < p.T ? t + 1 : t];
      const float e = forward_step(p, st, q, x, mslots, sslots, parity, m, s, c);
      if (j < p.K) ebuf[(t - t0) * p.K + j] = e;
      q = transit(p, e, j == m.i, s);
      x = xn;
    }
    x = obs[t1 - 1];
    for (int t = t1 - 1; t >= t0; --t) {
      const float2 xn = obs[t > 0 ? t - 1 : 0];
      Post v{0.f, 0.f, 0.f, MaxArg{-INFINITY, j}};
      if (j < p.K) {
        const float w = ebuf[(t - t0) * p.K + j] * bt;
        const float zp = (x.x - st.lp) * st.ip, za = (x.y - st.la) * st.ia;
        v.w = w;
        v.wp = -w * zp * st.ip;
        v.wa = -w * za * st.ia;
        v.m.v = log_lik(st, x) + logf(bt);
      }
      const Post r = block_reduce(v, pslots, parity);
      if (j == 0) dx[t] = make_float2(g * (r.wp / r.w), g * (r.wa / r.w));
      if (t > 0) {
        const float u = j < p.K ? expf(v.m.v - r.m.v) : 0.f;
        s = block_reduce(Sum2{u, j == r.m.i ? 0.f : u}, sslots, parity);
        bt = transit(p, u, j == r.m.i, s);
      }
      x = xn;
    }
  }
}

// dyn smem: T * (ceil(K / 32) + 1) words: the "stayed" bits of step t in
// bits[t * W .. t * W + W - 1], and (i1, i2) of d_{t-1} in pairs[t]
__global__ void __launch_bounds__(kMaxStates)
hmm_viterbi_kernel(Params p, int64_t* __restrict__ path) {
  extern __shared__ uint32_t vbuf[];
  __shared__ Top2 tslots[64];
  int parity = 0;
  const int b = blockIdx.x, j = threadIdx.x;
  const int W = (p.K + 31) >> 5;
  uint32_t* bits = vbuf;
  uint32_t* pairs = vbuf + (size_t)p.T * W;
  const float2* obs = p.obs + (size_t)b * p.T;
  const State st = load_state(p, j);
  const float lh = p.log_hold, lo = p.log_other;
  Top2 top{0.f, 0, 0.f, 0};
  float d = 0.f;   // d_{t-1}(j)
  float2 x = obs[0];
  for (int t = 0; t < p.T; ++t) {
    const float2 xn = obs[t + 1 < p.T ? t + 1 : t];
    const float l = j < p.K ? log_lik(st, x) : -INFINITY;
    bool stay = false;
    if (t == 0) {
      d = l;
    } else {
      // the best other state and its value, both relative to max d_{t-1}
      const bool is1 = j == top.i1;
      const int oi = is1 ? top.i2 : top.i1;
      const float sv = (d - top.v1) + lh, ov = ((is1 ? top.v2 : top.v1) - top.v1) + lo;
      stay = better(sv, j, ov, oi);
      d = j < p.K ? l + (stay ? sv : ov) : -INFINITY;
      const uint32_t word = __ballot_sync(~0u, stay && j < p.K);
      if ((j & 31) == 0) bits[(size_t)t * W + (j >> 5)] = word;
      if (j == 0) pairs[t] = (uint32_t)top.i1 | ((uint32_t)top.i2 << 16);
    }
    top = block_reduce(Top2{d, j, -INFINITY, (int)blockDim.x + j}, tslots, parity);
    x = xn;
  }
  __syncthreads();
  if (j == 0) {
    int64_t* out = path + (size_t)b * p.T;
    int s = top.i1;
    for (int t = p.T - 1; t > 0; --t) {
      out[t] = s;
      if (!((bits[(size_t)t * W + (s >> 5)] >> (s & 31)) & 1u)) {
        const uint32_t pr = pairs[t];
        const int i1 = (int)(pr & 0xFFFFu), i2 = (int)(pr >> 16);
        s = s == i1 ? i2 : i1;
      }
    }
    out[0] = s;
  }
}

}  // namespace hmm_
}  // namespace ddsp
