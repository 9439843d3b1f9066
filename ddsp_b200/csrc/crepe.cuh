// spectral_ops.PretrainedCREPE (spectral_ops.py:432-566) around its network: the frames
// the network reads, the Viterbi path of create_hmm's 360-state HMM, and the
// local-average f0 of activations_to_f0_and_confidence.  All three are forward only.
// The frames of losses.PretrainedCREPE (losses.py:418-486), which the embedding losses
// train through, also have a backward pass.
//
// Frames (crepe_frames_kernel).  One warp per frame of 1024 samples, 32 per lane, read
// once into registers: samples outside the audio are pad's zeros.  Mean and population
// variance about the mean (tf.nn.moments) are two passes in double, each lane summing
// its samples in order and the lanes combined by an xor butterfly, so every lane holds
// the same bits.  spectral_ops: std = sqrt(var), or 1e-8 where var = 0;
// out = (x - mean) / std.  losses (kEps): out = (x - mean) / (sqrt(var) + 1e-5).
//
// Frames backward (losses' normalisation only).  Per frame, with mu, s = sqrt(var),
// d = s + 1e-5, gbar = mean(g) and c = sum_j g_j (x_j - mu):
//   dx_k = (g_k - gbar) / d - c (x_k - mu) / (d^2 1024 s),
// the statistics in double as in the forward (tf.nn.moments stops the gradient of the
// mean inside the variance; the term it would add sums to zero).  A frame of variance
// 0 has c = 0 and s = 0: the second term is 0 / 0 = NaN on every sample the frame
// covers, as TensorFlow's infinite derivative of var**0.5 at 0 times 0 gives.  Samples
// no frame covers get 0.  No atomics: bit-reproducible.
//   hop >= 1024 (crepe_frames_bwd_disjoint_kernel): no sample is in two frames.  One
//     warp per frame computes its statistics and writes its samples, and zeroes the gap
//     up to the next frame (the audio's end after the last).
//   hop < 1024 (crepe_frames_bwd_overlap_kernel): a CTA owns kBwdOwn samples.  Its
//     warps compute the statistics of every frame that covers one of them into shared
//     memory, then each thread sums its sample's terms over those frames in increasing
//     frame order, in double.  A frame on a span boundary has its statistics computed
//     by both CTAs, with the same code and so the same bits.
//
// Viterbi (crepe_viterbi_kernel).  tfp's posterior_mode on create_hmm's model: uniform
// initial distribution, transition w(i, j) / rs_i with w = max(12 - |i - j|, 1e-5) and
// rs_i the true row sum (smaller near the edges), and the Multinomial(1, eye 0.1 +
// 0.9 / 360) emission, whose log-probability is a_s log 41 plus terms equal for every
// state (the lgammas and sum_i a_i log(0.9 / 360)), which a path's choice never sees.
//   delta_t(j) = l_t(j) + max_i (delta_{t-1}(i) - log rs_i + log w(i, j)).
// With u_i = delta_{t-1}(i) - log rs_i and g = argmax u (lowest index on ties), the
// max over i is the better of the 23 in-band i = j - 11 .. j + 11 (log(12 - |i - j|))
// and u_g + log 1e-5: if g is in j's band its in-band term u_g + log(12 - |g - j|) >=
// u_g > u_g + log 1e-5 beats every out-of-band term, and otherwise u_g + log 1e-5 IS
// the best out-of-band term, g being the lowest index attaining it.  Ties between the
// two go to the lower index, so every choice is tf.argmax's.  delta is kept relative to
// u_g, so it stays within a few tens of 0 for any T.
// One CTA per sequence, a thread per state, one __syncthreads per step (u and the warp
// maxima double-buffered).  A back pointer is 5 bits: the offset + 11 (0..22), or 23
// for "came from g_t".  Each warp stores its 32 pointers as 5 ballot bit-planes, so a
// step is a record of kRecordWords 32-bit words: 12 warps x 5 planes, then g_t.  The
// records go to the caller's workspace ([B, T - 1] records), not to shared memory,
// so T is unbounded.  The same launch then backtracks: the CTA stages kChunk records at
// a time into shared memory and thread 0 walks them.
//
// Decode (crepe_decode_kernel).  One warp per row: confidence = max, centre = first
// argmax unless given, window c - 4 .. c + 5 clamped into 0 .. 359 (edge bins repeat),
// f0_cent = sum(w cents) / sum(w) in double, f0 = 10 2^(f0_cent / 1200).  A window
// whose weights sum to 0 gives 0 / 0 = NaN, as the reference does.
#pragma once
#include <math.h>
#include <stdint.h>

#include "common.cuh"

namespace ddsp {
namespace crepe_ {

constexpr int kBins = DDSP_B200_CREPE_BINS;     // 360
constexpr int kFrame = DDSP_B200_CREPE_FRAME;   // 1024
constexpr int kPerLane = kFrame / 32;
constexpr int kFrameWarps = 8;

constexpr int kBand = 11;                        // |i - j| <= 11 has w = 12 - |i - j| >= 1
constexpr int kWarps = (kBins + 31) / 32;        // 12
constexpr int kThreads = 32 * kWarps;            // 384
constexpr int kPlanes = 5;                       // bits per back pointer
constexpr int kFromG = 2 * kBand + 1;            // the pointer code for "came from g_t"
constexpr int kRecordWords = kWarps * kPlanes + 1;
constexpr int kChunk = 64;                       // records staged per backtrack pass
constexpr int kDecodeWarps = 8;
constexpr double kLossEps = 1e-5;                // losses.PretrainedCREPE: std + 1e-5
constexpr int kBwdOwn = 1024;                    // samples a CTA owns (hop < kFrame)
constexpr int kBwdThreads = 256;
constexpr int kDisjointWarps = 4;                // 12 warps per SM at its registers

static_assert(kFrame % 32 == 0, "a lane reads kFrame / 32 samples");
static_assert(kFromG < (1 << kPlanes), "pointer codes fit kPlanes bits");

// ---- frames ---------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(~0u, v, o);
  return v;
}

// frames [B * F, kFrame]: frame r = b F + f reads padded samples f hop .. f hop + 1023,
// i.e. audio[b, f hop - pad_left + k] (zero outside 0 .. N - 1).  kEps: losses'
// normalisation, by sqrt(var) + 1e-5.
template <bool kEps>
__global__ void __launch_bounds__(32 * kFrameWarps)
crepe_frames_kernel(const float* __restrict__ audio, float* __restrict__ frames, int N,
                    int F, int64_t total, int hop, int pad_left) {
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * kFrameWarps;
  for (int64_t r = (int64_t)blockIdx.x * kFrameWarps + (threadIdx.x >> 5); r < total;
       r += stride) {
    const int64_t b = r / F, f = r - b * F;
    const float* x = audio + b * N;
    const int64_t start = f * hop - pad_left + lane;
    float v[kPerLane];
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < kPerLane; ++k) {
      const int64_t i = start + 32 * k;
      v[k] = (i >= 0 && i < N) ? x[i] : 0.f;
      s += (double)v[k];
    }
    const double mean = warp_sum(s) * (1.0 / kFrame);
    double q = 0.0;
#pragma unroll
    for (int k = 0; k < kPerLane; ++k) {
      const double d = (double)v[k] - mean;
      q = fma(d, d, q);
    }
    const double var = warp_sum(q) * (1.0 / kFrame);
    const double inv = kEps ? 1.0 / (sqrt(var) + kLossEps) : var > 0.0 ? 1.0 / sqrt(var) : 1e8;
    float* out = frames + r * kFrame + lane;
#pragma unroll
    for (int k = 0; k < kPerLane; ++k) out[32 * k] = (float)(((double)v[k] - mean) * inv);
  }
}

// ---- frames backward (losses' normalisation) ------------------------------------------
__device__ __forceinline__ int64_t i64min(int64_t a, int64_t b) { return a < b ? a : b; }
__device__ __forceinline__ int64_t i64max(int64_t a, int64_t b) { return a > b ? a : b; }

// What a sample's gradient needs of one frame: dx = (g - gbar) inv - coef (x - mu).
struct FrameGrad { double mu, inv, coef, gbar; };

// The statistics of the frame of padded samples start .. start + 1023 of x [N] (zero
// outside 0 .. N - 1), with upstream gradient g [1024]; every lane returns the same bits.
// v and w receive the lane's samples and gradients (sample start + lane + 32 k).
__device__ __forceinline__ FrameGrad frame_grad(const float* __restrict__ x,
                                                const float* __restrict__ g, int N,
                                                int64_t start, int lane, float (&v)[kPerLane],
                                                float (&w)[kPerLane]) {
  double s = 0.0, sg = 0.0;
#pragma unroll
  for (int k = 0; k < kPerLane; ++k) {
    const int64_t i = start + lane + 32 * k;
    v[k] = (i >= 0 && i < N) ? x[i] : 0.f;
    w[k] = g[lane + 32 * k];
    s += (double)v[k];
    sg += (double)w[k];
  }
  const double mu = warp_sum(s) * (1.0 / kFrame);
  double q = 0.0, c = 0.0;
#pragma unroll
  for (int k = 0; k < kPerLane; ++k) {
    const double d = (double)v[k] - mu;
    q = fma(d, d, q);
    c = fma((double)w[k], d, c);
  }
  const double sd = sqrt(warp_sum(q) * (1.0 / kFrame));
  c = warp_sum(c);
  const double inv = 1.0 / (sd + kLossEps);
  // c = 0 and sd = 0 on a frame of variance 0: NaN, as TensorFlow's gradient
  return FrameGrad{mu, inv, c * inv * inv / ((double)kFrame * sd), warp_sum(sg) * (1.0 / kFrame)};
}

__device__ __forceinline__ double frame_term(const FrameGrad& s, float g, float x) {
  return ((double)g - s.gbar) * s.inv - s.coef * ((double)x - s.mu);
}

// hop >= kFrame: warp r = b F + f writes frame f's samples of grad_audio [B, N], and
// zeroes the samples after it up to frame f + 1's first (or N).
__global__ void __launch_bounds__(32 * kDisjointWarps)
crepe_frames_bwd_disjoint_kernel(const float* __restrict__ audio,
                                 const float* __restrict__ grad_frames,
                                 float* __restrict__ grad_audio, int N, int F, int64_t total,
                                 int hop, int pad_left) {
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * kDisjointWarps;
  for (int64_t r = (int64_t)blockIdx.x * kDisjointWarps + (threadIdx.x >> 5); r < total;
       r += stride) {
    const int64_t b = r / F, f = r - b * F;
    const float* x = audio + b * N;
    const float* g = grad_frames + r * kFrame;
    float* dx = grad_audio + b * N;
    const int64_t start = f * hop - pad_left;
    float v[kPerLane], w[kPerLane];
    const FrameGrad st = frame_grad(x, g, N, start, lane, v, w);
#pragma unroll
    for (int k = 0; k < kPerLane; ++k) {
      const int64_t i = start + lane + 32 * k;
      if (i >= 0 && i < N) dx[i] = (float)(0.0 + frame_term(st, w[k], v[k]));
    }
    // frame 0 starts at or before sample 0, so only gaps after a frame remain
    const int64_t end = f + 1 < F ? i64min(start + hop, N) : (int64_t)N;
    for (int64_t i = i64max(start + kFrame, 0) + lane; i < end; i += 32) dx[i] = 0.f;
  }
}

// hop < kFrame: CTA t = b spans + s owns samples s kBwdOwn .. + kBwdOwn - 1 of item b.
// fg: the FrameGrad of every frame covering one of them, in dynamic shared memory.
__global__ void __launch_bounds__(kBwdThreads)
crepe_frames_bwd_overlap_kernel(const float* __restrict__ audio,
                                const float* __restrict__ grad_frames,
                                float* __restrict__ grad_audio, int N, int F, int spans,
                                int64_t total, int hop, int pad_left) {
  extern __shared__ FrameGrad fg[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t t = blockIdx.x; t < total; t += gridDim.x) {
    const int64_t b = t / spans;
    const int64_t k0 = (t - b * spans) * (int64_t)kBwdOwn;
    const int64_t k1 = i64min(k0 + kBwdOwn, N);
    const float* x = audio + b * N;
    const float* g = grad_frames + b * F * (int64_t)kFrame;
    // frames f with f hop - pad_left <= k1 - 1 and f hop - pad_left + 1023 >= k0
    const int64_t lo_num = k0 + pad_left - (kFrame - 1);
    const int64_t f_lo = lo_num <= 0 ? 0 : (lo_num + hop - 1) / hop;
    const int64_t f_hi = i64min((k1 - 1 + pad_left) / hop, (int64_t)F - 1);
    __syncthreads();   // the previous span has finished reading fg
    for (int64_t f = f_lo + warp; f <= f_hi; f += kBwdThreads / 32) {
      float v[kPerLane], w[kPerLane];
      const FrameGrad st = frame_grad(x, g + f * kFrame, N, f * hop - pad_left, lane, v, w);
      if (lane == 0) fg[f - f_lo] = st;
    }
    __syncthreads();
    for (int64_t i = k0 + threadIdx.x; i < k1; i += kBwdThreads) {
      const float xi = x[i];
      const int64_t num = i + pad_left - (kFrame - 1);
      const int64_t a = i64max(f_lo, num <= 0 ? 0 : (num + hop - 1) / hop);
      const int64_t e = i64min(f_hi, (i + pad_left) / hop);
      double acc = 0.0;
      for (int64_t f = a; f <= e; ++f)
        acc += frame_term(fg[f - f_lo], g[f * kFrame + (i + pad_left - f * hop)], xi);
      grad_audio[b * N + i] = (float)acc;
    }
  }
}

// Frames whose statistics one CTA of the overlap kernel keeps: those covering a span
// of kBwdOwn samples.
__host__ __device__ constexpr int bwd_frames_per_span(int hop) {
  return (kBwdOwn - 1 + kFrame - 1) / hop + 2;
}

// ---- argmax helpers -------------------------------------------------------------------
struct Arg { float v; int i; };   // maximum, lowest index on ties

__device__ __forceinline__ bool better(float va, int ia, float vb, int ib) {
  return va > vb || (va == vb && ia < ib);
}
__device__ __forceinline__ Arg combine(Arg a, Arg b) {
  return better(a.v, a.i, b.v, b.i) ? a : b;
}
__device__ __forceinline__ Arg warp_argmax(Arg a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    a = combine(a, Arg{__shfl_xor_sync(~0u, a.v, o), __shfl_xor_sync(~0u, a.i, o)});
  return a;
}

// ---- Viterbi --------------------------------------------------------------------------
// ptrs: [B, T - 1, kRecordWords] words, the record of step t >= 1 at t - 1.
__global__ void __launch_bounds__(kThreads, 1)
crepe_viterbi_kernel(const float* __restrict__ acts, int* __restrict__ centers, int T,
                     uint32_t* __restrict__ ptrs) {
  // u of the previous step, with kBand -inf entries on each side of the states
  __shared__ float ubuf[2][kThreads + 2 * kBand];
  __shared__ Arg slots[2][kWarps];
  __shared__ uint32_t chunk[kChunk * kRecordWords];
  const int j = threadIdx.x, lane = j & 31, warp = j >> 5;
  const bool live = j < kBins;
  const int64_t b = blockIdx.x;
  const float* a = acts + b * (int64_t)T * kBins + j;
  uint32_t* rec = ptrs + b * (int64_t)(T - 1) * kRecordWords;
  const float kLog41 = 3.7135720667043080f;    // log((0.1 + 0.9 / 360) / (0.9 / 360))
  const float kLogFloor = -11.512925464970229f;  // log(1e-5)
  const float log_w[kBand + 1] = {2.4849066497880004f, 2.3978952727983707f,  // log(12 - |d|)
                                  2.3025850929940457f, 2.1972245773362196f,
                                  2.0794415416798357f, 1.9459101490553132f,
                                  1.7917594692280550f, 1.6094379124341003f,
                                  1.3862943611198906f, 1.0986122886681098f,
                                  0.6931471805599453f, 0.0f};

  // log rs_j: the row sum of create_hmm's transition, in double
  float log_rs = 0.f;
  if (live) {
    double rs = 0.0;
    int in_band = 0;
    for (int d = -kBand; d <= kBand; ++d)
      if (j + d >= 0 && j + d < kBins) {
        rs += 12.0 - abs(d);
        ++in_band;
      }
    log_rs = (float)log(rs + (kBins - in_band) * 1e-5);
  }
  if (j < kBand) {
    ubuf[0][j] = ubuf[1][j] = -INFINITY;
    ubuf[0][kBand + kThreads + j] = ubuf[1][kBand + kThreads + j] = -INFINITY;
  }

  float delta = live ? a[0] * kLog41 : -INFINITY;   // the uniform initial term is a constant
  float a1 = live && T > 1 ? a[kBins] : 0.f;        // activations of steps t and t + 1
  float a2 = live && T > 2 ? a[2 * kBins] : 0.f;
  for (int t = 1; t < T; ++t) {
    float* u = ubuf[t & 1] + kBand;
    const float uj = live ? delta - log_rs : -INFINITY;
    u[j] = uj;
    const Arg wm = warp_argmax(Arg{uj, j});
    if (lane == 0) slots[t & 1][warp] = wm;
    const float l = a1 * kLog41;
    a1 = a2;
    a2 = live && t + 2 < T ? a[(int64_t)(t + 2) * kBins] : 0.f;
    __syncthreads();
    Arg g = slots[t & 1][0];
#pragma unroll
    for (int w = 1; w < kWarps; ++w) g = combine(g, slots[t & 1][w]);
    float best = -INFINITY;
    int bd = 0;
#pragma unroll
    for (int d = -kBand; d <= kBand; ++d) {
      const float c = u[j + d] + log_w[d < 0 ? -d : d];
      if (c > best) {
        best = c;
        bd = d;
      }
    }
    const float out = g.v + kLogFloor;
    const bool in_band = best > out || (best == out && j + bd < g.i);
    const int code = in_band ? bd + kBand : kFromG;
    delta = live ? l + ((in_band ? best : out) - g.v) : -INFINITY;
    uint32_t* r = rec + (int64_t)(t - 1) * kRecordWords;
#pragma unroll
    for (int k = 0; k < kPlanes; ++k) {
      const uint32_t word = __ballot_sync(~0u, (code >> k) & 1);
      if (lane == 0) r[warp * kPlanes + k] = word;
    }
    if (j == 0) r[kWarps * kPlanes] = (uint32_t)g.i;
  }

  // the most likely last state, then the walk back through the records
  const Arg wm = warp_argmax(Arg{delta, j});
  if (lane == 0) slots[T & 1][warp] = wm;
  __syncthreads();
  Arg e = slots[T & 1][0];
#pragma unroll
  for (int w = 1; w < kWarps; ++w) e = combine(e, slots[T & 1][w]);
  int* path = centers + b * (int64_t)T;
  int s = e.i;
  if (j == 0) path[T - 1] = s;
  for (int t1 = T - 1; t1 > 0; t1 -= kChunk) {   // records t0 .. t1 - 1 (steps t0+1 .. t1)
    const int t0 = t1 > kChunk ? t1 - kChunk : 0;
    const uint32_t* src = rec + (int64_t)t0 * kRecordWords;
    const int words = (t1 - t0) * kRecordWords;
    __syncthreads();   // the previous pass has finished reading chunk
    for (int i = j; i < words; i += kThreads) chunk[i] = src[i];
    __syncthreads();
    if (j == 0) {
      for (int t = t1 - 1; t >= t0; --t) {
        const uint32_t* rr = chunk + (t - t0) * kRecordWords;
        const uint32_t* planes = rr + (s >> 5) * kPlanes;
        int code = 0;
#pragma unroll
        for (int k = 0; k < kPlanes; ++k) code |= (int)((planes[k] >> (s & 31)) & 1u) << k;
        s = code == kFromG ? (int)rr[kWarps * kPlanes] : s + code - kBand;
        path[t] = s;
      }
    }
  }
}

// ---- decode ---------------------------------------------------------------------------
__global__ void __launch_bounds__(32 * kDecodeWarps)
crepe_decode_kernel(const float* __restrict__ acts, const int* __restrict__ centers,
                    float* __restrict__ f0, float* __restrict__ confidence, int64_t M) {
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * kDecodeWarps;
  for (int64_t r = (int64_t)blockIdx.x * kDecodeWarps + (threadIdx.x >> 5); r < M;
       r += stride) {
    const float* a = acts + r * kBins;
    Arg m{-INFINITY, kBins};
    for (int i = lane; i < kBins; i += 32) {
      const float v = a[i];
      if (better(v, i, m.v, m.i)) m = Arg{v, i};
    }
    m = warp_argmax(m);
    if (m.i == kBins) m.i = 0;   // every value NaN: tf.argmax's first index
    const int64_t c = centers ? (int64_t)centers[r] : (int64_t)m.i;
    double sw = 0.0, swc = 0.0;
    if (lane < 10) {
      const int64_t i = c - 4 + lane;
      const int idx = (int)(i > 0 ? (i < kBins - 1 ? i : kBins - 1) : 0);
      const double w = (double)a[idx];
      const double cents = (double)(float)(20.0 * idx + 1997.3794084376191);
      sw = w;
      swc = w * cents;
    }
    sw = warp_sum(sw);
    swc = warp_sum(swc);
    if (lane == 0) {
      f0[r] = (float)(10.0 * exp2((swc / sw) / 1200.0));
      confidence[r] = m.v;
    }
  }
}

}  // namespace crepe_
}  // namespace ddsp
