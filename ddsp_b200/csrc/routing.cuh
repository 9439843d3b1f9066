// Signal routing and the exponential-decay reverb: processors.Add, core.resample
// (core.py:573-714) and its backward, processors.Mix (processors.py:179-233) forward and backward,
// and ExpDecayReverb._get_ir (effects.py:144-151) forward and backward.
//
// Every gradient is written once per element, without float atomics or memset,
// and split sums are added in a fixed order, so each is bit-reproducible.
//
// resample_backward_kernel is the transpose of resample_kernel (above) in
// gather form.  Sample t of the forward reads frames lo(t) .. hi(t) (after the
// clamps), and both are non-decreasing in t, so the samples that reach frame j are
// one range [t0, t1): t0 the first t with hi(t) >= j, t1 the first t with
// lo(t) > j, found by bisection.  For each t in it the kernel recomputes the
// forward's float32 index and weights and adds every tap that lands on j,
// including the taps the clamps fold onto frames 0 and F - 1, in double.  G lanes
// share one frame (G = 32 when frames span many samples): lane l walks t0 + l,
// t0 + l + G, ..., and the lanes are summed by a fixed xor tree.
#pragma once
#include "taps.cuh"

namespace ddsp {

// processors.Add.get_signal (processors.py:174-176)
__global__ void __launch_bounds__(256)
add_kernel(const float* a, const float* b, float* out, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) out[i] = a[i] + b[i];
}

// core.resample / core.upsample_with_windows (core.py:573-714) as a stand-alone
// op: [B, F, C] -> [B, N, C].  method 0 = 'window' (Hann overlap-add ==
// two-tap raised cosine, SURVEY A.2), 1 = 'linear' (tf v1 bilinear,
// align_corners = !add_endpoint), 2 = 'nearest', 3 = 'cubic' (tf v1 bicubic).  Index math follows TF's
// float32 scale * index for linear / nearest; the window method needs an integer
// hop (checked by the caller, core.py:687-693).
__global__ void __launch_bounds__(256)
resample_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int F,
                int C, int N, int method, int add_endpoint) {
  const int64_t total = (int64_t)B * N * C;
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const float scale = (!add_endpoint && N > 1) ? (float)(F - 1) / (float)(N - 1)
                                               : (float)F / (float)N;
  const int hop = add_endpoint ? N / max(F, 1) : N / max(F - 1, 1);
  for (; idx < total; idx += stride) {
    const int c = (int)(idx % C);
    const int64_t bt = idx / C;
    const int t = (int)(bt % N);
    const int b = (int)(bt / N);
    const float* x = in + (size_t)b * F * C + c;
    float v;
    if (method == 0) {
      const int i = t / hop, r = t - i * hop;
      const int i1 = min(i + 1, F - 1);            // add_endpoint: frame F := F-1
      const float w1 = 0.5f - 0.5f * cospif((float)r / (float)hop);
      v = x[(size_t)i * C] * (1.0f - w1) + x[(size_t)i1 * C] * w1;
    } else if (method == 1) {
      const float src = (float)t * scale;
      const float fl = floorf(src);
      const int lo = max((int)fl, 0);
      const int hi = min((int)ceilf(src), F - 1);
      const float top = x[(size_t)min(lo, F - 1) * C], bot = x[(size_t)hi * C];
      v = __fadd_rn(top, __fmul_rn(__fsub_rn(bot, top), src - fl));
    } else if (method == 2) {
      const float src = (float)t * scale;
      const int i = min((int)(add_endpoint ? floorf(src) : roundf(src)), F - 1);
      v = x[(size_t)i * C];
    } else {
      // 'cubic': TensorFlow's legacy bicubic kernel (resize_bicubic_op.cc, Keys
      // A = -0.75, no half-pixel centres).  Its weights come from a 1025-entry
      // float32 table indexed by lrintf(delta * 1024); the same entries are
      // evaluated here in double and rounded to float32.
      const float src = (float)t * scale;
      const float fl = floorf(src);
      const int loc = (int)fl;
      const int off = (int)lrintf((src - fl) * 1024.0f);
      const double A = -0.75;
      const double xa = off * (1.0 / 1024.0), xb = (1024 - off) * (1.0 / 1024.0);
      const float w1 = (float)(((A + 2) * xa - (A + 3)) * xa * xa + 1);
      const float w2 = (float)(((A + 2) * xb - (A + 3)) * xb * xb + 1);
      const double ya = xa + 1.0, yb = xb + 1.0;
      const float w0 = (float)(((A * ya - 5 * A) * ya + 8 * A) * ya - 4 * A);
      const float w3 = (float)(((A * yb - 5 * A) * yb + 8 * A) * yb - 4 * A);
      const float v0 = x[(size_t)min(max(loc - 1, 0), F - 1) * C];
      const float v1 = x[(size_t)min(max(loc, 0), F - 1) * C];
      const float v2 = x[(size_t)min(max(loc + 1, 0), F - 1) * C];
      const float v3 = x[(size_t)min(max(loc + 2, 0), F - 1) * C];
      v = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(v0, w0), __fmul_rn(v1, w1)),
                              __fmul_rn(v2, w2)), __fmul_rn(v3, w3));
    }
    out[idx] = v;
  }
}

namespace rt_ {

constexpr int kThreads = 256;
constexpr int kIrBwdThreads = 512;

// d in [B, F, C] from d out [B, N, C]: G lanes (1 or a whole warp) per (b, j, c),
// grid-stride; for G = 32 the output index is warp-uniform.
template <int G>
__global__ void __launch_bounds__(kThreads)
resample_backward_kernel(const float* __restrict__ grad_out, float* __restrict__ grad_in,
                         int B, int C, ResampleGeom g) {
  static_assert(G == 1 || G == 32, "one lane or one warp per frame");
  const int64_t total = (int64_t)B * g.F * C;
  const int lane = threadIdx.x & (G - 1);
  const int64_t stride = (int64_t)gridDim.x * (kThreads / G);
  for (int64_t o = ((int64_t)blockIdx.x * kThreads + threadIdx.x) / G; o < total;
       o += stride) {
    const int c = (int)(o % C);
    const int64_t bj = o / C;
    const int j = (int)(bj % g.F);
    const int b = (int)(bj / g.F);
    const int t0 = resample_bound(g, j, true);
    const int t1 = resample_bound(g, j, false);
    const float* gr = grad_out + (size_t)b * g.N * C + c;
    double acc = 0.0;
    for (int t = t0 + lane; t < t1; t += G) {
      int idx[4];
      float w[4];
      const int n = resample_taps(g, t, idx, w);
      double wj = 0.0;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (k < n && idx[k] == j) wj += (double)w[k];
      acc += (double)__ldg(gr + (size_t)t * C) * wj;
    }
    if (G > 1) {
#pragma unroll
      for (int s = G / 2; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
    }
    if (lane == 0) grad_in[o] = (float)acc;
  }
}

// processors.Mix.get_signal: out = sqrt(|m|) s1 + (1 - sqrt(|m - 1|)) s2 in the
// reference's float32 operation order (no contraction).  s1, s2, out [B, N, C];
// m [B, N, 1].
__device__ __forceinline__ float mix_one(float m) { return sqrtf(fabsf(m)); }
__device__ __forceinline__ float mix_two(float m) {
  return __fsub_rn(1.0f, sqrtf(fabsf(__fsub_rn(m, 1.0f))));
}

__global__ void __launch_bounds__(kThreads)
mix_kernel(const float* __restrict__ s1, const float* __restrict__ s2,
           const float* __restrict__ mix, float* __restrict__ out, int64_t rows, int C) {
  const int64_t total = rows * C;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < total; i += stride) {
    const float m = __ldg(mix + i / C);
    out[i] = __fadd_rn(__fmul_rn(mix_one(m), __ldg(s1 + i)),
                       __fmul_rn(mix_two(m), __ldg(s2 + i)));
  }
}

// sign as TensorFlow's Abs gradient takes it: 0 at 0
__device__ __forceinline__ float sign0(float x) { return (float)((x > 0.f) - (x < 0.f)); }

// One thread per (b, t): d s1 = g sqrt|m|, d s2 = g (1 - sqrt|m - 1|), and
// d m = sum_c g s1 sign(m) / (2 sqrt|m|) - g s2 sign(m - 1) / (2 sqrt|m - 1|) in
// channel order.  At m = 0 or 1 the reference's autodiff multiplies 1 / 0 by a zero
// sign, and so does this: d m is NaN there.  NULL outputs are skipped.
__global__ void __launch_bounds__(kThreads)
mix_backward_kernel(const float* __restrict__ s1, const float* __restrict__ s2,
                    const float* __restrict__ mix, const float* __restrict__ grad,
                    float* __restrict__ d_s1, float* __restrict__ d_s2,
                    float* __restrict__ d_mix, int64_t rows, int C) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t r = (int64_t)blockIdx.x * kThreads + threadIdx.x; r < rows; r += stride) {
    const float m = __ldg(mix + r);
    const float a = mix_one(m), b = mix_two(m);
    const float bq = sqrtf(fabsf(__fsub_rn(m, 1.0f)));
    const float da = __fdiv_rn(0.5f, a) * sign0(m);
    const float db = -__fdiv_rn(0.5f, bq) * sign0(__fsub_rn(m, 1.0f));
    double dm = 0.0;
    for (int c = 0; c < C; ++c) {
      const int64_t i = r * C + c;
      const float gi = __ldg(grad + i);
      if (d_s1 != nullptr) d_s1[i] = __fmul_rn(gi, a);
      if (d_s2 != nullptr) d_s2[i] = __fmul_rn(gi, b);
      if (d_mix != nullptr)
        dm += (double)gi * ((double)__ldg(s1 + i) * (double)da +
                            (double)__ldg(s2 + i) * (double)db);
    }
    if (d_mix != nullptr) d_mix[r] = (float)dm;
  }
}

// ExpDecayReverb._get_ir: ir[r, t] = (gain_r * exp(-(2 + exp(decay_r)) * time_t)) * n_t
// in float32, time = tf.linspace(0, 1, L) (delta * t, the last point 1), n the one
// [1, L] noise row: `noise` when given, else Philox row 0 at (seed, offset), i.e.
// core.uniform_noise(1, L, seed, offset).
__device__ __forceinline__ float ir_time(int t, int L, float delta) {
  return t == L - 1 ? (L == 1 ? 0.0f : 1.0f) : __fmul_rn(delta, (float)t);
}

__device__ __forceinline__ float4 ir_noise(const float* __restrict__ noise, int q, int L,
                                           uint64_t seed, uint64_t offset) {
  if (noise == nullptr) return noise4((uint32_t)q, 0u, seed, offset);
  float v[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = 4 * q + k < L ? __ldg(noise + 4 * q + k) : 0.f;
  return make_float4(v[0], v[1], v[2], v[3]);
}

__device__ __forceinline__ float ir_decay(float t, float de) {
  return expf(__fmul_rn(-de, t));
}

// one thread per (row, 4 samples)
__global__ void __launch_bounds__(kThreads)
exp_decay_ir_kernel(const float* __restrict__ gain, const float* __restrict__ decay,
                    const float* __restrict__ noise, uint64_t seed, uint64_t offset,
                    float* __restrict__ ir, int rows, int L) {
  const int n4 = (L + 3) >> 2;
  const int64_t total = (int64_t)rows * n4;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  const float delta = L > 1 ? __fdiv_rn(1.0f, (float)(L - 1)) : 0.0f;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < total; i += stride) {
    const int r = (int)(i / n4);
    const int q = (int)(i - (int64_t)r * n4);
    const float gr = __ldg(gain + r);
    const float de = __fadd_rn(2.0f, expf(__ldg(decay + r)));
    const float4 nz = ir_noise(noise, q, L, seed, offset);
    const float n[4] = {nz.x, nz.y, nz.z, nz.w};
    float* o = ir + (size_t)r * L;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int t = 4 * q + k;
      if (t < L) o[t] = __fmul_rn(__fmul_rn(gr, ir_decay(ir_time(t, L, delta), de)), n[k]);
    }
  }
}

// One CTA per row: d gain_r = sum_t d_ir e n and
// d decay_r = -exp(decay_r) gain_r sum_t d_ir time e n, the noise regenerated, each
// thread's strided sum in double, then a fixed-order tree over the CTA.
__global__ void __launch_bounds__(kIrBwdThreads)
exp_decay_ir_backward_kernel(const float* __restrict__ gain, const float* __restrict__ decay,
                             const float* __restrict__ noise, uint64_t seed,
                             uint64_t offset, const float* __restrict__ grad_ir,
                             float* __restrict__ d_gain, float* __restrict__ d_decay,
                             int L) {
  __shared__ double s_g[kIrBwdThreads], s_d[kIrBwdThreads];
  const int r = blockIdx.x;
  const int n4 = (L + 3) >> 2;
  const float delta = L > 1 ? __fdiv_rn(1.0f, (float)(L - 1)) : 0.0f;
  const float dec = __ldg(decay + r);
  const float de = __fadd_rn(2.0f, expf(dec));
  const float* gr = grad_ir + (size_t)r * L;
  double sg = 0.0, sd = 0.0;
  for (int q = threadIdx.x; q < n4; q += kIrBwdThreads) {
    const float4 nz = ir_noise(noise, q, L, seed, offset);
    const float n[4] = {nz.x, nz.y, nz.z, nz.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int t = 4 * q + k;
      if (t < L) {
        const float tm = ir_time(t, L, delta);
        const double v = (double)__ldg(gr + t) * (double)ir_decay(tm, de) * (double)n[k];
        sg += v;
        sd += v * (double)tm;
      }
    }
  }
  s_g[threadIdx.x] = sg;
  s_d[threadIdx.x] = sd;
  __syncthreads();
  for (int s = kIrBwdThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      s_g[threadIdx.x] += s_g[threadIdx.x + s];
      s_d[threadIdx.x] += s_d[threadIdx.x + s];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    if (d_gain != nullptr) d_gain[r] = (float)s_g[0];
    if (d_decay != nullptr)
      d_decay[r] = (float)(-exp((double)dec) * (double)__ldg(gain + r) * s_d[0]);
  }
}

}  // namespace rt_
}  // namespace ddsp
