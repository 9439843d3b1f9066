// A-weighted loudness (spectral_ops.compute_loudness, spectral_ops.py:254-324) and
// RMS power (compute_power, spectral_ops.py:223-249) of framed audio, computed on-chip:
// the padded signal, the frames and the spectrum are never written to memory.
//
// loudness_kernel: one CTA takes a run of consecutive frames of one item, stages the
// audio span they cover in shared memory (padding is zeros made from indices), and
// gives each warp one frame at a time.  The warp windows its frame (periodic Hann),
// packs it as n_fft/2 complex points z_j = x_2j + i x_2j+1, runs an in-place radix-2
// FFT in its shared-memory slice and splits the result into the n_fft/2 + 1 bins of
// the real FFT.  The weighted power sum runs in a fixed order (per-lane strided sums,
// then a butterfly), and dB conversion happens in double.
//
// loudness_backward_kernel: a CTA owns a span of output samples and recomputes every
// frame that overlaps it (its halo included), so each d-audio sample is written once,
// by one thread, summing the frames in ascending order: no atomics, no memset, and
// the gradient is bit-reproducible.  Per frame it recomputes X, forms
// Y_k = (2 c / K) w_k X_k (halved at the interior bins, as spectral_l1_kernel's
// irfft_scale), and applies the transpose of the real FFT as an unnormalised
// inverse: an inverse split step, then an inverse complex FFT of n_fft/2 points.
//
// Twiddles e^{-i pi k / M} (M = n_fft / 2) are computed per CTA in double
// (sincospi) and stored as float; the Hann window is read from the same table.
#pragma once
#include "common.cuh"

namespace ddsp {
namespace ld_ {

constexpr int kLog2MaxFft = 14;
constexpr int kMaxFft = 1 << kLog2MaxFft;   // what one warp slice + twiddles fit
constexpr int kMinOwn = 4096;               // backward: samples a CTA owns (>= n_fft)
constexpr int kRmsThreads = 256;

struct LoudParams {
  const float* audio;      // [B, N]
  const float* weights;    // [M + 1] linear A-weighting, 10^(A_k / 10)
  int N, T, n_fft, M, log2M, hop, pad_left;
  double pmin, range_db, ref_db;
};

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

__device__ __forceinline__ int bitrev(int j, int log2M) {
  return log2M ? (int)(__brev((unsigned)j) >> (32 - log2M)) : 0;
}

// e^{-i pi k / M} for k in [0, M]
__device__ __forceinline__ float2 twiddle(const float2* tab, int k, int M) {
  return k == M ? make_float2(-1.f, 0.f) : tab[k];
}

// periodic Hann of length 2M at n: 0.5 - 0.5 cos(pi n / M)
__device__ __forceinline__ float hann(const float2* tab, int n, int M) {
  const float c = n < M ? tab[n].x : -tab[n - M].x;
  return 0.5f - 0.5f * c;
}

__device__ __forceinline__ void fill_twiddles(float2* tab, int M) {
  for (int k = threadIdx.x; k < M; k += blockDim.x) {
    double s, c;
    sincospi((double)k / (double)M, &s, &c);
    tab[k] = make_float2((float)c, (float)-s);
  }
}

// Windowed frame x[0, 2M) (x(n) gives the sample) packed into z in bit-reversed order.
template <typename X>
__device__ __forceinline__ void load_frame(float2* z, const float2* tab, int M, int log2M,
                                           int lane, X x) {
  for (int j = lane; j < M; j += 32)
    z[bitrev(j, log2M)] = make_float2(hann(tab, 2 * j, M) * x(2 * j),
                                      hann(tab, 2 * j + 1, M) * x(2 * j + 1));
}

// In-place decimation-in-time FFT (sign -1): bit-reversed input, natural output.
__device__ __forceinline__ void fft_dit(float2* z, const float2* tab, int M, int log2M,
                                        int lane) {
  for (int s = 0; s < log2M; ++s) {
    __syncwarp();
    const int half = 1 << s, shift = log2M - s;
    for (int bf = lane; bf < (M >> 1); bf += 32) {
      const int pos = bf & (half - 1);
      const int i0 = ((bf >> s) << (s + 1)) + pos, i1 = i0 + half;
      const float2 u = z[i0], v = cmul(z[i1], tab[pos << shift]);
      z[i0] = make_float2(u.x + v.x, u.y + v.y);
      z[i1] = make_float2(u.x - v.x, u.y - v.y);
    }
  }
  __syncwarp();
}

// In-place decimation-in-frequency inverse FFT (sign +1, unnormalised): natural
// input, bit-reversed output.
__device__ __forceinline__ void ifft_dif(float2* z, const float2* tab, int M, int log2M,
                                         int lane) {
  for (int s = log2M - 1; s >= 0; --s) {
    __syncwarp();
    const int half = 1 << s, shift = log2M - s;
    for (int bf = lane; bf < (M >> 1); bf += 32) {
      const int pos = bf & (half - 1);
      const int i0 = ((bf >> s) << (s + 1)) + pos, i1 = i0 + half;
      const float2 w = tab[pos << shift];
      const float2 u = z[i0], v = z[i1];
      z[i0] = make_float2(u.x + v.x, u.y + v.y);
      z[i1] = cmul(make_float2(u.x - v.x, u.y - v.y), make_float2(w.x, -w.y));
    }
  }
  __syncwarp();
}

// Bin k of the real FFT from the packed spectrum: zk = Z_k, zm = Z_{M-k}, tw = e^{-i pi k/M}.
__device__ __forceinline__ float2 split_bin(float2 zk, float2 zm, float2 tw) {
  const float2 e = make_float2(0.5f * (zk.x + zm.x), 0.5f * (zk.y - zm.y));
  const float2 o = make_float2(0.5f * (zk.y + zm.y), -0.5f * (zk.x - zm.x));
  const float2 t = cmul(tw, o);
  return make_float2(e.x + t.x, e.y + t.y);
}

// Packed inverse input V_a = (Y_a + conj Y_b) + i e (Y_a - conj Y_b), b = M - a,
// e = e^{+i pi a / M}.
__device__ __forceinline__ float2 unsplit_bin(float2 ya, float2 yb, float2 e) {
  const float2 d = cmul(e, make_float2(ya.x - yb.x, ya.y + yb.y));
  return make_float2(ya.x + yb.x - d.y, ya.y - yb.y + d.x);
}

// mean_k w_k |X_k|^2 over the M + 1 bins, the same value on every lane.
__device__ __forceinline__ float frame_power(const float2* z, const float2* tab,
                                             const float* __restrict__ w, int M, int lane) {
  float acc = 0.f;
  for (int k = lane; k <= M; k += 32) {
    const float2 X = split_bin(z[k & (M - 1)], z[(M - k) & (M - 1)], twiddle(tab, k, M));
    acc = fmaf(__ldg(w + k), X.x * X.x + X.y * X.y, acc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return acc / (float)(M + 1);
}

// core.power_to_db (core.py:258-272) in double; NaN propagates as in tf.maximum.
__device__ __forceinline__ double power_db_raw(double pw, double pmin, double ref_db) {
  return 10.0 * log10(pw < pmin ? pmin : pw) - ref_db;
}
__device__ __forceinline__ double clamp_db(double db, double range_db) {
  return db < -range_db ? -range_db : db;
}

__global__ void __launch_bounds__(256)
loudness_kernel(LoudParams p, float* __restrict__ out, int frames_per_cta, int span) {
  extern __shared__ float4 ld_smem[];
  float2* tab = reinterpret_cast<float2*>(ld_smem);
  const int n_warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float2* z = tab + (size_t)p.M * (1 + warp);
  float* sp = reinterpret_cast<float*>(tab + (size_t)p.M * (1 + n_warps));
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * frames_per_cta;
  const int t1 = min(p.T, t0 + frames_per_cta);
  const float* a = p.audio + (size_t)b * p.N;
  fill_twiddles(tab, p.M);
  const long long s0 = (long long)t0 * p.hop - p.pad_left;
  for (int i = threadIdx.x; i < span; i += blockDim.x) {
    const long long s = s0 + i;
    sp[i] = (s >= 0 && s < p.N) ? a[s] : 0.f;
  }
  __syncthreads();
  for (int t = t0 + warp; t < t1; t += n_warps) {
    const float* x = sp + (size_t)(t - t0) * p.hop;
    load_frame(z, tab, p.M, p.log2M, lane, [x](int n) { return x[n]; });
    fft_dit(z, tab, p.M, p.log2M, lane);
    const float pw = frame_power(z, tab, p.weights, p.M, lane);
    if (lane == 0)
      out[(size_t)b * p.T + t] =
          (float)clamp_db(power_db_raw((double)pw, p.pmin, p.ref_db), p.range_db);
    __syncwarp();
  }
}

// The d frame of frame t into z (bit-reversed, as the inverse FFT leaves it), already
// excluding the window.  Returns false (z untouched past the forward FFT) when a clamp
// is active or the upstream gradient is 0: the frame then contributes nothing.
__device__ __forceinline__ bool frame_grad(float2* z, const float2* tab, const LoudParams& p,
                                           const float* __restrict__ a, int t, float g,
                                           int lane) {
  const long long s0 = (long long)t * p.hop - p.pad_left;
  const int N = p.N;
  load_frame(z, tab, p.M, p.log2M, lane, [a, s0, N](int n) {
    const long long s = s0 + n;
    return (s >= 0 && s < N) ? __ldg(a + s) : 0.f;
  });
  fft_dit(z, tab, p.M, p.log2M, lane);
  const float pw = frame_power(z, tab, p.weights, p.M, lane);
  const double db = power_db_raw((double)pw, p.pmin, p.ref_db);
  // tf.maximum hands ties to its first argument: max(pmin, p) passes a gradient only
  // for p > pmin, max(db, -range_db) for db >= -range_db
  if (!((double)pw > p.pmin && db >= -p.range_db) || g == 0.f) return false;
  const double c = (double)g * 10.0 / (2.302585092994045684 * (double)pw);
  const float cK = (float)(c / (double)(p.M + 1));
  const int M = p.M;
  for (int k = lane; k <= (M >> 1); k += 32) {
    const int km = (M - k) & (M - 1);
    const float2 zk = z[k & (M - 1)], zm = z[km];
    const float2 xk = split_bin(zk, zm, twiddle(tab, k, M));
    const float2 xm = split_bin(zm, zk, twiddle(tab, M - k, M));
    const float sk = cK * __ldg(p.weights + k) * (k == 0 ? 2.f : 1.f);
    const float sm = cK * __ldg(p.weights + M - k) * (k == 0 ? 2.f : 1.f);
    const float2 yk = make_float2(sk * xk.x, sk * xk.y);
    const float2 ym = make_float2(sm * xm.x, sm * xm.y);
    const float2 tk = twiddle(tab, k, M), tm = twiddle(tab, M - k, M);
    z[k & (M - 1)] = unsplit_bin(yk, ym, make_float2(tk.x, -tk.y));
    if (km != (k & (M - 1))) z[km] = unsplit_bin(ym, yk, make_float2(tm.x, -tm.y));
  }
  ifft_dif(z, tab, M, p.log2M, lane);
  return true;
}

__global__ void __launch_bounds__(256)
loudness_backward_kernel(LoudParams p, const float* __restrict__ grad,
                         float* __restrict__ d_audio, int own) {
  extern __shared__ float4 ld_smem[];
  float2* tab = reinterpret_cast<float2*>(ld_smem);
  const int n_warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float2* z = tab + (size_t)p.M * (1 + warp);
  float* acc = reinterpret_cast<float*>(tab + (size_t)p.M * (1 + n_warps));
  int* active = reinterpret_cast<int*>(acc + own);
  const int b = blockIdx.y;
  const int a0 = blockIdx.x * own, n_own = min(p.N - a0, own);
  const float* a = p.audio + (size_t)b * p.N;
  fill_twiddles(tab, p.M);
  for (int i = threadIdx.x; i < n_own; i += blockDim.x) acc[i] = 0.f;
  // frames t with t hop <= q < t hop + n_fft for a padded index q in [q0, q1)
  const long long q0 = (long long)a0 + p.pad_left, q1 = q0 + n_own;
  const long long lo = q0 - p.n_fft + 1;
  const int t_lo = lo <= 0 ? 0 : (int)((lo + p.hop - 1) / p.hop);
  const int t_hi = (int)min((long long)p.T - 1, (q1 - 1) / p.hop);
  __syncthreads();
  for (int tb = t_lo; tb <= t_hi; tb += n_warps) {
    const int t = tb + warp;
    const bool on = t <= t_hi &&
                    frame_grad(z, tab, p, a, t, __ldg(grad + (size_t)b * p.T + t), lane);
    if (lane == 0) active[warp] = on;
    __syncthreads();
    for (int i = threadIdx.x; i < n_own; i += blockDim.x) {
      float s = acc[i];
      for (int w = 0; w < n_warps; ++w) {
        if (!active[w]) continue;
        const long long n = q0 + i - (long long)(tb + w) * p.hop;
        if (n < 0 || n >= p.n_fft) continue;
        const float2 v = tab[(size_t)p.M * (1 + w) + bitrev((int)n >> 1, p.log2M)];
        s = fmaf(hann(tab, (int)n, p.M), (n & 1) ? v.y : v.x, s);
      }
      acc[i] = s;
    }
    __syncthreads();
  }
  float* o = d_audio + (size_t)b * p.N + a0;
  for (int i = threadIdx.x; i < n_own; i += blockDim.x) o[i] = acc[i];
}

// compute_power: power_to_db(mean(frame^2)) per frame (in_db), or compute_rms_energy:
// mean(frame^2)^0.5; a warp per frame.
__global__ void __launch_bounds__(kRmsThreads)
rms_power_kernel(const float* __restrict__ audio, float* __restrict__ out, int N, int T,
                 long long total, int frame, int hop, int pad_left, int in_db, double pmin,
                 double range_db, double ref_db) {
  const int lane = threadIdx.x & 31;
  const long long stride = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long f = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; f < total;
       f += stride) {
    const long long b = f / T, t = f - b * T;
    const float* a = audio + b * N;
    const long long s0 = t * hop - pad_left;
    float acc = 0.f;
    for (int i = lane; i < frame; i += 32) {
      const long long s = s0 + i;
      const float x = (s >= 0 && s < N) ? __ldg(a + s) : 0.f;
      acc = fmaf(x, x, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    const double ms = (double)acc / frame;
    if (lane == 0)
      out[f] = (float)(in_db ? clamp_db(power_db_raw(ms, pmin, ref_db), range_db) : sqrt(ms));
  }
}

}  // namespace ld_
}  // namespace ddsp
