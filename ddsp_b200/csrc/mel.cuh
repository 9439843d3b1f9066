// Mel, log-mel and MFCC features (spectral_ops.compute_mel / compute_logmel /
// compute_mfcc, spectral_ops.py:73-133) computed on-chip: the frames and the spectrum
// are never written to memory, only the [B, T, C] features are.
//
// The STFT is tf.signal.stft's: frames of fft_size samples every hop (pad_end: zeros
// past the end, made from indices), the fft_size-point Hann window, zero padding to
// fft_length = 2M, and the real FFT's M + 1 bins.  The transform is loudness.cuh's:
// the warp packs its frame as M complex points, runs ld_::fft_dit in its
// shared-memory slice and reads bin k through ld_::split_bin.
//
// Projection: tf.signal.linear_to_mel_weight_matrix has at most two nonzero weights
// per bin, in adjacent bands, so the host passes it sparse (MelParams below) and
// band j sums W_kj |X_k| over its own bin range [band_lo[j], band_hi[j]) in ascending
// k, one lane per band.  The log is safe_log in double.  The MFCC is
// mfccs_from_log_mel_spectrograms' unnormalised DCT-II times rsqrt(2 bins), cut to
// the first C coefficients, from a per-CTA table of the 4 bins angles pi m / (2 bins)
// (c (2n + 1) is reduced mod 4 bins in integers, so every cosine is a table entry).
//
// mel_kernel: loudness_kernel's layout.  A CTA takes a run of frames of one item and
// stages their audio span in shared memory, one warp per frame at a time; when not
// even two frames' span fits next to the FFT slices, each warp reads its frame from
// global memory instead (one frame per CTA shares nothing anyway).
//
// mel_backward_kernel: loudness_backward_kernel's owned-span scheme.  A CTA owns a
// span of output samples and recomputes every frame overlapping it with that
// frame's mel values; per frame: the DCT transpose (MFCC), d mel = d logmel / mel on
// mel > 0 and 0 elsewhere (tf.where), d|X_k| from the sparse projection's transpose,
// Y_k = d|X_k| X_k / |X_k| (0 at |X_k| = 0, TensorFlow's div_no_nan), halved at the
// interior bins, then ld_::unsplit_bin + ld_::ifft_dif.  The first fft_size samples,
// times the window, are summed over the frames in ascending order, so every d-audio
// sample is written once: no atomics, no memset, bit-reproducible.
#pragma once
#include "loudness.cuh"

namespace ddsp {
namespace mel_ {

constexpr int kMaxBins = 1024;      // every fft_length fits one warp with these
constexpr int kMinOwn = 4096;       // backward: samples a CTA owns when they fit
constexpr int kOwnFloor = 1024;     // ... halved down to this where they do not
constexpr int kMel = 0, kLogMel = 1, kMfcc = 2;   // DDSP_B200_MEL / _LOGMEL / _MFCC

// The sparse mel matrix, laid out by the host as 32-bit words (include/ddsp_b200.h):
// [K] float2 (w_lo, w_hi), [K] int band, [bins] int band_lo, [bins] int band_hi.  Bin
// k weighs w_lo into band[k] (if >= 0) and w_hi into band[k] + 1 (if < bins).
struct MelParams {
  const float* audio;      // [B, N]
  const float* window;     // [fft_size]
  const float2* wpair;     // [K]
  const int* band;         // [K]
  const int* band_lo;      // [bins]
  const int* band_hi;      // [bins]
  int N, T, fft_size, M, log2M, hop, bins, C;
};

__device__ __forceinline__ float bin_mag(float2 X) { return sqrtf(fmaf(X.x, X.x, X.y * X.y)); }

// core.safe_log: log(where(x <= 0, 1e-5, x)), in double
__device__ __forceinline__ float safe_log(float m) {
  return (float)log(m <= 0.f ? 1e-5 : (double)m);
}

// 2 cos(pi m / (2 bins)) / sqrt(2 bins) for m in [0, 4 bins), in double
__device__ __forceinline__ void fill_dct(float* ctab, int bins) {
  const double s = 2.0 / sqrt(2.0 * bins);
  for (int m = threadIdx.x; m < 4 * bins; m += blockDim.x)
    ctab[m] = (float)(s * cospi((double)m / (2.0 * bins)));
}

// The windowed frame (x(n) gives sample n, n < fft_size) zero-padded to 2M and packed
// into z in bit-reversed order.
template <typename X>
__device__ __forceinline__ void load_frame(float2* z, const MelParams& p, int lane, X x) {
  for (int j = lane; j < p.M; j += 32) {
    const int n0 = 2 * j, n1 = n0 + 1;
    const float v0 = n0 < p.fft_size ? __ldg(p.window + n0) * x(n0) : 0.f;
    const float v1 = n1 < p.fft_size ? __ldg(p.window + n1) * x(n1) : 0.f;
    z[ld_::bitrev(j, p.log2M)] = make_float2(v0, v1);
  }
}

// mel_j = sum_k W_kj |X_k| over band j's bins, ascending, from the packed spectrum z.
__device__ __forceinline__ float band_mel(const float2* z, const float2* tab,
                                          const MelParams& p, int j) {
  const int M = p.M, k1 = __ldg(p.band_hi + j);
  float acc = 0.f;
  for (int k = __ldg(p.band_lo + j); k < k1; ++k) {
    const float2 X =
        ld_::split_bin(z[k & (M - 1)], z[(M - k) & (M - 1)], ld_::twiddle(tab, k, M));
    const float2 w = __ldg(p.wpair + k);
    acc = fmaf(__ldg(p.band + k) == j ? w.x : w.y, bin_mag(X), acc);
  }
  return acc;
}

// MFCC coefficient c from the log-mel row lm: c (2n + 1) mod 4 bins indexes ctab.
__device__ __forceinline__ float dct_coef(const float* lm, const float* ctab, int bins, int c) {
  const int period = 4 * bins, step = 2 * c;
  float acc = 0.f;
  for (int n = 0, m = c; n < bins; ++n) {
    acc = fmaf(lm[n], ctab[m], acc);
    m += step;
    if (m >= period) m -= period;
  }
  return acc;
}

// Its transpose: d logmel_n = sum_c g_c ctab[c (2n + 1) mod 4 bins].
__device__ __forceinline__ float dct_adjoint(const float* __restrict__ g, const float* ctab,
                                             int bins, int C, int n) {
  const int period = 4 * bins, step = 2 * n + 1;
  float acc = 0.f;
  for (int c = 0, m = 0; c < C; ++c) {
    acc = fmaf(__ldg(g + c), ctab[m], acc);
    m += step;
    if (m >= period) m -= period;
  }
  return acc;
}

// (256, 1): with no minimum ptxas holds the MEL instance to 32 registers and spills
template <int Mode>
__global__ void __launch_bounds__(256, 1)
mel_kernel(MelParams p, float* __restrict__ out, int frames_per_cta, int span) {
  extern __shared__ float4 mel_smem[];
  float2* tab = reinterpret_cast<float2*>(mel_smem);
  const int n_warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float2* z = tab + (size_t)p.M * (1 + warp);
  float* rows = reinterpret_cast<float*>(tab + (size_t)p.M * (1 + n_warps));
  float* lm = rows + (size_t)p.bins * warp;
  float* ctab = rows + (size_t)p.bins * n_warps;
  float* sp = ctab + (Mode == kMfcc ? 4 * p.bins : 0);
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * frames_per_cta;
  const int t1 = min(p.T, t0 + frames_per_cta);
  const float* a = p.audio + (size_t)b * p.N;
  ld_::fill_twiddles(tab, p.M);
  if (Mode == kMfcc) fill_dct(ctab, p.bins);
  const long long s0 = (long long)t0 * p.hop;
  for (int i = threadIdx.x; i < span; i += blockDim.x)
    sp[i] = s0 + i < p.N ? a[s0 + i] : 0.f;
  __syncthreads();
  for (int t = t0 + warp; t < t1; t += n_warps) {
    const long long st = (long long)t * p.hop;
    if (span) {
      const float* x = sp + (st - s0);
      load_frame(z, p, lane, [x](int n) { return x[n]; });
    } else {
      const int N = p.N;
      load_frame(z, p, lane, [a, st, N](int n) {
        return st + n < N ? __ldg(a + st + n) : 0.f;
      });
    }
    ld_::fft_dit(z, tab, p.M, p.log2M, lane);
    float* o = out + ((size_t)b * p.T + t) * p.C;
    for (int j = lane; j < p.bins; j += 32) {
      const float m = band_mel(z, tab, p, j);
      if (Mode == kMel) o[j] = m;
      else if (Mode == kLogMel) o[j] = safe_log(m);
      else lm[j] = safe_log(m);
    }
    if (Mode == kMfcc) {
      __syncwarp();
      for (int c = lane; c < p.C; c += 32) o[c] = dct_coef(lm, ctab, p.bins, c);
    }
    __syncwarp();
  }
}

// The d frame of frame t into z (bit-reversed, as the inverse FFT leaves it), without
// the window.  dm: the warp's [bins] row for d mel.
template <int Mode>
__device__ __forceinline__ void frame_grad(float2* z, const float2* tab, float* dm,
                                           const float* ctab, const MelParams& p,
                                           const float* __restrict__ a,
                                           const float* __restrict__ g, int t, int lane) {
  const long long st = (long long)t * p.hop;
  const int N = p.N, M = p.M;
  load_frame(z, p, lane, [a, st, N](int n) { return st + n < N ? __ldg(a + st + n) : 0.f; });
  ld_::fft_dit(z, tab, M, p.log2M, lane);
  for (int j = lane; j < p.bins; j += 32) {
    float d;
    if (Mode == kMel) {
      d = __ldg(g + j);
    } else {
      const float m = band_mel(z, tab, p, j);
      const float dl = Mode == kLogMel ? __ldg(g + j) : dct_adjoint(g, ctab, p.bins, p.C, j);
      d = m > 0.f ? dl / m : 0.f;
    }
    dm[j] = d;
  }
  __syncwarp();
  // d|X_k| = w_lo dm[band k] + w_hi dm[band k + 1]; Y_k = d|X_k| X_k / |X_k|, halved
  // inside (0, M) as the inverse split step's transpose wants (loudness frame_grad)
  auto grad_bin = [&](float2 X, int k) {
    const int j = __ldg(p.band + k);
    const float2 w = __ldg(p.wpair + k);
    float dmag = j >= 0 ? w.x * dm[j] : 0.f;
    if (j + 1 < p.bins) dmag = fmaf(w.y, dm[j + 1], dmag);
    const float mag = bin_mag(X);
    const float s = mag > 0.f ? dmag / mag * (k == 0 || k == M ? 1.f : 0.5f) : 0.f;
    return make_float2(s * X.x, s * X.y);
  };
  for (int k = lane; k <= (M >> 1); k += 32) {
    const int km = (M - k) & (M - 1);
    const float2 zk = z[k & (M - 1)], zm = z[km];
    const float2 tk = ld_::twiddle(tab, k, M), tm = ld_::twiddle(tab, M - k, M);
    const float2 yk = grad_bin(ld_::split_bin(zk, zm, tk), k);
    const float2 ym = grad_bin(ld_::split_bin(zm, zk, tm), M - k);
    z[k & (M - 1)] = ld_::unsplit_bin(yk, ym, make_float2(tk.x, -tk.y));
    if (km != (k & (M - 1))) z[km] = ld_::unsplit_bin(ym, yk, make_float2(tm.x, -tm.y));
  }
  ld_::ifft_dif(z, tab, M, p.log2M, lane);
}

template <int Mode>
__global__ void __launch_bounds__(256)
mel_backward_kernel(MelParams p, const float* __restrict__ grad, float* __restrict__ d_audio,
                    int own) {
  extern __shared__ float4 mel_smem[];
  float2* tab = reinterpret_cast<float2*>(mel_smem);
  const int n_warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float2* z = tab + (size_t)p.M * (1 + warp);
  float* rows = reinterpret_cast<float*>(tab + (size_t)p.M * (1 + n_warps));
  float* dm = rows + (size_t)p.bins * warp;
  float* ctab = rows + (size_t)p.bins * n_warps;
  float* acc = ctab + (Mode == kMfcc ? 4 * p.bins : 0);
  int* active = reinterpret_cast<int*>(acc + own);
  const int b = blockIdx.y;
  const int a0 = blockIdx.x * own, n_own = min(p.N - a0, own);
  const float* a = p.audio + (size_t)b * p.N;
  ld_::fill_twiddles(tab, p.M);
  if (Mode == kMfcc) fill_dct(ctab, p.bins);
  for (int i = threadIdx.x; i < n_own; i += blockDim.x) acc[i] = 0.f;
  // frames t with t hop <= q < t hop + fft_size for a sample q in [a0, a0 + n_own)
  const long long q0 = a0, q1 = q0 + n_own;
  const long long lo = q0 - p.fft_size + 1;
  const int t_lo = lo <= 0 ? 0 : (int)((lo + p.hop - 1) / p.hop);
  const int t_hi = (int)min((long long)p.T - 1, (q1 - 1) / p.hop);
  __syncthreads();
  for (int tb = t_lo; tb <= t_hi; tb += n_warps) {
    const int t = tb + warp;
    if (t <= t_hi)
      frame_grad<Mode>(z, tab, dm, ctab, p, a, grad + ((size_t)b * p.T + t) * p.C, t, lane);
    if (lane == 0) active[warp] = t <= t_hi;
    __syncthreads();
    for (int i = threadIdx.x; i < n_own; i += blockDim.x) {
      float s = acc[i];
      for (int w = 0; w < n_warps; ++w) {
        if (!active[w]) continue;
        const long long n = q0 + i - (long long)(tb + w) * p.hop;
        if (n < 0 || n >= p.fft_size) continue;
        const float2 v = tab[(size_t)p.M * (1 + w) + ld_::bitrev((int)n >> 1, p.log2M)];
        s = fmaf(__ldg(p.window + n), (n & 1) ? v.y : v.x, s);
      }
      acc[i] = s;
    }
    __syncthreads();
  }
  float* o = d_audio + (size_t)b * p.N + a0;
  for (int i = threadIdx.x; i < n_own; i += blockDim.x) o[i] = acc[i];
}

}  // namespace mel_
}  // namespace ddsp
