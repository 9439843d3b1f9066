// C ABI of the harmonic family: the harmonic and noise controls and their
// backward, the harmonic forward kernels and their backward.
#include "capi.cuh"
#include "controls.cuh"
#include "harmonic.cuh"
#include "harmonic_v4.cuh"
#include "harmonic_backward.cuh"
#include "controls_bwd.cuh"

namespace ddsp {

// Halves the frames per tile from FT until smem(FT, Kp) fits one CTA.  Returns the
// tile, or 0 with the error set when not even one frame fits.
static int fit_tile(const char* name, int FT, int K, int Kp, size_t (*smem)(int, int)) {
  while (FT > 1 && smem(FT, Kp) > kMaxDynSmem) FT = (FT + 1) / 2;
  DDSP_REQUIRE(smem(FT, Kp) <= kMaxDynSmem, 0,
               "%s: K=%d needs more shared memory than one CTA has", name, K);
  return FT;
}

}  // namespace ddsp

using namespace ddsp;

extern "C" {

int ddsp_b200_harmonic_controls(const float* amps_in, const float* hd_in,
                                const float* f0_hz, float* amps_out,
                                float* hd_out, int B, int F, int K,
                                float sample_rate, int flags, void* stream) {
  DDSP_REQUIRE(amps_in && hd_in && f0_hz && amps_out && hd_out,
               DDSP_B200_E_INVALID, "harmonic_controls: null pointer");
  DDSP_REQUIRE(B >= 0 && F >= 0 && K >= 1, DDSP_B200_E_INVALID,
               "harmonic_controls: bad shape B=%d F=%d K=%d", B, F, K);
  const int64_t rows = (int64_t)B * F;
  if (rows == 0) return 0;
  DDSP_REQUIRE(rows < (1ll << 31) / 32, DDSP_B200_E_INVALID,
               "harmonic_controls: B*F too large");
  int rc = check_overlap("harmonic_controls", {DDSP_OUT(amps_out, extent(B, F), amps_in),
                                               DDSP_OUT(hd_out, extent(B, F, K), hd_in)},
                         {DDSP_IN(amps_in, extent(B, F)), DDSP_IN(hd_in, extent(B, F, K)),
                          DDSP_IN(f0_hz, extent(B, F))});
  if (rc) return rc;
  const int threads = 256;
  const int blocks = (int)((rows * 32 + threads - 1) / threads);
  return launch("harmonic_controls", harmonic_controls_kernel, blocks, threads, 0,
                (cudaStream_t)stream, amps_in, hd_in, f0_hz, amps_out, hd_out, (int)rows, K,
                sample_rate * 0.5f, flags);
}

int ddsp_b200_harmonic_forward(const float* f0_hz, const float* amps,
                               const float* hd, float* audio, int B, int F,
                               int K, int N, float sample_rate, int amp_method,
                               int phase_mode, int accumulate, void* stream) {
  DDSP_REQUIRE(f0_hz && amps && audio, DDSP_B200_E_INVALID,
               "harmonic_forward: null pointer");
  int rc = harm_check("harmonic_forward", B, F, K, N, amp_method, sample_rate);
  if (rc) return rc;
  DDSP_REQUIRE(hd != nullptr || K == 1, DDSP_B200_E_INVALID,
               "harmonic_forward: harmonic_distribution is NULL but K=%d", K);
  DDSP_REQUIRE(phase_mode == DDSP_B200_PHASE_RECURRENCE ||
                   phase_mode == DDSP_B200_PHASE_DIRECT,
               DDSP_B200_E_INVALID, "harmonic_forward: bad phase_mode %d",
               phase_mode);
  // upsample_with_windows raises unless N % F == 0 and F < N (core.py:682-693);
  // the closed-form phase also needs an integer hop.
  DDSP_REQUIRE(N % F == 0, DDSP_B200_E_INVALID,
               "harmonic_forward: n_samples (%d) must be divisible by the "
               "number of frames (%d)", N, F);
  DDSP_REQUIRE(amp_method != DDSP_B200_AMP_WINDOW || F < N,
               DDSP_B200_E_INVALID,
               "harmonic_forward: window upsampling cannot downsample "
               "(frames %d >= timesteps %d)", F, N);
  if (B == 0) return 0;
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID,
               "harmonic_forward: B=%d exceeds the 65535 grid limit", B);

  rc = check_overlap("harmonic_forward", {DDSP_OUT(audio, extent(B, N))},
                     {DDSP_IN(f0_hz, extent(B, F)), DDSP_IN(amps, extent(B, F)),
                      DDSP_IN(hd, extent(B, F, K))});
  if (rc) return rc;
  HarmonicParams p = harm_params(f0_hz, amps, hd, audio, B, F, K, N, sample_rate,
                                 amp_method);
  p.accumulate = accumulate;
  cudaStream_t st = (cudaStream_t)stream;

  if (phase_mode == DDSP_B200_PHASE_RECURRENCE && harmonic_fused_supported(p)) {
    rc = launch_harmonic_v4(p, st);
    if (rc != 1) return rc;   // 1 = declined, fall through to the generic path
  }

  // frames per tile: ~2048 samples, enough CTAs to fill the chip, bounded smem
  int FT = std::max(1, 2048 / p.hop);
  const int64_t want_ctas = 4ll * num_sms();
  int ft_fill = (int)std::max<int64_t>(1, ((int64_t)B * F + want_ctas - 1) / want_ctas);
  FT = std::min(FT, std::max(ft_fill, std::min(4, F)));
  FT = std::min(FT, F);
  p.FT = fit_tile("harmonic_forward", FT, K, p.Kp, harm_smem_bytes);
  if (!p.FT) return DDSP_B200_E_UNSUPPORTED;
  const size_t smem = harm_smem_bytes(p.FT, p.Kp);
  auto kern = phase_mode == DDSP_B200_PHASE_DIRECT ? harmonic_generic_kernel<1>
                                                   : harmonic_generic_kernel<0>;
  return launch("harmonic_forward", kern, dim3((F + p.FT - 1) / p.FT, B), kHarmThreads,
                smem, st, p);
}

int ddsp_b200_streaming_harmonic_forward(const float* f0_hz, const float* amps,
                                         const float* hd, const float* initial_phase,
                                         float* audio, float* final_phase, int B,
                                         int F, int K, int N, float sample_rate,
                                         int amp_method, void* stream) {
  DDSP_REQUIRE(f0_hz && amps && audio, DDSP_B200_E_INVALID,
               "streaming_harmonic_forward: null pointer");
  int rc = harm_check("streaming_harmonic_forward", B, F, K, N, amp_method, sample_rate);
  if (rc) return rc;
  DDSP_REQUIRE(hd != nullptr || K == 1, DDSP_B200_E_INVALID,
               "streaming_harmonic_forward: harmonic_distribution is NULL but K=%d", K);
  DDSP_REQUIRE(N % F == 0, DDSP_B200_E_INVALID,
               "streaming_harmonic_forward: n_samples (%d) must be divisible by "
               "the number of frames (%d)", N, F);
  if (B == 0) return 0;
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID,
               "streaming_harmonic_forward: B=%d exceeds the 65535 grid limit", B);
  HarmonicParams p = harm_params(f0_hz, amps, hd, audio, B, F, K, N, sample_rate,
                                 amp_method);
  p.init_phase = initial_phase; p.final_phase = final_phase; p.mask_nyquist = 0;
  p.FT = fit_tile("streaming_harmonic_forward", std::max(1, std::min(F, 2048 / p.hop)),
                  K, p.Kp, harm_smem_bytes);
  if (!p.FT) return DDSP_B200_E_UNSUPPORTED;
  rc = check_overlap("streaming_harmonic_forward", {DDSP_OUT(audio, extent(B, N)),
                                                    DDSP_OUT(final_phase, extent(B))},
                     {DDSP_IN(f0_hz, extent(B, F)), DDSP_IN(amps, extent(B, F)),
                      DDSP_IN(hd, extent(B, F, K)), DDSP_IN(initial_phase, extent(B))});
  if (rc) return rc;
  const size_t smem = harm_smem_bytes(p.FT, p.Kp);
  dim3 grid((F + p.FT - 1) / p.FT, B);
  return launch("streaming_harmonic_forward", harmonic_generic_kernel<0>, grid,
                kHarmThreads, smem, (cudaStream_t)stream, p);
}

int ddsp_b200_noise_controls(const float* mag_in, float* mag_out, int64_t n,
                             float initial_bias, int apply_scale, void* stream) {
  DDSP_REQUIRE(mag_in && mag_out, DDSP_B200_E_INVALID,
               "noise_controls: null pointer");
  DDSP_REQUIRE(n >= 0, DDSP_B200_E_INVALID, "noise_controls: n < 0");
  if (n == 0) return 0;
  int rc = check_overlap("noise_controls", {DDSP_OUT(mag_out, extent(n), mag_in)},
                         {DDSP_IN(mag_in, extent(n))});
  if (rc) return rc;
  return launch("noise_controls", noise_controls_kernel, grid_for(n, 256), 256, 0,
                (cudaStream_t)stream, mag_in, mag_out, n, initial_bias, apply_scale);
}

int ddsp_b200_harmonic_backward_takes(int B, int F, int N) {
  if (F < 1) return 0;
  const int hop = N / F;
  return hop >= 64 && hop % 64 == 0 && hop <= 8192 && B <= 65535;
}

int ddsp_b200_harmonic_backward(const float* f0_hz, const float* grad_audio,
                                float* g0, float* g1, int B, int F, int K, int N,
                                float sample_rate, int amp_method, void* stream) {
  DDSP_REQUIRE(f0_hz && grad_audio && g0 && g1, DDSP_B200_E_INVALID,
               "harmonic_backward: null pointer");
  int rc = harm_check("harmonic_backward", B, F, K, N, amp_method, sample_rate);
  if (rc) return rc;
  DDSP_REQUIRE(N % F == 0, DDSP_B200_E_INVALID,
               "harmonic_backward: bad shape B=%d F=%d K=%d N=%d", B, F, K, N);
  if (B == 0) return 0;
  HarmonicParams p = harm_params(f0_hz, nullptr, nullptr, nullptr, B, F, K, N,
                                 sample_rate, amp_method);
  p.Kp = K;
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_UNSUPPORTED,
               "harmonic_backward: B=%d exceeds the 65535 grid limit", B);
  DDSP_REQUIRE(ddsp_b200_harmonic_backward_takes(B, F, N), DDSP_B200_E_UNSUPPORTED,
               "harmonic_backward: needs hop %% 64 == 0 (hop = %d)", p.hop);
  return launch_harmonic_backward(p, grad_audio, g0, g1, (cudaStream_t)stream);
}

int ddsp_b200_harmonic_backward_f0(const float* f0_hz, const float* amps,
                                   const float* hd, const float* grad_audio,
                                   float* d_f0, int B, int F, int K, int N,
                                   float sample_rate, int amp_method,
                                   void* workspace, size_t workspace_bytes,
                                   void* stream) {
  DDSP_REQUIRE(f0_hz && amps && grad_audio && d_f0, DDSP_B200_E_INVALID,
               "harmonic_backward_f0: null pointer");
  int rc = harm_check("harmonic_backward_f0", B, F, K, N, amp_method, sample_rate);
  if (rc) return rc;
  DDSP_REQUIRE(N % F == 0, DDSP_B200_E_INVALID,
               "harmonic_backward_f0: bad shape B=%d F=%d K=%d N=%d", B, F, K, N);
  DDSP_REQUIRE(hd != nullptr || K == 1, DDSP_B200_E_INVALID,
               "harmonic_backward_f0: harmonic_distribution is NULL but K=%d", K);
  if (B == 0) return 0;
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID,
               "harmonic_backward_f0: B=%d exceeds the 65535 grid limit", B);
  const size_t need = sizeof(float) * 3 * (size_t)B * F;
  DDSP_REQUIRE(workspace != nullptr && workspace_bytes >= need, DDSP_B200_E_WORKSPACE,
               "harmonic_backward_f0: workspace of %zu B needed, %zu given", need,
               workspace_bytes);
  HarmonicParams p = harm_params(f0_hz, amps, hd, nullptr, B, F, K, N, sample_rate,
                                 amp_method);
  p.FT = fit_tile("harmonic_backward_f0", std::max(1, std::min(F, 2048 / p.hop)), K,
                  p.Kp, harmonic_df0_smem);
  if (!p.FT) return DDSP_B200_E_UNSUPPORTED;
  const size_t smem = harmonic_df0_smem(p.FT, p.Kp);
  cudaStream_t st = (cudaStream_t)stream;
  float* sq = reinterpret_cast<float*>(workspace);
  auto kern = amp_method == DDSP_B200_AMP_WINDOW ? harmonic_df0_kernel<true>
                                                 : harmonic_df0_kernel<false>;
  rc = launch("harmonic_backward_f0", kern, dim3((F + p.FT - 1) / p.FT, B), kDf0Threads,
              smem, st, p, grad_audio, sq);
  if (rc) return rc;
  return launch("harmonic_backward_f0(finalize)", harmonic_df0_finalize, (B + 127) / 128,
                128, 0, st, sq, d_f0, B, F, p.hop, (float)p.inv_sr);
}

int ddsp_b200_harmonic_controls_backward(const float* amps_raw, const float* hd_raw,
                                         const float* f0_hz, const float* g0,
                                         const float* g1, float* d_amps_raw,
                                         float* d_hd_raw, int B, int F, int K,
                                         float sample_rate, int flags, void* stream) {
  DDSP_REQUIRE(amps_raw && hd_raw && f0_hz && g0 && g1 && d_amps_raw && d_hd_raw,
               DDSP_B200_E_INVALID, "harmonic_controls_backward: null pointer");
  DDSP_REQUIRE(B >= 0 && F >= 1 && K >= 1, DDSP_B200_E_INVALID,
               "harmonic_controls_backward: bad shape B=%d F=%d K=%d", B, F, K);
  const int64_t rows = (int64_t)B * F;
  if (rows == 0) return 0;
  DDSP_REQUIRE(rows < (1ll << 31) / 32, DDSP_B200_E_INVALID,
               "harmonic_controls_backward: B*F too large");
  const int threads = 256;
  const int blocks = (int)((rows * 32 + threads - 1) / threads);
  return launch("harmonic_controls_backward", harmonic_controls_backward_kernel, blocks,
                threads, 0, (cudaStream_t)stream, amps_raw, hd_raw, f0_hz, g0, g1,
                d_amps_raw, d_hd_raw, (int)rows, F, K, sample_rate * 0.5f, flags);
}

int ddsp_b200_harmonic_controls_vjp(const float* amps_raw, const float* hd_raw,
                                    const float* f0_hz, const float* d_amplitudes,
                                    const float* d_hd, float* d_amps_raw, float* d_hd_raw,
                                    int B, int F, int K, float sample_rate, int flags,
                                    void* stream) {
  DDSP_REQUIRE(amps_raw && hd_raw && f0_hz && d_amps_raw && d_hd_raw,
               DDSP_B200_E_INVALID, "harmonic_controls_vjp: null pointer");
  DDSP_REQUIRE(B >= 0 && F >= 1 && K >= 1, DDSP_B200_E_INVALID,
               "harmonic_controls_vjp: bad shape B=%d F=%d K=%d", B, F, K);
  const int64_t rows = (int64_t)B * F;
  if (rows == 0) return 0;
  DDSP_REQUIRE(rows < (1ll << 31) / 32, DDSP_B200_E_INVALID,
               "harmonic_controls_vjp: B*F too large");
  const int threads = 256;
  const int blocks = (int)((rows * 32 + threads - 1) / threads);
  return launch("harmonic_controls_vjp", harmonic_controls_vjp_kernel, blocks, threads, 0,
                (cudaStream_t)stream, amps_raw, hd_raw, f0_hz, d_amplitudes, d_hd,
                d_amps_raw, d_hd_raw, (int)rows, K, sample_rate * 0.5f, flags);
}

int ddsp_b200_noise_controls_backward(const float* mags_raw, const float* d_mags,
                                      float* d_raw, int64_t n, float initial_bias,
                                      void* stream) {
  DDSP_REQUIRE(mags_raw && d_mags && d_raw, DDSP_B200_E_INVALID,
               "noise_controls_backward: null pointer");
  DDSP_REQUIRE(n >= 0, DDSP_B200_E_INVALID, "noise_controls_backward: n < 0");
  if (n == 0) return 0;
  return launch("noise_controls_backward", noise_controls_backward_kernel, grid_for(n, 256),
                256, 0, (cudaStream_t)stream, mags_raw, d_mags, d_raw, n, initial_bias);
}

#ifdef DDSP_HV4_TIMING
// measurement builds only (tools/harm_timing.py): the harmonic_v4 phase counters
// summed since the previous call, [kMaxSMs][8 phases + warps counted] cycles; the
// counters are zeroed after the copy
int ddsp_b200_debug_harm_timing(unsigned long long* host_out) {
  const size_t bytes = sizeof(unsigned long long) * kMaxSMs * (ddsp::hv4::kTimingPhases + 1);
  cudaError_t e = cudaMemcpyFromSymbol(host_out, ddsp::hv4::g_hv4_timing, bytes);
  if (e != cudaSuccess) return DDSP_B200_E_CUDA;
  void* dev = nullptr;
  e = cudaGetSymbolAddress(&dev, ddsp::hv4::g_hv4_timing);
  if (e == cudaSuccess) e = cudaMemset(dev, 0, bytes);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  return e == cudaSuccess ? 0 : DDSP_B200_E_CUDA;
}
#endif

}  // extern "C"
