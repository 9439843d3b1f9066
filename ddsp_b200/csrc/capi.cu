// C ABI of libddsp_b200.so - argument validation + kernel launches.
// See include/ddsp_b200.h for the contract and the reference file:line each
// entry point replaces.
#include <stdarg.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "controls.cuh"
#include "harmonic.cuh"
#include "harmonic_v4.cuh"
#include "noise.cuh"
#include "noise_fused.cuh"
#include "noise_ring.cuh"
#include "host_pipeline.cuh"
#include "noise_backward.cuh"
#include "harmonic_backward.cuh"
#include "harmonic_bwd2.cuh"
#include "controls_bwd.cuh"
#include "oscbank.cuh"
#include "sinusoidal.cuh"
#include "longconv.cuh"
#include "spectral.cuh"
#include "mod_delay.cuh"
#include "fir_backward.cuh"
#include "routing.cuh"
#include "wavetable.cuh"
#include "loudness.cuh"
#include "mel.cuh"
#include "consistency.cuh"
#include "sinc.cuh"
#include "hmm.cuh"

namespace ddsp {

static thread_local char g_err[512] = "";
static thread_local uint64_t g_launches = 0;

void count_launch() { ++g_launches; }

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static inline int grid_for(int64_t n, int threads, int cap_per_sm = 8) {
  int64_t blocks = (n + threads - 1) / threads;
  int64_t cap = (int64_t)num_sms() * cap_per_sm;
  return (int)std::max<int64_t>(1, std::min(blocks, cap));
}

// The checks every harmonic entry point makes; `name` prefixes the messages.
static int harm_check(const char* name, int B, int F, int K, int N, int amp_method,
                      float sample_rate) {
  DDSP_REQUIRE(B >= 0 && F >= 1 && K >= 1 && N >= 1, DDSP_B200_E_INVALID,
               "%s: bad shape B=%d F=%d K=%d N=%d", name, B, F, K, N);
  DDSP_REQUIRE(amp_method == DDSP_B200_AMP_WINDOW || amp_method == DDSP_B200_AMP_LINEAR,
               DDSP_B200_E_INVALID, "%s: bad amp_method %d", name, amp_method);
  DDSP_REQUIRE(sample_rate > 0.f, DDSP_B200_E_INVALID,
               "%s: sample_rate must be positive", name);
  return 0;
}

// HarmonicParams of a harmonic entry point.  The caller sets the fields in which it
// differs: accumulate, ctl_flags, the phase pointers, mask_nyquist and Kp.
static HarmonicParams harm_params(const float* f0, const float* amps, const float* hd,
                                  float* audio, int B, int F, int K, int N,
                                  float sample_rate, int amp_method) {
  HarmonicParams p;
  p.f0 = f0; p.amps = amps; p.hd = hd; p.audio = audio;
  p.B = B; p.F = F; p.K = K; p.N = N; p.hop = N / F;
  p.sample_rate = sample_rate; p.nyquist = sample_rate * 0.5f;
  p.inv_sr = 1.0 / (double)sample_rate;
  p.amp_method = amp_method; p.accumulate = 0; p.ctl_flags = 0;
  p.init_phase = nullptr; p.final_phase = nullptr; p.mask_nyquist = 1;
  p.Kp = (K + 3) & ~3;
  return p;
}

// Halves the frames per tile from FT until smem(FT, Kp) fits one CTA.  Returns the
// tile, or 0 with the error set when not even one frame fits.
static int fit_tile(const char* name, int FT, int K, int Kp, size_t (*smem)(int, int)) {
  while (FT > 1 && smem(FT, Kp) > kMaxDynSmem) FT = (FT + 1) / 2;
  DDSP_REQUIRE(smem(FT, Kp) <= kMaxDynSmem, 0,
               "%s: K=%d needs more shared memory than one CTA has", name, K);
  return FT;
}

// core.py:1446-1457: F impulse responses over N samples have frames of ceil(N / F)
// samples, and framing the audio with that size (pad_end) must give F frames.
// Returns the frame size, or 0 with the error set.
static int ir_frame(int N, int F) {
  const int frame = (N + F - 1) / F;
  const int n_audio_frames = (N + frame - 1) / frame;
  DDSP_REQUIRE(n_audio_frames == F, 0,
               "Number of Audio frames (%d) and impulse response frames (%d) do "
               "not match. For small hop size = ceil(audio_size / n_ir_frames), "
               "number of impulse response frames must be a multiple of the "
               "audio size.", n_audio_frames, F);
  return frame;
}

// Workspaces are carved from the first 256-byte boundary at or after `p`.
template <typename T>
static T* align256(const void* p) {
  return reinterpret_cast<T*>(((uintptr_t)p + 255) & ~(uintptr_t)255);
}

}  // namespace ddsp

using namespace ddsp;

extern "C" {

int ddsp_b200_version(void) { return DDSP_B200_VERSION; }

const char* ddsp_b200_last_error(void) { return g_err; }

uint64_t ddsp_b200_launch_count(void) { return g_launches; }

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
  const int threads = 256;
  const int blocks = (int)((rows * 32 + threads - 1) / threads);
  harmonic_controls_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(
      amps_in, hd_in, f0_hz, amps_out, hd_out, (int)rows, K,
      sample_rate * 0.5f, flags);
  DDSP_CHECK_LAUNCH("harmonic_controls");
  return 0;
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
  rc = set_smem(kern, smem, "harmonic_forward");
  if (rc) return rc;
  kern<<<dim3((F + p.FT - 1) / p.FT, B), kHarmThreads, smem, st>>>(p);
  DDSP_CHECK_LAUNCH("harmonic_forward");
  return 0;
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
  const size_t smem = harm_smem_bytes(p.FT, p.Kp);
  rc = set_smem(harmonic_generic_kernel<0>, smem, "streaming_harmonic_forward");
  if (rc) return rc;
  dim3 grid((F + p.FT - 1) / p.FT, B);
  harmonic_generic_kernel<0><<<grid, kHarmThreads, smem, (cudaStream_t)stream>>>(p);
  DDSP_CHECK_LAUNCH("streaming_harmonic_forward");
  return 0;
}

int ddsp_b200_noise_controls(const float* mag_in, float* mag_out, int64_t n,
                             float initial_bias, int apply_scale, void* stream) {
  DDSP_REQUIRE(mag_in && mag_out, DDSP_B200_E_INVALID,
               "noise_controls: null pointer");
  DDSP_REQUIRE(n >= 0, DDSP_B200_E_INVALID, "noise_controls: n < 0");
  if (n == 0) return 0;
  noise_controls_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(
      mag_in, mag_out, n, initial_bias, apply_scale);
  DDSP_CHECK_LAUNCH("noise_controls");
  return 0;
}

int ddsp_b200_ir_size(int nb, int window_size) {
  if (nb < 2) return DDSP_B200_E_INVALID;
  return make_ir_geom(nb, window_size).S;
}

int ddsp_b200_frequency_impulse_response(const float* mags, float* ir,
                                         int64_t BF, int nb, int window_size,
                                         void* stream) {
  DDSP_REQUIRE(mags && ir, DDSP_B200_E_INVALID,
               "frequency_impulse_response: null pointer");
  DDSP_REQUIRE(nb >= 2 && BF >= 0, DDSP_B200_E_INVALID,
               "frequency_impulse_response: need n_frequencies >= 2 (got %d)", nb);
  if (BF == 0) return 0;
  IrGeom g = make_ir_geom(nb, window_size);
  const size_t smem = sizeof(float) * ((size_t)g.S0 + (size_t)kIrFrames * nb);
  DDSP_REQUIRE(smem <= kMaxDynSmem, DDSP_B200_E_UNSUPPORTED,
               "frequency_impulse_response: n_frequencies=%d too large", nb);
  int rc = set_smem(ir_kernel, smem, "frequency_impulse_response");
  if (rc) return rc;
  const int64_t blocks = (BF + kIrFrames - 1) / kIrFrames;
  DDSP_REQUIRE(blocks < (1ll << 31), DDSP_B200_E_INVALID,
               "frequency_impulse_response: too many frames");
  ir_kernel<<<(int)blocks, kIrThreads, smem, (cudaStream_t)stream>>>(mags, ir,
                                                                     BF, g);
  DDSP_CHECK_LAUNCH("frequency_impulse_response");
  return 0;
}

int ddsp_b200_fir_time_varying(const float* audio, const float* ir, float* out,
                               int B, int N, int F, int S, int ir_batch,
                               int padding, int delay_compensation,
                               int accumulate, void* stream) {
  DDSP_REQUIRE(audio && ir && out, DDSP_B200_E_INVALID,
               "fir_time_varying: null pointer");
  DDSP_REQUIRE(B >= 0 && N >= 1 && F >= 1 && S >= 1, DDSP_B200_E_INVALID,
               "fir_time_varying: bad shape B=%d N=%d F=%d S=%d", B, N, F, S);
  // core.py:1441-1443
  DDSP_REQUIRE(ir_batch == B || ir_batch == 1, DDSP_B200_E_INVALID,
               "Batch size of audio (%d) and impulse response (%d) must be the "
               "same.", B, ir_batch);
  DDSP_REQUIRE(padding == DDSP_B200_PAD_SAME || padding == DDSP_B200_PAD_VALID,
               DDSP_B200_E_INVALID,
               "Padding must be 'valid' or 'same' (got code %d)", padding);
  const int frame = ir_frame(N, F);
  if (!frame) return DDSP_B200_E_INVALID;
  if (B == 0) return 0;
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID,
               "fir_time_varying: B=%d exceeds the 65535 grid limit", B);
  // crop_and_compensate_delay (core.py:1338-1379)
  const int out_len = (padding == DDSP_B200_PAD_VALID) ? (N + S - 1) : N;
  const int start = delay_compensation < 0 ? ((S - 1) / 2 - 1)
                                           : delay_compensation;
  DDSP_REQUIRE(start >= 0, DDSP_B200_E_UNSUPPORTED,
               "fir_time_varying: impulse response of %d taps gives a negative "
               "automatic delay; pass delay_compensation >= 0", S);
  const size_t smem = sizeof(float) * ((size_t)kFirThreads + S - 1);
  DDSP_REQUIRE(smem <= kMaxDynSmem, DDSP_B200_E_UNSUPPORTED,
               "fir_time_varying: impulse response of %d taps is beyond the "
               "shared-memory FIR (long-IR convolution is not built yet)", S);
  int rc = set_smem(fir_kernel, smem, "fir_time_varying");
  if (rc) return rc;
  dim3 grid((out_len + kFirThreads - 1) / kFirThreads, B);
  fir_kernel<<<grid, kFirThreads, smem, (cudaStream_t)stream>>>(
      audio, ir, out, N, F, S, frame, ir_batch == 1 ? 0 : F * S, start, out_len,
      accumulate);
  DDSP_CHECK_LAUNCH("fir_time_varying");
  return 0;
}

int ddsp_b200_uniform_noise(float* out, int B, int N, uint64_t seed,
                            uint64_t offset, void* stream) {
  DDSP_REQUIRE(out, DDSP_B200_E_INVALID, "uniform_noise: null pointer");
  DDSP_REQUIRE(B >= 0 && N >= 0, DDSP_B200_E_INVALID, "uniform_noise: bad shape");
  if (B == 0 || N == 0) return 0;
  const int64_t n = (int64_t)B * ((N + 3) / 4);
  uniform_noise_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(
      out, B, N, seed, offset);
  DDSP_CHECK_LAUNCH("uniform_noise");
  return 0;
}

size_t ddsp_b200_filtered_noise_workspace(int B, int F, int nb, int N,
                                          int window_size) {
  if (nb < 2 || B <= 0 || F <= 0 || N <= 0) return 0;
  if (noise_fused_supported(F, nb, N, window_size)) return 0;
  IrGeom g = make_ir_geom(nb, window_size);
  // generic path: IR [B,F,S] + noise [B,N]
  return sizeof(float) * ((size_t)B * F * g.S + (size_t)B * N) + 256;
}

int ddsp_b200_filtered_noise_forward(const float* mags, const float* noise,
                                     uint64_t seed, uint64_t offset,
                                     float* audio, int B, int F, int nb, int N,
                                     int window_size, int accumulate,
                                     void* workspace, size_t workspace_bytes,
                                     void* stream) {
  DDSP_REQUIRE(mags && audio, DDSP_B200_E_INVALID,
               "filtered_noise_forward: null pointer");
  DDSP_REQUIRE(B >= 0 && F >= 1 && N >= 1, DDSP_B200_E_INVALID,
               "filtered_noise_forward: bad shape B=%d F=%d N=%d", B, F, N);
  DDSP_REQUIRE(nb >= 2, DDSP_B200_E_INVALID,
               "filtered_noise_forward: need n_frequencies >= 2 (got %d)", nb);
  if (!ir_frame(N, F)) return DDSP_B200_E_INVALID;
  if (B == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (noise_fused_supported(F, nb, N, window_size)) {
    return launch_noise_best(mags, noise, seed, offset, audio, B, F, nb, N,
                             window_size, accumulate, st);
  }
  const size_t need = ddsp_b200_filtered_noise_workspace(B, F, nb, N, window_size);
  DDSP_REQUIRE(workspace != nullptr && workspace_bytes >= need,
               DDSP_B200_E_WORKSPACE,
               "filtered_noise_forward: workspace of %zu B needed, %zu given",
               need, workspace_bytes);
  IrGeom g = make_ir_geom(nb, window_size);
  float* ir = align256<float>(workspace);
  float* nz = ir + (size_t)B * F * g.S;
  int rc = ddsp_b200_frequency_impulse_response(mags, ir, (int64_t)B * F, nb,
                                                window_size, stream);
  if (rc) return rc;
  const float* x = noise;
  if (x == nullptr) {
    rc = ddsp_b200_uniform_noise(nz, B, N, seed, offset, stream);
    if (rc) return rc;
    x = nz;
  }
  return ddsp_b200_fir_time_varying(x, ir, audio, B, N, F, g.S, B,
                                    DDSP_B200_PAD_SAME, -1, accumulate, stream);
}

static int decoder_forward_impl(const float* amps_raw, const float* hd_raw,
                                const float* f0_hz, const float* mags_raw,
                                const float* noise, uint64_t seed, uint64_t offset,
                                float* audio, int B, int F, int K, int nb, int N,
                                float sample_rate, int amp_method,
                                int harmonic_flags, int window_size,
                                float initial_bias, void* stream, int item_base) {
  DDSP_REQUIRE(amps_raw && hd_raw && f0_hz && mags_raw && audio,
               DDSP_B200_E_INVALID, "decoder_forward: null pointer");
  int rc = harm_check("decoder_forward", B, F, K, N, amp_method, sample_rate);
  if (rc) return rc;
  DDSP_REQUIRE(nb >= 2, DDSP_B200_E_INVALID,
               "decoder_forward: need n_frequencies >= 2 (got %d)", nb);
  DDSP_REQUIRE(harmonic_flags != 0 &&
                   (harmonic_flags & ~(DDSP_B200_CTL_SCALE | DDSP_B200_CTL_NYQUIST)) == 0,
               DDSP_B200_E_INVALID, "decoder_forward: bad harmonic_flags %d",
               harmonic_flags);
  if (B == 0) return 0;
  HarmonicParams p = harm_params(f0_hz, amps_raw, hd_raw, audio, B, F, K, N,
                                 sample_rate, amp_method);
  p.ctl_flags = harmonic_flags;
  // The single-pass pipeline exists for the decoder regime only; everything
  // else goes through get_controls + the two *_forward calls.
  DDSP_REQUIRE(N % F == 0 && B <= 65535 && harmonic_fused_supported(p) &&
                   noise_fused_supported(F, nb, N, window_size),
               DDSP_B200_E_UNSUPPORTED,
               "decoder_forward: shape outside the fused decoder path "
               "(needs hop %% 64 == 0, n_frequencies <= %d)", kNfMaxNb);
  cudaStream_t st = (cudaStream_t)stream;
  rc = launch_harmonic_v4(p, st);
  if (rc == 1) {
    set_error("decoder_forward: harmonic tile does not fit shared memory");
    return DDSP_B200_E_UNSUPPORTED;
  }
  if (rc) return rc;
  return launch_noise_best(mags_raw, noise, seed, offset, audio, B, F, nb, N,
                           window_size, /*accumulate=*/1, st, /*raw=*/1,
                           initial_bias, item_base, /*overlap_previous=*/1);
}

int ddsp_b200_decoder_forward(const float* amps_raw, const float* hd_raw,
                              const float* f0_hz, const float* mags_raw,
                              const float* noise, uint64_t seed, uint64_t offset,
                              float* audio, int B, int F, int K, int nb, int N,
                              float sample_rate, int amp_method,
                              int harmonic_flags, int window_size,
                              float initial_bias, void* stream) {
  return decoder_forward_impl(amps_raw, hd_raw, f0_hz, mags_raw, noise, seed, offset,
                              audio, B, F, K, nb, N, sample_rate, amp_method,
                              harmonic_flags, window_size, initial_bias, stream, 0);
}

// ---- host-buffer pipeline ---------------------------------------------------
#define DDSP_CUDA_TRY(expr, what)                                         \
  do {                                                                    \
    cudaError_t e__ = (expr);                                             \
    if (e__ != cudaSuccess) {                                             \
      ::ddsp::set_error("%s: %s", what, cudaGetErrorString(e__));         \
      return DDSP_B200_E_CUDA;                                            \
    }                                                                     \
  } while (0)

int ddsp_b200_host_pipeline_create(ddsp_b200_host_pipeline** out, int max_B, int F,
                                   int K, int nb, int N, int max_chunks) {
  DDSP_REQUIRE(out != nullptr, DDSP_B200_E_INVALID, "host_pipeline_create: null out");
  *out = nullptr;
  DDSP_REQUIRE(max_B >= 1 && F >= 1 && K >= 1 && nb >= 2 && N >= 1 && max_chunks >= 1,
               DDSP_B200_E_INVALID,
               "host_pipeline_create: bad shape max_B=%d F=%d K=%d nb=%d N=%d chunks=%d",
               max_B, F, K, nb, N, max_chunks);
  HostPipeline* hp = new HostPipeline();
  auto fail = [&](const char* what, cudaError_t e) {
    set_error("host_pipeline_create: %s: %s", what, cudaGetErrorString(e));
    host_pipeline_free(hp);
    return DDSP_B200_E_CUDA;
  };
  cudaError_t e = cudaGetDevice(&hp->device);
  if (e != cudaSuccess) { hp->device = -1; return fail("cudaGetDevice", e); }
  hp->max_B = max_B; hp->F = F; hp->K = K; hp->nb = nb; hp->N = N;
  hp->max_chunks = std::min(max_chunks, max_B);
  // every sub-buffer starts on a 256-byte boundary (TMA bulk copies want 16)
  auto pad = [](size_t n) { return (n + 63) & ~(size_t)63; };
  const size_t n_amps = pad((size_t)max_B * F), n_hd = pad((size_t)max_B * F * K),
               n_mags = pad((size_t)max_B * F * nb), n_audio = pad((size_t)max_B * N);
  const size_t total = 2 * n_amps + n_hd + n_mags + n_audio;
  if ((e = cudaMalloc(&hp->d_base, total * sizeof(float))) != cudaSuccess)
    return fail("cudaMalloc(staging)", e);
  hp->d_amps = hp->d_base;
  hp->d_f0 = hp->d_amps + n_amps;
  hp->d_hd = hp->d_f0 + n_amps;
  hp->d_mags = hp->d_hd + n_hd;
  hp->d_audio = hp->d_mags + n_mags;
  if ((e = cudaStreamCreateWithFlags(&hp->s_h2d, cudaStreamNonBlocking)) != cudaSuccess)
    return fail("cudaStreamCreate", e);
  if ((e = cudaStreamCreateWithFlags(&hp->s_h2d2, cudaStreamNonBlocking)) != cudaSuccess)
    return fail("cudaStreamCreate", e);
  if ((e = cudaStreamCreateWithFlags(&hp->s_d2h, cudaStreamNonBlocking)) != cudaSuccess)
    return fail("cudaStreamCreate", e);
  if ((e = cudaEventCreateWithFlags(&hp->ev_start, cudaEventDisableTiming)) != cudaSuccess)
    return fail("cudaEventCreate", e);
  if ((e = cudaEventCreateWithFlags(&hp->ev_done, cudaEventDisableTiming)) != cudaSuccess)
    return fail("cudaEventCreate", e);
  for (int c = 0; c < hp->max_chunks; ++c) {
    cudaEvent_t a = nullptr, b = nullptr;
    if ((e = cudaEventCreateWithFlags(&a, cudaEventDisableTiming)) != cudaSuccess)
      return fail("cudaEventCreate", e);
    hp->ev_h2d.push_back(a);
    if ((e = cudaEventCreateWithFlags(&b, cudaEventDisableTiming)) != cudaSuccess)
      return fail("cudaEventCreate", e);
    hp->ev_comp.push_back(b);
    cudaEvent_t a2 = nullptr;
    if ((e = cudaEventCreateWithFlags(&a2, cudaEventDisableTiming)) != cudaSuccess)
      return fail("cudaEventCreate", e);
    hp->ev_h2d2.push_back(a2);
  }
  *out = reinterpret_cast<ddsp_b200_host_pipeline*>(hp);
  return 0;
}

int ddsp_b200_host_pipeline_destroy(ddsp_b200_host_pipeline* handle) {
  host_pipeline_free(reinterpret_cast<HostPipeline*>(handle));
  return 0;
}

int ddsp_b200_decoder_forward_host(ddsp_b200_host_pipeline* handle,
                                   const float* amps_raw, const float* hd_raw,
                                   const float* f0_hz, const float* mags_raw,
                                   uint64_t seed, uint64_t offset, float* audio,
                                   int B, int n_chunks, float sample_rate,
                                   int amp_method, int harmonic_flags,
                                   int window_size, float initial_bias,
                                   void* stream) {
  HostPipeline* hp = reinterpret_cast<HostPipeline*>(handle);
  DDSP_REQUIRE(hp != nullptr, DDSP_B200_E_INVALID, "decoder_forward_host: null handle");
  DDSP_REQUIRE(amps_raw && hd_raw && f0_hz && mags_raw && audio, DDSP_B200_E_INVALID,
               "decoder_forward_host: null pointer");
  DDSP_REQUIRE(B >= 0 && B <= hp->max_B, DDSP_B200_E_INVALID,
               "decoder_forward_host: B=%d outside [0, %d]", B, hp->max_B);
  if (B == 0) return 0;
  int dev = 0;
  DDSP_CUDA_TRY(cudaGetDevice(&dev), "decoder_forward_host: cudaGetDevice");
  DDSP_REQUIRE(dev == hp->device, DDSP_B200_E_INVALID,
               "decoder_forward_host: pipeline belongs to device %d, current is %d",
               hp->device, dev);
  n_chunks = std::max(1, std::min(std::min(std::min(n_chunks, hp->max_chunks), B), 64));
  const int F = hp->F, K = hp->K, nb = hp->nb, N = hp->N;
  cudaStream_t st = (cudaStream_t)stream;
  // Order this call after whatever the caller queued on `st`, and after the
  // previous call's last device->host copy (the staging buffers are reused).
  DDSP_CUDA_TRY(cudaEventRecord(hp->ev_start, st), "decoder_forward_host: event");
  DDSP_CUDA_TRY(cudaStreamWaitEvent(hp->s_h2d, hp->ev_start, 0), "decoder_forward_host: wait");
  DDSP_CUDA_TRY(cudaStreamWaitEvent(hp->s_h2d2, hp->ev_start, 0), "decoder_forward_host: wait");
  if (hp->used) {
    DDSP_CUDA_TRY(cudaStreamWaitEvent(hp->s_h2d, hp->ev_done, 0), "decoder_forward_host: wait");
    DDSP_CUDA_TRY(cudaStreamWaitEvent(hp->s_h2d2, hp->ev_done, 0), "decoder_forward_host: wait");
  }
  hp->used = true;
  // Two host->device streams (harmonic_distribution on one; magnitudes and the
  // small per-frame vectors on the other): a copy has a fixed set-up cost however
  // small it is, and on one stream those set-ups do not overlap the previous
  // transfer - two streams keep the link busy while one of them sets up.  The
  // per-frame vectors go over once for the whole batch.
  DDSP_CUDA_TRY(cudaMemcpyAsync(hp->d_f0, f0_hz, sizeof(float) * (size_t)B * F,
                                cudaMemcpyHostToDevice, hp->s_h2d2), "decoder_forward_host: H2D f0");
  DDSP_CUDA_TRY(cudaMemcpyAsync(hp->d_amps, amps_raw, sizeof(float) * (size_t)B * F,
                                cudaMemcpyHostToDevice, hp->s_h2d2), "decoder_forward_host: H2D amps");
  // Chunk sizes halve: the call ends with the compute + device->host copy of the
  // LAST chunk (nothing left to overlap them with), so that one should be small,
  // while few chunks keep the per-chunk submission cost down.
  int sizes[64];
  int n_c = 0;
  for (int b0 = 0; b0 < B; ++n_c) {
    const int left = B - b0;
    sizes[n_c] = (n_c == n_chunks - 1 || n_c == 63) ? left : std::max(1, (left + 1) / 2);
    b0 += sizes[n_c];
  }
  // First queue EVERY host->device copy: the copy engines then never wait for
  // this thread to get through the launches and event calls of earlier chunks
  // (driver time per chunk can exceed a small chunk's transfer).
  for (int c = 0, b0 = 0; c < n_c; b0 += sizes[c], ++c) {
    const int nbi = sizes[c];
    const size_t o1 = (size_t)b0 * F;
    DDSP_CUDA_TRY(cudaMemcpyAsync(hp->d_hd + o1 * K, hd_raw + o1 * K,
                                  sizeof(float) * (size_t)nbi * F * K,
                                  cudaMemcpyHostToDevice, hp->s_h2d), "decoder_forward_host: H2D hd");
    DDSP_CUDA_TRY(cudaEventRecord(hp->ev_h2d[c], hp->s_h2d), "decoder_forward_host: event");
    DDSP_CUDA_TRY(cudaMemcpyAsync(hp->d_mags + o1 * nb, mags_raw + o1 * nb,
                                  sizeof(float) * (size_t)nbi * F * nb,
                                  cudaMemcpyHostToDevice, hp->s_h2d2), "decoder_forward_host: H2D mags");
    DDSP_CUDA_TRY(cudaEventRecord(hp->ev_h2d2[c], hp->s_h2d2), "decoder_forward_host: event");
  }
  for (int c = 0, b0 = 0; c < n_c; b0 += sizes[c], ++c) {
    const int nbi = sizes[c];
    const size_t o1 = (size_t)b0 * F;
    DDSP_CUDA_TRY(cudaStreamWaitEvent(st, hp->ev_h2d[c], 0), "decoder_forward_host: wait");
    DDSP_CUDA_TRY(cudaStreamWaitEvent(st, hp->ev_h2d2[c], 0), "decoder_forward_host: wait");
    int rc = decoder_forward_impl(hp->d_amps + o1, hp->d_hd + o1 * K, hp->d_f0 + o1,
                                  hp->d_mags + o1 * nb, nullptr, seed, offset,
                                  hp->d_audio + (size_t)b0 * N, nbi, F, K, nb, N,
                                  sample_rate, amp_method, harmonic_flags, window_size,
                                  initial_bias, stream, b0);
    if (rc) return rc;
    DDSP_CUDA_TRY(cudaEventRecord(hp->ev_comp[c], st), "decoder_forward_host: event");
    DDSP_CUDA_TRY(cudaStreamWaitEvent(hp->s_d2h, hp->ev_comp[c], 0), "decoder_forward_host: wait");
    DDSP_CUDA_TRY(cudaMemcpyAsync(audio + (size_t)b0 * N, hp->d_audio + (size_t)b0 * N,
                                  sizeof(float) * (size_t)nbi * N, cudaMemcpyDeviceToHost,
                                  hp->s_d2h), "decoder_forward_host: D2H audio");
  }
  DDSP_CUDA_TRY(cudaEventRecord(hp->ev_done, hp->s_d2h), "decoder_forward_host: event");
  // The caller's stream completes when the audio is in host memory.
  DDSP_CUDA_TRY(cudaStreamWaitEvent(st, hp->ev_done, 0), "decoder_forward_host: wait");
  return 0;
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
  DDSP_REQUIRE(p.hop % 64 == 0 && p.hop <= 8192 && B <= 65535,
               DDSP_B200_E_UNSUPPORTED,
               "harmonic_backward: needs hop %% 64 == 0 (hop = %d)", p.hop);
  cudaStream_t st = (cudaStream_t)stream;
  if (harmonic_backward2_supported(p))
    return launch_harmonic_backward2(p, grad_audio, g0, g1, st);
  const size_t gbytes = sizeof(float) * (size_t)B * F * K;
  DDSP_CUDA_TRY(cudaMemsetAsync(g0, 0, gbytes, st), "harmonic_backward: memset g0");
  DDSP_CUDA_TRY(cudaMemsetAsync(g1, 0, gbytes, st), "harmonic_backward: memset g1");
  p.FT = std::max(1, std::min(F, 2048 / p.hop));
  const size_t smem = harmonic_backward_smem(p.FT, p.hop);
  auto kern = amp_method == DDSP_B200_AMP_WINDOW ? harmonic_backward_kernel<true>
                                                 : harmonic_backward_kernel<false>;
  rc = set_smem(kern, smem, "harmonic_backward");
  if (rc) return rc;
  kern<<<dim3((F + p.FT - 1) / p.FT, B), kHbThreads, smem, st>>>(p, grad_audio, g0, g1);
  DDSP_CHECK_LAUNCH("harmonic_backward");
  return 0;
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
  rc = set_smem(kern, smem, "harmonic_backward_f0");
  if (rc) return rc;
  kern<<<dim3((F + p.FT - 1) / p.FT, B), kDf0Threads, smem, st>>>(p, grad_audio, sq);
  DDSP_CHECK_LAUNCH("harmonic_backward_f0");
  harmonic_df0_finalize<<<(B + 127) / 128, 128, 0, st>>>(sq, d_f0, B, F, p.hop,
                                                       (float)p.inv_sr);
  DDSP_CHECK_LAUNCH("harmonic_backward_f0(finalize)");
  return 0;
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
  harmonic_controls_backward_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(
      amps_raw, hd_raw, f0_hz, g0, g1, d_amps_raw, d_hd_raw, (int)rows, F, K,
      sample_rate * 0.5f, flags);
  DDSP_CHECK_LAUNCH("harmonic_controls_backward");
  return 0;
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
  harmonic_controls_vjp_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(
      amps_raw, hd_raw, f0_hz, d_amplitudes, d_hd, d_amps_raw, d_hd_raw, (int)rows, K,
      sample_rate * 0.5f, flags);
  DDSP_CHECK_LAUNCH("harmonic_controls_vjp");
  return 0;
}

int ddsp_b200_noise_controls_backward(const float* mags_raw, const float* d_mags,
                                      float* d_raw, int64_t n, float initial_bias,
                                      void* stream) {
  DDSP_REQUIRE(mags_raw && d_mags && d_raw, DDSP_B200_E_INVALID,
               "noise_controls_backward: null pointer");
  DDSP_REQUIRE(n >= 0, DDSP_B200_E_INVALID, "noise_controls_backward: n < 0");
  if (n == 0) return 0;
  noise_controls_backward_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(
      mags_raw, d_mags, d_raw, n, initial_bias);
  DDSP_CHECK_LAUNCH("noise_controls_backward");
  return 0;
}

// NoiseBwdParams of a filtered-noise (or frequency_filter) shape whose frame is
// `frame`; *n_tiles and *smem are what the launch needs (the caller checks them).
static NoiseBwdParams noise_bwd_params(const float* grad, const float* noise, uint64_t seed,
                                       uint64_t offset, float* dmags, int B, int F, int nb,
                                       int N, int frame, int window_size, long long* n_tiles,
                                       size_t* smem) {
  NoiseBwdParams p;
  p.grad = grad; p.noise = noise; p.dmags = dmags;
  p.seed = seed; p.offset = offset;
  p.B = B; p.F = F; p.nb = nb; p.N = N; p.frame = frame;
  p.g = make_ir_geom(nb, window_size);
  p.S = p.g.S;
  p.start = (p.S - 1) / 2 - 1;
  p.ylen = frame + p.S - 1;
  p.nh = p.g.S0 / 2 + 1;
  p.xS = (((frame + 15) & ~15) + 1) | 1;
  p.gS = (((frame + 15) & ~15) + p.S + 17) | 1;
  p.hS = (p.S + p.nh) | 1;
  p.tiles_per_item = (F + 31) / 32;
  *n_tiles = (long long)B * p.tiles_per_item;
  p.n_tiles = (int)std::min<long long>(*n_tiles, INT32_MAX);
  p.eo_tab = (nb == 65 && p.g.S0 == 128 && p.nh == 65) ? 1 : 0;
  *smem = sizeof(float) * (noise_bwd_eo_offset(p) +
                           (p.eo_tab ? (size_t)p.nh * kEoStride : 0));
  return p;
}

// Launches noise_backward_kernel on checked parameters.
static int noise_bwd_launch(const NoiseBwdParams& p, size_t smem, cudaStream_t st,
                            const char* name) {
  int rc = set_smem(noise_backward_kernel, smem, name);
  if (rc) return rc;
  const int per_sm = smem <= 100 * 1024 ? 2 : 1;
  const int grid = (int)std::min<long long>(p.n_tiles, (long long)num_sms() * per_sm);
  noise_backward_kernel<<<grid, kNbThreads, smem, st>>>(p);
  DDSP_CHECK_LAUNCH(name);
  return 0;
}

int ddsp_b200_filtered_noise_backward(const float* grad_audio, const float* noise,
                                      uint64_t seed, uint64_t offset, float* dmags,
                                      int B, int F, int nb, int N, int window_size,
                                      void* stream) {
  DDSP_REQUIRE(grad_audio && dmags, DDSP_B200_E_INVALID,
               "filtered_noise_backward: null pointer");
  DDSP_REQUIRE(B >= 0 && F >= 1 && N >= 1 && nb >= 2, DDSP_B200_E_INVALID,
               "filtered_noise_backward: bad shape B=%d F=%d nb=%d N=%d", B, F, nb, N);
  const int frame = ir_frame(N, F);
  if (!frame) return DDSP_B200_E_INVALID;
  if (B == 0) return 0;
  long long n_tiles;
  size_t smem;
  NoiseBwdParams p = noise_bwd_params(grad_audio, noise, seed, offset, dmags, B, F, nb, N,
                                      frame, window_size, &n_tiles, &smem);
  DDSP_REQUIRE(p.start >= 0, DDSP_B200_E_UNSUPPORTED,
               "filtered_noise_backward: impulse response too short");
  DDSP_REQUIRE(n_tiles < (1ll << 31), DDSP_B200_E_INVALID,
               "filtered_noise_backward: too many tiles");
  DDSP_REQUIRE(smem <= kMaxDynSmem, DDSP_B200_E_UNSUPPORTED,
               "filtered_noise_backward: shape needs %zu B of shared memory", smem);
  return noise_bwd_launch(p, smem, (cudaStream_t)stream, "filtered_noise_backward");
}

// ---- backward of the time-varying FIR and of the impulse-response synthesis ----
// The shared memory of ir_backward_kernel: the cosine table, padded to a float4, and
// kIrFrames rows of nb folded taps.
static size_t ir_backward_smem(const IrGeom& g) {
  return sizeof(float) * ((((size_t)g.S0 + 3) & ~(size_t)3) + (size_t)kIrFrames * g.nb);
}

// FirDirParams of a shape (frame from ir_frame); out is set by the caller.
static FirDirParams fir_dir_params(const float* x, const float* grad, int B, int N, int F,
                                   int S, int frame, int start, int out_len) {
  FirDirParams p;
  p.x = x; p.g = grad; p.out = nullptr;
  p.N = N; p.S = S; p.F = F; p.frame = frame; p.start = start; p.out_len = out_len;
  fir_dir_segments(frame, &p.n_chunk, &p.seg);
  p.segp = (p.seg + 15) & ~15;
  p.xS = p.segp + 1;
  p.gS = p.segp + kDirTaps + 1;
  p.n_rows = (long long)B * F * p.n_chunk;
  return p;
}

// Bytes of partial d IR sums a shape needs: none when every frame is one segment and
// every item has its own impulse response.
static size_t fir_dir_part_bytes(int B, int N, int F, int S, int ir_batch, int frame) {
  int n_chunk, seg;
  fir_dir_segments(frame, &n_chunk, &seg);
  (void)N;
  if (n_chunk == 1 && !(ir_batch == 1 && B > 1)) return 0;
  return sizeof(float) * (size_t)B * F * n_chunk * S;
}

// The checks of the FIR backward shared by both entry points, after the null-pointer
// and shape checks; sets *frame, *start and *out_len.  The caller returns 0 for B == 0.
static int fir_bwd_check(const char* name, int B, int N, int F, int S, int ir_batch,
                         int padding, int delay_compensation, int* frame, int* start,
                         int* out_len) {
  // core.py:1441-1443
  DDSP_REQUIRE(ir_batch == B || ir_batch == 1, DDSP_B200_E_INVALID,
               "Batch size of audio (%d) and impulse response (%d) must be the "
               "same.", B, ir_batch);
  DDSP_REQUIRE(padding == DDSP_B200_PAD_SAME || padding == DDSP_B200_PAD_VALID,
               DDSP_B200_E_INVALID,
               "Padding must be 'valid' or 'same' (got code %d)", padding);
  *frame = ir_frame(N, F);
  if (!*frame) return DDSP_B200_E_INVALID;
  if (B == 0) return 0;
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID, "%s: B=%d exceeds the 65535 grid limit",
               name, B);
  *out_len = (padding == DDSP_B200_PAD_VALID) ? (N + S - 1) : N;
  *start = delay_compensation < 0 ? ((S - 1) / 2 - 1) : delay_compensation;
  DDSP_REQUIRE(*start >= 0, DDSP_B200_E_UNSUPPORTED,
               "%s: impulse response of %d taps gives a negative automatic delay", name,
               S);
  DDSP_REQUIRE(sizeof(float) * ((size_t)kFadjThreads + S - 1) <= kMaxDynSmem,
               DDSP_B200_E_UNSUPPORTED,
               "%s: impulse response of %d taps is beyond the shared-memory FIR", name, S);
  int n_chunk, seg;
  fir_dir_segments(*frame, &n_chunk, &seg);
  DDSP_REQUIRE((long long)B * F * n_chunk / kDirRows < (1ll << 31) &&
                   (long long)ir_batch * F / kIrFrames < (1ll << 31),
               DDSP_B200_E_INVALID, "%s: too many frames", name);
  return 0;
}

// Launches d audio (when d_audio is set) and d IR (when d_ir is set) of a checked shape.
// `part` holds fir_dir_part_bytes of partial sums when that is not 0.
static int fir_bwd_launch(const float* audio, const float* ir, const float* grad,
                          float* d_audio, float* d_ir, int B, int N, int F, int S,
                          int ir_batch, int frame, int start, int out_len, float* part,
                          cudaStream_t st, const char* name) {
  if (d_audio) {
    const size_t smem = sizeof(float) * ((size_t)kFadjThreads + S - 1);
    int rc = set_smem(fir_adjoint_kernel, smem, name);
    if (rc) return rc;
    dim3 grid((N + kFadjThreads - 1) / kFadjThreads, B);
    fir_adjoint_kernel<<<grid, kFadjThreads, smem, st>>>(
        grad, ir, d_audio, N, S, frame, ir_batch == 1 ? 0 : F * S, start, out_len);
    DDSP_CHECK_LAUNCH(name);
  }
  if (d_ir) {
    FirDirParams p = fir_dir_params(audio, grad, B, N, F, S, frame, start, out_len);
    p.out = part ? part : d_ir;
    const size_t smem = fir_dir_smem(p);
    int rc = set_smem(fir_dir_kernel, smem, name);
    if (rc) return rc;
    dim3 grid((unsigned)((p.n_rows + kDirRows - 1) / kDirRows),
              (unsigned)((S + kDirTaps - 1) / kDirTaps));
    fir_dir_kernel<<<grid, kDirThreads, smem, st>>>(p);
    DDSP_CHECK_LAUNCH(name);
    if (part) {
      const long long n_out = (long long)ir_batch * F * S;
      fir_dir_reduce<<<grid_for(n_out, 256), 256, 0, st>>>(
          part, d_ir, B, F, S, p.n_chunk, ir_batch == 1 && B > 1, n_out);
      DDSP_CHECK_LAUNCH(name);
    }
  }
  return 0;
}

// The route of frequency_filter's d magnitudes: the fused noise_backward_kernel reads
// the audio as its noise when the padding is 'same', every item has its own magnitudes
// and the shape fits its shared memory; otherwise d IR (fir_dir_kernel) and the IR
// adjoint (ir_backward_kernel) through the workspace.
static bool freq_filter_fused(int B, int F, int nb, int N, int frame, int mags_batch,
                              int window_size, int padding) {
  if (padding != DDSP_B200_PAD_SAME || mags_batch != B) return false;
  long long n_tiles;
  size_t smem;
  noise_bwd_params(nullptr, nullptr, 0, 0, nullptr, B, F, nb, N, frame, window_size,
                   &n_tiles, &smem);
  return n_tiles < (1ll << 31) && smem <= kMaxDynSmem;
}

size_t ddsp_b200_fir_time_varying_backward_workspace(int B, int N, int F, int S,
                                                     int ir_batch) {
  if (B <= 0 || N <= 0 || F <= 0 || S <= 0 || (ir_batch != 1 && ir_batch != B)) return 0;
  const int frame = (N + F - 1) / F;
  if ((N + frame - 1) / frame != F) return 0;
  const size_t part = fir_dir_part_bytes(B, N, F, S, ir_batch, frame);
  return part ? part + 256 : 0;
}

int ddsp_b200_fir_time_varying_backward(const float* audio, const float* ir,
                                        const float* grad, float* d_audio, float* d_ir,
                                        int B, int N, int F, int S, int ir_batch,
                                        int padding, int delay_compensation,
                                        void* workspace, size_t workspace_bytes,
                                        void* stream) {
  const char* name = "fir_time_varying_backward";
  DDSP_REQUIRE(audio && ir && grad, DDSP_B200_E_INVALID, "%s: null pointer", name);
  DDSP_REQUIRE(B >= 0 && N >= 1 && F >= 1 && S >= 1, DDSP_B200_E_INVALID,
               "%s: bad shape B=%d N=%d F=%d S=%d", name, B, N, F, S);
  int frame = 0, start = 0, out_len = 0;
  int rc = fir_bwd_check(name, B, N, F, S, ir_batch, padding, delay_compensation, &frame,
                         &start, &out_len);
  if (rc || B == 0) return rc;
  const size_t need =
      d_ir ? ddsp_b200_fir_time_varying_backward_workspace(B, N, F, S, ir_batch) : 0;
  DDSP_REQUIRE(need == 0 || (workspace != nullptr && workspace_bytes >= need),
               DDSP_B200_E_WORKSPACE, "%s: workspace of %zu B needed, %zu given", name,
               need, workspace_bytes);
  return fir_bwd_launch(audio, ir, grad, d_audio, d_ir, B, N, F, S, ir_batch, frame, start,
                        out_len, need ? align256<float>(workspace) : nullptr,
                        (cudaStream_t)stream, name);
}

int ddsp_b200_frequency_impulse_response_backward(const float* d_ir, float* d_mags,
                                                  int64_t BF, int nb, int window_size,
                                                  void* stream) {
  DDSP_REQUIRE(d_ir && d_mags, DDSP_B200_E_INVALID,
               "frequency_impulse_response_backward: null pointer");
  DDSP_REQUIRE(nb >= 2 && BF >= 0, DDSP_B200_E_INVALID,
               "frequency_impulse_response_backward: need n_frequencies >= 2 (got %d)", nb);
  if (BF == 0) return 0;
  const IrGeom g = make_ir_geom(nb, window_size);
  const size_t smem = ir_backward_smem(g);
  DDSP_REQUIRE(smem <= kMaxDynSmem, DDSP_B200_E_UNSUPPORTED,
               "frequency_impulse_response_backward: n_frequencies=%d too large", nb);
  const int64_t blocks = (BF + kIrFrames - 1) / kIrFrames;
  DDSP_REQUIRE(blocks < (1ll << 31), DDSP_B200_E_INVALID,
               "frequency_impulse_response_backward: too many frames");
  int rc = set_smem(ir_backward_kernel, smem, "frequency_impulse_response_backward");
  if (rc) return rc;
  ir_backward_kernel<<<(int)blocks, kIrThreads, smem, (cudaStream_t)stream>>>(d_ir, d_mags,
                                                                              BF, g);
  DDSP_CHECK_LAUNCH("frequency_impulse_response_backward");
  return 0;
}

size_t ddsp_b200_frequency_filter_backward_workspace(int B, int F, int nb, int N,
                                                     int mags_batch, int window_size,
                                                     int padding) {
  if (B <= 0 || F <= 0 || N <= 0 || nb < 2 || (mags_batch != 1 && mags_batch != B))
    return 0;
  const int frame = (N + F - 1) / F;
  if ((N + frame - 1) / frame != F) return 0;
  if (freq_filter_fused(B, F, nb, N, frame, mags_batch, window_size, padding)) return 0;
  const int S = make_ir_geom(nb, window_size).S;
  // d IR [mags_batch, F, S], then the partial sums of fir_dir_kernel
  const size_t d_ir = (sizeof(float) * (size_t)mags_batch * F * S + 255) & ~(size_t)255;
  return 256 + d_ir + fir_dir_part_bytes(B, N, F, S, mags_batch, frame);
}

int ddsp_b200_frequency_filter_backward(const float* audio, const float* ir,
                                        const float* grad, float* d_audio, float* d_mags,
                                        int B, int F, int nb, int N, int mags_batch,
                                        int window_size, int padding, void* workspace,
                                        size_t workspace_bytes, void* stream) {
  const char* name = "frequency_filter_backward";
  DDSP_REQUIRE(audio && ir && grad, DDSP_B200_E_INVALID, "%s: null pointer", name);
  DDSP_REQUIRE(B >= 0 && F >= 1 && N >= 1 && nb >= 2, DDSP_B200_E_INVALID,
               "%s: bad shape B=%d F=%d nb=%d N=%d", name, B, F, nb, N);
  const IrGeom g = make_ir_geom(nb, window_size);
  const int S = g.S;
  int frame = 0, start = 0, out_len = 0;
  int rc = fir_bwd_check(name, B, N, F, S, mags_batch, padding, -1, &frame, &start,
                         &out_len);
  if (rc || B == 0) return rc;
  const bool fused =
      freq_filter_fused(B, F, nb, N, frame, mags_batch, window_size, padding);
  DDSP_REQUIRE(!d_mags || fused || ir_backward_smem(g) <= kMaxDynSmem,
               DDSP_B200_E_UNSUPPORTED, "%s: n_frequencies=%d too large", name, nb);
  const size_t need =
      d_mags ? ddsp_b200_frequency_filter_backward_workspace(B, F, nb, N, mags_batch,
                                                             window_size, padding)
             : 0;
  DDSP_REQUIRE(need == 0 || (workspace != nullptr && workspace_bytes >= need),
               DDSP_B200_E_WORKSPACE, "%s: workspace of %zu B needed, %zu given", name,
               need, workspace_bytes);
  cudaStream_t st = (cudaStream_t)stream;
  if (d_audio) {
    rc = fir_bwd_launch(audio, ir, grad, d_audio, nullptr, B, N, F, S, mags_batch, frame,
                        start, out_len, nullptr, st, name);
    if (rc) return rc;
  }
  if (!d_mags) return 0;
  if (fused) {
    long long n_tiles;
    size_t smem;
    NoiseBwdParams p = noise_bwd_params(grad, audio, 0, 0, d_mags, B, F, nb, N, frame,
                                        window_size, &n_tiles, &smem);
    return noise_bwd_launch(p, smem, st, name);
  }
  float* d_ir = align256<float>(workspace);
  float* part = d_ir + (((size_t)mags_batch * F * S + 63) & ~(size_t)63);
  rc = fir_bwd_launch(audio, ir, grad, nullptr, d_ir, B, N, F, S, mags_batch, frame, start,
                      out_len,
                      fir_dir_part_bytes(B, N, F, S, mags_batch, frame) ? part : nullptr, st,
                      name);
  if (rc) return rc;
  return ddsp_b200_frequency_impulse_response_backward(d_ir, d_mags, (int64_t)mags_batch * F,
                                                       nb, window_size, stream);
}

// ---- windowed-sinc filters (csrc/sinc.cuh) --------------------------------------------
int ddsp_b200_sinc_impulse_response(const float* cutoff, float* ir, int64_t BF, int S,
                                    float scale, int high_pass, void* stream) {
  const char* name = "sinc_impulse_response";
  DDSP_REQUIRE(cutoff && ir, DDSP_B200_E_INVALID, "%s: null pointer", name);
  DDSP_REQUIRE(BF >= 0 && S >= 1 && (S & 1), DDSP_B200_E_INVALID,
               "%s: bad shape BF=%lld S=%d (S must be odd)", name, (long long)BF, S);
  DDSP_REQUIRE(BF < (1ll << 31), DDSP_B200_E_INVALID, "%s: too many frames", name);
  if (BF == 0) return 0;
  sinc_ir_kernel<<<(unsigned)BF, kSincThreads, 0, (cudaStream_t)stream>>>(cutoff, ir, S, scale,
                                                                          high_pass);
  DDSP_CHECK_LAUNCH(name);
  return 0;
}

int ddsp_b200_sinc_impulse_response_backward(const float* cutoff, const float* d_ir,
                                             float* d_cutoff, int64_t BF, int S, float scale,
                                             int high_pass, void* stream) {
  const char* name = "sinc_impulse_response_backward";
  DDSP_REQUIRE(cutoff && d_ir && d_cutoff, DDSP_B200_E_INVALID, "%s: null pointer", name);
  DDSP_REQUIRE(BF >= 0 && S >= 1 && (S & 1), DDSP_B200_E_INVALID,
               "%s: bad shape BF=%lld S=%d (S must be odd)", name, (long long)BF, S);
  DDSP_REQUIRE(BF < (1ll << 31), DDSP_B200_E_INVALID, "%s: too many frames", name);
  if (BF == 0) return 0;
  sinc_ir_backward_kernel<<<(unsigned)BF, kSincThreads, 0, (cudaStream_t)stream>>>(
      cutoff, d_ir, d_cutoff, S, scale, high_pass);
  DDSP_CHECK_LAUNCH(name);
  return 0;
}

// The checks both sinc_filter entry points make after the null-pointer check; sets
// *frame, *start and *out_len.  The caller returns 0 for B == 0.
static int sinc_filter_check(const char* name, int B, int N, int F, int S, int cutoff_batch,
                             int padding, int* frame, int* start, int* out_len) {
  DDSP_REQUIRE(B >= 0 && N >= 1 && F >= 1 && S >= 1 && (S & 1), DDSP_B200_E_INVALID,
               "%s: bad shape B=%d N=%d F=%d S=%d (S must be odd)", name, B, N, F, S);
  // core.py:1441-1443
  DDSP_REQUIRE(cutoff_batch == B || cutoff_batch == 1, DDSP_B200_E_INVALID,
               "Batch size of audio (%d) and impulse response (%d) must be the "
               "same.", B, cutoff_batch);
  DDSP_REQUIRE(padding == DDSP_B200_PAD_SAME || padding == DDSP_B200_PAD_VALID,
               DDSP_B200_E_INVALID,
               "Padding must be 'valid' or 'same' (got code %d)", padding);
  *frame = ir_frame(N, F);
  if (!*frame) return DDSP_B200_E_INVALID;
  if (B == 0) return 0;
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID, "%s: B=%d exceeds the 65535 grid limit",
               name, B);
  DDSP_REQUIRE(S >= 3, DDSP_B200_E_UNSUPPORTED,
               "%s: %d tap gives a negative automatic delay (the reference's crop is "
               "empty); compose sinc_impulse_response and fft_convolve", name, S);
  DDSP_REQUIRE(S < 2048, DDSP_B200_E_UNSUPPORTED,
               "%s: %d taps is beyond the fused kernels (2047 at most); compose "
               "sinc_impulse_response and fft_convolve", name, S);
  DDSP_REQUIRE((long long)N + S + 4 * kSincTile < (1ll << 31), DDSP_B200_E_INVALID,
               "%s: N=%d is too long", name, N);
  *out_len = (padding == DDSP_B200_PAD_VALID) ? (N + S - 1) : N;
  *start = (S - 1) / 2 - 1;
  return 0;
}

int ddsp_b200_sinc_filter(const float* audio, const float* cutoff, float* out, int B, int N,
                          int F, int S, int cutoff_batch, float scale, int high_pass,
                          int padding, int accumulate, void* stream) {
  const char* name = "sinc_filter";
  DDSP_REQUIRE(audio && cutoff && out, DDSP_B200_E_INVALID, "%s: null pointer", name);
  int frame = 0, start = 0, out_len = 0;
  int rc = sinc_filter_check(name, B, N, F, S, cutoff_batch, padding, &frame, &start,
                             &out_len);
  if (rc || B == 0) return rc;
  const size_t smem = sinc_filter_smem(S);
  rc = set_smem(sinc_filter_kernel, smem, name);
  if (rc) return rc;
  SincFilterParams p;
  p.x = audio; p.cutoff = cutoff; p.out = out;
  p.N = N; p.F = F; p.frame = frame; p.S = S; p.cutoff_stride = cutoff_batch == 1 ? 0 : F;
  p.scale = scale; p.high_pass = high_pass ? 1 : 0; p.start = start; p.out_len = out_len;
  p.accumulate = accumulate ? 1 : 0;
  dim3 grid((out_len + kSincTile - 1) / kSincTile, B);
  sinc_filter_kernel<<<grid, kSincThreads, smem, (cudaStream_t)stream>>>(p);
  DDSP_CHECK_LAUNCH(name);
  return 0;
}

// Partial d cutoff sums the backward needs: none when every frame is one tile and every
// item has its own cutoff.
static size_t sinc_bwd_part_bytes(int B, int N, int F, int cutoff_batch, int frame) {
  int fpt, n_seg, seg, tiles;
  sinc_bwd_tiles(N, F, frame, &fpt, &n_seg, &seg, &tiles);
  if (n_seg == 1 && !(cutoff_batch == 1 && B > 1)) return 0;
  return sizeof(float) * (size_t)B * F * n_seg;
}

size_t ddsp_b200_sinc_filter_backward_workspace(int B, int N, int F, int S, int cutoff_batch) {
  if (B <= 0 || N <= 0 || F <= 0 || S <= 0 || (cutoff_batch != 1 && cutoff_batch != B))
    return 0;
  const int frame = (N + F - 1) / F;
  if ((N + frame - 1) / frame != F) return 0;
  const size_t part = sinc_bwd_part_bytes(B, N, F, cutoff_batch, frame);
  return part ? part + 256 : 0;
}

int ddsp_b200_sinc_filter_backward(const float* audio, const float* cutoff, const float* grad,
                                   float* d_audio, float* d_cutoff, int B, int N, int F,
                                   int S, int cutoff_batch, float scale, int high_pass,
                                   int padding, void* workspace, size_t workspace_bytes,
                                   void* stream) {
  const char* name = "sinc_filter_backward";
  DDSP_REQUIRE(audio && cutoff && grad, DDSP_B200_E_INVALID, "%s: null pointer", name);
  int frame = 0, start = 0, out_len = 0;
  int rc = sinc_filter_check(name, B, N, F, S, cutoff_batch, padding, &frame, &start,
                             &out_len);
  if (rc || B == 0) return rc;
  const size_t need =
      d_cutoff ? ddsp_b200_sinc_filter_backward_workspace(B, N, F, S, cutoff_batch) : 0;
  DDSP_REQUIRE(need == 0 || (workspace != nullptr && workspace_bytes >= need),
               DDSP_B200_E_WORKSPACE, "%s: workspace of %zu B needed, %zu given", name,
               need, workspace_bytes);
  if (!d_audio && !d_cutoff) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  SincBwdParams p;
  p.x = audio; p.cutoff = cutoff; p.g = grad; p.dx = d_audio;
  float* part = need ? align256<float>(workspace) : nullptr;
  p.dc = part ? part : d_cutoff;
  p.N = N; p.F = F; p.frame = frame; p.S = S; p.cutoff_stride = cutoff_batch == 1 ? 0 : F;
  p.scale = scale; p.high_pass = high_pass ? 1 : 0; p.start = start; p.out_len = out_len;
  sinc_bwd_tiles(N, F, frame, &p.fpt, &p.n_seg, &p.seg, &p.tiles);
  const size_t smem = sinc_bwd_smem(S);
  dim3 grid((unsigned)p.tiles, B);
  if (d_cutoff) {
    rc = set_smem(sinc_filter_backward_kernel<true>, smem, name);
    if (rc) return rc;
    sinc_filter_backward_kernel<true><<<grid, kSincThreads, smem, st>>>(p);
  } else {
    rc = set_smem(sinc_filter_backward_kernel<false>, smem, name);
    if (rc) return rc;
    sinc_filter_backward_kernel<false><<<grid, kSincThreads, smem, st>>>(p);
  }
  DDSP_CHECK_LAUNCH(name);
  if (part) {
    const long long n_out = (long long)cutoff_batch * F;
    sinc_dc_reduce<<<grid_for(n_out, 256), 256, 0, st>>>(part, d_cutoff, B, F, p.n_seg,
                                                         cutoff_batch == 1 && B > 1, n_out);
    DDSP_CHECK_LAUNCH(name);
  }
  return 0;
}

size_t ddsp_b200_oscillator_bank_workspace(int B, int N, int K) {
  if (B <= 0 || N <= 0 || K <= 0) return 0;
  const size_t n_chunks = ((size_t)N + kObChunk - 1) / kObChunk;
  return sizeof(unsigned long long) * (size_t)B * n_chunks * K + 256;
}

int ddsp_b200_oscillator_bank(const float* frequency_envelopes,
                              const float* amplitude_envelopes, float* out, int B,
                              int N, int K, float sample_rate, int sum_sinusoids,
                              void* workspace, size_t workspace_bytes,
                              void* stream) {
  DDSP_REQUIRE(frequency_envelopes && amplitude_envelopes && out,
               DDSP_B200_E_INVALID, "oscillator_bank: null pointer");
  DDSP_REQUIRE(B >= 0 && N >= 1 && K >= 1, DDSP_B200_E_INVALID,
               "oscillator_bank: bad shape B=%d N=%d K=%d", B, N, K);
  DDSP_REQUIRE(sample_rate > 0.f, DDSP_B200_E_INVALID,
               "oscillator_bank: sample_rate must be positive");
  if (B == 0) return 0;
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID,
               "oscillator_bank: B=%d exceeds the 65535 grid limit", B);
  const size_t need = ddsp_b200_oscillator_bank_workspace(B, N, K);
  DDSP_REQUIRE(workspace != nullptr && workspace_bytes >= need, DDSP_B200_E_WORKSPACE,
               "oscillator_bank: workspace of %zu B needed, %zu given", need,
               workspace_bytes);
  unsigned long long* sums = align256<unsigned long long>(workspace);
  const int n_chunks = (N + kObChunk - 1) / kObChunk;
  const double inv_sr = 1.0 / (double)sample_rate;
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(n_chunks, B);
  oscbank_chunk_sums<<<grid, kObThreads, 0, st>>>(frequency_envelopes, sums, N, K,
                                                 n_chunks, inv_sr);
  DDSP_CHECK_LAUNCH("oscillator_bank(chunk sums)");
  const int64_t BK = (int64_t)B * K;
  oscbank_scan_chunks<<<(int)((BK + kObThreads - 1) / kObThreads), kObThreads, 0, st>>>(
      sums, K, n_chunks, BK);
  DDSP_CHECK_LAUNCH("oscillator_bank(scan)");
  auto apply = sum_sinusoids ? oscbank_apply<true> : oscbank_apply<false>;
  apply<<<grid, kObThreads, 0, st>>>(frequency_envelopes, amplitude_envelopes, sums, out,
                                     N, K, n_chunks, inv_sr, sample_rate * 0.5f);
  DDSP_CHECK_LAUNCH("oscillator_bank(apply)");
  return 0;
}

// One cluster per (b, tile of kObbLanes oscillators) along x, batch along y.
static dim3 oscbank_backward_grid(int B, int K) {
  return dim3((unsigned)(kObbCluster * ((K + kObbLanes - 1) / kObbLanes)), (unsigned)B);
}

int ddsp_b200_oscillator_bank_backward(const float* frequency_envelopes,
                                       const float* amplitude_envelopes, const float* grad,
                                       float* d_frequency_envelopes,
                                       float* d_amplitude_envelopes, int B, int N, int K,
                                       float sample_rate, int sum_sinusoids, void* stream) {
  const bool empty = B == 0 || N == 0 || K == 0;
  DDSP_REQUIRE(empty || (frequency_envelopes && amplitude_envelopes && grad),
               DDSP_B200_E_INVALID, "oscillator_bank_backward: null pointer");
  DDSP_REQUIRE(B >= 0 && N >= 0 && K >= 0, DDSP_B200_E_INVALID,
               "oscillator_bank_backward: bad shape B=%d N=%d K=%d", B, N, K);
  DDSP_REQUIRE(sample_rate > 0.f, DDSP_B200_E_INVALID,
               "oscillator_bank_backward: sample_rate must be positive");
  DDSP_REQUIRE(sum_sinusoids == 0 || sum_sinusoids == 1, DDSP_B200_E_INVALID,
               "oscillator_bank_backward: sum_sinusoids must be 0 or 1, got %d",
               sum_sinusoids);
  if (empty || (!d_frequency_envelopes && !d_amplitude_envelopes)) return 0;
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID,
               "oscillator_bank_backward: B=%d exceeds the 65535 grid limit", B);
  auto kernel = sum_sinusoids ? oscbank_backward<kObbSum> : oscbank_backward<kObbFull>;
  kernel<<<oscbank_backward_grid(B, K), kObbLanes * kObbWarps, 0, (cudaStream_t)stream>>>(
      frequency_envelopes, amplitude_envelopes, grad, d_frequency_envelopes,
      d_amplitude_envelopes, N, K, 1.0 / (double)sample_rate, sample_rate * 0.5f,
      6.283185307179586 / (double)sample_rate);
  DDSP_CHECK_LAUNCH("oscillator_bank_backward");
  return 0;
}

size_t ddsp_b200_fft_convolve_lti_workspace(int B, int N, int S, int ir_batch) {
  if (B <= 0 || N <= 0 || S <= 0 || (ir_batch != 1 && ir_batch != B)) return 0;
  const lc::Geom g = lc::geom(N, S);
  const size_t z = (size_t)B * g.n_in * lc::M, h = (size_t)ir_batch * g.P * lc::M,
               w = (size_t)B * g.w_len;
  return sizeof(float2) * (z + h + w) + 256;
}

int ddsp_b200_fft_convolve_lti(const float* audio, const float* impulse_response,
                               float* out, int B, int N, int S, int ir_batch,
                               int start, int out_len, int accumulate, int flags,
                               void* workspace, size_t workspace_bytes, void* stream) {
  DDSP_REQUIRE(audio && impulse_response && out, DDSP_B200_E_INVALID,
               "fft_convolve_lti: null pointer");
  DDSP_REQUIRE(B >= 0 && N >= 1 && S >= 1, DDSP_B200_E_INVALID,
               "fft_convolve_lti: bad shape B=%d N=%d S=%d", B, N, S);
  // core.py:1441-1443
  DDSP_REQUIRE(ir_batch == B || ir_batch == 1, DDSP_B200_E_INVALID,
               "Batch size of audio (%d) and impulse response (%d) must be the same.",
               B, ir_batch);
  DDSP_REQUIRE(start >= 0 && out_len >= 0 &&
                   (long long)start + out_len <= (long long)N + S - 1,
               DDSP_B200_E_INVALID,
               "fft_convolve_lti: crop [%d, %d) leaves the convolution of length %lld",
               start, start + out_len, (long long)N + S - 1);
  if (B == 0 || out_len == 0) return 0;
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID,
               "fft_convolve_lti: B=%d exceeds the 65535 grid limit", B);
  const size_t need = ddsp_b200_fft_convolve_lti_workspace(B, N, S, ir_batch);
  DDSP_REQUIRE(workspace != nullptr && workspace_bytes >= need, DDSP_B200_E_WORKSPACE,
               "fft_convolve_lti: workspace of %zu B needed, %zu given", need,
               workspace_bytes);
  const lc::Geom g = lc::geom(N, S);
  float2* Z = align256<float2>(workspace);
  float2* H = Z + (size_t)B * g.n_in * lc::M;
  float2* W = H + (size_t)ir_batch * g.P * lc::M;
  cudaStream_t st = (cudaStream_t)stream;
  DDSP_REQUIRE((flags & ~3) == 0, DDSP_B200_E_INVALID,
               "fft_convolve_lti: bad flags %d", flags);
  lc::lc_fft_blocks<<<dim3(g.P, ir_batch), lc::THREADS, 0, st>>>(
      impulse_response, H, S, 0, g.P, 1, (flags & DDSP_B200_LTI_REVERSE_IR) ? 1 : 0);
  DDSP_CHECK_LAUNCH("fft_convolve_lti(ir spectra)");
  lc::lc_fft_blocks<<<dim3(g.n_in, B), lc::THREADS, 0, st>>>(
      audio, Z, N, g.n2, g.n_in, 0, (flags & DDSP_B200_LTI_REVERSE_AUDIO) ? 1 : 0);
  DDSP_CHECK_LAUNCH("fft_convolve_lti(audio spectra)");
  // w blocks the crop reads: positions [start, start + out_len) through the real
  // half and [start - n2, start + out_len - n2) through the imaginary half
  const int lo_pos = std::max(0, start - g.n2);
  const int hi_pos = std::min(g.w_len, start + out_len);      // exclusive
  const int j_first = lo_pos / lc::L;
  const int j_last = std::min(g.n_out - 1, (hi_pos - 1) / lc::L);
  const int n_blocks = j_last - j_first + 1;
  {
    int rc = set_smem(lc::lc_mac_ifft, lc::kMacSmem, "fft_convolve_lti");
    if (rc) return rc;
  }
  lc::lc_mac_ifft<<<dim3((n_blocks + lc::JT - 1) / lc::JT, B), lc::THREADS, lc::kMacSmem,
                    st>>>(
      Z, H, W, g.n_in, g.P, g.n_out, ir_batch == 1 ? 0 : g.P * lc::M, j_first, n_blocks);
  DDSP_CHECK_LAUNCH("fft_convolve_lti(multiply-accumulate + inverse)");
  const int cgrid = std::min((out_len + 255) / 256, 8 * num_sms());
  lc::lc_combine<<<dim3(cgrid, B), 256, 0, st>>>(W, out, g.n2, g.w_len, start, out_len,
                                               N + S - 1, accumulate, j_first * lc::L,
                                               (j_last + 1) * lc::L);
  DDSP_CHECK_LAUNCH("fft_convolve_lti(combine)");
  return 0;
}

int ddsp_b200_angular_cumsum(const float* angular_frequency, float* phase, int B,
                             int N, int C, int chunk_size, int mode,
                             void* workspace, size_t workspace_bytes, void* stream) {
  DDSP_REQUIRE(angular_frequency && phase, DDSP_B200_E_INVALID,
               "angular_cumsum: null pointer");
  DDSP_REQUIRE(B >= 0 && N >= 1 && C >= 1, DDSP_B200_E_INVALID,
               "angular_cumsum: bad shape B=%d N=%d C=%d", B, N, C);
  DDSP_REQUIRE(mode >= 0 && mode <= 2, DDSP_B200_E_INVALID,
               "angular_cumsum: bad mode %d", mode);
  DDSP_REQUIRE(mode != 2 || chunk_size >= 1, DDSP_B200_E_INVALID,
               "angular_cumsum: chunk_size must be positive");
  if (B == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (mode != 0) {
    const int64_t BC = (int64_t)B * C;
    tf_sequential_cumsum<<<(int)((BC + 127) / 128), 128, 0, st>>>(
        angular_frequency, nullptr, phase, B, N, C, mode, chunk_size, 0, 1.0f);
    DDSP_CHECK_LAUNCH("angular_cumsum(tf_sequential)");
    return 0;
  }
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID,
               "angular_cumsum: B=%d exceeds the 65535 grid limit", B);
  const size_t need = ddsp_b200_oscillator_bank_workspace(B, N, C);
  DDSP_REQUIRE(workspace != nullptr && workspace_bytes >= need, DDSP_B200_E_WORKSPACE,
               "angular_cumsum: workspace of %zu B needed, %zu given", need,
               workspace_bytes);
  unsigned long long* sums = align256<unsigned long long>(workspace);
  const int n_chunks = (N + kObChunk - 1) / kObChunk;
  const double inv_two_pi = 0.15915494309189535;
  dim3 grid(n_chunks, B);
  oscbank_chunk_sums<<<grid, kObThreads, 0, st>>>(angular_frequency, sums, N, C,
                                                 n_chunks, inv_two_pi);
  DDSP_CHECK_LAUNCH("angular_cumsum(chunk sums)");
  const int64_t BK = (int64_t)B * C;
  oscbank_scan_chunks<<<(int)((BK + kObThreads - 1) / kObThreads), kObThreads, 0, st>>>(
      sums, C, n_chunks, BK);
  DDSP_CHECK_LAUNCH("angular_cumsum(scan)");
  oscbank_phase_out<<<grid, kObThreads, 0, st>>>(angular_frequency, sums, phase, N, C,
                                                n_chunks, inv_two_pi);
  DDSP_CHECK_LAUNCH("angular_cumsum(apply)");
  return 0;
}

int ddsp_b200_angular_cumsum_backward(const float* grad, float* d_angular_frequency, int B,
                                      int N, int C, void* stream) {
  const bool empty = B == 0 || N == 0 || C == 0;
  DDSP_REQUIRE(empty || (grad && d_angular_frequency), DDSP_B200_E_INVALID,
               "angular_cumsum_backward: null pointer");
  DDSP_REQUIRE(B >= 0 && N >= 0 && C >= 0, DDSP_B200_E_INVALID,
               "angular_cumsum_backward: bad shape B=%d N=%d C=%d", B, N, C);
  if (empty) return 0;
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID,
               "angular_cumsum_backward: B=%d exceeds the 65535 grid limit", B);
  oscbank_backward<kObbCumsum>
      <<<oscbank_backward_grid(B, C), kObbLanes * kObbWarps, 0, (cudaStream_t)stream>>>(
          nullptr, nullptr, grad, d_angular_frequency, nullptr, N, C, 0.0, 0.f, 1.0);
  DDSP_CHECK_LAUNCH("angular_cumsum_backward");
  return 0;
}

int ddsp_b200_oscillator_bank_tf_sequential(const float* frequency_envelopes,
                                            const float* amplitude_envelopes,
                                            float* out, int B, int N, int K,
                                            float sample_rate, int use_angular_cumsum,
                                            int chunk_size, void* stream) {
  DDSP_REQUIRE(frequency_envelopes && amplitude_envelopes && out, DDSP_B200_E_INVALID,
               "oscillator_bank_tf_sequential: null pointer");
  DDSP_REQUIRE(B >= 0 && N >= 1 && K >= 1 && chunk_size >= 1 && sample_rate > 0.f,
               DDSP_B200_E_INVALID, "oscillator_bank_tf_sequential: bad arguments");
  if (B == 0) return 0;
  const int64_t BK = (int64_t)B * K;
  tf_sequential_cumsum<<<(int)((BK + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      frequency_envelopes, amplitude_envelopes, out, B, N, K,
      use_angular_cumsum ? 2 : 1, chunk_size, 1, sample_rate);
  DDSP_CHECK_LAUNCH("oscillator_bank_tf_sequential");
  return 0;
}

static int sinus_tile_frames(int F, int K) {
  int FT = std::min(16, F);
  while (FT > 1 && sf_smem(FT, K).total > kMaxDynSmem) FT = (FT + 1) / 2;
  return FT;
}

size_t ddsp_b200_sinusoidal_workspace(int B, int F, int K) {
  if (B <= 0 || F <= 0 || K <= 0) return 0;
  const int FT = sinus_tile_frames(F, K);
  const size_t n_tiles = ((size_t)F + FT - 1) / FT;
  return sizeof(unsigned long long) * (size_t)B * n_tiles * K + 256;
}

// The shape, method and workspace checks shared by the forward and the backward;
// `name` prefixes the messages.  The caller returns 0 for B == 0 afterwards.
static int sinus_check(const char* name, int B, int F, int K, int N, float sample_rate,
                       int amp_method, const void* workspace, size_t workspace_bytes,
                       size_t need) {
  DDSP_REQUIRE(B >= 0 && F >= 1 && K >= 1 && N >= 1, DDSP_B200_E_INVALID,
               "%s: bad shape B=%d F=%d K=%d N=%d", name, B, F, K, N);
  DDSP_REQUIRE(amp_method == DDSP_B200_AMP_WINDOW || amp_method == DDSP_B200_AMP_LINEAR,
               DDSP_B200_E_INVALID, "%s: bad amp_method %d", name, amp_method);
  DDSP_REQUIRE(N % F == 0, DDSP_B200_E_INVALID,
               "%s: n_samples (%d) must be divisible by the number "
               "of frames (%d)", name, N, F);
  DDSP_REQUIRE(amp_method != DDSP_B200_AMP_WINDOW || F < N, DDSP_B200_E_INVALID,
               "%s: window upsampling cannot downsample (frames %d "
               ">= timesteps %d)", name, F, N);
  DDSP_REQUIRE(sample_rate > 0.f, DDSP_B200_E_INVALID,
               "%s: sample_rate must be positive", name);
  if (B == 0) return 0;
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID,
               "%s: B=%d exceeds the 65535 grid limit", name, B);
  DDSP_REQUIRE(sf_smem(sinus_tile_frames(F, K), K).total <= kMaxDynSmem,
               DDSP_B200_E_UNSUPPORTED,
               "%s: K=%d needs more shared memory than one CTA has", name, K);
  DDSP_REQUIRE(workspace != nullptr && workspace_bytes >= need, DDSP_B200_E_WORKSPACE,
               "%s: workspace of %zu B needed, %zu given", name, need, workspace_bytes);
  return 0;
}

// Passes 1-2: the exclusive scan of the tile phase totals, into the workspace.
static int sinus_tile_offsets(const float* frequencies, unsigned long long* sums, int B,
                              int F, int K, int hop, int FT, double inv_sr,
                              cudaStream_t st, const char* name) {
  const int n_tiles = (F + FT - 1) / FT;
  sinus_tile_sums<<<dim3(n_tiles, B), kSfThreads, 0, st>>>(frequencies, sums, F, K, hop,
                                                           FT, n_tiles, inv_sr);
  DDSP_CHECK_LAUNCH(name);
  const int64_t BK = (int64_t)B * K;
  oscbank_scan_chunks<<<(int)((BK + kObThreads - 1) / kObThreads), kObThreads, 0, st>>>(
      sums, K, n_tiles, BK);
  DDSP_CHECK_LAUNCH(name);
  return 0;
}

int ddsp_b200_sinusoidal_forward(const float* frequencies, const float* amplitudes,
                                 float* audio, int B, int F, int K, int N,
                                 float sample_rate, int amp_method, int accumulate,
                                 void* workspace, size_t workspace_bytes,
                                 void* stream) {
  DDSP_REQUIRE(frequencies && amplitudes && audio, DDSP_B200_E_INVALID,
               "sinusoidal_forward: null pointer");
  int rc = sinus_check("sinusoidal_forward", B, F, K, N, sample_rate, amp_method, workspace,
                       workspace_bytes, ddsp_b200_sinusoidal_workspace(B, F, K));
  if (rc || B == 0) return rc;
  const int FT = sinus_tile_frames(F, K);
  const SfSmem L = sf_smem(FT, K);
  unsigned long long* sums = align256<unsigned long long>(workspace);
  const int n_tiles = (F + FT - 1) / FT;
  const int hop = N / F;
  const double inv_sr = 1.0 / (double)sample_rate;
  cudaStream_t st = (cudaStream_t)stream;
  rc = sinus_tile_offsets(frequencies, sums, B, F, K, hop, FT, inv_sr, st,
                          "sinusoidal_forward(tile offsets)");
  if (rc) return rc;
  auto kern = amp_method == DDSP_B200_AMP_WINDOW ? sinus_apply<true> : sinus_apply<false>;
  rc = set_smem(kern, L.total, "sinusoidal_forward");
  if (rc) return rc;
  kern<<<dim3(n_tiles, B), kSfThreads, L.total, st>>>(
      frequencies, amplitudes, sums, audio, F, K, N, hop, FT, n_tiles, inv_sr,
      sample_rate * 0.5f, accumulate);
  DDSP_CHECK_LAUNCH("sinusoidal_forward(apply)");
  return 0;
}

size_t ddsp_b200_sinusoidal_backward_workspace(int B, int F, int K) {
  if (B <= 0 || F <= 0 || K <= 0) return 0;
  return ddsp_b200_sinusoidal_workspace(B, F, K) + sizeof(float) * 5 * (size_t)B * F * K +
         256;
}

int ddsp_b200_sinusoidal_backward(const float* frequencies, const float* amplitudes,
                                  const float* grad_audio, float* d_frequencies,
                                  float* d_amplitudes, int B, int F, int K, int N,
                                  float sample_rate, int amp_method, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  DDSP_REQUIRE(frequencies && amplitudes && grad_audio && d_amplitudes, DDSP_B200_E_INVALID,
               "sinusoidal_backward: null pointer");
  int rc = sinus_check("sinusoidal_backward", B, F, K, N, sample_rate, amp_method,
                       workspace, workspace_bytes,
                       ddsp_b200_sinusoidal_backward_workspace(B, F, K));
  if (rc || B == 0) return rc;
  const int FT = sinus_tile_frames(F, K);
  const int n_tiles = (F + FT - 1) / FT;
  const int hop = N / F;
  const double inv_sr = 1.0 / (double)sample_rate;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* sums = align256<unsigned long long>(workspace);
  float* part = align256<float>(sums + (size_t)B * n_tiles * K);
  rc = sinus_tile_offsets(frequencies, sums, B, F, K, hop, FT, inv_sr, st,
                          "sinusoidal_backward(tile offsets)");
  if (rc) return rc;
  const int64_t BFK = (int64_t)B * F * K;
  const unsigned n_blocks = (unsigned)((BFK + 31) / 32);
  const bool phase = d_frequencies != nullptr;
  auto kern = amp_method == DDSP_B200_AMP_WINDOW
                  ? (phase ? sinus_bwd_frames<true, true> : sinus_bwd_frames<true, false>)
                  : (phase ? sinus_bwd_frames<false, true> : sinus_bwd_frames<false, false>);
  kern<<<n_blocks, kSbThreads, 0, st>>>(frequencies, amplitudes, grad_audio, sums, part, F,
                                        K, N, hop, FT, n_tiles, BFK, inv_sr,
                                        sample_rate * 0.5f);
  DDSP_CHECK_LAUNCH("sinusoidal_backward(frames)");
  sinus_bwd_finalize<<<dim3((K + 31) / 32, B), 32 * kSfinWarps, 0, st>>>(
      part, d_amplitudes, d_frequencies, F, K, hop, BFK, inv_sr);
  DDSP_CHECK_LAUNCH("sinusoidal_backward(finalize)");
  return 0;
}

int ddsp_b200_resample(const float* in, float* out, int B, int F, int C, int N,
                       int method, int add_endpoint, void* stream) {
  DDSP_REQUIRE(in && out, DDSP_B200_E_INVALID, "resample: null pointer");
  DDSP_REQUIRE(B >= 0 && F >= 1 && C >= 1 && N >= 1, DDSP_B200_E_INVALID,
               "resample: bad shape B=%d F=%d C=%d N=%d", B, F, C, N);
  DDSP_REQUIRE(method >= 0 && method <= 3, DDSP_B200_E_INVALID,
               "resample: bad method %d", method);
  if (method == 0) {
    // upsample_with_windows (core.py:676-693)
    const int n_frames = add_endpoint ? F + 1 : F;
    const int n_intervals = n_frames - 1;
    DDSP_REQUIRE(n_frames < N, DDSP_B200_E_INVALID,
                 "Upsample with windows cannot be used for downsampling"
                 "More input frames (%d) than output timesteps (%d)", n_frames, N);
    DDSP_REQUIRE(n_intervals > 0 && N % n_intervals == 0, DDSP_B200_E_INVALID,
                 "For upsampling, the target the number of timesteps must be "
                 "divisible by the number of input frames%s. (timesteps:%d, "
                 "frames:%d, add_endpoint=%s).", add_endpoint ? "" : " - 1", N,
                 n_frames, add_endpoint ? "True" : "False");
  }
  if (B == 0) return 0;
  const int64_t total = (int64_t)B * N * C;
  resample_kernel<<<grid_for(total, 256, 16), 256, 0, (cudaStream_t)stream>>>(
      in, out, B, F, C, N, method, add_endpoint);
  DDSP_CHECK_LAUNCH("resample");
  return 0;
}

int ddsp_b200_add(const float* a, const float* b, float* out, int64_t n,
                  void* stream) {
  DDSP_REQUIRE(a && b && out, DDSP_B200_E_INVALID, "add: null pointer");
  DDSP_REQUIRE(n >= 0, DDSP_B200_E_INVALID, "add: n < 0");
  if (n == 0) return 0;
  add_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(a, b, out, n);
  DDSP_CHECK_LAUNCH("add");
  return 0;
}

// ---- routing: resample backward, Mix, ExpDecayReverb impulse response -----------
int ddsp_b200_resample_backward(const float* grad_out, float* grad_in, int B, int F, int C,
                                int N, int method, int add_endpoint, void* stream) {
  DDSP_REQUIRE(grad_out && grad_in, DDSP_B200_E_INVALID, "resample_backward: null pointer");
  DDSP_REQUIRE(B >= 0 && F >= 1 && C >= 1 && N >= 1, DDSP_B200_E_INVALID,
               "resample_backward: bad shape B=%d F=%d C=%d N=%d", B, F, C, N);
  DDSP_REQUIRE(method >= 0 && method <= 3, DDSP_B200_E_INVALID,
               "resample_backward: bad method %d", method);
  if (method == 0) {
    // upsample_with_windows (core.py:676-693)
    const int n_frames = add_endpoint ? F + 1 : F;
    const int n_intervals = n_frames - 1;
    DDSP_REQUIRE(n_frames < N, DDSP_B200_E_INVALID,
                 "Upsample with windows cannot be used for downsampling"
                 "More input frames (%d) than output timesteps (%d)", n_frames, N);
    DDSP_REQUIRE(n_intervals > 0 && N % n_intervals == 0, DDSP_B200_E_INVALID,
                 "For upsampling, the target the number of timesteps must be "
                 "divisible by the number of input frames%s. (timesteps:%d, "
                 "frames:%d, add_endpoint=%s).", add_endpoint ? "" : " - 1", N,
                 n_frames, add_endpoint ? "True" : "False");
  }
  if (B == 0) return 0;
  const rt_::ResampleGeom g = rt_::resample_geom(F, N, method, add_endpoint);
  const int64_t total = (int64_t)B * F * C;
  if (N >= 8 * F) {   // long frames: a warp per frame
    rt_::resample_backward_kernel<32>
        <<<grid_for(total * 32, rt_::kThreads, 16), rt_::kThreads, 0, (cudaStream_t)stream>>>(
            grad_out, grad_in, B, C, g);
  } else {
    rt_::resample_backward_kernel<1>
        <<<grid_for(total, rt_::kThreads, 16), rt_::kThreads, 0, (cudaStream_t)stream>>>(
            grad_out, grad_in, B, C, g);
  }
  DDSP_CHECK_LAUNCH("resample_backward");
  return 0;
}

int ddsp_b200_mix_forward(const float* signal_one, const float* signal_two,
                          const float* mix_level, float* out, int B, int N, int C,
                          void* stream) {
  DDSP_REQUIRE(signal_one && signal_two && mix_level && out, DDSP_B200_E_INVALID,
               "mix_forward: null pointer");
  DDSP_REQUIRE(B >= 0 && N >= 1 && C >= 1, DDSP_B200_E_INVALID,
               "mix_forward: bad shape B=%d N=%d C=%d", B, N, C);
  if (B == 0) return 0;
  const int64_t total = (int64_t)B * N * C;
  rt_::mix_kernel<<<grid_for(total, rt_::kThreads), rt_::kThreads, 0, (cudaStream_t)stream>>>(
      signal_one, signal_two, mix_level, out, (int64_t)B * N, C);
  DDSP_CHECK_LAUNCH("mix_forward");
  return 0;
}

int ddsp_b200_mix_backward(const float* signal_one, const float* signal_two,
                           const float* mix_level, const float* grad_out,
                           float* grad_signal_one, float* grad_signal_two,
                           float* grad_mix_level, int B, int N, int C, void* stream) {
  DDSP_REQUIRE(signal_one && signal_two && mix_level && grad_out, DDSP_B200_E_INVALID,
               "mix_backward: null pointer");
  DDSP_REQUIRE(B >= 0 && N >= 1 && C >= 1, DDSP_B200_E_INVALID,
               "mix_backward: bad shape B=%d N=%d C=%d", B, N, C);
  if (B == 0 || (!grad_signal_one && !grad_signal_two && !grad_mix_level)) return 0;
  const int64_t rows = (int64_t)B * N;
  rt_::mix_backward_kernel<<<grid_for(rows, rt_::kThreads), rt_::kThreads, 0,
                             (cudaStream_t)stream>>>(
      signal_one, signal_two, mix_level, grad_out, grad_signal_one, grad_signal_two,
      grad_mix_level, rows, C);
  DDSP_CHECK_LAUNCH("mix_backward");
  return 0;
}

int ddsp_b200_exp_decay_ir(const float* gain, const float* decay, const float* noise,
                           uint64_t seed, uint64_t offset, float* ir, int rows, int L,
                           void* stream) {
  DDSP_REQUIRE(gain && decay && ir, DDSP_B200_E_INVALID, "exp_decay_ir: null pointer");
  DDSP_REQUIRE(rows >= 0 && L >= 1, DDSP_B200_E_INVALID,
               "exp_decay_ir: bad shape rows=%d L=%d", rows, L);
  if (rows == 0) return 0;
  const int64_t total = (int64_t)rows * ((L + 3) / 4);
  rt_::exp_decay_ir_kernel<<<grid_for(total, rt_::kThreads), rt_::kThreads, 0,
                             (cudaStream_t)stream>>>(gain, decay, noise, seed, offset, ir,
                                                     rows, L);
  DDSP_CHECK_LAUNCH("exp_decay_ir");
  return 0;
}

int ddsp_b200_exp_decay_ir_backward(const float* gain, const float* decay,
                                    const float* noise, uint64_t seed, uint64_t offset,
                                    const float* grad_ir, float* grad_gain,
                                    float* grad_decay, int rows, int L, void* stream) {
  DDSP_REQUIRE(gain && decay && grad_ir, DDSP_B200_E_INVALID,
               "exp_decay_ir_backward: null pointer");
  DDSP_REQUIRE(rows >= 0 && L >= 1, DDSP_B200_E_INVALID,
               "exp_decay_ir_backward: bad shape rows=%d L=%d", rows, L);
  if (rows == 0 || (!grad_gain && !grad_decay)) return 0;
  rt_::exp_decay_ir_backward_kernel<<<rows, rt_::kIrBwdThreads, 0, (cudaStream_t)stream>>>(
      gain, decay, noise, seed, offset, grad_ir, grad_gain, grad_decay, L);
  DDSP_CHECK_LAUNCH("exp_decay_ir_backward");
  return 0;
}


// ---- spectrogram-loss pieces -------------------------------------------------
int ddsp_b200_frame_window(const float* audio, const float* window, float* frames,
                           int B, int N, int n_frames, int frame_size, int frame_step,
                           void* stream) {
  DDSP_REQUIRE(audio && window && frames, DDSP_B200_E_INVALID, "frame_window: null pointer");
  DDSP_REQUIRE(B >= 0 && N >= 1 && n_frames >= 1 && frame_size >= 4 && frame_size % 4 == 0 &&
                   frame_step >= 1 && B <= 65535,
               DDSP_B200_E_INVALID, "frame_window: bad shape B=%d N=%d T=%d n=%d step=%d", B,
               N, n_frames, frame_size, frame_step);
  DDSP_REQUIRE((((uintptr_t)window | (uintptr_t)frames) & 15) == 0, DDSP_B200_E_INVALID,
               "frame_window: window / frames must be 16-byte aligned");
  if (B == 0) return 0;
  const long long quads = ((long long)n_frames * frame_size) / 4;
  dim3 grid((unsigned)((quads + 255) / 256), B);
  frame_window_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(audio, window, frames, N, n_frames,
                                                            frame_size, frame_step);
  DDSP_CHECK_LAUNCH("frame_window");
  return 0;
}

int ddsp_b200_frame_window_adjoint(const float* grad_frames, const float* window,
                                   float* grad_audio, int B, int N, int n_frames,
                                   int frame_size, int frame_step,
                                   const float* scale_device, int accumulate,
                                   void* stream) {
  DDSP_REQUIRE(grad_frames && window && grad_audio, DDSP_B200_E_INVALID,
               "frame_window_adjoint: null pointer");
  DDSP_REQUIRE(B >= 0 && N >= 1 && n_frames >= 1 && frame_size >= 1 && frame_step >= 1 &&
                   B <= 65535,
               DDSP_B200_E_INVALID, "frame_window_adjoint: bad shape");
  if (B == 0) return 0;
  dim3 grid((N + 255) / 256, B);
  frame_window_adjoint_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      grad_frames, window, grad_audio, N, n_frames, frame_size, frame_step,
      scale_device, accumulate);
  DDSP_CHECK_LAUNCH("frame_window_adjoint");
  return 0;
}

int ddsp_b200_spectral_l1(const float* stft_target, const float* stft_value,
                          float* grad_value, double* sums, int64_t n_bins_total,
                          float mag_weight, float logmag_weight, int n_bins,
                          int irfft_size, void* stream) {
  DDSP_REQUIRE(stft_target && stft_value && grad_value && sums, DDSP_B200_E_INVALID,
               "spectral_l1: null pointer");
  DDSP_REQUIRE(n_bins_total >= 1 && n_bins >= 1 && n_bins_total % n_bins == 0 &&
                   (irfft_size == 0 || irfft_size == -1 || irfft_size == 2 * (n_bins - 1)),
               DDSP_B200_E_INVALID, "spectral_l1: bad sizes (total %lld, bins %d, irfft %d)",
               (long long)n_bins_total, n_bins, irfft_size);
  DDSP_REQUIRE((((uintptr_t)stft_target | (uintptr_t)stft_value | (uintptr_t)grad_value) & 15) == 0,
               DDSP_B200_E_INVALID, "spectral_l1: tensors must be 16-byte aligned");
  const long long blocks = std::min<long long>((n_bins_total / 2 + 255) / 256 + 1, 8ll * num_sms());
  spectral_l1_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float2*>(stft_target), reinterpret_cast<const float2*>(stft_value),
      reinterpret_cast<float2*>(grad_value), sums, n_bins_total, mag_weight, logmag_weight,
      1.0f / (float)n_bins_total, 1e-5f, n_bins, irfft_size);
  DDSP_CHECK_LAUNCH("spectral_l1");
  return 0;
}

// ---- modulated delay ----------------------------------------------------------
int ddsp_b200_mod_delay_forward(const float* audio, const float* phase, const float* gain,
                                float* out, int B, int N, int max_length, float scale,
                                float offset, int add_dry, void* stream) {
  DDSP_REQUIRE(audio && phase && out, DDSP_B200_E_INVALID, "mod_delay_forward: null pointer");
  DDSP_REQUIRE(B >= 0 && B <= 65535 && N >= 1 && max_length >= 1 && max_length < (1 << 29),
               DDSP_B200_E_INVALID, "mod_delay_forward: bad shape B=%d N=%d max_length=%d",
               B, N, max_length);
  if (B == 0) return 0;
  dim3 grid((unsigned)((N + md_::kThreads - 1) / md_::kThreads), B);
  md_::mod_delay_forward_kernel<<<grid, md_::kThreads, 0, (cudaStream_t)stream>>>(
      audio, phase, gain, out, N, max_length, scale, offset, add_dry);
  DDSP_CHECK_LAUNCH("mod_delay_forward");
  return 0;
}

int ddsp_b200_mod_delay_backward(const float* audio, const float* phase, const float* gain,
                                 const float* grad_out, float* grad_audio, float* grad_gain,
                                 float* grad_phase, int B, int N, int max_length, float scale,
                                 float offset, int add_dry, void* stream) {
  DDSP_REQUIRE(audio && phase && grad_out, DDSP_B200_E_INVALID,
               "mod_delay_backward: null pointer");
  DDSP_REQUIRE(grad_gain == nullptr || gain != nullptr, DDSP_B200_E_INVALID,
               "mod_delay_backward: grad_gain asked for without a gain");
  DDSP_REQUIRE(B >= 0 && B <= 65535 && N >= 1 && max_length >= 1 && max_length < (1 << 29),
               DDSP_B200_E_INVALID, "mod_delay_backward: bad shape B=%d N=%d max_length=%d",
               B, N, max_length);
  if (B == 0 || (!grad_audio && !grad_gain && !grad_phase)) return 0;
  const size_t smem = grad_audio ? md_::backward_smem_bytes() : 0;
  int rc = set_smem(md_::mod_delay_backward_kernel, md_::backward_smem_bytes(),
                    "mod_delay_backward");
  if (rc) return rc;
  dim3 grid((unsigned)((N + md_::kTile - 1) / md_::kTile), B);
  md_::mod_delay_backward_kernel<<<grid, md_::kThreads, smem, (cudaStream_t)stream>>>(
      audio, phase, gain, grad_out, grad_audio, grad_gain, grad_phase, N, max_length, scale,
      offset, add_dry);
  DDSP_CHECK_LAUNCH("mod_delay_backward");
  return 0;
}

size_t ddsp_b200_wavetable_workspace(int B, int F) {
  if (B <= 0 || F <= 0) return 0;
  const size_t n_tiles = ((size_t)F + wt_::kFT - 1) / wt_::kFT;
  return sizeof(unsigned long long) * ((size_t)B * n_tiles + 3 * (size_t)B * F) + 4 * 256;
}

size_t ddsp_b200_wavetable_backward_workspace(int B, int F, int N, int Fw, int W) {
  if (B <= 0 || F <= 0 || N <= 0 || Fw <= 0 || W <= 0) return 0;
  const int n_seg = wt_::table_segments(N, Fw);
  size_t bytes = ddsp_b200_wavetable_workspace(B, F) + sizeof(float) * 6 * (size_t)B * F + 512;
  if (n_seg > 1) bytes += sizeof(float) * (size_t)B * Fw * n_seg * W + 256;
  return bytes;
}

// The checks the forward and the backward share; `name` prefixes the messages.  The
// caller returns 0 for B == 0 afterwards.
static int wt_check(const char* name, int B, int F, int N, int Fw, int W, float sample_rate,
                    int amp_method, const void* workspace, size_t workspace_bytes,
                    size_t need) {
  DDSP_REQUIRE(B >= 0 && F >= 1 && N >= 1 && Fw >= 1 && W >= 1, DDSP_B200_E_INVALID,
               "%s: bad shape B=%d F=%d N=%d Fw=%d W=%d", name, B, F, N, Fw, W);
  DDSP_REQUIRE(amp_method == DDSP_B200_AMP_WINDOW || amp_method == DDSP_B200_AMP_LINEAR,
               DDSP_B200_E_INVALID, "%s: bad amp_method %d", name, amp_method);
  DDSP_REQUIRE(N % F == 0, DDSP_B200_E_INVALID,
               "%s: n_samples (%d) must be divisible by the number of frames (%d)", name,
               N, F);
  DDSP_REQUIRE(amp_method != DDSP_B200_AMP_WINDOW || F < N, DDSP_B200_E_INVALID,
               "%s: window upsampling cannot downsample (frames %d >= timesteps %d)",
               name, F, N);
  DDSP_REQUIRE(sample_rate > 0.f, DDSP_B200_E_INVALID,
               "%s: sample_rate must be positive", name);
  DDSP_REQUIRE(W <= wt_::kMaxW, DDSP_B200_E_UNSUPPORTED,
               "%s: W=%d exceeds the %d wavetable columns supported", name, W, wt_::kMaxW);
  DDSP_REQUIRE((int64_t)Fw * wt_::table_segments(N, Fw) * wt_::table_col_tiles(W) < (1ll << 31),
               DDSP_B200_E_UNSUPPORTED, "%s: Fw=%d W=%d exceeds the grid limit", name, Fw,
               W);
  if (B == 0) return 0;
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID,
               "%s: B=%d exceeds the 65535 grid limit", name, B);
  DDSP_REQUIRE(workspace != nullptr && workspace_bytes >= need, DDSP_B200_E_WORKSPACE,
               "%s: workspace of %zu B needed, %zu given", name, need, workspace_bytes);
  return 0;
}

// Passes 1-3 of wavetable.cuh: the fixed-point phase P, A, D of every frame.
struct WtPhase {
  unsigned long long *sums, *P, *A, *D;
  void* end;
};
static WtPhase wt_phase_layout(void* workspace, int B, int F) {
  WtPhase w;
  const int n_tiles = (F + wt_::kFT - 1) / wt_::kFT;
  w.sums = align256<unsigned long long>(workspace);
  w.P = align256<unsigned long long>(w.sums + (size_t)B * n_tiles);
  w.A = align256<unsigned long long>(w.P + (size_t)B * F);
  w.D = align256<unsigned long long>(w.A + (size_t)B * F);
  w.end = w.D + (size_t)B * F;
  return w;
}
static int wt_frame_phases(const WtPhase& w, const float* f0, int B, int F, int hop,
                           float sample_rate, cudaStream_t st, const char* name) {
  const int n_tiles = (F + wt_::kFT - 1) / wt_::kFT;
  const double sr = (double)sample_rate;
  wt_::wt_tile_sums<<<dim3(n_tiles, B), wt_::kFT, 0, st>>>(f0, w.sums, F, hop, n_tiles, sr);
  DDSP_CHECK_LAUNCH(name);
  oscbank_scan_chunks<<<(B + kObThreads - 1) / kObThreads, kObThreads, 0, st>>>(
      w.sums, 1, n_tiles, (int64_t)B);
  DDSP_CHECK_LAUNCH(name);
  wt_::wt_frame_phase<<<dim3(n_tiles, B), wt_::kFT, 0, st>>>(f0, w.sums, w.P, w.A, w.D, F,
                                                             hop, n_tiles, sr);
  DDSP_CHECK_LAUNCH(name);
  return 0;
}

int ddsp_b200_wavetable_forward(const float* f0_hz, const float* amplitudes,
                                const float* wavetables, float* audio, int B, int F,
                                int N, int Fw, int W, float sample_rate, int amp_method,
                                void* workspace, size_t workspace_bytes, void* stream) {
  DDSP_REQUIRE(f0_hz && amplitudes && wavetables && audio, DDSP_B200_E_INVALID,
               "wavetable_forward: null pointer");
  int rc = wt_check("wavetable_forward", B, F, N, Fw, W, sample_rate, amp_method, workspace,
                    workspace_bytes, ddsp_b200_wavetable_workspace(B, F));
  if (rc || B == 0) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int hop = N / F;
  const WtPhase w = wt_phase_layout(workspace, B, F);
  rc = wt_frame_phases(w, f0_hz, B, F, hop, sample_rate, st, "wavetable_forward(phase)");
  if (rc) return rc;
  auto kern = amp_method == DDSP_B200_AMP_WINDOW ? wt_::wt_forward<true>
                                                 : wt_::wt_forward<false>;
  kern<<<dim3((unsigned)((N + wt_::kThreads - 1) / wt_::kThreads), B), wt_::kThreads, 0, st>>>(
      amplitudes, wavetables, w.P, w.A, w.D, audio, F, N, hop, Fw, W);
  DDSP_CHECK_LAUNCH("wavetable_forward");
  return 0;
}

int ddsp_b200_wavetable_backward(const float* f0_hz, const float* amplitudes,
                                 const float* wavetables, const float* grad_audio,
                                 float* d_f0, float* d_amplitudes, float* d_wavetables,
                                 int B, int F, int N, int Fw, int W, float sample_rate,
                                 int amp_method, void* workspace, size_t workspace_bytes,
                                 void* stream) {
  DDSP_REQUIRE(f0_hz && amplitudes && wavetables && grad_audio, DDSP_B200_E_INVALID,
               "wavetable_backward: null pointer");
  int rc = wt_check("wavetable_backward", B, F, N, Fw, W, sample_rate, amp_method, workspace,
                    workspace_bytes, ddsp_b200_wavetable_backward_workspace(B, F, N, Fw, W));
  if (rc || B == 0 || (!d_f0 && !d_amplitudes && !d_wavetables)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int hop = N / F;
  const bool window = amp_method == DDSP_B200_AMP_WINDOW;
  const WtPhase w = wt_phase_layout(workspace, B, F);
  float* part = align256<float>(w.end);                    // [5][B F]
  const int64_t BF = (int64_t)B * F;
  float* d_amp_scratch = align256<float>(part + 5 * (size_t)BF);
  float* tab_part = align256<float>(d_amp_scratch + (size_t)BF);
  rc = wt_frame_phases(w, f0_hz, B, F, hop, sample_rate, st, "wavetable_backward(phase)");
  if (rc) return rc;

  if (d_f0 || d_amplitudes) {
    const bool phase = d_f0 != nullptr;
    auto kern = window ? (phase ? wt_::wt_bwd_frames<true, true>
                                : wt_::wt_bwd_frames<true, false>)
                       : (phase ? wt_::wt_bwd_frames<false, true>
                                : wt_::wt_bwd_frames<false, false>);
    kern<<<(unsigned)((BF + 31) / 32), kSbThreads, 0, st>>>(
        amplitudes, wavetables, grad_audio, w.P, w.A, w.D, part, F, N, hop, Fw, W, BF);
    DDSP_CHECK_LAUNCH("wavetable_backward(frames)");
    // K = 1; sinus_bwd_finalize always writes d amplitudes
    sinus_bwd_finalize<<<dim3(1, B), 32 * kSfinWarps, 0, st>>>(
        part, d_amplitudes ? d_amplitudes : d_amp_scratch, d_f0, F, 1, hop, BF,
        1.0 / (double)sample_rate);
    DDSP_CHECK_LAUNCH("wavetable_backward(finalize)");
  }

  if (d_wavetables) {
    const int n_seg = wt_::table_segments(N, Fw);
    const size_t smem = wt_::table_smem_bytes(W);
    auto kern = window ? wt_::wt_bwd_table<true> : wt_::wt_bwd_table<false>;
    rc = set_smem(kern, smem, "wavetable_backward");
    if (rc) return rc;
    const unsigned gx = (unsigned)((int64_t)Fw * n_seg * wt_::table_col_tiles(W));
    kern<<<dim3(gx, B), wt_::kTabWarps * 32, smem, st>>>(
        amplitudes, grad_audio, w.P, w.A, w.D, n_seg > 1 ? tab_part : d_wavetables, F, N,
        hop, Fw, W, n_seg);
    DDSP_CHECK_LAUNCH("wavetable_backward(wavetables)");
    if (n_seg > 1) {
      const int64_t RW = (int64_t)B * Fw * W;
      wt_::wt_table_reduce<<<grid_for(RW, 256), 256, 0, st>>>(tab_part, d_wavetables, RW, W,
                                                            n_seg);
      DDSP_CHECK_LAUNCH("wavetable_backward(reduce)");
    }
  }
  return 0;
}

// ---- loudness and RMS power ----------------------------------------------------
// The checks every framing entry point makes (spectral_ops.pad and
// get_framed_lengths); sets *pad_left.  `name` prefixes the messages.
static int framing_check(const char* name, int B, int N, int n_frames, int frame, int hop,
                         int padding, int* pad_left) {
  DDSP_REQUIRE(B >= 0 && N >= 1 && n_frames >= 0 && frame >= 1 && hop >= 1,
               DDSP_B200_E_INVALID, "%s: bad shape B=%d N=%d T=%d frame=%d hop=%d", name, B,
               N, n_frames, frame, hop);
  DDSP_REQUIRE(padding == DDSP_B200_PAD_SAME || padding == DDSP_B200_PAD_VALID ||
                   padding == DDSP_B200_PAD_CENTER,
               DDSP_B200_E_INVALID, "%s: bad padding %d", name, padding);
  DDSP_REQUIRE(padding == DDSP_B200_PAD_VALID || hop <= frame, DDSP_B200_E_INVALID,
               "%s: frame_size (%d) must be greater than hop_size (%d)", name, frame, hop);
  *pad_left = padding == DDSP_B200_PAD_CENTER ? frame / 2 : 0;
  long long want;
  if (padding == DDSP_B200_PAD_SAME) {
    want = ((long long)N + hop - 1) / hop;
  } else {
    const long long padded = (long long)N + 2ll * *pad_left;
    want = padded >= frame ? 1 + (padded - frame) / hop : 0;
  }
  DDSP_REQUIRE(n_frames == want, DDSP_B200_E_INVALID, "%s: n_frames=%d, the padding gives %lld",
               name, n_frames, want);
  if (B == 0) return 0;
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID, "%s: B=%d exceeds the 65535 grid limit", name,
               B);
  return 0;
}

static size_t ld_fwd_smem(int M, int warps, int64_t span) {
  return sizeof(float2) * (size_t)M * (warps + 1) + sizeof(float) * (size_t)span;
}
static int ld_own(int n_fft) { return std::max(ld_::kMinOwn, n_fft); }
static size_t ld_bwd_smem(int M, int warps, int own) {
  return sizeof(float2) * (size_t)M * (warps + 1) + sizeof(float) * (size_t)own +
         sizeof(int) * warps;
}
// Warps per CTA: the most of 8, 4, 2, 1 whose slices fit both kernels.  n_fft up to
// ld_::kMaxFft always fits one.
static int ld_warps(int n_fft) {
  const int M = n_fft / 2;
  int w = 8;
  while (w > 1 && (ld_fwd_smem(M, w, n_fft) > kMaxDynSmem ||
                   ld_bwd_smem(M, w, ld_own(n_fft)) > kMaxDynSmem))
    w /= 2;
  return w;
}

static int loud_check(const char* name, int B, int N, int n_frames, int n_fft, int hop,
                      int padding, ld_::LoudParams* p) {
  int pad_left = 0;
  int rc = framing_check(name, B, N, n_frames, n_fft, hop, padding, &pad_left);
  if (rc) return rc;
  DDSP_REQUIRE(n_fft >= 2 && (n_fft & (n_fft - 1)) == 0, DDSP_B200_E_INVALID,
               "%s: n_fft (%d) must be a power of two", name, n_fft);
  DDSP_REQUIRE(n_fft <= ld_::kMaxFft, DDSP_B200_E_UNSUPPORTED,
               "%s: n_fft=%d exceeds the %d supported", name, n_fft, ld_::kMaxFft);
  p->N = N; p->T = n_frames; p->n_fft = n_fft; p->M = n_fft / 2; p->hop = hop;
  p->pad_left = pad_left;
  p->log2M = 0;
  while ((1 << p->log2M) < p->M) ++p->log2M;
  return 0;
}

static void db_params(ld_::LoudParams* p, float range_db, float ref_db) {
  p->pmin = pow(10.0, -(double)range_db / 10.0);
  p->range_db = (double)range_db;
  p->ref_db = (double)ref_db;
}

int ddsp_b200_loudness_forward(const float* audio, const float* weights, float* loudness,
                               int B, int N, int n_frames, int n_fft, int hop, int padding,
                               float range_db, float ref_db, void* stream) {
  DDSP_REQUIRE(audio && weights && (loudness || n_frames == 0), DDSP_B200_E_INVALID,
               "loudness_forward: null pointer");
  ld_::LoudParams p;
  int rc = loud_check("loudness_forward", B, N, n_frames, n_fft, hop, padding, &p);
  if (rc || B == 0 || n_frames == 0) return rc;
  p.audio = audio; p.weights = weights;
  db_params(&p, range_db, ref_db);
  const int warps = ld_warps(n_fft);
  int per_cta = 4 * warps;
  while (per_cta > 1 &&
         ld_fwd_smem(p.M, warps, (int64_t)(per_cta - 1) * hop + n_fft) > kMaxDynSmem)
    per_cta /= 2;
  const int span = (int)((int64_t)(per_cta - 1) * hop + n_fft);
  const size_t smem = ld_fwd_smem(p.M, warps, span);
  rc = set_smem(ld_::loudness_kernel, smem, "loudness_forward");
  if (rc) return rc;
  dim3 grid((unsigned)((n_frames + per_cta - 1) / per_cta), B);
  ld_::loudness_kernel<<<grid, 32 * warps, smem, (cudaStream_t)stream>>>(p, loudness, per_cta,
                                                                         span);
  DDSP_CHECK_LAUNCH("loudness_forward");
  return 0;
}

int ddsp_b200_loudness_backward(const float* audio, const float* weights,
                                const float* grad_loudness, float* grad_audio, int B, int N,
                                int n_frames, int n_fft, int hop, int padding, float range_db,
                                float ref_db, void* stream) {
  DDSP_REQUIRE(audio && weights && (grad_loudness || n_frames == 0) && grad_audio,
               DDSP_B200_E_INVALID, "loudness_backward: null pointer");
  ld_::LoudParams p;
  int rc = loud_check("loudness_backward", B, N, n_frames, n_fft, hop, padding, &p);
  if (rc || B == 0) return rc;
  p.audio = audio; p.weights = weights;
  db_params(&p, range_db, ref_db);
  const int warps = ld_warps(n_fft), own = ld_own(n_fft);
  const size_t smem = ld_bwd_smem(p.M, warps, own);
  rc = set_smem(ld_::loudness_backward_kernel, smem, "loudness_backward");
  if (rc) return rc;
  dim3 grid((unsigned)((N + own - 1) / own), B);
  ld_::loudness_backward_kernel<<<grid, 32 * warps, smem, (cudaStream_t)stream>>>(
      p, grad_loudness, grad_audio, own);
  DDSP_CHECK_LAUNCH("loudness_backward");
  return 0;
}

int ddsp_b200_rms_power(const float* audio, float* power_db, int B, int N, int n_frames,
                        int frame_size, int hop, int padding, int in_db, float range_db,
                        float ref_db, void* stream) {
  DDSP_REQUIRE(audio && (power_db || n_frames == 0), DDSP_B200_E_INVALID,
               "rms_power: null pointer");
  int pad_left = 0;
  int rc = framing_check("rms_power", B, N, n_frames, frame_size, hop, padding, &pad_left);
  if (rc || B == 0 || n_frames == 0) return rc;
  ld_::LoudParams d;
  db_params(&d, range_db, ref_db);
  const int64_t total = (int64_t)B * n_frames;
  ld_::rms_power_kernel<<<grid_for(total * 32, ld_::kRmsThreads), ld_::kRmsThreads, 0,
                          (cudaStream_t)stream>>>(audio, power_db, N, n_frames, total,
                                                  frame_size, hop, pad_left, in_db, d.pmin,
                                                  d.range_db, d.ref_db);
  DDSP_CHECK_LAUNCH("rms_power");
  return 0;
}

// ---- mel, log-mel and MFCC -------------------------------------------------------
// Twiddles and one FFT slice per warp, one [bins] row per warp, and the MFCC's
// 4 bins cosine table.
static size_t mel_fixed_smem(int M, int warps, int bins, int mode) {
  return sizeof(float2) * (size_t)M * (warps + 1) +
         sizeof(float) * (size_t)bins * (warps + (mode == DDSP_B200_MFCC ? 4 : 0));
}
static size_t mel_bwd_smem(int M, int warps, int bins, int mode, int own) {
  return mel_fixed_smem(M, warps, bins, mode) + sizeof(float) * (size_t)own +
         sizeof(int) * warps;
}
// Warps per CTA: the most of 8, 4, 2, 1 whose backward fits with the smallest owned
// span.  bins <= mel_::kMaxBins fits one warp at every fft_length.
static int mel_warps(int M, int bins, int mode) {
  int w = 8;
  while (w > 1 && mel_bwd_smem(M, w, bins, mode, mel_::kOwnFloor) > kMaxDynSmem) w /= 2;
  return w;
}
// Backward: samples a CTA owns, max(kMinOwn, fft_size) halved until it fits.
static int mel_own(int fft_size, int M, int warps, int bins, int mode) {
  int own = std::max(mel_::kMinOwn, fft_size);
  while (own > mel_::kOwnFloor && mel_bwd_smem(M, warps, bins, mode, own) > kMaxDynSmem)
    own /= 2;
  return own;
}

static int mel_check(const char* name, int B, int N, int n_frames, int fft_size,
                     int fft_length, int hop, int pad_end, int bins, int n_out, int mode,
                     mel_::MelParams* p) {
  DDSP_REQUIRE(B >= 0 && N >= 1 && n_frames >= 0 && fft_size >= 1 && hop >= 1,
               DDSP_B200_E_INVALID, "%s: bad shape B=%d N=%d T=%d fft_size=%d hop=%d", name,
               B, N, n_frames, fft_size, hop);
  DDSP_REQUIRE(pad_end == 0 || pad_end == 1, DDSP_B200_E_INVALID, "%s: bad pad_end %d", name,
               pad_end);
  DDSP_REQUIRE(mode == DDSP_B200_MEL || mode == DDSP_B200_LOGMEL || mode == DDSP_B200_MFCC,
               DDSP_B200_E_INVALID, "%s: bad mode %d", name, mode);
  DDSP_REQUIRE(bins >= 1 && (mode == DDSP_B200_MFCC ? n_out >= 0 && n_out <= bins
                                                    : n_out == bins),
               DDSP_B200_E_INVALID, "%s: bad bins=%d n_out=%d for mode %d", name, bins, n_out,
               mode);
  DDSP_REQUIRE(fft_length >= 1 && (fft_length & (fft_length - 1)) == 0, DDSP_B200_E_INVALID,
               "%s: fft_length (%d) must be a power of two", name, fft_length);
  DDSP_REQUIRE(fft_length >= 2 && fft_length <= ld_::kMaxFft, DDSP_B200_E_UNSUPPORTED,
               "%s: fft_length=%d is outside the 2..%d supported", name, fft_length,
               ld_::kMaxFft);
  DDSP_REQUIRE(fft_size <= fft_length, DDSP_B200_E_INVALID,
               "%s: fft_size (%d) exceeds fft_length (%d)", name, fft_size, fft_length);
  DDSP_REQUIRE(bins <= mel_::kMaxBins, DDSP_B200_E_UNSUPPORTED,
               "%s: bins=%d exceeds the %d supported", name, bins, mel_::kMaxBins);
  const long long want = pad_end ? ((long long)N + hop - 1) / hop
                                 : (N >= fft_size ? 1 + (long long)(N - fft_size) / hop : 0);
  DDSP_REQUIRE(n_frames == want, DDSP_B200_E_INVALID, "%s: n_frames=%d, the padding gives %lld",
               name, n_frames, want);
  if (B == 0) return 0;
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID, "%s: B=%d exceeds the 65535 grid limit", name,
               B);
  p->N = N; p->T = n_frames; p->fft_size = fft_size; p->M = fft_length / 2; p->hop = hop;
  p->bins = bins; p->C = n_out;
  p->log2M = 0;
  while ((1 << p->log2M) < p->M) ++p->log2M;
  return 0;
}

static void mel_tables(mel_::MelParams* p, const float* audio, const float* window,
                       const void* mel_table, int fft_length, int bins) {
  const int K = fft_length / 2 + 1;
  p->audio = audio; p->window = window;
  p->wpair = static_cast<const float2*>(mel_table);
  p->band = reinterpret_cast<const int*>(p->wpair + K);
  p->band_lo = p->band + K;
  p->band_hi = p->band_lo + bins;
}

int ddsp_b200_mel_forward(const float* audio, const float* window, const void* mel_table,
                          float* out, int B, int N, int n_frames, int fft_size, int fft_length,
                          int hop, int pad_end, int bins, int n_out, int mode, void* stream) {
  DDSP_REQUIRE(audio && window && mel_table && (out || n_frames == 0 || n_out == 0),
               DDSP_B200_E_INVALID, "mel_forward: null pointer");
  mel_::MelParams p;
  int rc = mel_check("mel_forward", B, N, n_frames, fft_size, fft_length, hop, pad_end, bins,
                     n_out, mode, &p);
  if (rc || B == 0 || n_frames == 0 || n_out == 0) return rc;
  mel_tables(&p, audio, window, mel_table, fft_length, bins);
  const int warps = mel_warps(p.M, bins, mode);
  const size_t fixed = mel_fixed_smem(p.M, warps, bins, mode);
  // stage the audio span of per_cta frames; when not even two fit, each warp reads
  // its own frame from global memory
  int per_cta = 4 * warps;
  while (per_cta > 1 &&
         fixed + sizeof(float) * ((int64_t)(per_cta - 1) * hop + fft_size) > kMaxDynSmem)
    per_cta /= 2;
  int span = (int)((int64_t)(per_cta - 1) * hop + fft_size);
  if (per_cta == 1) {
    per_cta = warps;
    span = 0;
  }
  const size_t smem = fixed + sizeof(float) * (size_t)span;
  auto kern = mode == DDSP_B200_MEL      ? mel_::mel_kernel<mel_::kMel>
              : mode == DDSP_B200_LOGMEL ? mel_::mel_kernel<mel_::kLogMel>
                                         : mel_::mel_kernel<mel_::kMfcc>;
  rc = set_smem(kern, smem, "mel_forward");
  if (rc) return rc;
  dim3 grid((unsigned)((n_frames + per_cta - 1) / per_cta), B);
  kern<<<grid, 32 * warps, smem, (cudaStream_t)stream>>>(p, out, per_cta, span);
  DDSP_CHECK_LAUNCH("mel_forward");
  return 0;
}

int ddsp_b200_mel_backward(const float* audio, const float* window, const void* mel_table,
                           const float* grad_out, float* grad_audio, int B, int N,
                           int n_frames, int fft_size, int fft_length, int hop, int pad_end,
                           int bins, int n_out, int mode, void* stream) {
  DDSP_REQUIRE(audio && window && mel_table && (grad_out || n_frames == 0 || n_out == 0) &&
                   grad_audio,
               DDSP_B200_E_INVALID, "mel_backward: null pointer");
  mel_::MelParams p;
  int rc = mel_check("mel_backward", B, N, n_frames, fft_size, fft_length, hop, pad_end, bins,
                     n_out, mode, &p);
  if (rc || B == 0 || n_frames == 0 || n_out == 0) return rc;
  mel_tables(&p, audio, window, mel_table, fft_length, bins);
  const int warps = mel_warps(p.M, bins, mode);
  const int own = mel_own(fft_size, p.M, warps, bins, mode);
  const size_t smem = mel_bwd_smem(p.M, warps, bins, mode, own);
  auto kern = mode == DDSP_B200_MEL      ? mel_::mel_backward_kernel<mel_::kMel>
              : mode == DDSP_B200_LOGMEL ? mel_::mel_backward_kernel<mel_::kLogMel>
                                         : mel_::mel_backward_kernel<mel_::kMfcc>;
  rc = set_smem(kern, smem, "mel_backward");
  if (rc) return rc;
  dim3 grid((unsigned)((N + own - 1) / own), B);
  kern<<<grid, 32 * warps, smem, (cudaStream_t)stream>>>(p, grad_out, grad_audio, own);
  DDSP_CHECK_LAUNCH("mel_backward");
  return 0;
}

// ---- consistency-loss mixture NLLs -------------------------------------------------
static int cons_rows(const char* name, int B, int T, int64_t* rows) {
  DDSP_REQUIRE((int64_t)B * T <= INT32_MAX, DDSP_B200_E_INVALID,
               "%s: B*T=%lld exceeds the 2^31 - 1 grid limit", name, (long long)B * T);
  *rows = (int64_t)B * T;
  return 0;
}

static int mix_check(const char* name, int B, int T, int Q, int J, float scale,
                     cons_::MixParams* p, int64_t* rows) {
  DDSP_REQUIRE(B >= 0 && T >= 0 && Q >= 0 && J >= 0, DDSP_B200_E_INVALID,
               "%s: bad shape B=%d T=%d Q=%d J=%d", name, B, T, Q, J);
  DDSP_REQUIRE(scale > 0.f && scale <= FLT_MAX, DDSP_B200_E_INVALID,
               "%s: scale must be positive and finite, got %g", name, (double)scale);
  DDSP_REQUIRE(J <= cons_::kMaxStaged, DDSP_B200_E_UNSUPPORTED,
               "%s: J=%d components exceed the %d supported", name, J, cons_::kMaxStaged);
  int rc = cons_rows(name, B, T, rows);
  if (rc) return rc;
  p->Q = Q;
  p->J = J;
  p->inv_scale = (float)(1.0 / scale);
  p->log_norm = (float)(std::log((double)scale) + 0.5 * std::log(2.0 * M_PI));
  return 0;
}

int ddsp_b200_mixture_nll_forward(const float* x, const float* mu, const float* lw,
                                  float* nll, int B, int T, int Q, int J, float scale,
                                  void* stream) {
  const bool empty = B == 0 || T == 0 || Q == 0 || J == 0;
  DDSP_REQUIRE(empty || (x && mu && lw && nll), DDSP_B200_E_INVALID,
               "mixture_nll_forward: null pointer");
  cons_::MixParams p;
  int64_t rows = 0;
  int rc = mix_check("mixture_nll_forward", B, T, Q, J, scale, &p, &rows);
  if (rc || rows == 0 || Q == 0 || J == 0) return rc;
  p.x = x; p.mu = mu; p.lw = lw;
  const size_t smem = sizeof(float) * 2 * (size_t)J;
  rc = set_smem(cons_::mixture_nll_kernel, smem, "mixture_nll_forward");
  if (rc) return rc;
  cons_::mixture_nll_kernel<<<(unsigned)rows, cons_::kThreads, smem, (cudaStream_t)stream>>>(
      p, nll);
  DDSP_CHECK_LAUNCH("mixture_nll_forward");
  return 0;
}

int ddsp_b200_mixture_nll_backward(const float* x, const float* mu, const float* lw,
                                   const float* grad, float* dx, float* dmu, float* dlw,
                                   int B, int T, int Q, int J, float scale, void* stream) {
  const bool empty = B == 0 || T == 0 || Q == 0 || J == 0;
  DDSP_REQUIRE(empty || (x && mu && lw && grad && dx && dmu && dlw), DDSP_B200_E_INVALID,
               "mixture_nll_backward: null pointer");
  cons_::MixParams p;
  int64_t rows = 0;
  int rc = mix_check("mixture_nll_backward", B, T, Q, J, scale, &p, &rows);
  if (rc || rows == 0 || Q == 0 || J == 0) return rc;
  p.x = x; p.mu = mu; p.lw = lw;
  const size_t smem = sizeof(float) * (4 * (size_t)J + 5 * cons_::kChunk);
  rc = set_smem(cons_::mixture_nll_backward_kernel, smem, "mixture_nll_backward");
  if (rc) return rc;
  cons_::mixture_nll_backward_kernel<<<(unsigned)rows, cons_::kThreads, smem,
                                       (cudaStream_t)stream>>>(p, grad, dx, dmu, dlw);
  DDSP_CHECK_LAUNCH("mixture_nll_backward");
  return 0;
}

// Half-width W of the comb window: the smallest W for which the terms |k - k0| > W
// sum to less than 2^-25 of the largest term, counting each with the weight 1 + |z_k|
// it carries into d nu / dq.  With k0 the nearest integer, |q - k0| <= 1/2 inside
// [1/2, G + 1/2], so term n = |k - k0| is at most exp(-n (n - 1) / (2 s^2)) of the
// largest (outside, every term is further: at most exp(-n^2 / (2 s^2))), twice for the
// two sides, and |z_k| <= (n + 1/2) / s.
static int comb_window(int G, double scale) {
  std::vector<double> tail(G + 2, 0.0);
  for (int n = G; n >= 1; --n)
    tail[n] = tail[n + 1] +
              2.0 * (1.0 + (n + 0.5) / scale) * std::exp(-0.5 * n * (n - 1.0) / (scale * scale));
  int W = 0;
  while (W < G && tail[W + 1] >= std::ldexp(1.0, -25)) ++W;
  return W;
}

static int comb_check(const char* name, int B, int T, int C, int P, int G, float scale,
                      cons_::CombParams* p, int64_t* rows) {
  DDSP_REQUIRE(B >= 0 && T >= 0 && C >= 0 && P >= 0 && G >= 1, DDSP_B200_E_INVALID,
               "%s: bad shape B=%d T=%d C=%d P=%d G=%d", name, B, T, C, P, G);
  DDSP_REQUIRE(scale > 0.f && scale <= FLT_MAX, DDSP_B200_E_INVALID,
               "%s: scale must be positive and finite, got %g", name, (double)scale);
  DDSP_REQUIRE(C <= cons_::kMaxStaged && P <= cons_::kMaxStaged, DDSP_B200_E_UNSUPPORTED,
               "%s: C=%d candidates or P=%d points exceed the %d supported", name, C, P,
               cons_::kMaxStaged);
  int rc = cons_rows(name, B, T, rows);
  if (rc) return rc;
  p->C = C;
  p->P = P;
  p->G = G;
  p->inv_scale = (float)(1.0 / scale);
  p->log_norm = (float)(std::log((double)G) + std::log((double)scale) +
                        0.5 * std::log(2.0 * M_PI));
  if (*rows && C && P) p->W = comb_window(G, scale);
  return 0;
}

int ddsp_b200_comb_nll_forward(const float* f0, const float* f, const float* a, float* out,
                               int B, int T, int C, int P, int G, float scale, void* stream) {
  const bool empty = B == 0 || T == 0 || C == 0 || P == 0;
  DDSP_REQUIRE(empty || (f0 && f && a && out), DDSP_B200_E_INVALID,
               "comb_nll_forward: null pointer");
  cons_::CombParams p;
  int64_t rows = 0;
  int rc = comb_check("comb_nll_forward", B, T, C, P, G, scale, &p, &rows);
  if (rc || rows == 0 || C == 0 || P == 0) return rc;
  p.f0 = f0; p.f = f; p.a = a;
  const size_t smem = sizeof(float) * (2 * (size_t)P + C + 1);
  rc = set_smem(cons_::comb_nll_kernel, smem, "comb_nll_forward");
  if (rc) return rc;
  cons_::comb_nll_kernel<<<(unsigned)rows, cons_::kThreads, smem, (cudaStream_t)stream>>>(
      p, out);
  DDSP_CHECK_LAUNCH("comb_nll_forward");
  return 0;
}

int ddsp_b200_comb_nll_backward(const float* f0, const float* f, const float* a,
                                const float* grad, float* d_f0, float* d_f, float* d_a,
                                int B, int T, int C, int P, int G, float scale,
                                void* stream) {
  const bool empty = B == 0 || T == 0 || C == 0 || P == 0;
  DDSP_REQUIRE(empty || (f0 && f && a && grad && d_f0 && d_f && d_a), DDSP_B200_E_INVALID,
               "comb_nll_backward: null pointer");
  cons_::CombParams p;
  int64_t rows = 0;
  int rc = comb_check("comb_nll_backward", B, T, C, P, G, scale, &p, &rows);
  if (rc || rows == 0 || C == 0 || P == 0) return rc;
  p.f0 = f0; p.f = f; p.a = a;
  const size_t smem = sizeof(float) * (2 * (size_t)P + 3 * (size_t)C + 1);
  rc = set_smem(cons_::comb_nll_backward_kernel, smem, "comb_nll_backward");
  if (rc) return rc;
  cons_::comb_nll_backward_kernel<<<(unsigned)rows, cons_::kThreads, smem,
                                    (cudaStream_t)stream>>>(p, grad, d_f0, d_f, d_a);
  DDSP_CHECK_LAUNCH("comb_nll_backward");
  return 0;
}

// ---- core.sinusoidal_to_harmonic ---------------------------------------------------
static int s2h_check(const char* name, int B, int T, int S, int K, float width,
                     float sample_rate, int normalize, cons_::S2HParams* p, int64_t* rows) {
  DDSP_REQUIRE(B >= 0 && T >= 0 && S >= 0 && K >= 0, DDSP_B200_E_INVALID,
               "%s: bad shape B=%d T=%d S=%d K=%d", name, B, T, S, K);
  DDSP_REQUIRE(width != 0.f, DDSP_B200_E_INVALID, "%s: harmonic_width must be nonzero",
               name);
  DDSP_REQUIRE(normalize == 0 || normalize == 1, DDSP_B200_E_INVALID,
               "%s: normalize must be 0 or 1, got %d", name, normalize);
  DDSP_REQUIRE(S <= cons_::kMaxStaged, DDSP_B200_E_UNSUPPORTED,
               "%s: S=%d sinusoids exceed the %d supported", name, S, cons_::kMaxStaged);
  int rc = cons_rows(name, B, T, rows);
  if (rc) return rc;
  p->S = S;
  p->K = K;
  p->width = width;
  p->nyquist = sample_rate * 0.5f;
  p->normalize = normalize;
  return 0;
}

int ddsp_b200_sinusoidal_to_harmonic(const float* sin_amps, const float* sin_freqs,
                                     const float* f0_hz, float* harm_amp, float* harm_dist,
                                     int B, int T, int S, int K, float width,
                                     float sample_rate, int normalize, void* stream) {
  const bool empty = B == 0 || T == 0;
  DDSP_REQUIRE(empty || (f0_hz && harm_amp && (S == 0 || (sin_amps && sin_freqs)) &&
                         (K == 0 || harm_dist)),
               DDSP_B200_E_INVALID, "sinusoidal_to_harmonic: null pointer");
  cons_::S2HParams p;
  int64_t rows = 0;
  int rc = s2h_check("sinusoidal_to_harmonic", B, T, S, K, width, sample_rate, normalize, &p,
                     &rows);
  if (rc || rows == 0) return rc;
  p.a = sin_amps; p.f = sin_freqs; p.f0 = f0_hz;
  const size_t smem = sizeof(float) * (2 * (size_t)S + cons_::kThreads + 1);
  rc = set_smem(cons_::sin_to_harm_kernel, smem, "sinusoidal_to_harmonic");
  if (rc) return rc;
  cons_::sin_to_harm_kernel<<<(unsigned)rows, cons_::kThreads, smem, (cudaStream_t)stream>>>(
      p, harm_amp, harm_dist);
  DDSP_CHECK_LAUNCH("sinusoidal_to_harmonic");
  return 0;
}

int ddsp_b200_sinusoidal_to_harmonic_backward(
    const float* sin_amps, const float* sin_freqs, const float* f0_hz, const float* grad_amp,
    const float* grad_dist, float* d_sin_amps, float* d_sin_freqs, float* d_f0_hz, int B,
    int T, int S, int K, float width, float sample_rate, int normalize, void* stream) {
  const bool empty = B == 0 || T == 0;
  DDSP_REQUIRE(empty || (f0_hz && grad_amp && d_f0_hz &&
                         (S == 0 || (sin_amps && sin_freqs && d_sin_amps && d_sin_freqs)) &&
                         (K == 0 || grad_dist)),
               DDSP_B200_E_INVALID, "sinusoidal_to_harmonic_backward: null pointer");
  cons_::S2HParams p;
  int64_t rows = 0;
  int rc = s2h_check("sinusoidal_to_harmonic_backward", B, T, S, K, width, sample_rate,
                     normalize, &p, &rows);
  if (rc || rows == 0) return rc;
  p.a = sin_amps; p.f = sin_freqs; p.f0 = f0_hz;
  const size_t smem =
      sizeof(float) * (4 * (size_t)S + 4 * cons_::kHarmChunk + cons_::kThreads + 1);
  rc = set_smem(cons_::sin_to_harm_backward_kernel, smem, "sinusoidal_to_harmonic_backward");
  if (rc) return rc;
  cons_::sin_to_harm_backward_kernel<<<(unsigned)rows, cons_::kThreads, smem,
                                       (cudaStream_t)stream>>>(
      p, grad_amp, grad_dist, d_sin_amps, d_sin_freqs, d_f0_hz);
  DDSP_CHECK_LAUNCH("sinusoidal_to_harmonic_backward");
  return 0;
}

// ---- losses.HmmTranscriber -----------------------------------------------------------
// The checks every HMM entry point makes, and its kernel parameters.
static int hmm_check(const char* name, const float* obs, const float* loc,
                     const float* scale, int B, int T, int K, double hold, double other,
                     hmm_::Params* p) {
  DDSP_REQUIRE(B >= 0 && T >= 1 && K >= 2, DDSP_B200_E_INVALID,
               "%s: bad shape B=%d T=%d K=%d", name, B, T, K);
  DDSP_REQUIRE(std::isfinite(hold) && std::isfinite(other) && hold >= 0.0 && other >= 0.0 &&
                   hold + other > 0.0,
               DDSP_B200_E_INVALID,
               "%s: hold=%g and other=%g must be finite, non-negative and not both 0",
               name, hold, other);
  DDSP_REQUIRE(K <= hmm_::kMaxStates, DDSP_B200_E_UNSUPPORTED,
               "%s: K=%d states exceed the %d supported", name, K, hmm_::kMaxStates);
  p->obs = reinterpret_cast<const float2*>(obs);
  p->loc = reinterpret_cast<const float2*>(loc);
  p->scale = reinterpret_cast<const float2*>(scale);
  p->T = T;
  p->K = K;
  p->hold = (float)hold;
  p->other = (float)other;
  p->log_hold = (float)std::log(hold);
  p->log_other = (float)std::log(other);
  p->log_init = -std::log((double)K);
  return 0;
}

static unsigned hmm_threads(int K) { return (unsigned)((K + 31) & ~31); }

int ddsp_b200_hmm_log_prob(const float* obs, const float* loc, const float* scale,
                           float* log_prob, int B, int T, int K, double hold, double other,
                           void* stream) {
  DDSP_REQUIRE(B == 0 || (obs && loc && scale && log_prob), DDSP_B200_E_INVALID,
               "hmm_log_prob: null pointer");
  hmm_::Params p;
  int rc = hmm_check("hmm_log_prob", obs, loc, scale, B, T, K, hold, other, &p);
  if (rc || B == 0) return rc;
  hmm_::hmm_log_prob_kernel<<<(unsigned)B, hmm_threads(K), 0, (cudaStream_t)stream>>>(
      p, log_prob);
  DDSP_CHECK_LAUNCH("hmm_log_prob");
  return 0;
}

int ddsp_b200_hmm_log_prob_backward(const float* obs, const float* loc, const float* scale,
                                    const float* grad, float* d_obs, float* checkpoints,
                                    int seg, int B, int T, int K, double hold, double other,
                                    void* stream) {
  DDSP_REQUIRE(B == 0 || (obs && loc && scale && grad && d_obs && checkpoints),
               DDSP_B200_E_INVALID, "hmm_log_prob_backward: null pointer");
  hmm_::Params p;
  int rc = hmm_check("hmm_log_prob_backward", obs, loc, scale, B, T, K, hold, other, &p);
  if (rc) return rc;
  DDSP_REQUIRE(seg >= 1 && (int64_t)seg * K <= hmm_::kSegFloats, DDSP_B200_E_INVALID,
               "hmm_log_prob_backward: seg=%d must be at least 1 with seg*K at most %d",
               seg, hmm_::kSegFloats);
  if (B == 0) return 0;
  const size_t smem = sizeof(float) * (size_t)seg * K;
  rc = set_smem(hmm_::hmm_backward_kernel, smem, "hmm_log_prob_backward");
  if (rc) return rc;
  hmm_::hmm_backward_kernel<<<(unsigned)B, hmm_threads(K), smem, (cudaStream_t)stream>>>(
      p, seg, grad, reinterpret_cast<float2*>(d_obs), checkpoints);
  DDSP_CHECK_LAUNCH("hmm_log_prob_backward");
  return 0;
}

int ddsp_b200_hmm_viterbi(const float* obs, const float* loc, const float* scale,
                          int64_t* path, int B, int T, int K, double hold, double other,
                          void* stream) {
  DDSP_REQUIRE(B == 0 || (obs && loc && scale && path), DDSP_B200_E_INVALID,
               "hmm_viterbi: null pointer");
  hmm_::Params p;
  int rc = hmm_check("hmm_viterbi", obs, loc, scale, B, T, K, hold, other, &p);
  if (rc) return rc;
  const size_t smem = sizeof(uint32_t) * (size_t)T * ((K + 31) / 32 + 1);
  DDSP_REQUIRE(smem <= hmm_::kViterbiBytes, DDSP_B200_E_UNSUPPORTED,
               "hmm_viterbi: T=%d steps of K=%d states need %zu B of back pointers, more "
               "than the %zu supported", T, K, smem, hmm_::kViterbiBytes);
  if (B == 0) return 0;
  rc = set_smem(hmm_::hmm_viterbi_kernel, smem, "hmm_viterbi");
  if (rc) return rc;
  hmm_::hmm_viterbi_kernel<<<(unsigned)B, hmm_threads(K), smem, (cudaStream_t)stream>>>(
      p, path);
  DDSP_CHECK_LAUNCH("hmm_viterbi");
  return 0;
}

#ifdef DDSP_NR_TIMING
// measurement builds only (tools/noise_timing.py): the noise_ring phase counters of
// the last launch, [kMaxSMs CTAs][32 warps][8 phases] cycles (rows past the grid stay 0)
int ddsp_b200_debug_noise_timing(unsigned* host_out) {
  cudaError_t e = cudaMemcpyFromSymbol(host_out, ddsp::nr_::g_nr_timing,
                                       sizeof(unsigned) * kMaxSMs * 32 * 8);
  return e == cudaSuccess ? 0 : DDSP_B200_E_CUDA;
}
#endif

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
