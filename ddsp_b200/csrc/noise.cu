// C ABI of the filtered-noise family: impulse responses, the time-varying FIR,
// uniform noise, filtered noise and their backward, and the fused decoder
// (harmonic_v4 through launch_harmonic_v4, then the noise kernel) with its
// host-buffer pipeline.
#include "capi.cuh"
#include "harmonic_common.cuh"
#include "noise.cuh"
#include "noise_fused.cuh"
#include "noise_ring.cuh"
#include "host_pipeline.cuh"
#include "noise_backward.cuh"
#include "fir_backward.cuh"

using namespace ddsp;

extern "C" {

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
  int rc = check_overlap("frequency_impulse_response", {DDSP_OUT(ir, extent(BF, g.S))},
                         {DDSP_IN(mags, extent(BF, nb))});
  if (rc) return rc;
  const int64_t blocks = (BF + kIrFrames - 1) / kIrFrames;
  DDSP_REQUIRE(blocks < (1ll << 31), DDSP_B200_E_INVALID,
               "frequency_impulse_response: too many frames");
  return launch("frequency_impulse_response", ir_kernel, (int)blocks, kIrThreads, smem,
                (cudaStream_t)stream, mags, ir, BF, g);
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
  int rc = check_overlap("fir_time_varying", {DDSP_OUT(out, extent(B, out_len))},
                         {DDSP_IN(audio, extent(B, N)),
                          DDSP_IN(ir, extent(ir_batch, F, S))});
  if (rc) return rc;
  dim3 grid((out_len + kFirThreads - 1) / kFirThreads, B);
  return launch("fir_time_varying", fir_kernel, grid, kFirThreads, smem,
                (cudaStream_t)stream, audio, ir, out, N, F, S, frame,
                ir_batch == 1 ? 0 : F * S, start, out_len, accumulate);
}

int ddsp_b200_uniform_noise(float* out, int B, int N, uint64_t seed,
                            uint64_t offset, void* stream) {
  DDSP_REQUIRE(out, DDSP_B200_E_INVALID, "uniform_noise: null pointer");
  DDSP_REQUIRE(B >= 0 && N >= 0, DDSP_B200_E_INVALID, "uniform_noise: bad shape");
  if (B == 0 || N == 0) return 0;
  const int64_t n = (int64_t)B * ((N + 3) / 4);
  return launch("uniform_noise", uniform_noise_kernel, grid_for(n, 256), 256, 0,
                (cudaStream_t)stream, out, B, N, seed, offset);
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
    int rc = check_overlap("filtered_noise_forward", {DDSP_OUT(audio, extent(B, N))},
                           {DDSP_IN(mags, extent(B, F, nb)), DDSP_IN(noise, extent(B, N))});
    if (rc) return rc;
    return launch_noise_best(mags, noise, seed, offset, audio, B, F, nb, N,
                             window_size, accumulate, st);
  }
  const size_t need = ddsp_b200_filtered_noise_workspace(B, F, nb, N, window_size);
  DDSP_REQUIRE(workspace != nullptr && workspace_bytes >= need,
               DDSP_B200_E_WORKSPACE,
               "filtered_noise_forward: workspace of %zu B needed, %zu given",
               need, workspace_bytes);
  int rc = check_overlap("filtered_noise_forward", {DDSP_OUT(audio, extent(B, N))},
                         {DDSP_IN(mags, extent(B, F, nb)), DDSP_IN(noise, extent(B, N))});
  if (rc) return rc;
  IrGeom g = make_ir_geom(nb, window_size);
  float* ir = align256<float>(workspace);
  float* nz = ir + (size_t)B * F * g.S;
  rc = ddsp_b200_frequency_impulse_response(mags, ir, (int64_t)B * F, nb, window_size,
                                            stream);
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
  rc = check_overlap("decoder_forward", {DDSP_OUT(audio, extent(B, N))},
                     {DDSP_IN(amps_raw, extent(B, F)), DDSP_IN(hd_raw, extent(B, F, K)),
                      DDSP_IN(f0_hz, extent(B, F)), DDSP_IN(mags_raw, extent(B, F, nb)),
                      DDSP_IN(noise, extent(B, N))});
  if (rc) return rc;
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
  const int per_sm = smem <= 100 * 1024 ? 2 : 1;
  const int grid = (int)std::min<long long>(p.n_tiles, (long long)num_sms() * per_sm);
  return launch(name, noise_backward_kernel, grid, kNbThreads, smem, st, p);
}

int ddsp_b200_filtered_noise_backward_takes(int F, int nb, int N, int window_size) {
  if (F < 1 || N < 1 || nb < 2) return 0;
  const int frame = (N + F - 1) / F;
  if ((N + frame - 1) / frame != F) return 0;
  long long n_tiles;
  size_t smem;
  const NoiseBwdParams p = noise_bwd_params(nullptr, nullptr, 0, 0, nullptr, 1, F, nb, N,
                                            frame, window_size, &n_tiles, &smem);
  return p.start >= 0 && smem <= kMaxDynSmem;
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
  DDSP_REQUIRE(ddsp_b200_filtered_noise_backward_takes(F, nb, N, window_size),
               DDSP_B200_E_UNSUPPORTED,
               p.start < 0 ? "filtered_noise_backward: impulse response too short"
                           : "filtered_noise_backward: shape needs %zu B of shared memory",
               smem);
  DDSP_REQUIRE(n_tiles < (1ll << 31), DDSP_B200_E_INVALID,
               "filtered_noise_backward: too many tiles");
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
  int rc = 0;
  if (d_audio) {
    const size_t smem = sizeof(float) * ((size_t)kFadjThreads + S - 1);
    dim3 grid((N + kFadjThreads - 1) / kFadjThreads, B);
    rc = launch(name, fir_adjoint_kernel, grid, kFadjThreads, smem, st, grad, ir, d_audio, N,
                S, frame, ir_batch == 1 ? 0 : F * S, start, out_len);
    if (rc) return rc;
  }
  if (d_ir) {
    FirDirParams p = fir_dir_params(audio, grad, B, N, F, S, frame, start, out_len);
    p.out = part ? part : d_ir;
    const size_t smem = fir_dir_smem(p);
    dim3 grid((unsigned)((p.n_rows + kDirRows - 1) / kDirRows),
              (unsigned)((S + kDirTaps - 1) / kDirTaps));
    rc = launch(name, fir_dir_kernel, grid, kDirThreads, smem, st, p);
    if (rc) return rc;
    if (part) {
      const long long n_out = (long long)ir_batch * F * S;
      rc = launch(name, fir_dir_reduce, grid_for(n_out, 256), 256, 0, st, part, d_ir, B, F, S,
                  p.n_chunk, ir_batch == 1 && B > 1, n_out);
    }
  }
  return rc;
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
  return launch("frequency_impulse_response_backward", ir_backward_kernel, (int)blocks,
                kIrThreads, smem, (cudaStream_t)stream, d_ir, d_mags, BF, g);
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

#ifdef DDSP_NR_TIMING
// measurement builds only (tools/noise_timing.py): the noise_ring phase counters of
// the last launch, [kMaxSMs CTAs][32 warps][8 phases] cycles (rows past the grid stay 0)
int ddsp_b200_debug_noise_timing(unsigned* host_out) {
  cudaError_t e = cudaMemcpyFromSymbol(host_out, ddsp::nr_::g_nr_timing,
                                       sizeof(unsigned) * kMaxSMs * 32 * 8);
  return e == cudaSuccess ? 0 : DDSP_B200_E_CUDA;
}
#endif

}  // extern "C"
