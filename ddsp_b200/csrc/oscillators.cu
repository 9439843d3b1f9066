// C ABI of the oscillator family: the oscillator bank, the harmonic oscillator bank,
// angular_cumsum, the sinusoidal and wavetable synthesizers and linear_lookup, forward and
// backward.
#include "capi.cuh"
#include "harmonic_bank.cuh"
#include "lookup.cuh"
#include "oscbank.cuh"
#include "sinusoidal.cuh"
#include "wavetable.cuh"

using namespace ddsp;

extern "C" {

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
  int rc = check_overlap("oscillator_bank",
                         {DDSP_OUT(out, extent(B, N, sum_sinusoids ? 1 : K))},
                         {DDSP_IN(frequency_envelopes, extent(B, N, K)),
                          DDSP_IN(amplitude_envelopes, extent(B, N, K))});
  if (rc) return rc;
  unsigned long long* sums = align256<unsigned long long>(workspace);
  const int n_chunks = (N + kObChunk - 1) / kObChunk;
  const double inv_sr = 1.0 / (double)sample_rate;
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(n_chunks, B);
  rc = launch("oscillator_bank(chunk sums)", oscbank_chunk_sums, grid, kObThreads, 0, st,
              frequency_envelopes, sums, N, K, n_chunks, inv_sr);
  if (rc) return rc;
  const int64_t BK = (int64_t)B * K;
  rc = launch("oscillator_bank(scan)", oscbank_scan_chunks,
              (int)((BK + kObThreads - 1) / kObThreads), kObThreads, 0, st, sums, K,
              n_chunks, BK);
  if (rc) return rc;
  auto apply = sum_sinusoids ? oscbank_apply<true> : oscbank_apply<false>;
  return launch("oscillator_bank(apply)", apply, grid, kObThreads, 0, st,
                frequency_envelopes, amplitude_envelopes, sums, out, N, K, n_chunks, inv_sr,
                sample_rate * 0.5f);
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
  return launch("oscillator_bank_backward", kernel, oscbank_backward_grid(B, K),
                kObbLanes * kObbWarps, 0, (cudaStream_t)stream, frequency_envelopes,
                amplitude_envelopes, grad, d_frequency_envelopes, d_amplitude_envelopes, N,
                K, 1.0 / (double)sample_rate, sample_rate * 0.5f,
                6.283185307179586 / (double)sample_rate);
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
    int rc = check_overlap("angular_cumsum", {DDSP_OUT(phase, extent(B, N, C))},
                           {DDSP_IN(angular_frequency, extent(B, N, C))});
    if (rc) return rc;
    const int64_t BC = (int64_t)B * C;
    return launch("angular_cumsum(tf_sequential)", tf_sequential_cumsum,
                  (int)((BC + 127) / 128), 128, 0, st, angular_frequency, nullptr, phase, B,
                  N, C, mode, chunk_size, 0, 1.0f);
  }
  DDSP_REQUIRE(B <= 65535, DDSP_B200_E_INVALID,
               "angular_cumsum: B=%d exceeds the 65535 grid limit", B);
  const size_t need = ddsp_b200_oscillator_bank_workspace(B, N, C);
  DDSP_REQUIRE(workspace != nullptr && workspace_bytes >= need, DDSP_B200_E_WORKSPACE,
               "angular_cumsum: workspace of %zu B needed, %zu given", need,
               workspace_bytes);
  int rc = check_overlap("angular_cumsum", {DDSP_OUT(phase, extent(B, N, C))},
                         {DDSP_IN(angular_frequency, extent(B, N, C))});
  if (rc) return rc;
  unsigned long long* sums = align256<unsigned long long>(workspace);
  const int n_chunks = (N + kObChunk - 1) / kObChunk;
  const double inv_two_pi = 0.15915494309189535;
  dim3 grid(n_chunks, B);
  rc = launch("angular_cumsum(chunk sums)", oscbank_chunk_sums, grid, kObThreads, 0, st,
              angular_frequency, sums, N, C, n_chunks, inv_two_pi);
  if (rc) return rc;
  const int64_t BK = (int64_t)B * C;
  rc = launch("angular_cumsum(scan)", oscbank_scan_chunks,
              (int)((BK + kObThreads - 1) / kObThreads), kObThreads, 0, st, sums, C,
              n_chunks, BK);
  if (rc) return rc;
  return launch("angular_cumsum(apply)", oscbank_phase_out, grid, kObThreads, 0, st,
                angular_frequency, sums, phase, N, C, n_chunks, inv_two_pi);
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
  return launch("angular_cumsum_backward", oscbank_backward<kObbCumsum>,
                oscbank_backward_grid(B, C), kObbLanes * kObbWarps, 0, (cudaStream_t)stream,
                nullptr, nullptr, grad, d_angular_frequency, nullptr, N, C, 0.0, 0.f, 1.0);
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
  int rc = check_overlap("oscillator_bank_tf_sequential", {DDSP_OUT(out, extent(B, N, K))},
                         {DDSP_IN(frequency_envelopes, extent(B, N, K)),
                          DDSP_IN(amplitude_envelopes, extent(B, N, K))});
  if (rc) return rc;
  if (B == 0) return 0;
  const int64_t BK = (int64_t)B * K;
  return launch("oscillator_bank_tf_sequential", tf_sequential_cumsum,
                (int)((BK + 127) / 128), 128, 0, (cudaStream_t)stream, frequency_envelopes,
                amplitude_envelopes, out, B, N, K, use_angular_cumsum ? 2 : 1, chunk_size,
                1, sample_rate);
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
  int rc = launch(name, sinus_tile_sums, dim3(n_tiles, B), kSfThreads, 0, st, frequencies,
                  sums, F, K, hop, FT, n_tiles, inv_sr);
  if (rc) return rc;
  const int64_t BK = (int64_t)B * K;
  return launch(name, oscbank_scan_chunks, (int)((BK + kObThreads - 1) / kObThreads),
                kObThreads, 0, st, sums, K, n_tiles, BK);
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
  rc = check_overlap("sinusoidal_forward", {DDSP_OUT(audio, extent(B, N))},
                     {DDSP_IN(frequencies, extent(B, F, K)),
                      DDSP_IN(amplitudes, extent(B, F, K))});
  if (rc) return rc;
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
  return launch("sinusoidal_forward(apply)", kern, dim3(n_tiles, B), kSfThreads, L.total,
                st, frequencies, amplitudes, sums, audio, F, K, N, hop, FT, n_tiles, inv_sr,
                sample_rate * 0.5f, accumulate);
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
  rc = launch("sinusoidal_backward(frames)", kern, n_blocks, kSbThreads, 0, st, frequencies,
              amplitudes, grad_audio, sums, part, F, K, N, hop, FT, n_tiles, BFK, inv_sr,
              sample_rate * 0.5f);
  if (rc) return rc;
  return launch("sinusoidal_backward(finalize)", sinus_bwd_finalize, dim3((K + 31) / 32, B),
                32 * kSfinWarps, 0, st, part, d_amplitudes, d_frequencies, F, K, hop, BFK,
                inv_sr);
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
  int rc = launch(name, wt_::wt_tile_sums, dim3(n_tiles, B), wt_::kFT, 0, st, f0, w.sums, F,
                  hop, n_tiles, sr);
  if (rc) return rc;
  rc = launch(name, oscbank_scan_chunks, (B + kObThreads - 1) / kObThreads, kObThreads, 0,
              st, w.sums, 1, n_tiles, (int64_t)B);
  if (rc) return rc;
  return launch(name, wt_::wt_frame_phase, dim3(n_tiles, B), wt_::kFT, 0, st, f0, w.sums,
                w.P, w.A, w.D, F, hop, n_tiles, sr);
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
  rc = check_overlap("wavetable_forward", {DDSP_OUT(audio, extent(B, N))},
                     {DDSP_IN(f0_hz, extent(B, F)), DDSP_IN(amplitudes, extent(B, F)),
                      DDSP_IN(wavetables, extent(B, Fw, W))});
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int hop = N / F;
  const WtPhase w = wt_phase_layout(workspace, B, F);
  rc = wt_frame_phases(w, f0_hz, B, F, hop, sample_rate, st, "wavetable_forward(phase)");
  if (rc) return rc;
  auto kern = amp_method == DDSP_B200_AMP_WINDOW ? wt_::wt_forward<true>
                                                 : wt_::wt_forward<false>;
  return launch("wavetable_forward", kern,
                dim3((unsigned)((N + wt_::kThreads - 1) / wt_::kThreads), B), wt_::kThreads,
                0, st, amplitudes, wavetables, w.P, w.A, w.D, audio, F, N, hop, Fw, W);
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
    rc = launch("wavetable_backward(frames)", kern, (unsigned)((BF + 31) / 32), kSbThreads,
                0, st, amplitudes, wavetables, grad_audio, w.P, w.A, w.D, part, F, N, hop,
                Fw, W, BF);
    if (rc) return rc;
    // K = 1; sinus_bwd_finalize always writes d amplitudes
    rc = launch("wavetable_backward(finalize)", sinus_bwd_finalize, dim3(1, B),
                32 * kSfinWarps, 0, st, part, d_amplitudes ? d_amplitudes : d_amp_scratch,
                d_f0, F, 1, hop, BF, 1.0 / (double)sample_rate);
    if (rc) return rc;
  }

  if (d_wavetables) {
    const int n_seg = wt_::table_segments(N, Fw);
    const size_t smem = wt_::table_smem_bytes(W);
    auto kern = window ? wt_::wt_bwd_table<true> : wt_::wt_bwd_table<false>;
    const unsigned gx = (unsigned)((int64_t)Fw * n_seg * wt_::table_col_tiles(W));
    rc = launch("wavetable_backward(wavetables)", kern, dim3(gx, B), wt_::kTabWarps * 32,
                smem, st, amplitudes, grad_audio, w.P, w.A, w.D,
                n_seg > 1 ? tab_part : d_wavetables, F, N, hop, Fw, W, n_seg);
    if (rc) return rc;
    if (n_seg > 1) {
      const int64_t RW = (int64_t)B * Fw * W;
      rc = launch("wavetable_backward(reduce)", wt_::wt_table_reduce, grid_for(RW, 256),
                  256, 0, st, tab_part, d_wavetables, RW, W, n_seg);
      if (rc) return rc;
    }
  }
  return 0;
}

// ---- core.harmonic_oscillator_bank (harmonic_bank.cuh) ----------------------------------
int ddsp_b200_harmonic_oscillator_bank_backward_takes(int B, int N, int K) {
  return B >= 0 && B <= 65535 && N >= 1 && K >= 1;
}

static int hob_check(const char* name, int B, int N, int K, float sample_rate) {
  DDSP_REQUIRE(B >= 0 && N >= 1 && K >= 1, DDSP_B200_E_INVALID,
               "%s: bad shape B=%d N=%d K=%d", name, B, N, K);
  DDSP_REQUIRE(sample_rate > 0.f, DDSP_B200_E_INVALID, "%s: sample_rate must be positive",
               name);
  return 0;
}

int ddsp_b200_harmonic_oscillator_bank(const float* frequency,
                                       const float* amplitude_envelopes,
                                       const float* initial_phase, float* audio,
                                       float* final_phase, int B, int N, int K,
                                       float sample_rate, int use_angular_cumsum,
                                       void* stream) {
  int rc = hob_check("harmonic_oscillator_bank", B, N, K, sample_rate);
  if (rc || B == 0) return rc;
  DDSP_REQUIRE(frequency && amplitude_envelopes && audio, DDSP_B200_E_INVALID,
               "harmonic_oscillator_bank: null pointer");
  rc = check_overlap("harmonic_oscillator_bank", {DDSP_OUT(audio, extent(B, N)),
                                                  DDSP_OUT(final_phase, extent(B))},
                     {DDSP_IN(frequency, extent(B, N)),
                      DDSP_IN(amplitude_envelopes, extent(B, N, K)),
                      DDSP_IN(initial_phase, extent(B))});
  if (rc) return rc;
  return launch("harmonic_oscillator_bank", hob_::hob_forward, dim3(B, hob_::n_spans(N)),
                hob_::kThreads, 0, (cudaStream_t)stream, frequency, amplitude_envelopes,
                initial_phase, audio, final_phase, N, K, 1.0 / (double)sample_rate,
                use_angular_cumsum ? 0 : 1);
}

int ddsp_b200_harmonic_oscillator_bank_backward(
    const float* frequency, const float* amplitude_envelopes, const float* initial_phase,
    const float* grad_audio, const float* grad_final_phase, float* d_frequency,
    float* d_amplitude_envelopes, float* d_initial_phase, int B, int N, int K,
    float sample_rate, void* stream) {
  int rc = hob_check("harmonic_oscillator_bank_backward", B, N, K, sample_rate);
  if (rc || B == 0) return rc;
  DDSP_REQUIRE(ddsp_b200_harmonic_oscillator_bank_backward_takes(B, N, K),
               DDSP_B200_E_UNSUPPORTED,
               "harmonic_oscillator_bank_backward: B=%d exceeds the 65535 clusters of its grid",
               B);
  DDSP_REQUIRE(frequency && amplitude_envelopes && grad_audio, DDSP_B200_E_INVALID,
               "harmonic_oscillator_bank_backward: null pointer");
  if (!d_frequency && !d_amplitude_envelopes && !d_initial_phase) return 0;
  return launch("harmonic_oscillator_bank_backward", hob_::hob_backward, dim3(hob_::kCl, B),
                hob_::kBwWarps * 32, 0, (cudaStream_t)stream, frequency,
                amplitude_envelopes, initial_phase, grad_audio, grad_final_phase,
                d_frequency, d_amplitude_envelopes, d_initial_phase, N, K,
                1.0 / (double)sample_rate, 6.283185307179586 / (double)sample_rate);
}

// ---- core.linear_lookup (lookup.cuh) -------------------------------------------------
static int ll_check(const char* name, int B, int N, int W, int per_sample) {
  DDSP_REQUIRE(B >= 0 && N >= 1 && W >= 1 && (per_sample == 0 || per_sample == 1),
               DDSP_B200_E_INVALID, "%s: bad shape B=%d N=%d W=%d per_sample=%d", name, B,
               N, W, per_sample);
  DDSP_REQUIRE(W <= DDSP_B200_LOOKUP_MAX_W, DDSP_B200_E_UNSUPPORTED,
               "%s: W=%d exceeds the %d wavetable columns supported", name, W,
               (int)DDSP_B200_LOOKUP_MAX_W);
  DDSP_REQUIRE((int64_t)B * N < (1ll << 31) * (int64_t)ll_::kThreads, DDSP_B200_E_INVALID,
               "%s: B=%d N=%d exceeds the grid limit", name, B, N);
  return 0;
}

int ddsp_b200_linear_lookup_forward(const float* phase, const float* wavetables, float* out,
                                    int B, int N, int W, int per_sample, void* stream) {
  DDSP_REQUIRE(phase && wavetables && out, DDSP_B200_E_INVALID,
               "linear_lookup_forward: null pointer");
  int rc = ll_check("linear_lookup_forward", B, N, W, per_sample);
  if (rc || B == 0) return rc;
  rc = check_overlap("linear_lookup_forward", {DDSP_OUT(out, extent(B, N))},
                     {DDSP_IN(phase, extent(B, N)),
                      DDSP_IN(wavetables, extent(B, per_sample ? N : 1, W))});
  if (rc) return rc;
  auto kern = per_sample ? ll_::ll_samples<true, false> : ll_::ll_samples<false, false>;
  const int64_t rows = (int64_t)B * N;
  return launch("linear_lookup_forward", kern,
                (unsigned)((rows + ll_::kThreads - 1) / ll_::kThreads), ll_::kThreads, 0,
                (cudaStream_t)stream, phase, wavetables, nullptr, out, rows, N, W);
}

int ddsp_b200_linear_lookup_backward(const float* phase, const float* wavetables,
                                     const float* grad, float* d_phase, float* d_wavetables,
                                     int B, int N, int W, int per_sample, void* stream) {
  DDSP_REQUIRE(phase && wavetables && grad, DDSP_B200_E_INVALID,
               "linear_lookup_backward: null pointer");
  int rc = ll_check("linear_lookup_backward", B, N, W, per_sample);
  if (rc || B == 0) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t rows = (int64_t)B * N;
  if (d_phase) {
    auto kern = per_sample ? ll_::ll_samples<true, true> : ll_::ll_samples<false, true>;
    rc = launch("linear_lookup_backward(phase)", kern,
                (unsigned)((rows + ll_::kThreads - 1) / ll_::kThreads), ll_::kThreads, 0,
                st, phase, wavetables, grad, d_phase, rows, N, W);
    if (rc) return rc;
  }
  if (!d_wavetables) return 0;
  if (per_sample) {
    return launch("linear_lookup_backward(wavetables)", ll_::ll_dtab_rows,
                  grid_for(rows * 32, ll_::kThreads), ll_::kThreads, 0, st, phase, grad,
                  d_wavetables, rows, W);
  }
  const size_t smem = wt_::table_smem_bytes(W);
  return launch("linear_lookup_backward(wavetables)", ll_::ll_dtab_items,
                dim3((unsigned)(ll_::kCl * wt_::table_col_tiles(W)), std::min(B, 65535)),
                wt_::kTabWarps * 32, smem, st, phase, grad, d_wavetables, B, N, W);
}

}  // extern "C"
