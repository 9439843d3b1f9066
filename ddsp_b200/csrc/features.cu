// C ABI of the feature family: framing, the spectral loss, loudness, RMS power,
// mel, log-mel and MFCC, forward and backward, and CREPE's frames, Viterbi path and f0.
#include "capi.cuh"
#include "spectral.cuh"
#include "spectral_terms.cuh"
#include "loudness.cuh"
#include "mel.cuh"
#include "crepe.cuh"

using namespace ddsp;

extern "C" {

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
  int rc = check_overlap("frame_window",
                         {DDSP_OUT(frames, extent(B, n_frames, frame_size))},
                         {DDSP_IN(audio, extent(B, N)),
                          DDSP_IN(window, extent(frame_size))});
  if (rc) return rc;
  if (B == 0) return 0;
  const long long quads = ((long long)n_frames * frame_size) / 4;
  dim3 grid((unsigned)((quads + 255) / 256), B);
  return launch("frame_window", frame_window_kernel, grid, 256, 0, (cudaStream_t)stream,
                audio, window, frames, N, n_frames, frame_size, frame_step);
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
  int rc = check_overlap("frame_window_adjoint", {DDSP_OUT(grad_audio, extent(B, N))},
                         {DDSP_IN(grad_frames, extent(B, n_frames, frame_size)),
                          DDSP_IN(window, extent(frame_size)),
                          DDSP_IN(scale_device, extent(1))});
  if (rc) return rc;
  if (B == 0) return 0;
  dim3 grid((N + 255) / 256, B);
  return launch("frame_window_adjoint", frame_window_adjoint_kernel, grid, 256, 0,
                (cudaStream_t)stream, grad_frames, window, grad_audio, N, n_frames,
                frame_size, frame_step, scale_device, accumulate);
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
  int rc = check_overlap("spectral_l1",
                         {DDSP_OUT(grad_value, extent(n_bins_total, 2), stft_value)},
                         {DDSP_IN(stft_target, extent(n_bins_total, 2)),
                          DDSP_IN(stft_value, extent(n_bins_total, 2))});
  if (rc) return rc;
  const long long blocks = std::min<long long>((n_bins_total / 2 + 255) / 256 + 1, 8ll * num_sms());
  return launch("spectral_l1", spectral_l1_kernel, (unsigned)blocks, 256, 0,
                (cudaStream_t)stream, reinterpret_cast<const float2*>(stft_target),
                reinterpret_cast<const float2*>(stft_value),
                reinterpret_cast<float2*>(grad_value), sums, n_bins_total, mag_weight,
                logmag_weight, 1.0f / (float)n_bins_total, 1e-5f, n_bins, irfft_size);
}

int ddsp_b200_spectral_terms(const float* stft_target, const float* stft_value,
                             float* grad_value, double* sums, int B, int T, int F, int terms,
                             int loss_type, float mag_weight, float delta_time_weight,
                             float delta_freq_weight, float cumsum_freq_weight,
                             float logmag_weight, void* stream) {
  DDSP_REQUIRE(stft_target && stft_value && grad_value && sums, DDSP_B200_E_INVALID,
               "spectral_terms: null pointer");
  DDSP_REQUIRE(B >= 0 && B <= 65535 && T >= 1 && F >= 2, DDSP_B200_E_INVALID,
               "spectral_terms: bad shape B=%d T=%d F=%d", B, T, F);
  DDSP_REQUIRE(terms >= 1 && terms <= st_::kAllTerms, DDSP_B200_E_INVALID,
               "spectral_terms: bad terms %d", terms);
  DDSP_REQUIRE(loss_type == DDSP_B200_LOSS_L1 || loss_type == DDSP_B200_LOSS_L2,
               DDSP_B200_E_INVALID, "spectral_terms: bad loss_type %d", loss_type);
  DDSP_REQUIRE((((uintptr_t)stft_target | (uintptr_t)stft_value | (uintptr_t)grad_value) & 7) == 0,
               DDSP_B200_E_INVALID, "spectral_terms: STFTs must be 8-byte aligned");
  const size_t bytes = sizeof(float2) * (size_t)B * T * F;
  DDSP_REQUIRE(!(terms & DDSP_B200_TERM_DELTA_TIME) ||
                   !(overlaps(grad_value, bytes, stft_target, bytes) ||
                     overlaps(grad_value, bytes, stft_value, bytes)),
               DDSP_B200_E_INVALID,
               "spectral_terms: with delta_time, grad_value must not overlap either STFT");
  DDSP_REQUIRE(F <= st_::kMaxBins, DDSP_B200_E_UNSUPPORTED,
               "spectral_terms: F=%d bins exceed the %d per frame supported", F, st_::kMaxBins);
  int rc = check_overlap("spectral_terms",
                         {DDSP_OUT(grad_value, extent(B, T, 2 * F), stft_target, stft_value)},
                         {DDSP_IN(stft_target, extent(B, T, 2 * F)),
                          DDSP_IN(stft_value, extent(B, T, 2 * F))});
  if (rc) return rc;
  if (B == 0) return 0;
  // per-term weight / element count; delta_time has none when T = 1
  const double counts[5] = {(double)B * T * F, (double)B * (T - 1) * F,
                            (double)B * T * (F - 1), (double)B * T * F, (double)B * T * F};
  const float weights[5] = {mag_weight, delta_time_weight, delta_freq_weight,
                            cumsum_freq_weight, logmag_weight};
  st_::Coeffs k;
  for (int j = 0; j < 5; ++j) k.c[j] = counts[j] > 0 ? (float)(weights[j] / counts[j]) : 0.f;
  const int rows = st_::tile_rows(T, F);
  const size_t smem = st_::tile_smem(rows, F, terms);
  st_::Kernel kern = st_::pick<1>(terms, loss_type == DDSP_B200_LOSS_L2);
  dim3 grid((unsigned)((T + rows - 1) / rows), B);
  return launch("spectral_terms", kern, grid, st_::kThreads, smem, (cudaStream_t)stream,
                reinterpret_cast<const float2*>(stft_target),
                reinterpret_cast<const float2*>(stft_value),
                reinterpret_cast<float2*>(grad_value), sums, T, F, rows, k);
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
  rc = check_overlap("loudness_forward", {DDSP_OUT(loudness, extent(B, n_frames))},
                     {DDSP_IN(audio, extent(B, N)),
                      DDSP_IN(weights, extent(n_fft / 2 + 1))});
  if (rc) return rc;
  p.audio = audio; p.weights = weights;
  db_params(&p, range_db, ref_db);
  const int warps = ld_warps(n_fft);
  int per_cta = 4 * warps;
  while (per_cta > 1 &&
         ld_fwd_smem(p.M, warps, (int64_t)(per_cta - 1) * hop + n_fft) > kMaxDynSmem)
    per_cta /= 2;
  const int span = (int)((int64_t)(per_cta - 1) * hop + n_fft);
  const size_t smem = ld_fwd_smem(p.M, warps, span);
  dim3 grid((unsigned)((n_frames + per_cta - 1) / per_cta), B);
  return launch("loudness_forward", ld_::loudness_kernel, grid, 32 * warps, smem,
                (cudaStream_t)stream, p, loudness, per_cta, span);
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
  dim3 grid((unsigned)((N + own - 1) / own), B);
  return launch("loudness_backward", ld_::loudness_backward_kernel, grid, 32 * warps, smem,
                (cudaStream_t)stream, p, grad_loudness, grad_audio, own);
}

int ddsp_b200_rms_power(const float* audio, float* power_db, int B, int N, int n_frames,
                        int frame_size, int hop, int padding, int in_db, float range_db,
                        float ref_db, void* stream) {
  DDSP_REQUIRE(audio && (power_db || n_frames == 0), DDSP_B200_E_INVALID,
               "rms_power: null pointer");
  int pad_left = 0;
  int rc = framing_check("rms_power", B, N, n_frames, frame_size, hop, padding, &pad_left);
  if (rc || B == 0 || n_frames == 0) return rc;
  rc = check_overlap("rms_power", {DDSP_OUT(power_db, extent(B, n_frames))},
                     {DDSP_IN(audio, extent(B, N))});
  if (rc) return rc;
  ld_::LoudParams d;
  db_params(&d, range_db, ref_db);
  const int64_t total = (int64_t)B * n_frames;
  return launch("rms_power", ld_::rms_power_kernel, grid_for(total * 32, ld_::kRmsThreads),
                ld_::kRmsThreads, 0, (cudaStream_t)stream, audio, power_db, N, n_frames,
                total, frame_size, hop, pad_left, in_db, d.pmin, d.range_db, d.ref_db);
}

// ---- CREPE: frames, Viterbi path, f0 and confidence ------------------------------
// The framing of losses.PretrainedCREPE.frame_audio (CENTER pads 512 zeros on both
// sides, VALID nothing; any hop, N >= 0); sets *pad_left.
static int crepe_loss_check(const char* name, int B, int N, int n_frames, int hop,
                            int padding, int* pad_left) {
  DDSP_REQUIRE(B >= 0 && N >= 0 && n_frames >= 0 && hop >= 1, DDSP_B200_E_INVALID,
               "%s: bad shape B=%d N=%d T=%d hop=%d", name, B, N, n_frames, hop);
  DDSP_REQUIRE(padding == DDSP_B200_PAD_VALID || padding == DDSP_B200_PAD_CENTER,
               DDSP_B200_E_INVALID, "%s: bad padding %d (CENTER or VALID)", name, padding);
  *pad_left = padding == DDSP_B200_PAD_CENTER ? crepe_::kFrame / 2 : 0;
  const long long padded = (long long)N + 2ll * *pad_left;
  const long long want = padded >= crepe_::kFrame ? 1 + (padded - crepe_::kFrame) / hop : 0;
  DDSP_REQUIRE(n_frames == want, DDSP_B200_E_INVALID, "%s: n_frames=%d, the padding gives %lld",
               name, n_frames, want);
  return 0;
}

static int crepe_loss_frames(const float* audio, float* frames, int B, int N, int n_frames,
                             int hop, int padding, void* stream) {
  int pad_left = 0;
  int rc = crepe_loss_check("crepe_frames", B, N, n_frames, hop, padding, &pad_left);
  if (rc) return rc;
  DDSP_REQUIRE((audio || N == 0 || B == 0) && (frames || n_frames == 0 || B == 0),
               DDSP_B200_E_INVALID, "crepe_frames: null pointer");
  if (B == 0 || n_frames == 0) return 0;
  rc = check_overlap("crepe_frames",
                     {DDSP_OUT(frames, extent(B, n_frames, crepe_::kFrame))},
                     {DDSP_IN(audio, extent(B, N))});
  if (rc) return rc;
  const int64_t total = (int64_t)B * n_frames;
  const int threads = 32 * crepe_::kFrameWarps;
  return launch("crepe_frames", crepe_::crepe_frames_kernel<true>,
                grid_for(total * 32, threads, 16), threads, 0, (cudaStream_t)stream, audio,
                frames, N, n_frames, total, hop, pad_left);
}

int ddsp_b200_crepe_frames(const float* audio, float* frames, int B, int N, int n_frames,
                           int hop, int padding, void* stream) {
  if (padding & DDSP_B200_CREPE_LOSS_FRAMES)
    return crepe_loss_frames(audio, frames, B, N, n_frames, hop,
                             padding & ~DDSP_B200_CREPE_LOSS_FRAMES, stream);
  DDSP_REQUIRE(audio && (frames || n_frames == 0 || B == 0), DDSP_B200_E_INVALID,
               "crepe_frames: null pointer");
  int pad_left = 0;
  // the kernel strides over all B * n_frames frames, so the batch has no grid limit
  // and is checked here alone
  DDSP_REQUIRE(B >= 0, DDSP_B200_E_INVALID, "crepe_frames: bad shape B=%d", B);
  int rc = framing_check("crepe_frames", B > 0, N, n_frames, crepe_::kFrame, hop, padding,
                         &pad_left);
  if (rc || B == 0 || n_frames == 0) return rc;
  rc = check_overlap("crepe_frames",
                     {DDSP_OUT(frames, extent(B, n_frames, crepe_::kFrame))},
                     {DDSP_IN(audio, extent(B, N))});
  if (rc) return rc;
  const int64_t total = (int64_t)B * n_frames;
  const int threads = 32 * crepe_::kFrameWarps;
  return launch("crepe_frames", crepe_::crepe_frames_kernel<false>,
                grid_for(total * 32, threads, 16), threads, 0, (cudaStream_t)stream, audio,
                frames, N, n_frames, total, hop, pad_left);
}

int ddsp_b200_crepe_frames_backward(const float* audio, const float* grad_frames,
                                    float* grad_audio, int B, int N, int n_frames, int hop,
                                    int padding, void* stream) {
  int pad_left = 0;
  int rc = crepe_loss_check("crepe_frames_backward", B, N, n_frames, hop,
                            padding & ~DDSP_B200_CREPE_LOSS_FRAMES, &pad_left);
  if (rc) return rc;
  DDSP_REQUIRE(B == 0 || N == 0 || (audio && grad_audio && (grad_frames || n_frames == 0)),
               DDSP_B200_E_INVALID, "crepe_frames_backward: null pointer");
  if (B == 0 || N == 0) return 0;
  rc = check_overlap("crepe_frames_backward", {DDSP_OUT(grad_audio, extent(B, N))},
                     {DDSP_IN(audio, extent(B, N)),
                      DDSP_IN(grad_frames, extent(B, n_frames, crepe_::kFrame))});
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  if (hop >= crepe_::kFrame && n_frames > 0) {
    const int64_t total = (int64_t)B * n_frames;
    const int threads = 32 * crepe_::kDisjointWarps;
    return launch("crepe_frames_backward", crepe_::crepe_frames_bwd_disjoint_kernel,
                  grid_for(total * 32, threads, 16), threads, 0, s, audio, grad_frames,
                  grad_audio, N, n_frames, total, hop, pad_left);
  }
  const int spans = (N + crepe_::kBwdOwn - 1) / crepe_::kBwdOwn;
  const int64_t total = (int64_t)B * spans;
  const size_t smem = sizeof(crepe_::FrameGrad) * crepe_::bwd_frames_per_span(hop);
  const int blocks = (int)std::min<int64_t>(total, 16ll * num_sms());
  return launch("crepe_frames_backward", crepe_::crepe_frames_bwd_overlap_kernel, blocks,
                crepe_::kBwdThreads, smem, s, audio, grad_frames, grad_audio, N, n_frames,
                spans, total, hop, pad_left);
}

size_t ddsp_b200_crepe_viterbi_workspace_bytes(int B, int T) {
  if (B <= 0 || T <= 1) return 0;
  return sizeof(uint32_t) * crepe_::kRecordWords * (size_t)B * (size_t)(T - 1);
}

int ddsp_b200_crepe_viterbi(const float* activations, int* centers, void* workspace,
                            size_t workspace_bytes, int B, int T, void* stream) {
  DDSP_REQUIRE(B >= 0 && T >= 1, DDSP_B200_E_INVALID, "crepe_viterbi: bad shape B=%d T=%d",
               B, T);
  DDSP_REQUIRE(B == 0 || (activations && centers), DDSP_B200_E_INVALID,
               "crepe_viterbi: null pointer");
  const size_t need = ddsp_b200_crepe_viterbi_workspace_bytes(B, T);
  DDSP_REQUIRE(workspace_bytes >= need && (need == 0 || workspace), DDSP_B200_E_WORKSPACE,
               "crepe_viterbi: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  DDSP_REQUIRE(((uintptr_t)workspace & 3) == 0, DDSP_B200_E_INVALID,
               "crepe_viterbi: workspace must be 4-byte aligned");
  if (B == 0) return 0;
  return launch("crepe_viterbi", crepe_::crepe_viterbi_kernel, B, crepe_::kThreads, 0,
                (cudaStream_t)stream, activations, centers, T,
                static_cast<uint32_t*>(workspace));
}

int ddsp_b200_crepe_decode(const float* activations, const int* centers, float* f0,
                           float* confidence, int64_t M, void* stream) {
  DDSP_REQUIRE(M >= 0, DDSP_B200_E_INVALID, "crepe_decode: bad shape M=%lld", (long long)M);
  DDSP_REQUIRE(M == 0 || (activations && f0 && confidence), DDSP_B200_E_INVALID,
               "crepe_decode: null pointer");
  if (M == 0) return 0;
  int rc = check_overlap("crepe_decode", {DDSP_OUT(f0, extent(M)),
                                          DDSP_OUT(confidence, extent(M))},
                         {DDSP_IN(activations, extent(M, DDSP_B200_CREPE_BINS))});
  if (rc) return rc;
  const int threads = 32 * crepe_::kDecodeWarps;
  return launch("crepe_decode", crepe_::crepe_decode_kernel, grid_for(M * 32, threads, 16),
                threads, 0, (cudaStream_t)stream, activations, centers, f0, confidence, M);
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
  rc = check_overlap("mel_forward", {DDSP_OUT(out, extent(B, n_frames, n_out))},
                     {DDSP_IN(audio, extent(B, N)), DDSP_IN(window, extent(fft_size))});
  if (rc) return rc;
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
  dim3 grid((unsigned)((n_frames + per_cta - 1) / per_cta), B);
  return launch("mel_forward", kern, grid, 32 * warps, smem, (cudaStream_t)stream, p, out,
                per_cta, span);
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
  dim3 grid((unsigned)((N + own - 1) / own), B);
  return launch("mel_backward", kern, grid, 32 * warps, smem, (cudaStream_t)stream, p,
                grad_out, grad_audio, own);
}

}  // extern "C"
