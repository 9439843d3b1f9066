// C ABI of the effects and routing family: windowed-sinc filters, the LTI FFT
// convolution, resample, Add, Mix, the exponential-decay impulse response and
// the modulated delay, forward and backward.
#include "capi.cuh"
#include "longconv.cuh"
#include "mod_delay.cuh"
#include "routing.cuh"
#include "sinc.cuh"

using namespace ddsp;

extern "C" {

// ---- windowed-sinc filters (csrc/sinc.cuh) --------------------------------------------
int ddsp_b200_sinc_impulse_response(const float* cutoff, float* ir, int64_t BF, int S,
                                    float scale, int high_pass, void* stream) {
  const char* name = "sinc_impulse_response";
  DDSP_REQUIRE(cutoff && ir, DDSP_B200_E_INVALID, "%s: null pointer", name);
  DDSP_REQUIRE(BF >= 0 && S >= 1 && (S & 1), DDSP_B200_E_INVALID,
               "%s: bad shape BF=%lld S=%d (S must be odd)", name, (long long)BF, S);
  DDSP_REQUIRE(BF < (1ll << 31), DDSP_B200_E_INVALID, "%s: too many frames", name);
  if (BF == 0) return 0;
  int rc = check_overlap(name, {DDSP_OUT(ir, extent(BF, S))},
                         {DDSP_IN(cutoff, extent(BF))});
  if (rc) return rc;
  return launch(name, sinc_ir_kernel, (unsigned)BF, kSincThreads, 0, (cudaStream_t)stream,
                cutoff, ir, S, scale, high_pass);
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
  return launch(name, sinc_ir_backward_kernel, (unsigned)BF, kSincThreads, 0,
                (cudaStream_t)stream, cutoff, d_ir, d_cutoff, S, scale, high_pass);
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
  rc = check_overlap(name, {DDSP_OUT(out, extent(B, out_len))},
                     {DDSP_IN(audio, extent(B, N)),
                      DDSP_IN(cutoff, extent(cutoff_batch, F))});
  if (rc) return rc;
  const size_t smem = sinc_filter_smem(S);
  SincFilterParams p;
  p.x = audio; p.cutoff = cutoff; p.out = out;
  p.N = N; p.F = F; p.frame = frame; p.S = S; p.cutoff_stride = cutoff_batch == 1 ? 0 : F;
  p.scale = scale; p.high_pass = high_pass ? 1 : 0; p.start = start; p.out_len = out_len;
  p.accumulate = accumulate ? 1 : 0;
  dim3 grid((out_len + kSincTile - 1) / kSincTile, B);
  return launch(name, sinc_filter_kernel, grid, kSincThreads, smem, (cudaStream_t)stream,
                p);
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
  auto kern = d_cutoff ? sinc_filter_backward_kernel<true> : sinc_filter_backward_kernel<false>;
  rc = launch(name, kern, dim3((unsigned)p.tiles, B), kSincThreads, smem, st, p);
  if (rc) return rc;
  if (part) {
    const long long n_out = (long long)cutoff_batch * F;
    rc = launch(name, sinc_dc_reduce, grid_for(n_out, 256), 256, 0, st, part, d_cutoff, B,
                F, p.n_seg, cutoff_batch == 1 && B > 1, n_out);
    if (rc) return rc;
  }
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
  int rc = launch("fft_convolve_lti(ir spectra)", lc::lc_fft_blocks, dim3(g.P, ir_batch),
                  lc::THREADS, 0, st, impulse_response, H, S, 0, g.P, 1,
                  (flags & DDSP_B200_LTI_REVERSE_IR) ? 1 : 0);
  if (rc) return rc;
  rc = launch("fft_convolve_lti(audio spectra)", lc::lc_fft_blocks, dim3(g.n_in, B),
              lc::THREADS, 0, st, audio, Z, N, g.n2, g.n_in, 0,
              (flags & DDSP_B200_LTI_REVERSE_AUDIO) ? 1 : 0);
  if (rc) return rc;
  // w blocks the crop reads: positions [start, start + out_len) through the real
  // half and [start - n2, start + out_len - n2) through the imaginary half
  const int lo_pos = std::max(0, start - g.n2);
  const int hi_pos = std::min(g.w_len, start + out_len);      // exclusive
  const int j_first = lo_pos / lc::L;
  const int j_last = std::min(g.n_out - 1, (hi_pos - 1) / lc::L);
  const int n_blocks = j_last - j_first + 1;
  rc = launch("fft_convolve_lti(multiply-accumulate + inverse)", lc::lc_mac_ifft,
              dim3((n_blocks + lc::JT - 1) / lc::JT, B), lc::THREADS, lc::kMacSmem, st, Z,
              H, W, g.n_in, g.P, g.n_out, ir_batch == 1 ? 0 : g.P * lc::M, j_first,
              n_blocks);
  if (rc) return rc;
  const int cgrid = std::min((out_len + 255) / 256, 8 * num_sms());
  return launch("fft_convolve_lti(combine)", lc::lc_combine, dim3(cgrid, B), 256, 0, st, W,
                out, g.n2, g.w_len, start, out_len, N + S - 1, accumulate, j_first * lc::L,
                (j_last + 1) * lc::L);
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
  int rc = check_overlap("resample", {DDSP_OUT(out, extent(B, N, C))},
                         {DDSP_IN(in, extent(B, F, C))});
  if (rc) return rc;
  if (B == 0) return 0;
  const int64_t total = (int64_t)B * N * C;
  return launch("resample", resample_kernel, grid_for(total, 256, 16), 256, 0,
                (cudaStream_t)stream, in, out, B, F, C, N, method, add_endpoint);
}

int ddsp_b200_add(const float* a, const float* b, float* out, int64_t n,
                  void* stream) {
  DDSP_REQUIRE(a && b && out, DDSP_B200_E_INVALID, "add: null pointer");
  DDSP_REQUIRE(n >= 0, DDSP_B200_E_INVALID, "add: n < 0");
  if (n == 0) return 0;
  int rc = check_overlap("add", {DDSP_OUT(out, extent(n), a, b)},
                         {DDSP_IN(a, extent(n)), DDSP_IN(b, extent(n))});
  if (rc) return rc;
  return launch("add", add_kernel, grid_for(n, 256), 256, 0, (cudaStream_t)stream, a, b,
                out, n);
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
  const int lanes = N >= 8 * F ? 32 : 1;   // long frames: a warp per frame
  auto kern = lanes == 32 ? rt_::resample_backward_kernel<32> : rt_::resample_backward_kernel<1>;
  return launch("resample_backward", kern, grid_for(total * lanes, rt_::kThreads, 16),
                rt_::kThreads, 0, (cudaStream_t)stream, grad_out, grad_in, B, C, g);
}

int ddsp_b200_mix_forward(const float* signal_one, const float* signal_two,
                          const float* mix_level, float* out, int B, int N, int C,
                          void* stream) {
  DDSP_REQUIRE(signal_one && signal_two && mix_level && out, DDSP_B200_E_INVALID,
               "mix_forward: null pointer");
  DDSP_REQUIRE(B >= 0 && N >= 1 && C >= 1, DDSP_B200_E_INVALID,
               "mix_forward: bad shape B=%d N=%d C=%d", B, N, C);
  int rc = check_overlap("mix_forward",
                         {DDSP_OUT(out, extent(B, N, C), signal_one, signal_two, mix_level)},
                         {DDSP_IN(signal_one, extent(B, N, C)),
                          DDSP_IN(signal_two, extent(B, N, C)),
                          DDSP_IN(mix_level, extent(B, N))});
  if (rc) return rc;
  if (B == 0) return 0;
  const int64_t total = (int64_t)B * N * C;
  return launch("mix_forward", rt_::mix_kernel, grid_for(total, rt_::kThreads),
                rt_::kThreads, 0, (cudaStream_t)stream, signal_one, signal_two, mix_level,
                out, (int64_t)B * N, C);
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
  return launch("mix_backward", rt_::mix_backward_kernel, grid_for(rows, rt_::kThreads),
                rt_::kThreads, 0, (cudaStream_t)stream, signal_one, signal_two, mix_level,
                grad_out, grad_signal_one, grad_signal_two, grad_mix_level, rows, C);
}

int ddsp_b200_exp_decay_ir(const float* gain, const float* decay, const float* noise,
                           uint64_t seed, uint64_t offset, float* ir, int rows, int L,
                           void* stream) {
  DDSP_REQUIRE(gain && decay && ir, DDSP_B200_E_INVALID, "exp_decay_ir: null pointer");
  DDSP_REQUIRE(rows >= 0 && L >= 1, DDSP_B200_E_INVALID,
               "exp_decay_ir: bad shape rows=%d L=%d", rows, L);
  int rc = check_overlap("exp_decay_ir", {DDSP_OUT(ir, extent(rows, L))},
                         {DDSP_IN(gain, extent(rows)), DDSP_IN(decay, extent(rows)),
                          DDSP_IN(noise, extent(L))});
  if (rc) return rc;
  if (rows == 0) return 0;
  const int64_t total = (int64_t)rows * ((L + 3) / 4);
  return launch("exp_decay_ir", rt_::exp_decay_ir_kernel, grid_for(total, rt_::kThreads),
                rt_::kThreads, 0, (cudaStream_t)stream, gain, decay, noise, seed, offset,
                ir, rows, L);
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
  return launch("exp_decay_ir_backward", rt_::exp_decay_ir_backward_kernel, rows,
                rt_::kIrBwdThreads, 0, (cudaStream_t)stream, gain, decay, noise, seed,
                offset, grad_ir, grad_gain, grad_decay, L);
}

// ---- modulated delay ----------------------------------------------------------
int ddsp_b200_mod_delay_forward(const float* audio, const float* phase, const float* gain,
                                float* out, int B, int N, int max_length, float scale,
                                float offset, int add_dry, void* stream) {
  DDSP_REQUIRE(audio && phase && out, DDSP_B200_E_INVALID, "mod_delay_forward: null pointer");
  DDSP_REQUIRE(B >= 0 && B <= 65535 && N >= 1 && max_length >= 1 && max_length < (1 << 29),
               DDSP_B200_E_INVALID, "mod_delay_forward: bad shape B=%d N=%d max_length=%d",
               B, N, max_length);
  int rc = check_overlap("mod_delay_forward", {DDSP_OUT(out, extent(B, N), phase, gain)},
                         {DDSP_IN(audio, extent(B, N)), DDSP_IN(phase, extent(B, N)),
                          DDSP_IN(gain, extent(B, N))});
  if (rc) return rc;
  if (B == 0) return 0;
  dim3 grid((unsigned)((N + md_::kThreads - 1) / md_::kThreads), B);
  return launch("mod_delay_forward", md_::mod_delay_forward_kernel, grid, md_::kThreads, 0,
                (cudaStream_t)stream, audio, phase, gain, out, N, max_length, scale, offset,
                add_dry);
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
  dim3 grid((unsigned)((N + md_::kTile - 1) / md_::kTile), B);
  return launch("mod_delay_backward", md_::mod_delay_backward_kernel, grid, md_::kThreads,
                smem, (cudaStream_t)stream, audio, phase, gain, grad_out, grad_audio,
                grad_gain, grad_phase, N, max_length, scale, offset, add_dry);
}

}  // extern "C"
