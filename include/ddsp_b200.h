/*
 * ddsp_b200.h - C ABI of libddsp_b200.so (hand-written sm_90a kernels for the
 * DDSP Harmonic + FilteredNoise decoder signal path).
 *
 * The reference (magenta/ddsp v3.7.0) has no FFI: its operator API is the Python
 * Processor / ProcessorGroup protocol (ddsp/processors.py:37-158).  Every entry
 * point below replaces one or more reference *functions*; the file:line each one
 * stands for is cited.  The Python layer in ddsp_b200/ binds these with ctypes
 * and re-creates the reference classes on top (see INTEGRATION.md).
 *
 * Conventions
 *   - All tensors are contiguous row-major float32 in DEVICE memory of the
 *     current CUDA device.  Controls are [B, F, C]; audio is [B, N].
 *   - The caller allocates every input, output and workspace.  The library never
 *     allocates, frees or retains a pointer past the call (one exception, with
 *     explicit create/destroy: ddsp_b200_host_pipeline and ddsp_b200_gru, below).
 *   - `stream` is a cudaStream_t passed as void*.  Calls are asynchronous and
 *     re-entrant; there is no global mutable state (the last-error string is
 *     thread-local).
 *   - Return value: 0 = ok, negative = DDSP_B200_E_* below.  Shape/argument
 *     errors are detected BEFORE any launch.
 *   - Aliasing: each forward entry point says which outputs may BE which inputs (the
 *     same pointer and extent) or may overlap them at all; every other overlap of a
 *     float output with a float input, partial ones included, is E_INVALID, after the
 *     other argument checks and before any launch.
 *   - The *_workspace, *_workspace_bytes, *_takes and ddsp_b200_ir_size queries
 *     are pure host functions: they launch nothing and set no error.
 *
 * The Python binding (ddsp_b200/_lib.py) is derived from this file at import:
 * every ddsp_b200_* prototype and every DDSP_B200_* integer constant.  A C type
 * it does not know stops the import, so a new type needs a line there.
 */
#ifndef DDSP_B200_H_
#define DDSP_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DDSP_B200_VERSION 200 /* 0.2.0 */

enum {
  DDSP_B200_OK = 0,
  DDSP_B200_E_INVALID = -1,   /* bad argument / shape (maps to ValueError)    */
  DDSP_B200_E_UNSUPPORTED = -2, /* valid in the reference, not built here yet */
  DDSP_B200_E_CUDA = -3,      /* CUDA runtime error (launch failed)           */
  DDSP_B200_E_WORKSPACE = -4  /* workspace too small                          */
};

/* amp_method: how frame-rate amplitudes become audio-rate (core.py:573-714). */
enum {
  DDSP_B200_AMP_WINDOW = 0,   /* upsample_with_windows, Hann OLA (default)    */
  DDSP_B200_AMP_LINEAR = 1    /* tf v1 bilinear, add_endpoint=True            */
};

/* phase_mode of the oscillator bank.  Both accumulate *wrapped* phase exactly
 * (64-bit fixed-point turns), i.e. the intent of core.angular_cumsum
 * (core.py:799-866); they differ only in how sin(k*phi) is evaluated. */
enum {
  DDSP_B200_PHASE_RECURRENCE = 0, /* Reinsch recurrence over harmonics (fast) */
  DDSP_B200_PHASE_DIRECT = 1      /* one sin per oscillator (validation)      */
};

/* flags of ddsp_b200_harmonic_controls */
enum {
  DDSP_B200_CTL_SCALE = 1,            /* apply exp_sigmoid (scale_fn)          */
  DDSP_B200_CTL_NYQUIST = 2           /* normalize_below_nyquist=True          */
};

/* padding of ddsp_b200_fir_time_varying (core.py:1338-1379); the framing entry points
 * (loudness, rms_power: spectral_ops.pad) also take CENTER */
enum { DDSP_B200_PAD_SAME = 0, DDSP_B200_PAD_VALID = 1, DDSP_B200_PAD_CENTER = 2 };

int ddsp_b200_version(void);
/* Thread-local description of the last non-zero return on this thread. */
const char* ddsp_b200_last_error(void);
/* Number of kernels this THREAD has launched through the library so far
 * (thread-local diagnostic counter; bench.py reports it as gpu_launches). */
uint64_t ddsp_b200_launch_count(void);

/* Harmonic.get_controls (synths.py:94-121): exp_sigmoid (core.py:386-404) on
 * amplitudes and harmonic_distribution, Nyquist mask + row normalisation
 * (core.normalize_harmonics, core.py:894-907; safe_divide core.py:207-210).
 * amps_in/out [B,F,1]; hd_in/out [B,F,K]; f0_hz [B,F,1].  amps_out may be amps_in
 * and hd_out may be hd_in (in place); neither may overlap another input. */
int ddsp_b200_harmonic_controls(const float* amps_in, const float* hd_in,
                                const float* f0_hz, float* amps_out,
                                float* hd_out, int B, int F, int K,
                                float sample_rate, int flags, void* stream);

/* Harmonic.get_signal = core.harmonic_synthesis (core.py:1048-1111) with
 * harmonic_shifts=None: get_harmonic_frequencies (1028-1045), resample 'linear'
 * of f0*k (573-642), resample amp*hd by amp_method (645-714), oscillator_bank
 * (911-962) incl. audio-rate remove_above_nyquist (869-891).
 * f0_hz [B,F,1], amps [B,F,1], hd [B,F,K] or NULL (K must be 1), audio [B,N].
 * N must be a multiple of F.  accumulate!=0: audio += result (fused Add).
 * audio must not overlap f0_hz, amps or hd. */
int ddsp_b200_harmonic_forward(const float* f0_hz, const float* amps,
                               const float* hd, float* audio, int B, int F,
                               int K, int N, float sample_rate, int amp_method,
                               int phase_mode, int accumulate, void* stream);

/* core.streaming_harmonic_synthesis after its normalize_harmonics call =
 * resample f0 ('linear') and amplitudes (amp_method) + harmonic_oscillator_bank
 * (core.py:1151-1163, 966-1025): phase = cumsum(omega) + initial_phase, harmonic
 * k uses k * phase, NO audio-rate Nyquist mask, and the phase after the last
 * sample is returned (wrapped cumsum in [0, 2 pi) + initial_phase, as
 * angular_cumsum gives).  hd must already be normalize_harmonics'ed
 * (ddsp_b200_harmonic_controls with DDSP_B200_CTL_NYQUIST only).
 * initial_phase [B] radians or NULL; final_phase [B] or NULL.  Neither audio nor
 * final_phase may overlap an input. */
int ddsp_b200_streaming_harmonic_forward(const float* f0_hz, const float* amps,
                                         const float* hd, const float* initial_phase,
                                         float* audio, float* final_phase, int B,
                                         int F, int K, int N, float sample_rate,
                                         int amp_method, void* stream);

/* FilteredNoise.get_controls (synths.py:165-179): exp_sigmoid(x + bias).  mag_out
 * may be mag_in (in place). */
int ddsp_b200_noise_controls(const float* mag_in, float* mag_out, int64_t n,
                             float initial_bias, int apply_scale, void* stream);

/* core.frequency_impulse_response + apply_window_to_impulse_response
 * (core.py:1534-1565, 1477-1531).  mags [BF, nb] -> ir [BF, S] with
 * S = ddsp_b200_ir_size(nb, window_size).  ir must not overlap mags. */
int ddsp_b200_ir_size(int nb, int window_size);
int ddsp_b200_frequency_impulse_response(const float* mags, float* ir,
                                         int64_t BF, int nb, int window_size,
                                         void* stream);

/* core.fft_convolve (core.py:1382-1473) restated as the equivalent direct-form
 * time-varying FIR (get_fft_size / rfft / irfft / overlap_and_add /
 * crop_and_compensate_delay folded into index math).  audio [B,N]; ir
 * [ir_batch(1 or B), F, S]; out [B, N] ('same') or [B, N+S-1] ('valid').
 * delay_compensation < 0 -> (S-1)/2 - 1 as in the reference.
 * accumulate!=0: out += result.  out must not overlap audio or ir. */
int ddsp_b200_fir_time_varying(const float* audio, const float* ir, float* out,
                               int B, int N, int F, int S, int ir_batch,
                               int padding, int delay_compensation,
                               int accumulate, void* stream);

/* Uniform noise in [-1, 1): Philox4x32-10, counter = (i/4, b, offset), key =
 * seed.  Stands in for tf.random.uniform at synths.py:192-193. out [B,N]. */
int ddsp_b200_uniform_noise(float* out, int B, int N, uint64_t seed,
                            uint64_t offset, void* stream);

/* FilteredNoise.get_signal (synths.py:181-196) = noise -> frequency_filter
 * (core.py:1628-1655), fused: IRs are built in shared memory, never in HBM.
 * mags [B,F,nb]; noise [B,N] or NULL (NULL: in-kernel Philox(seed, offset));
 * audio [B,N].  accumulate!=0: audio += result (the fused processors.Add,
 * processors.py:174-176).  workspace: ddsp_b200_filtered_noise_workspace()
 * bytes (0 for the fused path; may be NULL then).  audio must not overlap mags or
 * noise. */
size_t ddsp_b200_filtered_noise_workspace(int B, int F, int nb, int N,
                                          int window_size);
int ddsp_b200_filtered_noise_forward(const float* mags, const float* noise,
                                     uint64_t seed, uint64_t offset,
                                     float* audio, int B, int F, int nb, int N,
                                     int window_size, int accumulate,
                                     void* workspace, size_t workspace_bytes,
                                     void* stream);

/* The whole `ae.gin` decoder (ae.gin:47-72) from RAW network outputs in two
 * launches: ProcessorGroup.__call__ (processors.py:121-131) for the DAG
 * Harmonic -> FilteredNoise -> Add with scale_fn = exp_sigmoid.  Both
 * get_controls (synths.py:94-121, 165-179) are applied while the frame tiles
 * are staged in shared memory (controls never reach HBM), the noise kernel adds
 * into the harmonic audio (processors.py:174-176).  harmonic_flags:
 * DDSP_B200_CTL_SCALE | DDSP_B200_CTL_NYQUIST as in harmonic_controls.
 * Returns DDSP_B200_E_UNSUPPORTED outside the decoder regime (hop % 64 == 0,
 * n_frequencies <= 80); callers then use the per-processor entry points.
 * audio must not overlap an input. */
int ddsp_b200_decoder_forward(const float* amps_raw, const float* hd_raw,
                              const float* f0_hz, const float* mags_raw,
                              const float* noise, uint64_t seed, uint64_t offset,
                              float* audio, int B, int F, int K, int nb, int N,
                              float sample_rate, int amp_method,
                              int harmonic_flags, int window_size,
                              float initial_bias, void* stream);

/* The same decoder for HOST buffers - what a caller of the reference's
 * ProcessorGroup.__call__ holds when its network outputs are numpy arrays
 * (processors_test.py:35-42) and it wants numpy audio back.  The batch is cut
 * into at most n_chunks groups of items whose sizes halve (16, 8, 4, 4 of 32:
 * the tail of the call is the last chunk's compute + copy-out, so it is kept
 * small); chunk c's host->device copies, its two kernels and its device->host
 * audio copy run on three streams and overlap with the neighbouring chunks', so
 * the call costs about max(H2D, compute, D2H) instead of their sum.  Results are identical to ddsp_b200_decoder_forward on the whole
 * batch (the Philox item index of a chunk's rows is offset accordingly).
 *
 * The pipeline handle owns one device staging allocation for max_B items of
 * shape (F, K, nb, N), two copy streams and the events - with ddsp_b200_gru, the only objects this
 * library ever allocates; *_destroy releases them.  A handle belongs to the
 * device that was current at creation and serialises its own calls.
 * amps_raw/f0_hz [B,F,1], hd_raw [B,F,K], mags_raw [B,F,nb], audio [B,N]: HOST
 * pointers, pinned (cudaHostAlloc / cudaHostRegister) for the copies to be
 * asynchronous.  The call returns once everything is queued; `stream` completes
 * when the audio is in host memory. */
typedef struct ddsp_b200_host_pipeline ddsp_b200_host_pipeline;
int ddsp_b200_host_pipeline_create(ddsp_b200_host_pipeline** out, int max_B, int F,
                                   int K, int nb, int N, int max_chunks);
int ddsp_b200_host_pipeline_destroy(ddsp_b200_host_pipeline* pipeline);
int ddsp_b200_decoder_forward_host(ddsp_b200_host_pipeline* pipeline,
                                   const float* amps_raw, const float* hd_raw,
                                   const float* f0_hz, const float* mags_raw,
                                   uint64_t seed, uint64_t offset, float* audio,
                                   int B, int n_chunks, float sample_rate,
                                   int amp_method, int harmonic_flags,
                                   int window_size, float initial_bias,
                                   void* stream);

/* Backward of Harmonic.get_signal w.r.t. the frame-rate harmonic amplitudes
 * ha = amplitudes * harmonic_distribution (the transpose of core.py:1096-1111;
 * the reference gets it from TF autodiff).  grad_audio [B,N] -> g0, g1 [B,F,K]:
 *   g0[i,k] = sum_{t in frame i} grad(t) w0(r) m_k(t) sin(k phi(t)),  g1 with w1;
 *   dL/dha[i,k] = g0[i,k] + g1[i-1,k] (+ g1[F-1,k] when i == F-1).
 * The frame-rate recombination is left to the caller.  d f0 is not built.
 * Shapes beyond ddsp_b200_harmonic_backward_takes(B, F, N) are E_UNSUPPORTED: it is
 * 1 for a hop N / F that is a multiple of 64 up to 8192 and B <= 65535, else 0. */
int ddsp_b200_harmonic_backward_takes(int B, int F, int N);
int ddsp_b200_harmonic_backward(const float* f0_hz, const float* grad_audio,
                                float* g0, float* g1, int B, int F, int K, int N,
                                float sample_rate, int amp_method, void* stream);

/* d f0 of core.harmonic_synthesis (what the reference gets from TF autodiff through
 * the phase cumsum, core.py:947-958; needed by models/inverse_synthesis.py:84-117).
 * f0_hz, amps [B,F,1], hd [B,F,K] are synthesizer CONTROLS; grad_audio [B,N] ->
 * d_f0 [B,F].  workspace: 12 * B * F bytes (per-frame partial sums). */
int ddsp_b200_harmonic_backward_f0(const float* f0_hz, const float* amps,
                                   const float* hd, const float* grad_audio,
                                   float* d_f0, int B, int F, int K, int N,
                                   float sample_rate, int amp_method,
                                   void* workspace, size_t workspace_bytes,
                                   void* stream);

/* Backward of Harmonic.get_controls (synths.py:94-121) fused with the frame-rate
 * recombination of ddsp_b200_harmonic_backward's g0 / g1: from the RAW network
 * outputs (amps_raw [B,F,1], hd_raw [B,F,K]) and f0_hz to d amps_raw, d hd_raw -
 * exp_sigmoid' (core.py:386-404), the Nyquist mask and the row normalisation
 * (core.py:894-907, 207-210) transposed.  flags as ddsp_b200_harmonic_controls. */
int ddsp_b200_harmonic_controls_backward(const float* amps_raw, const float* hd_raw,
                                         const float* f0_hz, const float* g0,
                                         const float* g1, float* d_amps_raw,
                                         float* d_hd_raw, int B, int F, int K,
                                         float sample_rate, int flags, void* stream);

/* The vector-Jacobian product of Harmonic.get_controls (synths.py:94-121) for ANY
 * upstream gradient: d_amplitudes [B,F,1] on the scaled amplitudes and d_hd [B,F,K] on
 * the normalised harmonic distribution - what a loss on the controls themselves
 * produces, summed with the synthesizer's own gradient.  Either may be NULL: zeros,
 * and not read.  From the RAW inputs amps_raw [B,F,1], hd_raw [B,F,K] and f0_hz
 * [B,F,1] to d_amps_raw [B,F,1] and d_hd_raw [B,F,K], every element written.
 * flags as ddsp_b200_harmonic_controls (without DDSP_B200_CTL_SCALE the inputs are
 * already scaled and only the mask and the normalisation are transposed).  f0_hz gets
 * no gradient: the Nyquist mask is piecewise constant.  One launch. */
int ddsp_b200_harmonic_controls_vjp(const float* amps_raw, const float* hd_raw,
                                    const float* f0_hz, const float* d_amplitudes,
                                    const float* d_hd, float* d_amps_raw, float* d_hd_raw,
                                    int B, int F, int K, float sample_rate, int flags,
                                    void* stream);

/* Backward of FilteredNoise.get_controls (synths.py:165-179):
 * d raw = d magnitudes * exp_sigmoid'(raw + initial_bias), n elements. */
int ddsp_b200_noise_controls_backward(const float* mags_raw, const float* d_mags,
                                      float* d_raw, int64_t n, float initial_bias,
                                      void* stream);

/* Backward of FilteredNoise.get_signal w.r.t. magnitudes (controls): the
 * transpose of core.frequency_filter (core.py:1628-1655) for the same noise
 * (caller-supplied, or the Philox stream of (seed, offset)).
 * grad_audio [B,N] -> dmags [B,F,nb].  Shapes beyond
 * ddsp_b200_filtered_noise_backward_takes(F, nb, N, window_size) are E_UNSUPPORTED: it
 * is 1 for a valid shape whose impulse response has at least 3 taps and whose tiles of
 * 32 frames (noise, gradient and taps) fit one CTA's shared memory, else 0. */
int ddsp_b200_filtered_noise_backward_takes(int F, int nb, int N, int window_size);
int ddsp_b200_filtered_noise_backward(const float* grad_audio, const float* noise,
                                      uint64_t seed, uint64_t offset, float* dmags,
                                      int B, int F, int nb, int N, int window_size,
                                      void* stream);

/* Backward of ddsp_b200_fir_time_varying for the upstream gradient grad [B, out_len]
 * (out_len = N for 'same', N+S-1 for 'valid'): d_audio [B,N] and d_ir
 * [ir_batch,F,S], each skipped when NULL.  A shared impulse response (ir_batch 1)
 * gets the sum over the batch.  Same arguments, checks and status codes as the
 * forward (E_UNSUPPORTED for a negative automatic delay).  No atomics: both
 * gradients are bit-reproducible.  workspace: ddsp_b200_fir_time_varying_backward_
 * workspace(B,N,F,S,ir_batch) bytes (needed only when d_ir is set; 0 when every
 * frame is at most 256 samples and the impulse responses are per item). */
size_t ddsp_b200_fir_time_varying_backward_workspace(int B, int N, int F, int S,
                                                     int ir_batch);
int ddsp_b200_fir_time_varying_backward(const float* audio, const float* ir,
                                        const float* grad, float* d_audio, float* d_ir,
                                        int B, int N, int F, int S, int ir_batch,
                                        int padding, int delay_compensation,
                                        void* workspace, size_t workspace_bytes,
                                        void* stream);

/* Backward of ddsp_b200_frequency_impulse_response: d_ir [BF, S] -> d_mags [BF, nb].
 * Same limits as the forward (nb <= 5120). */
int ddsp_b200_frequency_impulse_response_backward(const float* d_ir, float* d_mags,
                                                  int64_t BF, int nb, int window_size,
                                                  void* stream);

/* Backward of core.frequency_filter (core.py:1628-1655): audio [B,N], the forward's
 * impulse responses ir [mags_batch,F,S] and grad [B, out_len] -> d_audio [B,N] and
 * d_mags [mags_batch,F,nb], each skipped when NULL (shared magnitudes, mags_batch 1,
 * get the sum over the batch).  d_mags takes the fused filtered-noise backward kernel
 * (the audio as its noise) for 'same' padding and per-item magnitudes when the shape
 * fits it, and d IR plus the IR adjoint through the workspace otherwise.
 * workspace: ddsp_b200_frequency_filter_backward_workspace(...) bytes (needed only
 * when d_mags is set; 0 on the fused route). */
size_t ddsp_b200_frequency_filter_backward_workspace(int B, int F, int nb, int N,
                                                     int mags_batch, int window_size,
                                                     int padding);
int ddsp_b200_frequency_filter_backward(const float* audio, const float* ir,
                                        const float* grad, float* d_audio, float* d_mags,
                                        int B, int F, int nb, int N, int mags_batch,
                                        int window_size, int padding, void* workspace,
                                        size_t workspace_bytes, void* stream);

/* core.sinc_impulse_response (core.py:1576-1625): cutoff [BF] -> ir [BF, S] for
 * S = 2 (window_size / 2) + 1 taps (odd).  The cutoff is multiplied by `scale` in
 * float32 first (1, or float32(2 / sample_rate)); high_pass != 0 gives delta - h.
 * ir must not overlap cutoff. */
int ddsp_b200_sinc_impulse_response(const float* cutoff, float* ir, int64_t BF, int S,
                                    float scale, int high_pass, void* stream);
/* Its backward: d_ir [BF, S] -> d_cutoff [BF] (the gradient of the unscaled cutoff). */
int ddsp_b200_sinc_impulse_response_backward(const float* cutoff, const float* d_ir,
                                             float* d_cutoff, int64_t BF, int S, float scale,
                                             int high_pass, void* stream);

/* core.sinc_filter (core.py:1658-1690) fused: fft_convolve of audio [B,N] with the
 * sinc impulse responses of cutoff [cutoff_batch, F] (cutoff_batch 1 or B), automatic
 * delay compensation, taps built in shared memory and never stored.  out [B, N] for
 * 'same', [B, N+S-1] for 'valid'; accumulate != 0: out += result.  The reference's
 * errors for batch, frames and padding; E_UNSUPPORTED for S < 3 (an empty crop) and
 * S >= 2048.  out must not overlap audio or cutoff. */
int ddsp_b200_sinc_filter(const float* audio, const float* cutoff, float* out, int B, int N,
                          int F, int S, int cutoff_batch, float scale, int high_pass,
                          int padding, int accumulate, void* stream);
/* Backward of ddsp_b200_sinc_filter for grad [B, out_len]: d_audio [B,N] and d_cutoff
 * [cutoff_batch, F], each skipped when NULL; a shared cutoff gets the sum over the
 * batch.  Same checks as the forward.  No atomics: both gradients are bit-reproducible.
 * workspace: ddsp_b200_sinc_filter_backward_workspace(B,N,F,S,cutoff_batch) bytes
 * (needed only when d_cutoff is set; 0 when frames are at most 1024 samples and the
 * cutoffs are per item). */
size_t ddsp_b200_sinc_filter_backward_workspace(int B, int N, int F, int S, int cutoff_batch);
int ddsp_b200_sinc_filter_backward(const float* audio, const float* cutoff, const float* grad,
                                   float* d_audio, float* d_cutoff, int B, int N, int F,
                                   int S, int cutoff_batch, float scale, int high_pass,
                                   int padding, void* workspace, size_t workspace_bytes,
                                   void* stream);

/* core.oscillator_bank (core.py:911-962) on audio-rate envelopes [B,N,K]:
 * Nyquist mask, exact wrapped phase accumulation (three-pass chunked scan in
 * 64-bit fixed point), amp * sin(phase), summed over k when sum_sinusoids != 0
 * (out [B,N]) or not (out [B,N,K]).  workspace: *_workspace(B,N,K) bytes.
 * out must not overlap either envelope. */
size_t ddsp_b200_oscillator_bank_workspace(int B, int N, int K);
int ddsp_b200_oscillator_bank(const float* frequency_envelopes,
                              const float* amplitude_envelopes, float* out, int B,
                              int N, int K, float sample_rate, int sum_sinusoids,
                              void* workspace, size_t workspace_bytes,
                              void* stream);
/* Backward of ddsp_b200_oscillator_bank for grad [B,N] (sum_sinusoids = 1) or [B,N,K]
 * (0): TensorFlow's gradients of core.py:911-962.  With m = [f < sr/2] (the forward's
 * float32 mask, which passes no gradient) and phi_t = (2 pi / sr) sum_{u<=t} f_u (the
 * forward's exact phase, bit for bit):
 *   d_amplitude_envelopes[t,k] = g m sin(phi_t),
 *   d_frequency_envelopes[t,k] = (2 pi / sr) sum_{u>=t} g_u a_u m_u cos(phi_u)
 * (the suffix summed in double, rounded once).  use_angular_cumsum does not change the
 * gradient.  Each gradient is skipped when its pointer is NULL (d_frequency_envelopes =
 * NULL skips the suffix scan and the cosine); d_amplitude_envelopes does not depend on
 * whether d_frequency_envelopes is asked for.  No workspace and no atomics: one
 * thread-block cluster per (b, 32 oscillators) exchanges segment totals in distributed
 * shared memory, so both gradients are bit-reproducible.  Checks as the forward's, plus
 * sum_sinusoids in {0, 1}; B, N or K = 0 is a no-op (NULL pointers allowed then). */
int ddsp_b200_oscillator_bank_backward(const float* frequency_envelopes,
                                       const float* amplitude_envelopes, const float* grad,
                                       float* d_frequency_envelopes,
                                       float* d_amplitude_envelopes, int B, int N, int K,
                                       float sample_rate, int sum_sinusoids, void* stream);

/* core.fft_convolve (core.py:1382-1473) with ONE impulse response per item of any
 * length (the LTI case: effects.Reverb, effects.py:103-117, 48000 taps): uniformly
 * partitioned overlap-save convolution, 1024-sample blocks, hand-written 2048-point
 * FFTs.  audio [B,N], impulse_response [ir_batch (1 or B), S] -> out [B,out_len] =
 * full convolution [start, start + out_len) (crop_and_compensate_delay,
 * core.py:1338-1379; start + out_len <= N + S - 1).  workspace:
 * ddsp_b200_fft_convolve_lti_workspace(B, N, S, ir_batch) bytes.
 * flags: DDSP_B200_LTI_REVERSE_AUDIO / _IR read that operand back to front - the
 * backward pass is the same convolution on time-reversed signals:
 *   d audio = (g * reverse(ir)) [S-1-start, +N),  d ir = (g * reverse(audio)) [N-1-start, +S).
 * out may overlap audio or impulse_response in any way: both are transformed into the
 * workspace by launches that end before out is written. */
enum { DDSP_B200_LTI_REVERSE_AUDIO = 1, DDSP_B200_LTI_REVERSE_IR = 2 };
size_t ddsp_b200_fft_convolve_lti_workspace(int B, int N, int S, int ir_batch);
int ddsp_b200_fft_convolve_lti(const float* audio, const float* impulse_response,
                               float* out, int B, int N, int S, int ir_batch,
                               int start, int out_len, int accumulate, int flags,
                               void* workspace, size_t workspace_bytes, void* stream);

/* core.angular_cumsum (core.py:799-866) and tf.cumsum (core.py:955) on
 * [B,N,C] float32 (C = product of the trailing axes).  mode:
 *   0  exact: the wrapped running sum in 64-bit fixed point (what angular_cumsum
 *      approximates), radians in [0, 2 pi); three-pass scan, workspace =
 *      ddsp_b200_oscillator_bank_workspace(B,N,C) bytes;
 *   1  tf_sequential, tf.cumsum: float32 running sum in the reference's order;
 *   2  tf_sequential, angular_cumsum: float32, chunked by chunk_size with the
 *      reference's mod-2pi stitching (debug mode: reproduces TensorFlow's own
 *      float32 error, one thread per (b, c) - small shapes).
 * phase must not overlap angular_frequency.
 * ddsp_b200_oscillator_bank_tf_sequential is core.oscillator_bank evaluated that
 * way end to end (omega = f * 2pi / sr in float32, modes 1 / 2, Nyquist mask,
 * amp * sin(phase)); out is [B,N,K], the sum over k is left to the caller.  Its out
 * must not overlap either envelope. */
int ddsp_b200_angular_cumsum(const float* angular_frequency, float* phase, int B,
                             int N, int C, int chunk_size, int mode,
                             void* workspace, size_t workspace_bytes, void* stream);
/* Backward of ddsp_b200_angular_cumsum (mode 0) for grad [B,N,C]: floormod has
 * derivative 1, so d_angular_frequency[t] = sum_{u>=t} grad[u] along N, summed in
 * double and rounded once.  No workspace, no atomics (the oscillator-bank backward's
 * cluster scan); B, N or C = 0 is a no-op (NULL pointers allowed then). */
int ddsp_b200_angular_cumsum_backward(const float* grad, float* d_angular_frequency, int B,
                                      int N, int C, void* stream);
int ddsp_b200_oscillator_bank_tf_sequential(const float* frequency_envelopes,
                                            const float* amplitude_envelopes,
                                            float* out, int B, int N, int K,
                                            float sample_rate, int use_angular_cumsum,
                                            int chunk_size, void* stream);

/* core.harmonic_oscillator_bank (core.py:966-1025): frequency [B,N] (Hz, one f0 per
 * sample), amplitude_envelopes [B,N,K], initial_phase [B] radians or NULL (0) ->
 * audio [B,N] = sum_k a[t,k] sin(k phi_t), phi_t = initial_phase + (2 pi / sr) sum_{u<=t}
 * f_u, with no Nyquist mask.  The phase is accumulated exactly in 64-bit fixed-point turns
 * (one scan per item) and harmonic k's is the wrapping product k phi.  final_phase [B] (or
 * NULL) is phi after the last sample: with use_angular_cumsum != 0 the wrapped sum in
 * [0, 2 pi) plus initial_phase, else the unwrapped sum (accumulated exactly, rounded once)
 * plus initial_phase.  The audio does not depend on use_angular_cumsum.  B = 0 is a no-op.
 * No workspace.  Neither audio nor final_phase may overlap an input. */
int ddsp_b200_harmonic_oscillator_bank(const float* frequency,
                                       const float* amplitude_envelopes,
                                       const float* initial_phase, float* audio,
                                       float* final_phase, int B, int N, int K,
                                       float sample_rate, int use_angular_cumsum,
                                       void* stream);
/* Its backward for grad_audio [B,N] and grad_final_phase [B] (NULL: 0).  With
 * c_t = g_t sum_k k a[t,k] cos(k phi_t) on the forward's exact phase:
 *   d_amplitude_envelopes[t,k] = g_t sin(k phi_t),
 *   d_frequency[t] = (2 pi / sr) (sum_{u>=t} c_u + g_phi),
 *   d_initial_phase = sum_u c_u + g_phi
 * (floormod passes gradient 1; the sums in double in a fixed order, rounded once).  A NULL
 * output is not computed; without d_frequency and d_initial_phase there is no cosine and no
 * suffix scan.  No atomics: bit-reproducible.  Checks as the forward's.
 * The forward takes any B; the backward runs one thread-block cluster per item and takes
 * B <= 65535 (more is E_UNSUPPORTED):
 * ddsp_b200_harmonic_oscillator_bank_backward_takes(B, N, K) says whether a shape is taken.
 * No workspace: one thread-block cluster per item exchanges segment totals. */
int ddsp_b200_harmonic_oscillator_bank_backward_takes(int B, int N, int K);
int ddsp_b200_harmonic_oscillator_bank_backward(
    const float* frequency, const float* amplitude_envelopes, const float* initial_phase,
    const float* grad_audio, const float* grad_final_phase, float* d_frequency,
    float* d_amplitude_envelopes, float* d_initial_phase, int B, int N, int K,
    float sample_rate, void* stream);

/* Frame-rate oscillator bank with per-sinusoid frequencies: the fusion of
 * resample(frequencies) + resample(amplitudes, amp_method) + oscillator_bank
 * for synths.Sinusoidal.get_signal (synths.py:305-323) and for
 * core.harmonic_synthesis with harmonic_shifts (core.py:1084-1111; the caller
 * forms f0 * k * (1 + shifts) and amp * hd at frame rate, as the reference does).
 * frequencies, amplitudes [B,F,K] -> audio [B,N] (summed over k), N % F == 0.
 * workspace: ddsp_b200_sinusoidal_workspace(B,F,K) bytes.  audio must not overlap
 * frequencies or amplitudes. */
size_t ddsp_b200_sinusoidal_workspace(int B, int F, int K);
int ddsp_b200_sinusoidal_forward(const float* frequencies, const float* amplitudes,
                                 float* audio, int B, int F, int K, int N,
                                 float sample_rate, int amp_method, int accumulate,
                                 void* workspace, size_t workspace_bytes,
                                 void* stream);

/* Its backward: for the upstream gradient grad_audio [B,N], writes
 * d_amplitudes [B,F,K] and, when d_frequencies [B,F,K] is not NULL, the
 * gradient to the frequencies through the phase (a NULL d_frequencies skips
 * the phase path: no cos, no phase sums, no frame scan).  The Nyquist mask is
 * the forward's own float32 decision with subgradient 0, as tf.where gives.
 * Same validation and error codes as the forward.  No atomics: the gradients
 * are bit-reproducible.
 * workspace: ddsp_b200_sinusoidal_backward_workspace(B,F,K) bytes. */
size_t ddsp_b200_sinusoidal_backward_workspace(int B, int F, int K);
int ddsp_b200_sinusoidal_backward(const float* frequencies, const float* amplitudes,
                                  const float* grad_audio, float* d_frequencies,
                                  float* d_amplitudes, int B, int F, int K, int N,
                                  float sample_rate, int amp_method, void* workspace,
                                  size_t workspace_bytes, void* stream);

/* core.resample / core.upsample_with_windows (core.py:573-714) stand-alone:
 * in [B,F,C] -> out [B,N,C].  method: 0 'window', 1 'linear', 2 'nearest',
 * 3 'cubic' (tf.compat.v1 bicubic, Keys A = -0.75).  add_endpoint as in the
 * reference.  4-D inputs [B,F,n_freq,C] are the 3-D case with n_freq*C channels
 * (the reference resizes the n_freq axis to itself, core.py:616-621).  out must not
 * overlap in. */
int ddsp_b200_resample(const float* in, float* out, int B, int F, int C, int N,
                       int method, int add_endpoint, void* stream);

/* Pieces of losses.SpectralLoss (losses.py:130-243) around cuFFT.
 * frame_window: tf.signal.stft's framing + periodic Hann window with pad_end=True
 * (spectral_ops.py:34-47): audio [B,N] -> frames [B, n_frames, frame_size],
 * frames[b,t,i] = window[i] * audio[b, t*frame_step + i] (0 past the end).
 * frame_window_adjoint: its transpose, grad_frames -> grad_audio [B,N], times the
 * optional DEVICE scalar *scale_device (NULL = 1), added to grad_audio when
 * accumulate != 0 (the FFT sizes of the multi-scale loss share one buffer).
 * spectral_l1: for complex STFTs [n_bins_total] (interleaved re/im) of target and
 * value: sums[0] += sum |mag_t - mag_v|, sums[1] += sum |safe_log mag_t -
 * safe_log mag_v| (core.py:213-216), and grad_value = d/dX_v of
 * mag_weight * mean|.| + logmag_weight * mean|.| (losses.py:102-127, 'L1').
 * n_bins = bins per frame.  irfft_size = 0: grad_value is the plain gradient;
 * irfft_size = 2 (n_bins - 1): it is pre-scaled so that irfft(grad_value,
 * irfft_size) is the gradient w.r.t. the real frames (the transpose of rfft);
 * irfft_size = -1: the same for an UNNORMALISED inverse transform (no 1/n pass).
 * sums must be zeroed by the caller.  frames must not overlap audio or window;
 * grad_audio must not overlap grad_frames, window or *scale_device; spectral_l1's
 * grad_value may be stft_value (in place) and must not overlap stft_target. */
int ddsp_b200_frame_window(const float* audio, const float* window, float* frames,
                           int B, int N, int n_frames, int frame_size, int frame_step,
                           void* stream);
int ddsp_b200_frame_window_adjoint(const float* grad_frames, const float* window,
                                   float* grad_audio, int B, int N, int n_frames,
                                   int frame_size, int frame_step,
                                   const float* scale_device, int accumulate,
                                   void* stream);
int ddsp_b200_spectral_l1(const float* stft_target, const float* stft_value,
                          float* grad_value, double* sums, int64_t n_bins_total,
                          float mag_weight, float logmag_weight, int n_bins,
                          int irfft_size, void* stream);

/* spectral_terms: every spectrogram term of losses.SpectralLoss (losses.py:194-234)
 * for complex STFTs [B, T, F] (interleaved re/im, F = fft_size/2 + 1) of target and
 * value, 'L1' or 'L2'.  For each term in `terms` (DDSP_B200_TERM_* flags) it adds
 * the sum of |d| (L1) or d^2 (L2), d = target term - value term, to sums[bit index]
 * (mag 0, delta_time 1, delta_freq 2, cumsum_freq 3, logmag 4; the caller zeroes
 * them), and writes to grad_value d/dX_v of sum weight * mean(term), pre-scaled for
 * an unnormalised inverse transform (spectral_l1's irfft_size = -1).  The terms of
 * m = |X|: mag m, delta_time core.diff(m, axis=1), delta_freq core.diff(m, axis=2),
 * cumsum_freq cumsum(m, axis=2), logmag safe_log(m).  grad_value may be
 * stft_value or stft_target (in place) unless delta_time is active, when it must
 * overlap neither STFT.
 * F > DDSP_B200_SPECTRAL_TERMS_MAX_BINS (fft_size 8192) is E_UNSUPPORTED. */
enum {
  DDSP_B200_TERM_MAG = 1,
  DDSP_B200_TERM_DELTA_TIME = 2,
  DDSP_B200_TERM_DELTA_FREQ = 4,
  DDSP_B200_TERM_CUMSUM_FREQ = 8,
  DDSP_B200_TERM_LOGMAG = 16
};
enum { DDSP_B200_LOSS_L1 = 0, DDSP_B200_LOSS_L2 = 1 };
enum { DDSP_B200_SPECTRAL_TERMS_MAX_BINS = 4097 /* frame rows one CTA stages */ };
int ddsp_b200_spectral_terms(const float* stft_target, const float* stft_value,
                             float* grad_value, double* sums, int B, int T, int F, int terms,
                             int loss_type, float mag_weight, float delta_time_weight,
                             float delta_freq_weight, float cumsum_freq_weight,
                             float logmag_weight, void* stream);

/* processors.Add.get_signal (processors.py:174-176).  out may be a or b (in place). */
int ddsp_b200_add(const float* a, const float* b, float* out, int64_t n,
                  void* stream);

/* Modulated delay: core.variable_length_delay (core.py:1285-1314) and
 * effects.ModDelay.get_signal (effects.py:328-394).
 *   out[b,t] = (add_dry ? audio[b,t] : 0) + gain[b,t] * delay[b,t],
 *   delay[b,t] = (1 - frac) v_{j0} + frac v_{j0+1},  pos = phase' * max_length,
 *   phase' = phase[b,t] * scale + offset (two float32 roundings, no FMA),
 *   j0 = floor(pos), frac = pos - j0,  v_j = audio[b, t - j] for 0 <= j < max_length
 *   (0 for t - j < 0), v_{max_length} = audio[b, t] (the reference's wrap column),
 *   v_j = 0 for j < 0 or j > max_length.
 * audio, phase, out: [B, N]; gain: [B, N] or NULL (= 1).  core.variable_length_delay
 * is scale = 1, offset = 0, gain = NULL, add_dry = 0.  1 <= max_length < 2^29.
 * out must not overlap audio; it may be phase or gain.
 *
 * backward: for the upstream gradient grad_out [B, N], writes any of
 *   grad_audio [B, N]  (d out / d audio, dry path included),
 *   grad_gain  [B, N]  (= grad_out * delay; needs gain),
 *   grad_phase [B, N]  (w.r.t. `phase`, i.e. times scale; 0 where pos is an integer:
 *                       TensorFlow's subgradients of |.| and relu at 0);
 * a NULL output is not computed.  No atomics: every element is written once and
 * the result is bit-reproducible. */
int ddsp_b200_mod_delay_forward(const float* audio, const float* phase, const float* gain,
                                float* out, int B, int N, int max_length, float scale,
                                float offset, int add_dry, void* stream);
int ddsp_b200_mod_delay_backward(const float* audio, const float* phase, const float* gain,
                                 const float* grad_out, float* grad_audio, float* grad_gain,
                                 float* grad_phase, int B, int N, int max_length, float scale,
                                 float offset, int add_dry, void* stream);

/* Transpose of ddsp_b200_resample: grad_out [B,N,C] -> grad_in [B,F,C], same
 * arguments and checks.  Every tap of the forward (its float32 index and weight,
 * the clamped taps included) is added in double; bit-reproducible. */
int ddsp_b200_resample_backward(const float* grad_out, float* grad_in, int B, int F, int C,
                                int N, int method, int add_endpoint, void* stream);

/* processors.Mix.get_signal (processors.py:217-233):
 *   out = sqrt(|m|) * s1 + (1 - sqrt(|m - 1|)) * s2
 * in float32, in that operation order.  signal_one, signal_two, out: [B,N,C];
 * mix_level m: [B,N,1], broadcast over C.
 * backward: writes any of grad_signal_one, grad_signal_two [B,N,C] and
 * grad_mix_level [B,N,1] (summed over C in channel order); NULL outputs are not
 * computed.  grad_mix_level is NaN where m is exactly 0 or 1, as the reference's
 * autodiff gives it (0 * inf).  The forward's out may be signal_one, signal_two or,
 * with C = 1, mix_level (in place); with C > 1 it must not overlap mix_level. */
int ddsp_b200_mix_forward(const float* signal_one, const float* signal_two,
                          const float* mix_level, float* out, int B, int N, int C,
                          void* stream);
int ddsp_b200_mix_backward(const float* signal_one, const float* signal_two,
                           const float* mix_level, const float* grad_out,
                           float* grad_signal_one, float* grad_signal_two,
                           float* grad_mix_level, int B, int N, int C, void* stream);

/* effects.ExpDecayReverb._get_ir (effects.py:144-151), on the scaled gain:
 *   ir[r,t] = (gain[r] * exp(-(2 + exp(decay[r])) * time[t])) * noise[t]
 * in float32, time = tf.linspace(0, 1, L).  gain, decay: [rows]; ir: [rows, L];
 * noise: one [L] row shared by every row, or NULL for the Philox stream's batch row
 * 0 at (seed, offset) (= ddsp_b200_uniform_noise(1, L, seed, offset)).
 * backward: for grad_ir [rows, L], writes any of
 *   grad_gain[r]  = sum_t grad_ir e n,
 *   grad_decay[r] = -exp(decay[r]) gain[r] sum_t grad_ir time e n
 * (NULL outputs are not computed); the noise is regenerated, the sums are in double
 * in a fixed order.  The forward's ir must not overlap gain, decay or noise. */
int ddsp_b200_exp_decay_ir(const float* gain, const float* decay, const float* noise,
                           uint64_t seed, uint64_t offset, float* ir, int rows, int L,
                           void* stream);
int ddsp_b200_exp_decay_ir_backward(const float* gain, const float* decay,
                                    const float* noise, uint64_t seed, uint64_t offset,
                                    const float* grad_ir, float* grad_gain,
                                    float* grad_decay, int rows, int L, void* stream);

/* core.wavetable_synthesis (core.py:1238-1282) with the tables kept at frame rate:
 *   audio[b,t] = amp(t) * ((1 - frac) T_t[j0] + frac T_t[(j0 + 1) mod W]),
 *   pos = phi(t) W, j0 = floor(pos), phi(t) = sum_{s<t} f0(s) / sr mod 1,
 * with phi exact (64-bit fixed-point turns of the linearly interpolated f0).
 * f0_hz, amplitudes: [B,F], N % F == 0; amplitudes upsampled with amp_method
 * ('window' needs F < N).  wavetables: [B,Fw,W]; Fw == 1 is a static table, Fw > 1
 * is interpolated in time with core.resample's 'linear' taps (add_endpoint), any
 * Fw.  1 <= W <= 1048576, else E_UNSUPPORTED; B <= 65535.
 * workspace: ddsp_b200_wavetable_workspace(B,F) bytes.
 * backward: for grad_audio [B,N], writes any of d_f0 [B,F], d_amplitudes [B,F] and
 * d_wavetables [B,Fw,W]; a NULL output is not computed.  d_f0 follows TensorFlow's
 * subgradients: 0 where pos is an integer.  Table entries no sample reads are 0.
 * No atomics: the gradients are bit-reproducible.
 * workspace: ddsp_b200_wavetable_backward_workspace(B,F,N,Fw,W) bytes.
 * The forward's audio must not overlap f0_hz, amplitudes or wavetables. */
size_t ddsp_b200_wavetable_workspace(int B, int F);
int ddsp_b200_wavetable_forward(const float* f0_hz, const float* amplitudes,
                                const float* wavetables, float* audio, int B, int F,
                                int N, int Fw, int W, float sample_rate, int amp_method,
                                void* workspace, size_t workspace_bytes, void* stream);
size_t ddsp_b200_wavetable_backward_workspace(int B, int F, int N, int Fw, int W);
int ddsp_b200_wavetable_backward(const float* f0_hz, const float* amplitudes,
                                 const float* wavetables, const float* grad_audio,
                                 float* d_f0, float* d_amplitudes, float* d_wavetables,
                                 int B, int F, int N, int Fw, int W, float sample_rate,
                                 int amp_method, void* workspace, size_t workspace_bytes,
                                 void* stream);

/* core.linear_lookup (core.py:1168-1214): phase [B,N] reads wavetables [B,W]
 * (per_sample = 0, one table per item) or [B,N,W] (per_sample = 1) -> out [B,N] =
 * sum_{j=0..W} relu(1 - |phase - lin_j| W) T[j mod W], lin = float32 linspace(0, 1, W + 1),
 * every step in float32 as the reference computes it; phases outside [0, 1] are not
 * wrapped.  W <= DDSP_B200_LOOKUP_MAX_W (more is E_UNSUPPORTED).
 * The backward writes d_phase [B,N] (TensorFlow's subgradients: 0 on a grid point of a
 * power-of-two W) and d_wavetables (the table's shape); a NULL output is not computed.
 * No atomics and no workspace: bit-reproducible.  The forward's out must not overlap
 * phase or wavetables. */
enum { DDSP_B200_LOOKUP_MAX_W = 4194304 /* the four candidate columns stay exact */ };
int ddsp_b200_linear_lookup_forward(const float* phase, const float* wavetables, float* out,
                                    int B, int N, int W, int per_sample, void* stream);
int ddsp_b200_linear_lookup_backward(const float* phase, const float* wavetables,
                                     const float* grad, float* d_phase, float* d_wavetables,
                                     int B, int N, int W, int per_sample, void* stream);

/* spectral_ops.compute_loudness (spectral_ops.py:254-324) on audio [B,N]: frames of
 * n_fft samples every hop under `padding` (DDSP_B200_PAD_*; CENTER pads n_fft/2 zeros
 * on both sides, SAME pads the end to (ceil(N/hop) - 1) hop + n_fft, VALID nothing),
 * periodic Hann window, loudness[b,t] = power_to_db(mean_k weights[k] |X_k|^2) with
 * ref_db and range_db.  weights: [n_fft/2 + 1] device floats, the linear A-weighting.
 * n_frames must be the frame count of that padding (1 + (padded - n_fft) / hop, or
 * ceil(N/hop) for SAME).  n_fft is a power of two, hop <= n_fft unless VALID;
 * n_fft > 16384 is E_UNSUPPORTED.  B <= 65535.
 * backward: grad_audio [B,N] for grad_loudness [B,T], with tf.maximum's tie rule (no
 * gradient through an active clamp).  No atomics: bit-reproducible.  The forward's
 * loudness must not overlap audio or weights. */
int ddsp_b200_loudness_forward(const float* audio, const float* weights, float* loudness,
                               int B, int N, int n_frames, int n_fft, int hop, int padding,
                               float range_db, float ref_db, void* stream);
int ddsp_b200_loudness_backward(const float* audio, const float* weights,
                                const float* grad_loudness, float* grad_audio, int B, int N,
                                int n_frames, int n_fft, int hop, int padding, float range_db,
                                float ref_db, void* stream);
/* spectral_ops.compute_power (spectral_ops.py:223-249): power_db[b,t] =
 * power_to_db(mean(frame^2)) with frames of any frame_size every hop, padded as above
 * (CENTER pads frame_size/2 zeros on both sides).  in_db == 0 writes
 * compute_rms_energy's mean(frame^2)^0.5 instead.  Forward only.
 * power_db must not overlap audio. */
int ddsp_b200_rms_power(const float* audio, float* power_db, int B, int N, int n_frames,
                        int frame_size, int hop, int padding, int in_db, float range_db,
                        float ref_db, void* stream);

/* spectral_ops.PretrainedCREPE (spectral_ops.py:432-566) around its network.  All three
 * are forward only, with no atomics: bit-reproducible.
 * ddsp_b200_crepe_frames: the network's input frames [B * n_frames, 1024] of audio [B,N]:
 *   pad (padding DDSP_B200_PAD_*: CENTER pads 512 zeros on both sides, SAME pads the end
 *   to (ceil(N/hop) - 1) hop + 1024, VALID nothing), frames of 1024 every hop
 *   (tf.signal.frame, pad_end=False), each normalised to (x - mean) / std with the mean
 *   and population variance of tf.nn.moments, summed in double, and std = 1e-8 where the
 *   variance is 0.  n_frames must be that padding's frame count (0 for VALID audio
 *   shorter than a frame); hop <= 1024 unless VALID.  B = 0 or n_frames = 0 returns after
 *   the checks without a launch.
 * ddsp_b200_crepe_viterbi: centers [B,T] (int32), HiddenMarkovModel.posterior_mode of
 *   activations [B,T,360] under create_hmm's model (uniform start, transitions
 *   max(12 - |i - j|, 1e-5) over their row sums, Multinomial(1, eye 0.1 + 0.9/360)
 *   emissions); every tie goes to the lowest state index, as tf.argmax's.  workspace:
 *   ddsp_b200_crepe_viterbi_workspace_bytes(B, T) bytes of back pointers (E_WORKSPACE if
 *   smaller; 0 for T = 1, when it may be null), 4-byte aligned.  B >= 0, T >= 1, both
 *   otherwise unbounded; B = 0 returns after the checks without a launch.
 * ddsp_b200_crepe_decode: activations_to_f0_and_confidence of activations [M,360]:
 *   confidence [M] = the row max, f0 [M] = 10 2^(c / 1200) Hz with c the weighted mean of
 *   the float32 cents linspace(0, 7180, 360) + 1997.3794084376191 over bins
 *   centre - 4 .. centre + 5, each clamped into 0 .. 359.  The centre is the row's first
 *   argmax, or centers[m] (int32, any value) when centers is not null.  Weights summing
 *   to 0 give NaN (0 / 0), as in the reference.  M >= 0; M = 0 launches nothing.
 * crepe_frames' frames must not overlap audio; crepe_decode's f0 and confidence must
 * not overlap activations.
 *
 * losses.PretrainedCREPE.frame_audio (losses.py:455-468), the frames the embedding losses
 * train through: padding DDSP_B200_PAD_CENTER or _VALID OR'ed with
 * DDSP_B200_CREPE_LOSS_FRAMES makes ddsp_b200_crepe_frames normalise each frame to
 * (x - mean) / (sqrt(var) + 1e-5) instead (a frame of variance 0 becomes zeros).  In
 * that mode any hop >= 1 is taken with either padding, N may be 0 (CENTER then gives one
 * frame of zeros, and audio may be null), and n_frames must be
 * 1 + (N + 2 pad - 1024) / hop (pad = 512 for CENTER, 0 for VALID), or 0 when that
 * padded length is below 1024.  SAME is E_INVALID.
 * ddsp_b200_crepe_frames_backward: grad_audio [B,N] of that normalisation for
 *   grad_frames [B * n_frames, 1024], the same B, N, n_frames, hop and padding (with or
 *   without the flag).  Every element of grad_audio is written, 0 where no frame reads
 *   the sample.  Per frame with mu, s = sqrt(var), gbar = mean(g) and
 *   c = sum_j g_j (x_j - mu):
 *     dx_k = (g_k - gbar) / (s + 1e-5) - c (x_k - mu) / ((s + 1e-5)^2 1024 s),
 *   statistics in double; overlapping frames (hop < 1024) add in increasing frame order.
 *   A frame of variance 0 makes every sample it covers NaN, as TensorFlow's gradient of
 *   var**0.5 at 0 does.  No atomics and no workspace: bit-reproducible.  grad_audio must
 *   not overlap audio or grad_frames.  B = 0 or N = 0 returns after the checks without a
 *   launch; B and N are otherwise unbounded. */
enum { DDSP_B200_CREPE_BINS = 360, DDSP_B200_CREPE_FRAME = 1024 };
enum { DDSP_B200_CREPE_LOSS_FRAMES = 256 /* OR'ed into crepe_frames' padding */ };
int ddsp_b200_crepe_frames(const float* audio, float* frames, int B, int N, int n_frames,
                           int hop, int padding, void* stream);
int ddsp_b200_crepe_frames_backward(const float* audio, const float* grad_frames,
                                    float* grad_audio, int B, int N, int n_frames, int hop,
                                    int padding, void* stream);
size_t ddsp_b200_crepe_viterbi_workspace_bytes(int B, int T);
int ddsp_b200_crepe_viterbi(const float* activations, int* centers, void* workspace,
                            size_t workspace_bytes, int B, int T, void* stream);
int ddsp_b200_crepe_decode(const float* activations, const int* centers, float* f0,
                           float* confidence, int64_t M, void* stream);

/* output stage of ddsp_b200_mel_forward / _backward */
enum { DDSP_B200_MEL = 0, DDSP_B200_LOGMEL = 1, DDSP_B200_MFCC = 2 };

/* spectral_ops.compute_mel / compute_logmel / compute_mfcc (spectral_ops.py:73-133) on
 * audio [B,N]: tf.signal.stft frames of fft_size samples every hop (pad_end = 1 pads
 * zeros past the end, n_frames = ceil(N / hop); pad_end = 0 pads nothing, n_frames =
 * 1 + (N - fft_size) / hop, or 0 when N < fft_size), times window[fft_size], zero
 * padded to fft_length (a power of two >= fft_size), real FFT of K = fft_length/2 + 1
 * bins; mel[t,j] = sum_k W[k,j] |X_k|.  mode MEL writes out[B,T,bins] = mel, LOGMEL
 * log(mel <= 0 ? 1e-5 : mel), MFCC the first n_out coefficients of the log-mel's
 * unnormalised DCT-II times rsqrt(2 bins), out[B,T,n_out] (n_out == bins otherwise).
 * mel_table: W in sparse form, 3K + 2 bins 32-bit words: [K] float pairs (w_lo, w_hi),
 * [K] int32 band, [bins] int32 band_lo, [bins] int32 band_hi.  Bin k weighs w_lo into
 * band[k] (when >= 0) and w_hi into band[k] + 1 (when < bins), band j sums its bins
 * k in [band_lo[j], band_hi[j]), and band[] must lie in {j - 1, j} there.  fft_length
 * outside 2..16384 and bins > 1024 are E_UNSUPPORTED.  B <= 65535.  B = 0, n_frames = 0
 * and n_out = 0 return before any launch (backward: grad_audio is then not written).
 * backward: grad_audio [B,N] for grad_out [B,T,C], TensorFlow's gradient (no gradient
 * through mel <= 0 in the log, none through |X_k| = 0).  No atomics: bit-reproducible.
 * The forward's out must not overlap audio or window. */
int ddsp_b200_mel_forward(const float* audio, const float* window, const void* mel_table,
                          float* out, int B, int N, int n_frames, int fft_size, int fft_length,
                          int hop, int pad_end, int bins, int n_out, int mode, void* stream);
int ddsp_b200_mel_backward(const float* audio, const float* window, const void* mel_table,
                           const float* grad_out, float* grad_audio, int B, int N,
                           int n_frames, int fft_size, int fft_length, int hop, int pad_end,
                           int bins, int n_out, int mode, void* stream);

/* Limits of the loss kernels, which run one CTA per row (a frame, or a Wasserstein row):
 * rows on the grid's x axis, and the components, candidates, points or sinusoids the
 * consistency kernels stage per frame. */
enum { DDSP_B200_MAX_ROWS = 2147483647, DDSP_B200_CONSISTENCY_MAX_STAGED = 4096 };

/* Mixture NLL of the consistency losses (losses.KDEConsistencyLoss.nll and
 * TWMLoss's p(harmonics | sinusoids), losses.py:759-813, 982-990): per frame (b, t),
 *   nll[b,t,q] = -logsumexp_j(lw[b,t,j] - ((x[b,t,q] - mu[b,t,j]) / scale)^2 / 2)
 *                + log(scale) + log(2 pi) / 2
 * for x [B,T,Q], mu and lw [B,T,J] (lw: log-weights, normalised by the caller), the
 * logsumexp shifted by its largest term.  1 <= J <= 4096 is staged per frame; J > 4096
 * is E_UNSUPPORTED.  Q is unbounded.  scale must be positive and finite.  B*T <=
 * 2^31 - 1.  B, T, Q or J = 0 return before any launch and write nothing; the
 * pointers may then be null.
 * backward: for g [B,T,Q], with responsibilities r_qj and z_qj = (x_q - mu_j) / scale,
 *   dx = g_q / scale sum_j r_qj z_qj, dmu = -1/scale sum_q g_q r_qj z_qj,
 *   dlw = -sum_q g_q r_qj;
 * every sum in a fixed order, no atomics: bit-reproducible.  The forward's nll must not
 * overlap x, mu or lw. */
int ddsp_b200_mixture_nll_forward(const float* x, const float* mu, const float* lw,
                                  float* nll, int B, int T, int Q, int J, float scale,
                                  void* stream);
int ddsp_b200_mixture_nll_backward(const float* x, const float* mu, const float* lw,
                                   const float* grad, float* dx, float* dmu, float* dlw,
                                   int B, int T, int Q, int J, float scale, void* stream);

/* Harmonic-comb NLL of TWMLoss's p(sinusoids | harmonics), amplitude-reduced
 * (losses.py:956-977): for candidates f0 [B,T,C], points f and amplitudes a [B,T,P],
 *   out[b,t,c] = safe_divide(sum_p a_p nu(safe_divide(f_p, f0_c)), sum_p a_p),
 *   nu(q) = -logsumexp_{k=1..G}(-log G - ((q - k) / scale)^2 / 2) + log(scale)
 *           + log(2 pi) / 2,
 * safe_divide's zero denominators being the constant 1e-7.  Only the comb terms within
 * a window around the nearest k are summed, its half-width chosen from scale and G so
 * that the omitted terms stay below 2^-25 of the sum.  1 <= C, P <= 4096 (more is
 * E_UNSUPPORTED), G >= 1, scale positive and finite, B*T <= 2^31 - 1.  B, T, C or P = 0
 * return before any launch and write nothing; the pointers may then be null.
 * backward: d_f0 [B,T,C], d_f and d_a [B,T,P] for g [B,T,C]; no gradient through a
 * safe_divide denominator that was 0 (d_f0 = 0 at f0 = 0).  Fixed-order sums, no
 * atomics: bit-reproducible.  The forward's out must not overlap f0, f or a. */
int ddsp_b200_comb_nll_forward(const float* f0, const float* f, const float* a, float* out,
                               int B, int T, int C, int P, int G, float scale, void* stream);
int ddsp_b200_comb_nll_backward(const float* f0, const float* f, const float* a,
                                const float* grad, float* d_f0, float* d_f, float* d_a,
                                int B, int T, int C, int P, int G, float scale,
                                void* stream);

/* core.sinusoidal_to_harmonic (core.py:733-781): for sinusoids sin_amps and sin_freqs
 * [B,T,S] and f0_hz [B,T,1], per frame with den = f0 (1e-7 where f0 = 0) and k = 1..K,
 *   w_ks = exp(-(|(sin_freqs_s - f0 k) / den| / width)^2),
 *   W_ks = w_ks / sum_s w_ks where normalize and that sum is > 1, else w_ks,
 *   HA_k = sum_s W_ks sin_amps_s, 0 where f0 k >= sample_rate / 2,
 *   harm_amp [B,T,1] = sum_k HA_k,  harm_dist [B,T,K] = HA_k / harm_amp
 *   (1e-7 for a zero harm_amp).
 * width must be nonzero (0 is E_INVALID; a negative width acts as its magnitude),
 * normalize 0 or 1.  S <= 4096 sinusoids are staged per frame; more is E_UNSUPPORTED.
 * K is unbounded.  B*T <= 2^31 - 1.  No workspace.  B = 0 or T = 0 returns before any
 * launch and writes nothing (the pointers may then be null).  Otherwise one launch
 * writes every output: S = 0 gives harm_amp = 0 and harm_dist = 0; K = 0 gives
 * harm_amp = 0.  Arrays of zero elements may be null.
 * backward: for grad_amp [B,T,1] and grad_dist [B,T,K], d_sin_amps and d_sin_freqs
 * [B,T,S] and d_f0_hz [B,T,1], all written, zeros where nothing contributes (K = 0 or
 * S = 0).  TensorFlow's gradient: none through a safe_divide denominator that took its
 * 1e-7 (f0 = 0, harm_amp = 0), sign(0) = 0 in |q|, none to the branch of normalize's
 * where that was not taken, none through harmonics at or above Nyquist.  Every sum in a
 * fixed order, no atomics: bit-reproducible.  The forward's harm_amp and harm_dist must
 * not overlap an input. */
int ddsp_b200_sinusoidal_to_harmonic(const float* sin_amps, const float* sin_freqs,
                                     const float* f0_hz, float* harm_amp, float* harm_dist,
                                     int B, int T, int S, int K, float width,
                                     float sample_rate, int normalize, void* stream);
int ddsp_b200_sinusoidal_to_harmonic_backward(
    const float* sin_amps, const float* sin_freqs, const float* f0_hz, const float* grad_amp,
    const float* grad_dist, float* d_sin_amps, float* d_sin_freqs, float* d_f0_hz, int B,
    int T, int S, int K, float width, float sample_rate, int normalize, void* stream);

/* losses.HmmTranscriber (losses.py:247-345): tfp's HiddenMarkovModel over K states with
 * a uniform initial distribution, transitions hold on the diagonal and other elsewhere,
 * and observations obs [B,T,2] (pitch, amps) under MultivariateNormalDiag(loc_j, scale_j),
 * loc and scale [K,2] (scale positive).
 *   ddsp_b200_hmm_log_prob: log_prob [B] = log p(obs_b), the forward algorithm in O(K)
 *     per step, its normalisers summed in double.
 *   ddsp_b200_hmm_log_prob_backward: d_obs [B,T,2] = grad_b * d log_prob_b / d obs, from
 *     the posterior marginals; loc and scale are constants.  checkpoints is scratch of
 *     B * ceil(T / seg) * K floats: the kernel re-runs the forward and keeps its state
 *     there every seg steps; 1 <= seg and seg * K <= DDSP_B200_HMM_SEGMENT_FLOATS
 *     (E_INVALID otherwise).  No atomics: bit-reproducible.
 *   ddsp_b200_hmm_viterbi: path [B,T] (int64), the most likely state sequence; ties go to
 *     the lowest state index.  The back pointers stay in shared memory, which bounds
 *     4 T (ceil(K / 32) + 1) <= DDSP_B200_HMM_VITERBI_BYTES (E_UNSUPPORTED otherwise):
 *     K = 1024 takes T <= 1551, K = 128 T <= 10240.  ddsp_b200_hmm_viterbi_takes(T, K) is
 *     1 for T >= 1 steps of K >= 1 states within that bound, else 0.
 * All three take B >= 0, T >= 1, 2 <= K <= DDSP_B200_HMM_MAX_STATES (more is
 * E_UNSUPPORTED), hold and other finite, non-negative and not both 0.  B = 0 returns
 * after the checks without a launch (the pointers may then be null).  hmm_log_prob's
 * log_prob must not overlap obs, loc or scale. */
enum {
  DDSP_B200_HMM_MAX_STATES = 1024,      /* one CTA runs the states, a thread each      */
  DDSP_B200_HMM_SEGMENT_FLOATS = 49152, /* the backward's segment buffer (192 KiB)     */
  DDSP_B200_HMM_VITERBI_BYTES = 204800  /* the Viterbi back pointers (200 KiB)         */
};
int ddsp_b200_hmm_viterbi_takes(int T, int K);
int ddsp_b200_hmm_log_prob(const float* obs, const float* loc, const float* scale,
                           float* log_prob, int B, int T, int K, double hold, double other,
                           void* stream);
int ddsp_b200_hmm_log_prob_backward(const float* obs, const float* loc, const float* scale,
                                    const float* grad, float* d_obs, float* checkpoints,
                                    int seg, int B, int T, int K, double hold, double other,
                                    void* stream);
int ddsp_b200_hmm_viterbi(const float* obs, const float* loc, const float* scale,
                          int64_t* path, int B, int T, int K, double hold, double other,
                          void* stream);

/* losses.wasserstein_distance (losses.py:641-686): for R rows of values u [R,Nu] and
 * v [R,Nv] with weights wu [R,Nu] and wv [R,Nv], s = sort(concat(u, v)) (stable: u before
 * v, lower index first; -0 ties with +0, NaNs sort last), N = Nu + Nv and i = 0 .. N-2,
 *   out[r] = (sum_i (s_{i+1} - s_i) |U_i - V_i|^p)^(1/p),
 *   U_i = sum_k wu_k [u_k <= s_i],  V_i = sum_k wv_k [v_k <= s_i].
 * The CDFs are raw cumulative weights, not normalised, as the reference computes them.
 * p positive and finite; Nu, Nv <= DDSP_B200_WASSERSTEIN_MAX_SIDE (more is
 * E_UNSUPPORTED); R <= DDSP_B200_MAX_ROWS.  No workspace.  R, Nu or Nv = 0 returns after
 * the checks without a launch and writes nothing (the pointers may then be null).  One CTA per row sorts, scans and sums in
 * shared memory: nothing but out is written.
 * backward: for grad [R], du [R,Nu], dv [R,Nv], dwu [R,Nu] and dwv [R,Nv], all written.
 * With c_i = |U_i - V_i|^p, S = sum_i delta_i c_i, G = grad (1/p) S^(1/p - 1) and
 * g_i = G delta_i p |U_i - V_i|^(p-1) sgn(U_i - V_i):
 *   the element sorted to position j gets G c_{j-1} [j >= 1] - G c_j [j <= N-2],
 *   dwu_k = sum_{i: s_i >= u_k} g_i,  dwv_k = -sum_{i: s_i >= v_k} g_i.
 * An exact U_i = V_i at p < 1, or S = 0 at p > 1, gives NaN (0 * inf) as autograd does;
 * at p = 1 everything finite stays finite.  Fixed-order scans and sums, no atomics:
 * bit-reproducible.  The forward's out must not overlap u, v, wu or wv. */
enum { DDSP_B200_WASSERSTEIN_MAX_SIDE = 4096 /* values per side one CTA sorts */ };
int ddsp_b200_wasserstein_forward(const float* u, const float* v, const float* wu,
                                  const float* wv, float* out, int64_t R, int Nu, int Nv,
                                  float p, void* stream);
int ddsp_b200_wasserstein_backward(const float* u, const float* v, const float* wu,
                                   const float* wv, const float* grad, float* du, float* dv,
                                   float* dwu, float* dwv, int64_t R, int Nu, int Nv, float p,
                                   void* stream);

/* training/nn.py:375-557, the note functions of the MIDI autoencoder.
 * ddsp_b200_note_mask: the dense mask [B, T_out, R] of get_note_mask (onset null) or
 *   get_note_mask_from_onset (onset [B,T]) for q [B,T] (channel 0 of a 3-D q_pitch).
 *   Edge rule: frame 0 opens region 0; frame t in 1 .. T-2 opens a new region iff
 *   |q_t - q_{t-1}| > 0 (NaN never does); the last frame joins the region before it.
 *   T_out = T, except T = 1 gives two rows, both region 0.  Onset rule: frame t >= 1
 *   adds (int)onset_t (truncation) to the region count, T_out = T; non-finite onsets and
 *   onsets of magnitude 2^31 or more are outside the contract.  Row t is 1 at its region
 *   index when 0 <= index < R and the note is on, else 0.  note_on_only: with the edge
 *   rule a region is on iff the reference's mask-weighted sum of q over all T frames is
 *   > 0, decided in double (a non-finite frame outside the region makes it NaN: off);
 *   with the onset rule a frame is on iff q_t > 0.  workspace: scratch of at least
 *   B * min(R, T) bytes with the edge rule and note_on_only, else none (E_WORKSPACE if
 *   smaller).  B >= 0, T >= 1, R >= 0; B = 0 or R = 0
 *   returns after the checks without a launch.
 * ddsp_b200_note_moments: for x [B,T,D] and any float mask [B,T,N],
 *   L_n = sum_t m_tn, Ls_n = L_n or 1e-7 where L_n = 0,
 *   mean [B,N,D] = sum_t m_tn x_td / Ls_n, std [B,N,D] = (sum_t ((x_td - mean) m_tn)^2 / Ls_n)^0.5
 *   (two passes; std may be null), and, when pooled_mean is not null, pooled_mean [B,T,D] =
 *   sum_n m_tn mean_nd and (pooled_std not null, which needs std) pooled_std = sum_n m_tn std_nd.
 *   One launch, or two when pooling.  N = 0 writes zero pooled values.
 * ddsp_b200_note_moments_backward: dx [B,T,D] from any of grad_mean, grad_std [B,N,D] and
 *   grad_pooled_mean, grad_pooled_std [B,T,D] (null for none; a std gradient needs std):
 *   with Gmu = grad_mean + sum_t m grad_pooled_mean, Gs = grad_std + sum_t m grad_pooled_std,
 *   Gv = Gs 0.5 / std, GQ = Gv / Ls, r_tnd = (x_td - mean_nd) m_tn,
 *   Gmu' = Gmu - 2 GQ sum_t m_tn r_tnd, dx_td = sum_n m_tn (Gmu'_nd / Ls_n + 2 GQ_nd r_tnd);
 *   without a std gradient the GQ terms are skipped.  std = 0 under a std gradient gives NaN
 *   (0 * inf) through the whole (b, d), as autograd does.  workspace: scratch of at least
 *   8 B N D + 256 bytes when B, N and D are positive (E_WORKSPACE if smaller).  Two launches.
 * Both moment entry points take B >= 0, T >= 1, N, D >= 0 and at most 2^31 - 1 CTAs (B
 * times the tiles of 32 notes or frames by 64 dims); B = 0 or D = 0 returns after the
 * checks without a launch.  All three: no atomics, fixed summation orders,
 * bit-reproducible.  No output of note_mask or note_moments may overlap an input. */
int ddsp_b200_note_mask(const float* q, const float* onset, float* mask, void* workspace,
                        size_t workspace_bytes, int B, int T, int R, int note_on_only,
                        void* stream);
int ddsp_b200_note_moments(const float* x, const float* mask, float* mean, float* std,
                           float* pooled_mean, float* pooled_std, int B, int T, int N, int D,
                           void* stream);
int ddsp_b200_note_moments_backward(const float* x, const float* mask, const float* mean,
                                    const float* std, const float* grad_mean,
                                    const float* grad_std, const float* grad_pooled_mean,
                                    const float* grad_pooled_std, float* dx, void* workspace,
                                    size_t workspace_bytes, int B, int T, int N, int D,
                                    void* stream);

/* training/heuristics.py, DDSP controls to notes.
 * ddsp_b200_note_heuristic: the binary mask [B,T] (one byte per frame, 0 or 1) of one or
 *   more of heuristics.py's binarizers, one CTA per item.  stages is a bit mask:
 *   DDSP_B200_HEURISTIC_POOL: pooled outliers of v = log(x) (log_values, amplitudes) or
 *     v = x + shift in float32 (power): frame t is on iff mean(w) - num_devs std(w) < v_t
 *     for its window w of pool_width padded values (population std), decided in double
 *     on deviations from v_t; a window with a non-finite value is off; with
 *     pool_positive also v_t > 0.
 *   DDSP_B200_HEURISTIC_STRIDED: strided_freq_change's transitions for the n_widths
 *     widths in `widths` (HOST memory, read before the launch), in order, on the float32
 *     hz_to_midi(f0); a frame is turned off where the padded window of the transitions
 *     before this width is all on and |midi(first) - midi(last)| > 0.75.
 *   DDSP_B200_HEURISTIC_F0_POSITIVE: and f0 > 0.
 *   With neither POOL nor STRIDED the mask starts from `on` [B,T] (nonzero bytes are on;
 *   mask may be on), else from the AND of the two.
 *   DDSP_B200_HEURISTIC_REMOVE_SHORT: then remove_short(min_samples, glue_back): a run of
 *     on frames that an off frame ends is cleared when shorter than min_samples; with
 *     glue_back an off frame is set on instead when the run before the next off frame is
 *     shorter than min_samples.
 *   Pads (DDSP_B200_HEURISTIC_PAD_*) repeat the edge values truncated toward zero; front
 *   pads width - 1 frames before, center width / 2 before and the rest after, end
 *   width - 1 after.  status [B]: 0, or DDSP_B200_HEURISTIC_POOL_EDGE /
 *   DDSP_B200_HEURISTIC_PITCH_EDGE where a padded vector has a non-finite first or last
 *   value (the reference raises); that item's mask row is all 0.  workspace:
 *   ddsp_b200_note_heuristic_workspace_bytes(B, T) bytes (E_WORKSPACE if smaller).
 * ddsp_b200_note_segments: the note table of the runs of nonzero bytes of mask [B,T]:
 *   notes [B, (T+1)/2] records (16-byte aligned), the first count[b] of them the notes in
 *   order and the rest zero.  f0 is the run's mean of f0 (summed in double, rounded once
 *   to float) or, with median, np.median's (the middle value, or the float32 mean of the
 *   two middle values; NaN when the run holds a NaN).  pitch is round-half-even of the
 *   float32 hz_to_midi(f0), -2^31 for a non-finite value.
 * Both take B >= 0 and 1 <= T <= DDSP_B200_NOTE_HEURISTIC_MAX_T
 * (ddsp_b200_note_heuristic_takes(T); more is E_UNSUPPORTED); B = 0 returns after the
 * checks.  No output may overlap an input (except mask on), no atomics, bit-reproducible. */
enum {
  DDSP_B200_HEURISTIC_POOL = 1,
  DDSP_B200_HEURISTIC_STRIDED = 2,
  DDSP_B200_HEURISTIC_F0_POSITIVE = 4,
  DDSP_B200_HEURISTIC_REMOVE_SHORT = 8,
  DDSP_B200_HEURISTIC_PAD_FRONT = 0,
  DDSP_B200_HEURISTIC_PAD_CENTER = 1,
  DDSP_B200_HEURISTIC_PAD_END = 2,
  DDSP_B200_HEURISTIC_POOL_EDGE = 1,
  DDSP_B200_HEURISTIC_PITCH_EDGE = 2,
  DDSP_B200_HEURISTIC_MAX_WIDTHS = 8,
  DDSP_B200_NOTE_HEURISTIC_MAX_T = 268435456 /* 2^28 frames: int counts and positions */
};
typedef struct {
  int start, stop; /* frames [start, stop) */
  int pitch;
  float f0;
} ddsp_b200_note;
size_t ddsp_b200_note_heuristic_workspace_bytes(int B, int T);
int ddsp_b200_note_heuristic_takes(int T);
int ddsp_b200_note_heuristic(const float* x, const float* f0, const unsigned char* on,
                             unsigned char* mask, int* status, void* workspace,
                             size_t workspace_bytes, int B, int T, int stages, int log_values,
                             float shift, int pool_width, int pool_pad, int pool_positive,
                             double num_devs, const int* widths, int n_widths,
                             int strided_pad, int min_samples, int glue_back, void* stream);
int ddsp_b200_note_segments(const unsigned char* mask, const float* f0, ddsp_b200_note* notes,
                            int* count, int B, int T, int median, void* stream);

/* training/postprocessing.py and colab_utils.get_tuning_factor / auto_tune: adjusting
 * controls for tone transfer.  Every input is float64 (float32 values widened exactly);
 * flags make the kernels round the reference's float32 steps to float32, so that the
 * caller's cast of a result back to float32 is exact.  Forward only, no atomics,
 * bit-reproducible.  No output may overlap an input or another output.
 * ddsp_b200_detect_notes: [B,T] (n = B T) in two launches.  smooth's box filter of
 *   conf ** exponent (numpy's fast paths for 2, 0.5, 1, -1, 0; in float32 with
 *   DETECT_CONF_F32), converted to float32, over `smoothing` taps of float32(1 / k) with
 *   TF 'SAME' zero padding ((k-1)/2 taps left), summed in float32 tap by tap.  ratio =
 *   smoothed (loudness - min_db) / ((mean - min_db) weight), the mean over all n frames
 *   summed in double over a partition fixed by n; in float32 with DETECT_LOUD_F32.
 *   mask = ratio >= note_threshold.  DETECT_SMOOTH_ONLY writes the smoothed input into
 *   ratio (loudness and mask may be NULL).  workspace:
 *   ddsp_b200_detect_notes_workspace_bytes(n) bytes (E_WORKSPACE if smaller).
 * ddsp_b200_quantile_fit: np.nanpercentile(col, 100 q) then np.maximum.accumulate, for
 *   each of F columns of `sorted` [F, n_rows] (ascending, NaN last; counts[f] non-NaN
 *   values, 0 gives NaN), into quantiles [nq, F]: numpy 2.3's linear method, b - a in
 *   float32 with QUANTILE_F32.
 * ddsp_b200_quantile_transform: QuantileTransformer._transform_col of every column of
 *   x [n, F] into out [n, F], forward or inverse, QUANTILE_UNIFORM or QUANTILE_NORMAL,
 *   with np.interp's rules on the column's quantiles [nq, F] and references [nq]
 *   (1 <= nq <= DDSP_B200_QUANTILE_MAX_N).  The 'normal' forward output is clipped to
 *   [ppf(1e-7 - eps), ppf(1 - (1e-7 - eps))], computed on the device.  QUANTILE_F32: x is a float32 column (the forward result is
 *   rounded to float32 before the bounds, and scipy's float32 ppf).
 * ddsp_b200_tuning_factor: get_tuning_factor on the N masked frames f0 [N] and conf [N]
 *   for n_factors <= DDSP_B200_TUNING_MAX_FACTORS factors: costs [2, n_factors] (the
 *   mean weighted distance, the mean weighted note change) and index [1], np.argmin of
 *   their normalised sum, in two launches.
 * ddsp_b200_auto_tune: out [T] = f0 - amount midi_diff.  chromatic: midi_diff =
 *   (f0 - tuning_factor) % 1, less 1 above 0.5 (in float32 with AUTO_TUNE_F32); else
 *   the major scale s with the least mean distance of the N masked frames f0_on to its
 *   nearest note (scale_cost [12], scale_index [1]), and each frame's difference to its
 *   nearest note of scale s. */
enum {
  DDSP_B200_DETECT_SMOOTH_ONLY = 1,
  DDSP_B200_DETECT_CONF_F32 = 2,
  DDSP_B200_DETECT_LOUD_F32 = 4,
  DDSP_B200_QUANTILE_F32 = 1,
  DDSP_B200_QUANTILE_UNIFORM = 0,
  DDSP_B200_QUANTILE_NORMAL = 1,
  DDSP_B200_QUANTILE_MAX_N = 8192,  /* quantiles and references of a column in shared memory */
  DDSP_B200_TUNING_MAX_FACTORS = 128,
  DDSP_B200_SCALE_NOTES = 70,
  DDSP_B200_AUTO_TUNE_F32 = 1
};
size_t ddsp_b200_detect_notes_workspace_bytes(int64_t n);
int ddsp_b200_detect_notes(const double* loudness, const double* conf, double* ratio,
                           unsigned char* mask, void* workspace, size_t workspace_bytes, int B,
                           int T, int smoothing, double exponent, double weight, double min_db,
                           double note_threshold, int flags, void* stream);
int ddsp_b200_quantile_fit(const double* sorted, const int64_t* counts, const double* q,
                           double* quantiles, int64_t n_rows, int F, int nq, int flags,
                           void* stream);
int ddsp_b200_quantile_transform(const double* x, const double* quantiles,
                                 const double* references, double* out, int64_t n, int F,
                                 int nq, int inverse, int distribution, int flags,
                                 void* stream);
int ddsp_b200_tuning_factor(const double* f0, const double* conf, const double* factors,
                            double* costs, int* index, int64_t N, int n_factors, void* stream);
int ddsp_b200_auto_tune(const double* f0, const double* f0_on, double* scale_cost,
                        int* scale_index, double* out, int64_t T, int64_t N,
                        double tuning_factor, double amount, int chromatic, int flags,
                        void* stream);

/* training/data_preparation/synthetic_data.py generate_notes_v2: InverseSynthesis's
 * synthetic notes, drawn from numpy's legacy RandomState (MT19937) in the reference's
 * order, as the reference's float64 arrays before its TF steps: harm_amp [B, T],
 * harm_dist [B, T, K], f0_midi [B, T], mags [B, T, M], and (get_controls) the harm_amp
 * divisor [B], drawn once per stream after all of its items.
 *   Seeds mode (seeds [B] non-NULL, each in [0, 2^32)): item b is
 *   np.random.seed(seeds[b]); generate_notes_v2(n_batch=1), one CTA per item, whatever B
 *   and b; key, pos and gauss are ignored.
 *   State mode (seeds NULL): generate_notes_v2(n_batch=B) continuing numpy's state, key
 *   [624] words, pos [2] = (pos, has_gauss) and gauss [1] the cached Gaussian, all
 *   device memory read before and written after the call; one CTA walks the items in
 *   order and every item gets the one divisor.
 * Elementary float64 steps round as numpy's do; cos, sin, pow and log are CUDA's (ulps),
 * and every integer decision is the reference's.  B >= 0; 1 <= min_note_length <=
 * max_note_length; T, K, M >= 1 and within ddsp_b200_synthetic_notes_takes(T, K, M)
 * (T <= DDSP_B200_SYNTHETIC_MAX_T, K and M <= DDSP_B200_SYNTHETIC_MAX_BANDS; more is
 * E_UNSUPPORTED).  No output may overlap an input or another output.  No atomics,
 * bit-reproducible. */
enum {
  DDSP_B200_SYNTHETIC_MAX_T = 8192,     /* a note's blend in shared memory */
  DDSP_B200_SYNTHETIC_MAX_BANDS = 4096  /* a note's two distributions in shared memory */
};
int ddsp_b200_synthetic_notes_takes(int T, int K, int M);
int ddsp_b200_synthetic_notes(const int64_t* seeds, unsigned int* key, int* pos, double* gauss,
                              double* harm_amp, double* harm_dist, double* f0_midi,
                              double* mags, double* divisor, int B, int T, int K, int M,
                              int min_note_length, int max_note_length, double p_silent,
                              double p_vibrato, int get_controls, void* stream);

/* The recurrence of tf.keras.layers.GRU (TF2 defaults: reset_after=True, gate columns
 * z | r | h), as decoders.RnnFcDecoder runs it (nn.Rnn, nn.py:866-879):
 *   z = sigmoid(x W_z + b_z + h U_z + c_z),  r = sigmoid(x W_r + b_r + h U_r + c_r),
 *   h~ = tanh(x W_h + b_h + r * (h U_h + c_h)),  h' = z * h + (1 - z) * h~.
 * Only the sequential part is here; the caller computes x W + b before the forward and
 * the weight, bias and input gradients from d_pre and d_rec after the backward.
 *
 * A handle belongs to one layer on the device that was current at creation and owns
 * the recurrent weights packed for the kernels (6 H^2 + 3 H floats of device memory,
 * freed by _destroy).  units = H must be a multiple of 32 from 32 to 512
 * (ddsp_b200_gru_takes(H); any other H is E_UNSUPPORTED).  Launches of one handle
 * must be ordered on one stream: _load rewrites what later launches read.
 *
 * _load packs recurrent_kernel U [H, 3H] and recurrent_bias c [3H] (one launch).
 * _forward (one launch): gates [B, T, 4H] holds x W + b in its first 3H columns and
 *   receives what the backward reads, z | r | h~ | h U_h + c_h; states [B, T + 1, H]
 *   holds h_0 in row 0 and receives h_1 .. h_T.  gates must not overlap states.
 * _backward (one launch): grad_out [B, T, H] = dL/dh_1 .. h_T -> d_pre [B, T, 3H], the
 *   gradient of x W + b, and d_rec [B, T + 1, 3H], the gradient of h U + c in rows
 *   0 .. T-1 and zeros in row T, from the forward's gates and states and the weights of
 *   the last _load.  Row b (T + 1) + t of d_rec pairs with the same row of states (h_t),
 *   so dU = states^T d_rec is one GEMM over both flat buffers.  d_pre and d_rec overlap
 *   no operand.
 * B = 0 or T = 0 launches nothing.  FP32 in a fixed order: bit-reproducible, and item
 * b's results depend on item b alone.
 * _clusters: how many thread-block clusters of the B-item forward (backward != 0:
 * backward) launch the device runs at once, as its occupancy calculator answered at
 * creation (a pure host query; 0 for a null handle or B < 1). */
typedef struct ddsp_b200_gru ddsp_b200_gru;
int ddsp_b200_gru_takes(int units);
int ddsp_b200_gru_create(ddsp_b200_gru** out, int units);
int ddsp_b200_gru_destroy(ddsp_b200_gru* gru);
int ddsp_b200_gru_clusters(const ddsp_b200_gru* gru, int B, int backward);
int ddsp_b200_gru_load(ddsp_b200_gru* gru, const float* recurrent_kernel,
                       const float* recurrent_bias, void* stream);
int ddsp_b200_gru_forward(ddsp_b200_gru* gru, float* gates, float* states, int B, int T,
                          void* stream);
int ddsp_b200_gru_backward(ddsp_b200_gru* gru, const float* gates, const float* states,
                           const float* grad_out, float* d_pre, float* d_rec, int B, int T,
                           void* stream);

/* nn.Normalize followed by a ReLU, as every site of nn.ResNet runs them (nn.py:699-839),
 * on x [B, HW, C] channels-last (NHWC with H and W flattened) with the C channels in G
 * groups (G = 1 'layer', 32 'group', C 'instance'; normalize_op, nn.py:561-575):
 *   y = max(0, (x - mean) rstd scale[c] + shift[c]),  rstd = 1 / sqrt(var + eps),
 * mean and population variance of each (item, group) over HW and its C / G channels.
 * C must be a multiple of 4 from 4 to 2048 and G must divide it
 * (ddsp_b200_norm_relu_takes(C, G); anything else is E_UNSUPPORTED).  x, y, dy and dx
 * are 16-byte aligned (E_INVALID otherwise).
 * _forward (one launch) writes y [B, HW, C] and the per-(item, group) mean and rstd
 *   [B, G], float32 buffers that autograd.NormReluFn allocates, which are all the
 *   backward needs besides x.
 * _backward (two launches): dy -> dx [B, HW, C] and dscale, dshift [C] summed over
 *   B and HW.  The ReLU mask is recomputed from x with the forward's arithmetic; its
 *   gradient at an input of exactly 0 is 0.  The workspace holds
 *   DDSP_B200_NORM_CLUSTER B 2 C floats (each CTA's per-channel partial sums).
 * No output overlaps an input or another output.  B = 0 or HW = 0 launches nothing
 * and writes nothing.  FP32 with every sum in a fixed order and no atomics:
 * bit-reproducible, and item b's y and dx depend on item b alone. */
#define DDSP_B200_NORM_CLUSTER 8   /* CTAs per item */
int ddsp_b200_norm_relu_takes(int C, int G);
int ddsp_b200_norm_relu_forward(const float* x, const float* scale, const float* shift,
                                void* y, void* mean, void* rstd, int B, int HW, int C, int G,
                                float eps, void* stream);
int ddsp_b200_norm_relu_backward(const float* x, const float* scale, const float* shift,
                                 const float* mean, const float* rstd, const float* dy,
                                 float* dx, float* dscale, float* dshift, void* workspace,
                                 size_t workspace_bytes, int B, int HW, int C, int G,
                                 void* stream);

/* The residual site of nn.DilatedConvStack (nn.py:1153-1324) on the same cluster
 * geometry and statistics pass, over y (the convolution's output) and x (the residual
 * stream), both [B, T, C]:
 *   x_next = x + xh s + h,  r = relu(x_next),
 * with xh = (y - mean) rstd of y's (item, group) statistics as above for G >= 1, or
 * xh = y for G = 0 (norm_type None).  ddsp_b200_norm_residual_takes(C, G): C a multiple
 * of 4 from 4 to 2048, and G = 0 or a divisor of C (anything else is E_UNSUPPORTED).
 * s and h are per channel when ld = 0: scale and shift [C] (nn.Normalize).  When ld > 0
 * (a multiple of 4, at least C) they are per row: item b's row t reads C values from
 * scale + (b T + t) ld and from shift + (b T + t) ld, so a FiLM Dense output [B, T, ld]
 * is read in place (nn.ConditionalNorm: scale = out, shift = out + C).  A null scale with
 * ld > 0 is s = 1 (shift_only).  Row operands (y, x, x_next, r, dy, dx, gx, gr, and the
 * per-row scale, shift, dscale and dshift) are 16-byte aligned (E_INVALID otherwise).
 * _forward (one launch) writes x_next, r unless it is null, and for G >= 1 the
 *   per-(item, group) mean and rstd [B, G] (null for G = 0).
 * _backward: g = gx + gr 1[x_next > 0] (gr may be null, and then x_next too; the
 *   gradient at x_next = 0 is 0) is dx [B, T, C], and dy is the normalization's
 *   backward of g s, with xh recomputed from y with the forward's arithmetic.  ld = 0:
 *   two launches, dscale = sum g xh and dshift = sum g [C] over B and T, through a
 *   workspace of DDSP_B200_NORM_CLUSTER B 2 C floats.  ld > 0: one launch, which writes
 *   g xh per row to dscale (null when scale is) and g to dshift at the forward's offsets
 *   and stride (other columns of the rows are not written; dscale and dshift are
 *   disjoint column blocks); no workspace.
 * No output overlaps an input or another output.  B = 0 or T = 0 launches nothing and
 * writes nothing.  FP32 with every sum in a fixed order and no atomics: bit-reproducible,
 * and item b's outputs depend on item b alone. */
int ddsp_b200_norm_residual_takes(int C, int G);
int ddsp_b200_norm_residual_forward(const float* y, const float* x, const float* scale,
                                    const float* shift, int ld, void* x_next, void* r,
                                    void* mean, void* rstd, int B, int T, int C, int G,
                                    float eps, void* stream);
int ddsp_b200_norm_residual_backward(const float* y, const float* scale, int ld,
                                     const float* x_next, const float* mean, const float* rstd,
                                     const float* gx, const float* gr, float* dy, float* dx,
                                     float* dscale, float* dshift, void* workspace,
                                     size_t workspace_bytes, int B, int T, int C, int G,
                                     void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DDSP_B200_H_ */
