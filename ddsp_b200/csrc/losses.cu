// C ABI of the loss family: the consistency mixture and comb NLLs,
// sinusoidal_to_harmonic, the HMM, the Wasserstein distance and the note functions of
// the MIDI autoencoder, forward and backward, and its controls-to-notes heuristics.
#include "capi.cuh"
#include "consistency.cuh"
#include "heuristics.cuh"
#include "hmm.cuh"
#include "notes.cuh"
#include "wasserstein.cuh"

using namespace ddsp;

extern "C" {

// ---- consistency-loss mixture NLLs -------------------------------------------------
static int cons_rows(const char* name, int B, int T, int64_t* rows) {
  DDSP_REQUIRE((int64_t)B * T <= DDSP_B200_MAX_ROWS, DDSP_B200_E_INVALID,
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
  rc = check_overlap("mixture_nll_forward", {DDSP_OUT(nll, extent(rows, Q))},
                     {DDSP_IN(x, extent(rows, Q)), DDSP_IN(mu, extent(rows, J)),
                      DDSP_IN(lw, extent(rows, J))});
  if (rc) return rc;
  p.x = x; p.mu = mu; p.lw = lw;
  const size_t smem = sizeof(float) * 2 * (size_t)J;
  return launch("mixture_nll_forward", cons_::mixture_nll_kernel, (unsigned)rows,
                cons_::kThreads, smem, (cudaStream_t)stream, p, nll);
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
  return launch("mixture_nll_backward", cons_::mixture_nll_backward_kernel, (unsigned)rows,
                cons_::kThreads, smem, (cudaStream_t)stream, p, grad, dx, dmu, dlw);
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
  rc = check_overlap("comb_nll_forward", {DDSP_OUT(out, extent(rows, C))},
                     {DDSP_IN(f0, extent(rows, C)), DDSP_IN(f, extent(rows, P)),
                      DDSP_IN(a, extent(rows, P))});
  if (rc) return rc;
  p.f0 = f0; p.f = f; p.a = a;
  const size_t smem = sizeof(float) * (2 * (size_t)P + C + 1);
  return launch("comb_nll_forward", cons_::comb_nll_kernel, (unsigned)rows, cons_::kThreads,
                smem, (cudaStream_t)stream, p, out);
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
  return launch("comb_nll_backward", cons_::comb_nll_backward_kernel, (unsigned)rows,
                cons_::kThreads, smem, (cudaStream_t)stream, p, grad, d_f0, d_f, d_a);
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
  rc = check_overlap("sinusoidal_to_harmonic", {DDSP_OUT(harm_amp, extent(rows)),
                                                DDSP_OUT(harm_dist, extent(rows, K))},
                     {DDSP_IN(sin_amps, extent(rows, S)),
                      DDSP_IN(sin_freqs, extent(rows, S)), DDSP_IN(f0_hz, extent(rows))});
  if (rc) return rc;
  p.a = sin_amps; p.f = sin_freqs; p.f0 = f0_hz;
  const size_t smem = sizeof(float) * (2 * (size_t)S + cons_::kThreads + 1);
  return launch("sinusoidal_to_harmonic", cons_::sin_to_harm_kernel, (unsigned)rows,
                cons_::kThreads, smem, (cudaStream_t)stream, p, harm_amp, harm_dist);
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
  return launch("sinusoidal_to_harmonic_backward", cons_::sin_to_harm_backward_kernel,
                (unsigned)rows, cons_::kThreads, smem, (cudaStream_t)stream, p, grad_amp,
                grad_dist, d_sin_amps, d_sin_freqs, d_f0_hz);
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
  rc = check_overlap("hmm_log_prob", {DDSP_OUT(log_prob, extent(B))},
                     {DDSP_IN(obs, extent(B, T, 2)), DDSP_IN(loc, extent(K, 2)),
                      DDSP_IN(scale, extent(K, 2))});
  if (rc) return rc;
  return launch("hmm_log_prob", hmm_::hmm_log_prob_kernel, (unsigned)B, hmm_threads(K), 0,
                (cudaStream_t)stream, p, log_prob);
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
  return launch("hmm_log_prob_backward", hmm_::hmm_backward_kernel, (unsigned)B,
                hmm_threads(K), smem, (cudaStream_t)stream, p, seg, grad,
                reinterpret_cast<float2*>(d_obs), checkpoints);
}

// Shared bytes of the Viterbi back pointers of T steps of K states.
static size_t hmm_viterbi_smem(int T, int K) {
  return sizeof(uint32_t) * (size_t)T * ((K + 31) / 32 + 1);
}

int ddsp_b200_hmm_viterbi_takes(int T, int K) {
  return T >= 1 && K >= 1 && hmm_viterbi_smem(T, K) <= hmm_::kViterbiBytes;
}

int ddsp_b200_hmm_viterbi(const float* obs, const float* loc, const float* scale,
                          int64_t* path, int B, int T, int K, double hold, double other,
                          void* stream) {
  DDSP_REQUIRE(B == 0 || (obs && loc && scale && path), DDSP_B200_E_INVALID,
               "hmm_viterbi: null pointer");
  hmm_::Params p;
  int rc = hmm_check("hmm_viterbi", obs, loc, scale, B, T, K, hold, other, &p);
  if (rc) return rc;
  const size_t smem = hmm_viterbi_smem(T, K);
  DDSP_REQUIRE(ddsp_b200_hmm_viterbi_takes(T, K), DDSP_B200_E_UNSUPPORTED,
               "hmm_viterbi: T=%d steps of K=%d states need %zu B of back pointers, more "
               "than the %zu supported", T, K, smem, hmm_::kViterbiBytes);
  if (B == 0) return 0;
  return launch("hmm_viterbi", hmm_::hmm_viterbi_kernel, (unsigned)B, hmm_threads(K), smem,
                (cudaStream_t)stream, p, path);
}

// ---- losses.wasserstein_distance ------------------------------------------------------
static int ws_check(const char* name, int64_t R, int Nu, int Nv, float p, ws_::Params* wp) {
  DDSP_REQUIRE(R >= 0 && Nu >= 0 && Nv >= 0, DDSP_B200_E_INVALID,
               "%s: bad shape R=%lld Nu=%d Nv=%d", name, (long long)R, Nu, Nv);
  DDSP_REQUIRE(p > 0.f && p <= FLT_MAX, DDSP_B200_E_INVALID,
               "%s: p must be positive and finite, got %g", name, (double)p);
  DDSP_REQUIRE(Nu <= ws_::kMaxSide && Nv <= ws_::kMaxSide, DDSP_B200_E_UNSUPPORTED,
               "%s: Nu=%d or Nv=%d elements exceed the %d supported per side", name, Nu, Nv,
               ws_::kMaxSide);
  DDSP_REQUIRE(R <= DDSP_B200_MAX_ROWS, DDSP_B200_E_INVALID,
               "%s: R=%lld exceeds the 2^31 - 1 grid limit", name, (long long)R);
  wp->Nu = Nu;
  wp->Nv = Nv;
  wp->p = p;
  wp->inv_p = (float)(1.0 / (double)p);
  return 0;
}

int ddsp_b200_wasserstein_forward(const float* u, const float* v, const float* wu,
                                  const float* wv, float* out, int64_t R, int Nu, int Nv,
                                  float p, void* stream) {
  const bool empty = R == 0 || Nu == 0 || Nv == 0;
  DDSP_REQUIRE(empty || (u && v && wu && wv && out), DDSP_B200_E_INVALID,
               "wasserstein_forward: null pointer");
  ws_::Params wp;
  int rc = ws_check("wasserstein_forward", R, Nu, Nv, p, &wp);
  if (rc || empty) return rc;
  rc = check_overlap("wasserstein_forward", {DDSP_OUT(out, extent(R))},
                     {DDSP_IN(u, extent(R, Nu)), DDSP_IN(v, extent(R, Nv)),
                      DDSP_IN(wu, extent(R, Nu)), DDSP_IN(wv, extent(R, Nv))});
  if (rc) return rc;
  wp.u = u; wp.v = v; wp.wu = wu; wp.wv = wv;
  const int m = ws_::padded(Nu + Nv);
  const size_t smem = ws_::smem_bytes(m);
  return launch("wasserstein_forward", ws_::wasserstein_kernel, (unsigned)R,
                ws_::threads_for(m), smem, (cudaStream_t)stream, wp, out);
}

int ddsp_b200_wasserstein_backward(const float* u, const float* v, const float* wu,
                                   const float* wv, const float* grad, float* du, float* dv,
                                   float* dwu, float* dwv, int64_t R, int Nu, int Nv, float p,
                                   void* stream) {
  const bool empty = R == 0 || Nu == 0 || Nv == 0;
  DDSP_REQUIRE(empty || (u && v && wu && wv && grad && du && dv && dwu && dwv),
               DDSP_B200_E_INVALID, "wasserstein_backward: null pointer");
  ws_::Params wp;
  int rc = ws_check("wasserstein_backward", R, Nu, Nv, p, &wp);
  if (rc || empty) return rc;
  wp.u = u; wp.v = v; wp.wu = wu; wp.wv = wv;
  const int m = ws_::padded(Nu + Nv);
  const size_t smem = ws_::smem_bytes(m);
  return launch("wasserstein_backward", ws_::wasserstein_backward_kernel, (unsigned)R,
                ws_::threads_for(m), smem, (cudaStream_t)stream, wp, grad, du, dv, dwu,
                dwv);
}

// ---- nn.get_note_mask, get_note_moments, pool_over_notes ---------------------------------
// Region decisions of the edge rule with note_on_only: one byte per region that can hold a
// frame (min(R, T)) per item.
static size_t note_mask_regions(int B, int T, int R, int onset, int note_on_only) {
  if (onset || !note_on_only || B <= 0 || T <= 0 || R <= 0) return 0;
  return (size_t)B * (size_t)(R < T ? R : T);
}

int ddsp_b200_note_mask(const float* q, const float* onset, float* mask, void* workspace,
                        size_t workspace_bytes, int B, int T, int R, int note_on_only,
                        void* stream) {
  DDSP_REQUIRE(B >= 0 && T >= 1 && R >= 0, DDSP_B200_E_INVALID,
               "note_mask: bad shape B=%d T=%d R=%d", B, T, R);
  DDSP_REQUIRE(note_on_only == 0 || note_on_only == 1, DDSP_B200_E_INVALID,
               "note_mask: note_on_only must be 0 or 1, got %d", note_on_only);
  const bool empty = B == 0 || R == 0;
  DDSP_REQUIRE(empty || (q && mask), DDSP_B200_E_INVALID, "note_mask: null pointer");
  const size_t need = note_mask_regions(B, T, R, onset != nullptr, note_on_only);
  DDSP_REQUIRE(workspace_bytes >= need && (need == 0 || workspace), DDSP_B200_E_WORKSPACE,
               "note_mask: workspace of %zu B is smaller than the %zu B needed",
               workspace_bytes, need);
  if (empty) return 0;
  int rc = check_overlap("note_mask",
                         {DDSP_OUT(mask, extent(B, onset || T > 1 ? T : 2, R))},
                         {DDSP_IN(q, extent(B, T)), DDSP_IN(onset, extent(B, T))});
  if (rc) return rc;
  notes_::MaskParams p;
  p.q = q;
  p.onset = onset;
  p.on = static_cast<uint8_t*>(workspace);
  p.T = T;
  p.T_out = onset || T > 1 ? T : 2;
  p.R = R;
  p.Rf = R < T ? R : T;
  p.note_on_only = note_on_only;
  auto kern = onset ? notes_::note_mask_kernel<true> : notes_::note_mask_kernel<false>;
  return launch("note_mask", kern, (unsigned)B, notes_::kMaskThreads, 0, (cudaStream_t)stream,
                p, mask);
}

// The shape checks of the moments entry points, and the CTA count of a grid of tiles of
// `rows` rows (notes or frames) by D dims per item.
static int notes_check(const char* name, int B, int T, int N, int D, notes_::Params* p) {
  DDSP_REQUIRE(B >= 0 && T >= 1 && N >= 0 && D >= 0, DDSP_B200_E_INVALID,
               "%s: bad shape B=%d T=%d N=%d D=%d", name, B, T, N, D);
  p->T = T;
  p->N = N;
  p->D = D;
  p->tiles_d = (D + notes_::kDTile - 1) / notes_::kDTile;
  return 0;
}

static int notes_grid(const char* name, int B, int rows, notes_::Params* p, unsigned* grid) {
  p->tiles_r = (rows + notes_::kTile - 1) / notes_::kTile;
  const int64_t ctas = (int64_t)B * p->tiles_r * p->tiles_d;
  DDSP_REQUIRE(ctas <= DDSP_B200_MAX_ROWS, DDSP_B200_E_INVALID,
               "%s: %lld tiles exceed the 2^31 - 1 grid limit", name, (long long)ctas);
  *grid = (unsigned)ctas;
  return 0;
}

int ddsp_b200_note_moments(const float* x, const float* mask, float* mean, float* stdev,
                           float* pooled_mean, float* pooled_std, int B, int T, int N, int D,
                           void* stream) {
  notes_::Params p;
  int rc = notes_check("note_moments", B, T, N, D, &p);
  if (rc) return rc;
  const bool empty = B == 0 || N == 0 || D == 0;
  DDSP_REQUIRE(empty || (x && mask && mean), DDSP_B200_E_INVALID,
               "note_moments: null pointer");
  DDSP_REQUIRE(empty || !pooled_std || (stdev && pooled_mean), DDSP_B200_E_INVALID,
               "note_moments: pooled_std needs std and pooled_mean");
  unsigned grid_n = 0, grid_t = 0;
  rc = notes_grid("note_moments", B, N, &p, &grid_n);
  if (rc) return rc;
  notes_::Params pt = p;
  rc = notes_grid("note_moments", B, T, &pt, &grid_t);
  if (rc) return rc;
  if (B == 0 || D == 0) return 0;
  // `stdev` is the header's `std`, a name the std namespace takes here
  rc = check_overlap("note_moments",
                     {DDSP_OUT(mean, extent(B, N, D)),
                      Operand{"std", stdev, extent(B, N, D), ""},
                      DDSP_OUT(pooled_mean, extent(B, T, D)),
                      DDSP_OUT(pooled_std, extent(B, T, D))},
                     {DDSP_IN(x, extent(B, T, D)), DDSP_IN(mask, extent(B, T, N))});
  if (rc) return rc;
  if (N == 0) {   // nothing to pool: the pooled sums are zero
    const size_t bytes = sizeof(float) * (size_t)B * T * D;
    if (pooled_mean)
      DDSP_CUDA_TRY(cudaMemsetAsync(pooled_mean, 0, bytes, (cudaStream_t)stream), "note_moments");
    if (pooled_std)
      DDSP_CUDA_TRY(cudaMemsetAsync(pooled_std, 0, bytes, (cudaStream_t)stream), "note_moments");
    return 0;
  }
  p.x = pt.x = x;
  p.m = pt.m = mask;
  auto moments = stdev ? notes_::note_moments_kernel<true> : notes_::note_moments_kernel<false>;
  rc = launch("note_moments", moments, grid_n, notes_::kThreads, 0, (cudaStream_t)stream, p,
              mean, stdev);
  if (rc) return rc;
  if (!pooled_mean) return 0;
  const notes_::OverN o{mean, stdev, nullptr};
  auto pool = pooled_std ? notes_::note_over_n_kernel<notes_::kPoolBoth>
                         : notes_::note_over_n_kernel<notes_::kPoolMean>;
  return launch("note_pool", pool, grid_t, notes_::kThreads, 0, (cudaStream_t)stream, pt, o,
                pooled_mean, pooled_std);
}

// The backward's A and C, [B,N,D] floats each, from a 256-byte boundary.
static size_t note_backward_bytes(int B, int N, int D) {
  if (B <= 0 || N <= 0 || D <= 0) return 0;
  return 2 * sizeof(float) * (size_t)B * N * D + 256;
}

int ddsp_b200_note_moments_backward(const float* x, const float* mask, const float* mean,
                                    const float* stdev, const float* grad_mean,
                                    const float* grad_std, const float* grad_pooled_mean,
                                    const float* grad_pooled_std, float* dx, void* workspace,
                                    size_t workspace_bytes, int B, int T, int N, int D,
                                    void* stream) {
  notes_::Params p;
  int rc = notes_check("note_moments_backward", B, T, N, D, &p);
  if (rc) return rc;
  const bool empty = B == 0 || D == 0;
  DDSP_REQUIRE(empty || (x && dx && (N == 0 || (mask && mean))), DDSP_B200_E_INVALID,
               "note_moments_backward: null pointer");
  const bool with_std = grad_std || grad_pooled_std;
  DDSP_REQUIRE(!with_std || stdev || N == 0, DDSP_B200_E_INVALID,
               "note_moments_backward: a std gradient needs std");
  const size_t need = note_backward_bytes(B, N, D);
  DDSP_REQUIRE(workspace_bytes >= need && (need == 0 || workspace), DDSP_B200_E_WORKSPACE,
               "note_moments_backward: workspace of %zu B is smaller than the %zu B needed",
               workspace_bytes, need);
  unsigned grid_n = 0, grid_t = 0;
  rc = notes_grid("note_moments_backward", B, N, &p, &grid_n);
  if (rc) return rc;
  notes_::Params pt = p;
  rc = notes_grid("note_moments_backward", B, T, &pt, &grid_t);
  if (rc) return rc;
  if (empty) return 0;
  if (N == 0) {   // x enters no note
    DDSP_CUDA_TRY(cudaMemsetAsync(dx, 0, sizeof(float) * (size_t)B * T * D,
                                  (cudaStream_t)stream), "note_moments_backward");
    return 0;
  }
  p.x = pt.x = x;
  p.m = pt.m = mask;
  float* A = align256<float>(workspace);
  float* C = A + (size_t)B * N * D;
  const notes_::Grads g{mean, stdev, grad_mean, grad_std, grad_pooled_mean, grad_pooled_std};
  auto moments = with_std ? notes_::note_moments_backward_kernel<true>
                          : notes_::note_moments_backward_kernel<false>;
  rc = launch("note_moments_backward", moments, grid_n, notes_::kThreads, 0,
              (cudaStream_t)stream, p, g, A, with_std ? C : nullptr);
  if (rc) return rc;
  const notes_::OverN o{A, C, mean};
  auto over_n = with_std ? notes_::note_over_n_kernel<notes_::kDxBoth>
                         : notes_::note_over_n_kernel<notes_::kDxMean>;
  return launch("note_moments_backward", over_n, grid_t, notes_::kThreads, 0,
                (cudaStream_t)stream, pt, o, dx, nullptr);
}

// ---- heuristics: binarizers and the note table ------------------------------------------
// The workspace of note_heuristic: per item, the pooled values and MIDI pitches (floats),
// T + 1 counts and T transition bytes, each region 256-byte aligned.
static size_t heur_region(int B, int64_t per_item, size_t elem) {
  return ((size_t)B * (size_t)per_item * elem + 255) & ~(size_t)255;
}

size_t ddsp_b200_note_heuristic_workspace_bytes(int B, int T) {
  if (B <= 0 || T <= 0) return 0;
  return 256 + 2 * heur_region(B, T, sizeof(float)) + heur_region(B, (int64_t)T + 1, sizeof(int)) +
         heur_region(B, T, 1);
}

int ddsp_b200_note_heuristic_takes(int T) {
  return T >= 1 && T <= DDSP_B200_NOTE_HEURISTIC_MAX_T;
}

static int heur_pad(const char* what, int pad) {
  DDSP_REQUIRE(pad == DDSP_B200_HEURISTIC_PAD_FRONT || pad == DDSP_B200_HEURISTIC_PAD_CENTER ||
                   pad == DDSP_B200_HEURISTIC_PAD_END,
               DDSP_B200_E_INVALID, "note_heuristic: unrecognized %s pad mode %d", what, pad);
  return 0;
}

int ddsp_b200_note_heuristic(const float* x, const float* f0, const unsigned char* on,
                             unsigned char* mask, int* status, void* workspace,
                             size_t workspace_bytes, int B, int T, int stages, int log_values,
                             float shift, int pool_width, int pool_pad, int pool_positive,
                             double num_devs, const int* widths, int n_widths,
                             int strided_pad, int min_samples, int glue_back, void* stream) {
  DDSP_REQUIRE(B >= 0 && T >= 1, DDSP_B200_E_INVALID, "note_heuristic: bad shape B=%d T=%d",
               B, T);
  DDSP_REQUIRE(ddsp_b200_note_heuristic_takes(T), DDSP_B200_E_UNSUPPORTED,
               "note_heuristic: T=%d frames exceed the %d supported", T,
               DDSP_B200_NOTE_HEURISTIC_MAX_T);
  DDSP_REQUIRE(stages >= 0 && stages <= 15, DDSP_B200_E_INVALID,
               "note_heuristic: bad stage mask %d", stages);
  const bool pool = stages & heur_::kPool, strided = stages & heur_::kStrided;
  const bool uses_f0 = stages & (heur_::kStrided | heur_::kF0Pos);
  DDSP_REQUIRE(B == 0 || ((!pool || x) && (!uses_f0 || f0) && (pool || strided || on) &&
                          mask && status),
               DDSP_B200_E_INVALID, "note_heuristic: null pointer");
  if (pool) {
    DDSP_REQUIRE(pool_width >= 1, DDSP_B200_E_INVALID,
                 "note_heuristic: frame_width must be at least 1, got %d", pool_width);
    DDSP_REQUIRE(num_devs == num_devs, DDSP_B200_E_INVALID, "note_heuristic: num_devs is NaN");
    int rc = heur_pad("pooled", pool_pad);
    if (rc) return rc;
  }
  if (strided) {
    DDSP_REQUIRE(n_widths >= 0 && n_widths <= DDSP_B200_HEURISTIC_MAX_WIDTHS &&
                     (n_widths == 0 || widths),
                 DDSP_B200_E_INVALID, "note_heuristic: %d frame widths, at most %d", n_widths,
                 DDSP_B200_HEURISTIC_MAX_WIDTHS);
    for (int i = 0; i < n_widths; ++i)
      DDSP_REQUIRE(widths[i] >= 1, DDSP_B200_E_INVALID,
                   "note_heuristic: frame widths must be at least 1, got %d", widths[i]);
    int rc = heur_pad("strided", strided_pad);
    if (rc) return rc;
  }
  const size_t need = ddsp_b200_note_heuristic_workspace_bytes(B, T);
  DDSP_REQUIRE(workspace_bytes >= need && (need == 0 || workspace), DDSP_B200_E_WORKSPACE,
               "note_heuristic: workspace of %zu B is smaller than the %zu B needed",
               workspace_bytes, need);
  if (B == 0) return 0;
  const size_t mb = (size_t)B * T;
  DDSP_REQUIRE(!overlaps(mask, mb, x, pool ? mb * 4 : 0) &&
                   !overlaps(mask, mb, f0, uses_f0 ? mb * 4 : 0) &&
                   !overlaps(status, 4 * (size_t)B, x, pool ? mb * 4 : 0) &&
                   !overlaps(status, 4 * (size_t)B, f0, uses_f0 ? mb * 4 : 0) &&
                   !overlaps(status, 4 * (size_t)B, on, pool || strided ? 0 : mb) &&
                   !overlaps(status, 4 * (size_t)B, mask, mb),
               DDSP_B200_E_INVALID, "note_heuristic: mask and status must not overlap the "
               "inputs or each other");
  DDSP_REQUIRE((const void*)mask == (const void*)on || !overlaps(mask, mb, on, pool || strided ? 0 : mb),
               DDSP_B200_E_INVALID, "note_heuristic: mask must be on or not overlap it");
  heur_::Params p;
  p.x = x;
  p.f0 = f0;
  p.on = on;
  p.mask = mask;
  p.status = status;
  char* ws = align256<char>(workspace);
  p.val = reinterpret_cast<float*>(ws);
  ws += heur_region(B, T, sizeof(float));
  p.midi = reinterpret_cast<float*>(ws);
  ws += heur_region(B, T, sizeof(float));
  p.cnt = reinterpret_cast<int*>(ws);
  ws += heur_region(B, (int64_t)T + 1, sizeof(int));
  p.tr = reinterpret_cast<uint8_t*>(ws);
  p.T = T;
  p.stages = stages;
  p.log_values = log_values != 0;
  p.shift = shift;
  p.pool_width = pool_width;
  p.pool_pad = pool_pad;
  p.pool_positive = pool_positive != 0;
  p.num_devs = num_devs;
  p.n_widths = strided ? n_widths : 0;
  for (int i = 0; i < heur_::kMaxWidths; ++i) p.widths[i] = i < p.n_widths ? widths[i] : 1;
  p.strided_pad = strided_pad;
  p.min_samples = min_samples;
  p.glue_back = glue_back != 0;
  return launch("note_heuristic", heur_::note_heuristic_kernel, (unsigned)B,
                heur_::kMaskThreads, 0, (cudaStream_t)stream, p);
}

int ddsp_b200_note_segments(const unsigned char* mask, const float* f0, ddsp_b200_note* notes,
                            int* count, int B, int T, int median, void* stream) {
  DDSP_REQUIRE(B >= 0 && T >= 1, DDSP_B200_E_INVALID, "note_segments: bad shape B=%d T=%d",
               B, T);
  DDSP_REQUIRE(ddsp_b200_note_heuristic_takes(T), DDSP_B200_E_UNSUPPORTED,
               "note_segments: T=%d frames exceed the %d supported", T,
               DDSP_B200_NOTE_HEURISTIC_MAX_T);
  DDSP_REQUIRE(median == 0 || median == 1, DDSP_B200_E_INVALID,
               "note_segments: median must be 0 or 1, got %d", median);
  DDSP_REQUIRE(B == 0 || (mask && f0 && notes && count), DDSP_B200_E_INVALID,
               "note_segments: null pointer");
  DDSP_REQUIRE((uintptr_t)notes % 16 == 0, DDSP_B200_E_INVALID,
               "note_segments: notes must be 16-byte aligned");
  if (B == 0) return 0;
  const int cap = (T + 1) / 2;
  const size_t mb = (size_t)B * T, nb = (size_t)B * cap * sizeof(ddsp_b200_note);
  DDSP_REQUIRE(!overlaps(notes, nb, mask, mb) && !overlaps(notes, nb, f0, 4 * mb) &&
                   !overlaps(count, 4 * (size_t)B, mask, mb) &&
                   !overlaps(count, 4 * (size_t)B, f0, 4 * mb) &&
                   !overlaps(count, 4 * (size_t)B, notes, nb),
               DDSP_B200_E_INVALID, "note_segments: notes and count must not overlap the "
               "inputs or each other");
  heur_::SegParams p;
  p.mask = mask;
  p.f0 = f0;
  p.notes = reinterpret_cast<int4*>(notes);
  p.count = count;
  p.T = T;
  p.cap = cap;
  p.median = median;
  return launch("note_segments", heur_::note_segments_kernel, (unsigned)B,
                heur_::kMaskThreads, 0, (cudaStream_t)stream, p);
}

}  // extern "C"
