// C ABI of the tone-transfer adjustment kernels (postprocessing.cuh): detect_notes and
// smooth, the QuantileTransformer fit and transform, get_tuning_factor and auto_tune.
#include "capi.cuh"
#include "postprocessing.cuh"

using namespace ddsp;

// The byte range of n elements of T (0 for a negative count).
template <typename T>
static size_t span(int64_t n) {
  return n > 0 ? (size_t)n * sizeof(T) : 0;
}

#define POST_DISJOINT(fn, a, a_bytes, b, b_bytes)                                  \
  DDSP_REQUIRE(!overlaps((a), (a_bytes), (b), (b_bytes)), DDSP_B200_E_INVALID,      \
               "%s: %s must not overlap %s", (fn), #a, #b)

extern "C" {

// ---- detect_notes / smooth -----------------------------------------------------------
// The fixed partition of the mean: chunks of at least kMinChunk frames, at most
// kPartials of them; it depends on n alone.
static int64_t detect_chunk(int64_t n) {
  return std::max<int64_t>(post_::kMinChunk, (n + post_::kPartials - 1) / post_::kPartials);
}

size_t ddsp_b200_detect_notes_workspace_bytes(int64_t n) {
  if (n <= 0) return 0;
  return 256 + (((size_t)post_::kPartials * sizeof(double) + 255) & ~(size_t)255) +
         (size_t)n * sizeof(float);
}

int ddsp_b200_detect_notes(const double* loudness, const double* conf, double* ratio,
                           unsigned char* mask, void* workspace, size_t workspace_bytes, int B,
                           int T, int smoothing, double exponent, double weight, double min_db,
                           double note_threshold, int flags, void* stream) {
  const char* fn = "detect_notes";
  DDSP_REQUIRE(B >= 0 && T >= 1, DDSP_B200_E_INVALID, "%s: bad shape B=%d T=%d", fn, B, T);
  DDSP_REQUIRE(smoothing >= 1, DDSP_B200_E_INVALID,
               "%s: the filter size must be at least 1, got %d", fn, smoothing);
  DDSP_REQUIRE(flags >= 0 && flags <= 7, DDSP_B200_E_INVALID, "%s: bad flags %d", fn, flags);
  const bool smooth_only = flags & DDSP_B200_DETECT_SMOOTH_ONLY;
  DDSP_REQUIRE(B == 0 || (conf && ratio && (smooth_only || (loudness && mask))),
               DDSP_B200_E_INVALID, "%s: null pointer", fn);
  const int64_t n = (int64_t)B * T;
  const size_t need = ddsp_b200_detect_notes_workspace_bytes(n);
  DDSP_REQUIRE(workspace_bytes >= need && (need == 0 || workspace), DDSP_B200_E_WORKSPACE,
               "%s: workspace of %zu B is smaller than the %zu B needed", fn, workspace_bytes,
               need);
  if (B == 0) return 0;
  const size_t nd = span<double>(n), nb = smooth_only ? 0 : (size_t)n;
  const size_t nl = smooth_only ? 0 : nd;
  POST_DISJOINT(fn, ratio, nd, conf, nd);
  POST_DISJOINT(fn, ratio, nd, loudness, nl);
  POST_DISJOINT(fn, mask, nb, conf, nd);
  POST_DISJOINT(fn, mask, nb, loudness, nl);
  POST_DISJOINT(fn, mask, nb, ratio, nd);
  POST_DISJOINT(fn, workspace, need, conf, nd);
  POST_DISJOINT(fn, workspace, need, loudness, nl);
  POST_DISJOINT(fn, workspace, need, ratio, nd);
  POST_DISJOINT(fn, workspace, need, mask, nb);
  post_::DetectParams p;
  p.loud = loudness;
  p.conf = conf;
  p.ratio = ratio;
  p.mask = mask;
  char* ws = align256<char>(workspace);
  p.partial = reinterpret_cast<double*>(ws);
  p.powed = reinterpret_cast<float*>(ws + (((size_t)post_::kPartials * sizeof(double) + 255) &
                                           ~(size_t)255));
  p.n = n;
  p.chunk = detect_chunk(n);
  p.n_partials = (int)((n + p.chunk - 1) / p.chunk);
  p.T = T;
  p.k = smoothing;
  p.flags = flags;
  p.exponent = exponent;
  p.weight = weight;
  p.min_db = min_db;
  p.note_threshold = note_threshold;
  cudaStream_t s = (cudaStream_t)stream;
  int rc = launch("detect_notes (prepare)", post_::detect_prepare_kernel,
                  (unsigned)p.n_partials, post_::kThreads, 0, s, p);
  if (rc) return rc;
  return launch("detect_notes", post_::detect_notes_kernel, grid_for(n, post_::kThreads),
                post_::kThreads, 0, s, p);
}

// ---- QuantileTransformer ---------------------------------------------------------------
int ddsp_b200_quantile_fit(const double* sorted, const int64_t* counts, const double* q,
                           double* quantiles, int64_t n_rows, int F, int nq, int flags,
                           void* stream) {
  const char* fn = "quantile_fit";
  DDSP_REQUIRE(n_rows >= 0 && F >= 0 && nq >= 1, DDSP_B200_E_INVALID,
               "%s: bad shape n_rows=%lld F=%d nq=%d", fn, (long long)n_rows, F, nq);
  DDSP_REQUIRE(F <= 65535, DDSP_B200_E_UNSUPPORTED, "%s: %d columns, at most 65535", fn, F);
  DDSP_REQUIRE(flags == 0 || flags == DDSP_B200_QUANTILE_F32, DDSP_B200_E_INVALID,
               "%s: bad flags %d", fn, flags);
  DDSP_REQUIRE(F == 0 || (sorted && counts && q && quantiles), DDSP_B200_E_INVALID,
               "%s: null pointer", fn);
  if (F == 0) return 0;
  const size_t out = span<double>((int64_t)nq * F);
  POST_DISJOINT(fn, quantiles, out, sorted, span<double>(n_rows * F));
  POST_DISJOINT(fn, quantiles, out, counts, span<int64_t>(F));
  POST_DISJOINT(fn, quantiles, out, q, span<double>(nq));
  post_::FitParams p;
  p.sorted = sorted;
  p.counts = counts;
  p.q = q;
  p.quantiles = quantiles;
  p.n_rows = n_rows;
  p.F = F;
  p.nq = nq;
  p.f32 = flags & DDSP_B200_QUANTILE_F32;
  return launch(fn, post_::quantile_fit_kernel, (unsigned)F, post_::kThreads, 0,
                (cudaStream_t)stream, p);
}

int ddsp_b200_quantile_transform(const double* x, const double* quantiles,
                                 const double* references, double* out, int64_t n, int F,
                                 int nq, int inverse, int distribution, int flags,
                                 void* stream) {
  const char* fn = "quantile_transform";
  DDSP_REQUIRE(n >= 0 && F >= 0 && nq >= 1, DDSP_B200_E_INVALID,
               "%s: bad shape n=%lld F=%d nq=%d", fn, (long long)n, F, nq);
  DDSP_REQUIRE(nq <= DDSP_B200_QUANTILE_MAX_N, DDSP_B200_E_UNSUPPORTED,
               "%s: %d quantiles, at most %d", fn, nq, DDSP_B200_QUANTILE_MAX_N);
  DDSP_REQUIRE(F <= 65535, DDSP_B200_E_UNSUPPORTED, "%s: %d columns, at most 65535", fn, F);
  DDSP_REQUIRE(inverse == 0 || inverse == 1, DDSP_B200_E_INVALID, "%s: inverse must be 0 or 1",
               fn);
  DDSP_REQUIRE(distribution == DDSP_B200_QUANTILE_UNIFORM ||
                   distribution == DDSP_B200_QUANTILE_NORMAL,
               DDSP_B200_E_INVALID, "%s: unknown output distribution %d", fn, distribution);
  DDSP_REQUIRE(flags == 0 || flags == DDSP_B200_QUANTILE_F32, DDSP_B200_E_INVALID,
               "%s: bad flags %d", fn, flags);
  DDSP_REQUIRE(n == 0 || F == 0 || (x && quantiles && references && out), DDSP_B200_E_INVALID,
               "%s: null pointer", fn);
  if (n == 0 || F == 0) return 0;
  const size_t nb = span<double>(n * F);
  POST_DISJOINT(fn, out, nb, x, nb);
  POST_DISJOINT(fn, out, nb, quantiles, span<double>((int64_t)nq * F));
  POST_DISJOINT(fn, out, nb, references, span<double>(nq));
  post_::TransformParams p;
  p.x = x;
  p.quantiles = quantiles;
  p.references = references;
  p.out = out;
  p.n = n;
  p.F = F;
  p.nq = nq;
  p.inverse = inverse;
  p.normal = distribution == DDSP_B200_QUANTILE_NORMAL;
  p.f32 = flags & DDSP_B200_QUANTILE_F32;
  const size_t smem = 2 * (size_t)nq * sizeof(double);
  const int64_t row_blocks = (n + post_::kThreads - 1) / post_::kThreads;
  const int64_t cap = std::max<int64_t>(1, (int64_t)num_sms() * 8 / F);
  const dim3 grid((unsigned)std::min(row_blocks, cap), (unsigned)F);
  return launch(fn, post_::quantile_transform_kernel, grid, post_::kThreads, smem,
                (cudaStream_t)stream, p);
}

// ---- get_tuning_factor / auto_tune -----------------------------------------------------
int ddsp_b200_tuning_factor(const double* f0, const double* conf, const double* factors,
                            double* costs, int* index, int64_t N, int n_factors, void* stream) {
  const char* fn = "tuning_factor";
  DDSP_REQUIRE(N >= 0, DDSP_B200_E_INVALID, "%s: bad frame count %lld", fn, (long long)N);
  DDSP_REQUIRE(n_factors >= 1 && n_factors <= DDSP_B200_TUNING_MAX_FACTORS, DDSP_B200_E_INVALID,
               "%s: %d tuning factors, 1 to %d", fn, n_factors, DDSP_B200_TUNING_MAX_FACTORS);
  DDSP_REQUIRE((N == 0 || (f0 && conf)) && factors && costs && index, DDSP_B200_E_INVALID,
               "%s: null pointer", fn);
  const size_t cb = span<double>(2 * (int64_t)n_factors), nb = span<double>(N);
  POST_DISJOINT(fn, costs, cb, f0, nb);
  POST_DISJOINT(fn, costs, cb, conf, nb);
  POST_DISJOINT(fn, costs, cb, factors, span<double>(n_factors));
  POST_DISJOINT(fn, index, sizeof(int), f0, nb);
  POST_DISJOINT(fn, index, sizeof(int), conf, nb);
  POST_DISJOINT(fn, index, sizeof(int), factors, span<double>(n_factors));
  POST_DISJOINT(fn, index, sizeof(int), costs, cb);
  post_::TuningParams p;
  p.f0 = f0;
  p.conf = conf;
  p.factors = factors;
  p.costs = costs;
  p.index = index;
  p.N = N;
  p.n_factors = n_factors;
  cudaStream_t s = (cudaStream_t)stream;
  int rc = launch("tuning_factor (costs)", post_::tuning_costs_kernel, (unsigned)n_factors,
                  post_::kThreads, 0, s, p);
  if (rc) return rc;
  return launch(fn, post_::tuning_argmin_kernel, 1, 32, 0, s, p);
}

int ddsp_b200_auto_tune(const double* f0, const double* f0_on, double* scale_cost,
                        int* scale_index, double* out, int64_t T, int64_t N,
                        double tuning_factor, double amount, int chromatic, int flags,
                        void* stream) {
  const char* fn = "auto_tune";
  DDSP_REQUIRE(T >= 0 && N >= 0, DDSP_B200_E_INVALID, "%s: bad shape T=%lld N=%lld", fn,
               (long long)T, (long long)N);
  DDSP_REQUIRE(chromatic == 0 || chromatic == 1, DDSP_B200_E_INVALID,
               "%s: chromatic must be 0 or 1", fn);
  DDSP_REQUIRE(flags == 0 || (flags == DDSP_B200_AUTO_TUNE_F32 && chromatic),
               DDSP_B200_E_INVALID, "%s: bad flags %d (float32 is chromatic only)", fn, flags);
  DDSP_REQUIRE((T == 0 || (f0 && out)) &&
                   (chromatic || ((N == 0 || f0_on) && scale_cost && scale_index)),
               DDSP_B200_E_INVALID, "%s: null pointer", fn);
  const size_t tb = span<double>(T), nb = span<double>(N);
  const size_t cb = chromatic ? 0 : span<double>(12), ib = chromatic ? 0 : sizeof(int);
  POST_DISJOINT(fn, out, tb, f0, tb);
  POST_DISJOINT(fn, out, tb, f0_on, chromatic ? 0 : nb);
  POST_DISJOINT(fn, scale_cost, cb, f0, tb);
  POST_DISJOINT(fn, scale_cost, cb, f0_on, nb);
  POST_DISJOINT(fn, scale_cost, cb, out, tb);
  POST_DISJOINT(fn, scale_index, ib, f0, tb);
  POST_DISJOINT(fn, scale_index, ib, f0_on, nb);
  POST_DISJOINT(fn, scale_index, ib, out, tb);
  POST_DISJOINT(fn, scale_index, ib, scale_cost, cb);
  post_::AutoTuneParams p;
  p.f0 = f0;
  p.f0_on = f0_on;
  p.scale_cost = scale_cost;
  p.scale_index = scale_index;
  p.out = out;
  p.T = T;
  p.N = N;
  p.tuning_factor = tuning_factor;
  p.amount = amount;
  p.chromatic = chromatic;
  p.f32 = flags & DDSP_B200_AUTO_TUNE_F32;
  cudaStream_t s = (cudaStream_t)stream;
  int rc = 0;
  if (!chromatic) {
    rc = launch("auto_tune (scales)", post_::scale_costs_kernel, 12, post_::kThreads, 0, s, p);
    if (rc) return rc;
  }
  if (T > 0 || !chromatic)
    rc = launch(fn, post_::auto_tune_kernel, grid_for(std::max<int64_t>(T, 1), post_::kThreads),
                post_::kThreads, 0, s, p);
  return rc;
}

}  // extern "C"
