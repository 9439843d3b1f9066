// C ABI of the synthetic training data of InverseSynthesis (synthetic_notes.cuh):
// generate_notes_v2's float64 rows, in seeds mode or from numpy's global state.
#include "capi.cuh"
#include "synthetic_notes.cuh"

using namespace ddsp;

#define SYNTH_DISJOINT(fn, a, a_bytes, b, b_bytes)                                  \
  DDSP_REQUIRE(!overlaps((a), (a_bytes), (b), (b_bytes)), DDSP_B200_E_INVALID,      \
               "%s: %s must not overlap %s", (fn), #a, #b)

extern "C" {

int ddsp_b200_synthetic_notes_takes(int T, int K, int M) {
  return T >= 1 && K >= 1 && M >= 1 && T <= DDSP_B200_SYNTHETIC_MAX_T &&
         K <= DDSP_B200_SYNTHETIC_MAX_BANDS && M <= DDSP_B200_SYNTHETIC_MAX_BANDS;
}

int ddsp_b200_synthetic_notes(const int64_t* seeds, unsigned int* key, int* pos, double* gauss,
                              double* harm_amp, double* harm_dist, double* f0_midi,
                              double* mags, double* divisor, int B, int T, int K, int M,
                              int min_note_length, int max_note_length, double p_silent,
                              double p_vibrato, int get_controls, void* stream) {
  const char* fn = "synthetic_notes";
  DDSP_REQUIRE(B >= 0 && T >= 1 && K >= 1 && M >= 1, DDSP_B200_E_INVALID,
               "%s: bad shape B=%d T=%d K=%d M=%d", fn, B, T, K, M);
  DDSP_REQUIRE(ddsp_b200_synthetic_notes_takes(T, K, M), DDSP_B200_E_UNSUPPORTED,
               "%s: T=%d K=%d M=%d; at most T=%d and K, M=%d", fn, T, K, M,
               DDSP_B200_SYNTHETIC_MAX_T, DDSP_B200_SYNTHETIC_MAX_BANDS);
  DDSP_REQUIRE(min_note_length >= 1 && min_note_length <= max_note_length,
               DDSP_B200_E_INVALID, "%s: note lengths must satisfy 1 <= %d <= %d", fn,
               min_note_length, max_note_length);
  DDSP_REQUIRE(get_controls == 0 || get_controls == 1, DDSP_B200_E_INVALID,
               "%s: get_controls must be 0 or 1", fn);
  const bool state = seeds == nullptr;
  DDSP_REQUIRE(!state || (key && pos && gauss), DDSP_B200_E_INVALID,
               "%s: state mode needs key, pos and gauss", fn);
  if (B == 0 && !state) return 0;
  DDSP_REQUIRE(B == 0 || (harm_amp && harm_dist && f0_midi && mags), DDSP_B200_E_INVALID,
               "%s: null pointer", fn);
  DDSP_REQUIRE(!get_controls || B == 0 || divisor, DDSP_B200_E_INVALID,
               "%s: get_controls needs divisor", fn);
  const size_t bt = extent(B, T) * 8, btk = extent(B, T, K) * 8, btm = extent(B, T, M) * 8;
  const size_t nd = get_controls ? extent(B) * 8 : 0, ns = state ? 0 : extent(B) * 8;
  const size_t nk = state ? 624 * 4 : 0, np_ = state ? 2 * sizeof(int) : 0;
  const size_t ng = state ? 8 : 0;
  const void* outs[] = {harm_amp, harm_dist, f0_midi, mags, divisor, key, pos, gauss};
  const size_t out_bytes[] = {bt, btk, bt, btm, nd, nk, np_, ng};
  const char* names[] = {"harm_amp", "harm_dist", "f0_midi", "mags",
                         "divisor", "key", "pos", "gauss"};
  for (int i = 0; i < 8; ++i) {
    SYNTH_DISJOINT(fn, outs[i], out_bytes[i], seeds, ns);
    for (int j = 0; j < i; ++j)
      DDSP_REQUIRE(!overlaps(outs[i], out_bytes[i], outs[j], out_bytes[j]),
                   DDSP_B200_E_INVALID, "%s: %s must not overlap %s", fn, names[i],
                   names[j]);
  }
  synth_::Params p;
  p.seeds = seeds;
  p.key = reinterpret_cast<uint32_t*>(key);
  p.pos = pos;
  p.gauss = gauss;
  p.harm_amp = harm_amp;
  p.harm_dist = harm_dist;
  p.f0_midi = f0_midi;
  p.mags = mags;
  p.divisor = divisor;
  p.B = B;
  p.T = T;
  p.K = K;
  p.M = M;
  p.min_len = min_note_length;
  p.max_len = max_note_length;
  p.get_controls = get_controls;
  p.p_silent = p_silent;
  p.p_vibrato = p_vibrato;
  const size_t smem = synth_::smem_bytes(T, K, M);
  const unsigned grid = state ? 1u : (unsigned)B;
  return launch(fn, synth_::synthetic_notes_kernel, grid, synth_::kThreads, smem,
                (cudaStream_t)stream, p);
}

}  // extern "C"
