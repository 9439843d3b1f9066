// Host helpers that the entry points of several kernel families (one .cu each)
// share.  A family's own helpers stay in its unit; the harmonic checks are in
// harmonic_common.cuh.
#pragma once

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <initializer_list>
#include <vector>

#include "common.cuh"

namespace ddsp {

static inline int grid_for(int64_t n, int threads, int cap_per_sm = 8) {
  int64_t blocks = (n + threads - 1) / threads;
  int64_t cap = (int64_t)num_sms() * cap_per_sm;
  return (int)std::max<int64_t>(1, std::min(blocks, cap));
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

// Whether the byte ranges [a, a + a_bytes) and [b, b + b_bytes) share a byte (a null
// pointer or an empty range shares none).
inline bool overlaps(const void* a, size_t a_bytes, const void* b, size_t b_bytes) {
  return a && b && a_bytes && b_bytes && (uintptr_t)a < (uintptr_t)b + b_bytes &&
         (uintptr_t)b < (uintptr_t)a + a_bytes;
}

// Elements of an extent given as a product of shape arguments; a negative factor
// (an invalid shape, refused by the entry point's own checks) counts as empty.
inline size_t extent(int64_t a, int64_t b = 1, int64_t c = 1) {
  return (a <= 0 || b <= 0 || c <= 0) ? 0 : (size_t)a * (size_t)b * (size_t)c;
}

// Workspaces are carved from the first 256-byte boundary at or after `p`.
template <typename T>
static T* align256(const void* p) {
  return reinterpret_cast<T*>(((uintptr_t)p + 255) & ~(uintptr_t)255);
}

// A float operand of an entry point: its C parameter name, first element and extent in
// elements.  An output's `may_be` lists, comma-separated, the inputs it may BE.
struct Operand {
  const char* name;
  const void* p;
  size_t n;
  const char* may_be;
};

// Whether the comma-separated list `names` holds `name`.
inline bool lists(const char* names, const char* name) {
  const size_t len = strlen(name);
  for (const char* s = names + strspn(names, ", "); *s; s += strspn(s, ", ")) {
    const size_t n = strcspn(s, ", ");
    if (n == len && !strncmp(s, name, n)) return true;
    s += n;
  }
  return false;
}

// E_INVALID, before any launch, when a float output of entry point `fn` overlaps one
// of its float inputs: a kernel whose threads read inputs that other threads write
// would race.  An output may be an input its `may_be` lists (an elementwise kernel in
// place), but only exactly: same first element and extent.  Walks outputs x inputs in
// order and reports the first pair that overlaps.
inline int check_overlap(const char* fn, std::initializer_list<Operand> outs,
                         std::initializer_list<Operand> ins) {
  for (const Operand& o : outs)
    for (const Operand& i : ins) {
      const bool may_be = lists(o.may_be, i.name);
      if (may_be && o.p == i.p && o.n == i.n) continue;
      if (!overlaps(o.p, sizeof(float) * o.n, i.p, sizeof(float) * i.n)) continue;
      if (may_be)
        set_error("%s: %s must be %s or not overlap it", fn, o.name, i.name);
      else
        set_error("%s: %s must not overlap %s", fn, o.name, i.name);
      return DDSP_B200_E_INVALID;
    }
  return 0;
}

}  // namespace ddsp

// Operands of check_overlap, named after their C parameter.  DDSP_OUT's trailing
// arguments name the inputs the output may be.
#define DDSP_IN(x, n) (::ddsp::Operand{#x, (x), (size_t)(n), ""})
#define DDSP_OUT(x, n, ...) (::ddsp::Operand{#x, (x), (size_t)(n), #__VA_ARGS__})

#define DDSP_CUDA_TRY(expr, what)                                       \
  do {                                                                    \
    cudaError_t e__ = (expr);                                             \
    if (e__ != cudaSuccess) {                                             \
      ::ddsp::set_error("%s: %s", what, cudaGetErrorString(e__));         \
      return DDSP_B200_E_CUDA;                                            \
    }                                                                     \
  } while (0)
