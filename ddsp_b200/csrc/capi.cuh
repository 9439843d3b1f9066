// Host helpers that the entry points of several kernel families (one .cu each)
// share.  A family's own helpers stay in its unit; the harmonic checks are in
// harmonic_common.cuh.
#pragma once

#include <algorithm>
#include <cfloat>
#include <cmath>
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

// Workspaces are carved from the first 256-byte boundary at or after `p`.
template <typename T>
static T* align256(const void* p) {
  return reinterpret_cast<T*>(((uintptr_t)p + 255) & ~(uintptr_t)255);
}

}  // namespace ddsp

#define DDSP_CUDA_TRY(expr, what)                                         \
  do {                                                                    \
    cudaError_t e__ = (expr);                                             \
    if (e__ != cudaSuccess) {                                             \
      ::ddsp::set_error("%s: %s", what, cudaGetErrorString(e__));         \
      return DDSP_B200_E_CUDA;                                            \
    }                                                                     \
  } while (0)
