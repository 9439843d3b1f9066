// DDSP controls to notes (training/heuristics.py): the binarizers amp_pooled_outliers,
// power_pooled_outliers, strided_freq_change, remove_short and their compositions
// midi_heuristic / midi_heuristic_power, and the note table of segment_notes.
//
// Binarizer.  One CTA of kMaskThreads per item walks the frames in chunks of one frame
// per thread, stage by stage, with the stages a bit mask:
//   kPool     pooled outliers of v = log(x) (amplitudes) or v = x + shift (power): frame t
//             is on iff mean(w) - num_devs * std(w) < v_t over its padded window w.  The
//             log is correctly rounded (through double).  The statistics are double, two
//             passes over deviations from v_t itself, so a constant window gives exactly
//             0 < 0: off.  A non-finite value in the window
//             turns it off (the reference's std is NaN there).  With pool_positive, also
//             v_t > 0.
//   kStrided  strided_freq_change's transition vector, starting all on: for each width in
//             order, frame t is turned off where the padded window of the vector as it
//             stood before this width is all on and |midi(first) - midi(last)| > 0.75.
//             "All on" is a difference of a block-scanned count of off frames.
//   kF0Pos    and f0 > 0.
//   kRemoveShort  remove_short on the result: a scan places every off frame, so each
//             frame finds the off frames before and after its run.
// Pads repeat int() of the edge values (truncation toward zero).  A non-finite edge value
// of a padded vector is the reference's OverflowError / ValueError: the item's status is
// set and its mask row is all off.  The values, MIDI pitches, counts and positions live
// in a caller-sized global workspace (ddsp_b200_note_heuristic_workspace_bytes).
//
// Note table.  One CTA per item: a scan numbers the runs of on frames, the first and last
// frame of each run write its start and stop, then one warp per note picks its f0 (the
// double sum of the run rounded once to float, or the exact median by a bitwise radix
// select over the run) and its pitch, round-half-even of the float32 hz_to_midi.
#pragma once
#include "common.cuh"
#include "notes.cuh"

namespace ddsp {
namespace heur_ {

using notes_::kMaskThreads;
using notes_::kMaskWarps;

constexpr int kMaxWidths = 8;
constexpr int kPool = 1, kStrided = 2, kF0Pos = 4, kRemoveShort = 8;
constexpr int kPadFront = 0, kPadCenter = 1, kPadEnd = 2;
constexpr int kStatusPoolEdge = 1, kStatusPitchEdge = 2;

// Frames the window of frame t reaches before it under each pad mode.
__host__ __device__ __forceinline__ int pad_before(int mode, int width) {
  return mode == kPadFront ? width - 1 : mode == kPadCenter ? width / 2 : 0;
}

struct Params {
  const float* x;             // [B, T] amplitudes or power (kPool)
  const float* f0;            // [B, T] Hz (kStrided, kF0Pos)
  const uint8_t* on;          // [B, T] input mask when neither kPool nor kStrided
  uint8_t* mask;              // [B, T] out
  int* status;                // [B] out
  float* val;                 // [B, T] workspace: pooled values
  float* midi;                // [B, T] workspace: hz_to_midi(f0)
  int* cnt;                   // [B, T + 1] workspace: counts and positions
  uint8_t* tr;                // [B, T] workspace: transitions
  int T, stages;
  int log_values;             // v = log(x), else v = x + shift
  float shift;
  int pool_width, pool_pad, pool_positive;
  double num_devs;
  int n_widths, widths[kMaxWidths], strided_pad;
  int min_samples, glue_back;
};

// core.hz_to_midi in float32 in the reference's op order:
// 12 * (log(f) / log(2) - log(440) / log(2)) + 69, and 0 where f <= 0.  The logs are
// correctly rounded (through double); no contraction into FMA.
__device__ __forceinline__ float hz_to_midi(float f) {
  if (f <= 0.f) return 0.f;
  const float ln2 = (float)0.69314718055994530942;
  const float c = __fdiv_rn((float)6.0867747269123065 /* log(440) */, ln2);
  const float l = __fdiv_rn((float)log((double)f), ln2);
  return __fadd_rn(__fmul_rn(12.f, __fsub_rn(l, c)), 69.f);
}

// np.round(x).astype(np.int32): half to even; NaN and out-of-range give x86's
// integer-indefinite value -2^31.
__device__ __forceinline__ int round_pitch(float m) {
  const float r = rintf(m);
  return (r >= -2147483648.f && r < 2147483648.f) ? (int)r : INT_MIN;
}

// Value at padded position i (frame index, may be outside [0, T)).
__device__ __forceinline__ float padded(const float* v, int T, float e0, float e1, int i) {
  return i < 0 ? e0 : i >= T ? e1 : v[i];
}

__global__ void __launch_bounds__(kMaskThreads)
note_heuristic_kernel(Params p) {
  __shared__ int itot[kMaskWarps + 1];
  const int64_t b = blockIdx.x;
  const int T = p.T;
  const float* x = p.x + b * T;
  const float* f0 = p.f0 + b * T;
  uint8_t* mask = p.mask + b * T;
  float* val = p.val + b * T;
  float* midi = p.midi + b * T;
  int* cnt = p.cnt + b * (T + 1);
  uint8_t* tr = p.tr + b * T;

  if (p.stages & kPool) {
    for (int t = threadIdx.x; t < T; t += kMaskThreads)
      val[t] = p.log_values ? (float)log((double)x[t]) : __fadd_rn(x[t], p.shift);
  }
  if (p.stages & kStrided) {
    for (int t = threadIdx.x; t < T; t += kMaskThreads) {
      midi[t] = hz_to_midi(f0[t]);
      tr[t] = 1;
    }
  }
  __syncthreads();
  int status = 0;
  if ((p.stages & kPool) && !(isfinite(val[0]) && isfinite(val[T - 1])))
    status = kStatusPoolEdge;
  if ((p.stages & kStrided) && p.n_widths > 0 && !(isfinite(midi[0]) && isfinite(midi[T - 1])))
    status = kStatusPitchEdge;
  if (threadIdx.x == 0) p.status[b] = status;
  if (status) {
    for (int t = threadIdx.x; t < T; t += kMaskThreads) mask[t] = 0;
    return;
  }

  // pooled outliers, or the input mask
  if (p.stages & kPool) {
    const float e0 = truncf(val[0]), e1 = truncf(val[T - 1]);
    const int W = p.pool_width, lo0 = pad_before(p.pool_pad, W);
    for (int t = threadIdx.x; t < T; t += kMaskThreads) {
      const float vt = val[t];
      const double xt = (double)vt;
      double s = 0.0;
      bool finite = true;
      for (int k = 0; k < W; ++k) {
        const float w = padded(val, T, e0, e1, t - lo0 + k);
        finite = finite && isfinite(w);
        s += (double)w - xt;
      }
      bool on = false;
      if (finite) {
        const double mean = s / W;
        double q = 0.0;
        for (int k = 0; k < W; ++k) {
          const double d = ((double)padded(val, T, e0, e1, t - lo0 + k) - xt) - mean;
          q = fma(d, d, q);
        }
        on = mean - p.num_devs * sqrt(q / W) < 0.0;
      }
      if (p.pool_positive) on = on && vt > 0.f;
      mask[t] = on;
    }
  } else if (!(p.stages & kStrided)) {
    for (int t = threadIdx.x; t < T; t += kMaskThreads) mask[t] = p.on[b * T + t] != 0;
  } else {
    for (int t = threadIdx.x; t < T; t += kMaskThreads) mask[t] = 1;
  }

  if (p.stages & kStrided) {
    const float m0 = truncf(midi[0]), m1 = truncf(midi[T - 1]);
    for (int wi = 0; wi < p.n_widths; ++wi) {
      const int W = p.widths[wi], lo0 = pad_before(p.strided_pad, W);
      // cnt[i] = off frames among 0 .. i-1 of the vector before this width
      if (threadIdx.x == 0) cnt[0] = 0;
      int carry = 0;
      for (int t0 = 0; t0 < T; t0 += kMaskThreads) {
        const int t = t0 + threadIdx.x;
        int total;
        const int c = notes_::scan_int(t < T && !tr[t], carry, itot, &total);
        carry = total;
        if (t < T) cnt[t + 1] = c;
      }
      __syncthreads();
      const bool old0 = cnt[1] == 0, old1 = cnt[T] == cnt[T - 1];
      for (int t = threadIdx.x; t < T; t += kMaskThreads) {
        const int lo = t - lo0, hi = lo + W - 1;
        const int a = max(lo, 0), z = min(hi, T - 1);
        const bool all = (lo >= 0 || old0) && (hi < T || old1) && cnt[z + 1] == cnt[a];
        const bool change = fabsf(__fsub_rn(padded(midi, T, m0, m1, lo),
                                            padded(midi, T, m0, m1, hi))) > 0.75f;
        tr[t] = cnt[t + 1] == cnt[t] && !(all && change);
      }
      __syncthreads();
    }
    for (int t = threadIdx.x; t < T; t += kMaskThreads)
      mask[t] = mask[t] && tr[t] && (!(p.stages & kF0Pos) || f0[t] > 0.f);
  } else if (p.stages & kF0Pos) {
    for (int t = threadIdx.x; t < T; t += kMaskThreads) mask[t] = mask[t] && f0[t] > 0.f;
  }
  __syncthreads();

  if (p.stages & kRemoveShort) {
    // cnt[k] = frame of the k-th off frame
    int carry = 0, n_off = 0;
    for (int t0 = 0; t0 < T; t0 += kMaskThreads) {
      const int t = t0 + threadIdx.x;
      const bool off = t < T && !mask[t];
      int total;
      const int c = notes_::scan_int(off, carry, itot, &total);
      carry = total;
      if (off) cnt[c - 1] = t;
    }
    n_off = carry;
    __syncthreads();
    carry = 0;
    for (int t0 = 0; t0 < T; t0 += kMaskThreads) {
      const int t = t0 + threadIdx.x;
      const bool in = t < T;
      const bool on = in && mask[t];
      int total;
      // off frames before t
      const int before = notes_::scan_int(in && !on, carry, itot, &total) - (in && !on);
      carry = total;
      if (!in) continue;
      if (!p.glue_back) {
        // a run that an off frame ends is cleared when shorter than min_samples
        if (on && before < n_off) {
          const int prev = before > 0 ? cnt[before - 1] : -1;
          if (cnt[before] - prev - 1 < p.min_samples) mask[t] = 0;
        }
      } else if (!on && before + 1 < n_off) {
        // the next off frame glues [this frame, it) when its run is short
        if (cnt[before + 1] - t - 1 < p.min_samples) mask[t] = 1;
      }
    }
  }
}

// ---- note table --------------------------------------------------------------------
struct SegParams {
  const uint8_t* mask;   // [B, T]
  const float* f0;       // [B, T]
  int4* notes;           // [B, cap] {start, stop, pitch, f0 bits}
  int* count;            // [B]
  int T, cap, median;
};

__device__ __forceinline__ uint32_t order_key(float v) {
  const uint32_t u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float key_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// The k-th smallest (0-based) of f[lo, hi), no NaN among them, by the warp: a bitwise
// radix select, 32 counting passes over the run.
__device__ uint32_t warp_select(const float* f, int lo, int hi, int k) {
  const int lane = threadIdx.x & 31;
  uint32_t prefix = 0;
  for (int bit = 31; bit >= 0; --bit) {
    int c = 0;
    for (int i = lo + lane; i < hi; i += 32)
      c += ((order_key(f[i]) ^ prefix) >> bit) == 0;   // same high bits, this bit 0
    c = __reduce_add_sync(0xffffffffu, c);
    if (k >= c) {
      k -= c;
      prefix |= 1u << bit;
    }
  }
  return prefix;
}

__global__ void __launch_bounds__(kMaskThreads)
note_segments_kernel(SegParams p) {
  __shared__ int itot[kMaskWarps + 1];
  const int64_t b = blockIdx.x;
  const int T = p.T;
  const uint8_t* m = p.mask + b * T;
  const float* f0 = p.f0 + b * T;
  int4* notes = p.notes + b * p.cap;

  int n = 0;
  for (int t0 = 0; t0 < T; t0 += kMaskThreads) {
    const int t = t0 + threadIdx.x;
    const bool on = t < T && m[t];
    const bool first = on && (t == 0 || !m[t - 1]);
    const bool last = on && (t == T - 1 || !m[t + 1]);
    int total;
    const int idx = notes_::scan_int(first, n, itot, &total) - 1;
    n = total;
    if (first) notes[idx].x = t;
    if (last) notes[idx].y = t + 1;
  }
  __syncthreads();
  if (threadIdx.x == 0) p.count[b] = n;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = warp; j < n; j += kMaskWarps) {
    const int lo = notes[j].x, hi = notes[j].y, len = hi - lo;
    float pick;
    if (!p.median) {
      double s = 0.0;
      for (int i = lo + lane; i < hi; i += 32) s += (double)f0[i];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      pick = (float)(s / len);
    } else {
      bool nan = false;
      for (int i = lo + lane; i < hi; i += 32) nan = nan || isnan(f0[i]);
      if (__any_sync(0xffffffffu, nan)) {
        pick = __int_as_float(0x7fffffff);
      } else {
        const float a = key_value(warp_select(f0, lo, hi, (len - 1) / 2));
        // np.median averages the two middle values in float32
        pick = len & 1 ? a
                       : __fmul_rn(__fadd_rn(a, key_value(warp_select(f0, lo, hi, len / 2))),
                                   0.5f);
      }
    }
    if (lane == 0) {
      notes[j].z = round_pitch(hz_to_midi(pick));
      notes[j].w = __float_as_int(pick);
    }
  }
  for (int j = n + threadIdx.x; j < p.cap; j += kMaskThreads) notes[j] = make_int4(0, 0, 0, 0);
}

}  // namespace heur_
}  // namespace ddsp
