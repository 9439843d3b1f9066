// 1-D Wasserstein distance of two weighted point sets per row (losses.wasserstein_distance,
// losses.py:641-686), forward and backward, one CTA per row.
//
// For row r with values u [Nu], v [Nv] and weights wu, wv, let s = sort(concat(u, v)),
// N = Nu + Nv, delta_i = s_{i+1} - s_i and, for i = 0 .. N-2,
//   D_i = U_i - V_i,  U_i = sum_k wu_k [u_k <= s_i],  V_i likewise,
//   out[r] = (sum_i delta_i |D_i|^p)^(1/p).
// The CDFs are the raw cumulative weights: the reference's normalisation by the weight
// totals is computed and discarded (losses.py:673, 683), so it is not applied here.
//
// Order.  Each element is staged as a 64-bit key: an order-preserving map of its float
// bits in the high word (-0 is mapped to +0 and every NaN to one positive NaN, so NaNs
// sort last) and its concat index in the low word.  One bitonic sort of the keys gives
// TensorFlow's order, which is stable in concat order (u before v, lower index first),
// and decides which element of a tie group takes which value gradient.  The padding to a
// power of two sorts after everything.
//
// CDFs.  A block scan of the signed weights (+wu, -wv) in sorted order gives the running
// difference P_j.  U_i and V_i count every element equal to s_i, so D_i is P read at the
// end of s_i's tie group, found by a reverse min-scan of the group ends.
//
// Backward, with c_i = |D_i|^p, S = sum_i delta_i c_i, G = grad (1/p) S^(1/p - 1) and
// g_i = G delta_i p |D_i|^(p-1) sgn(D_i) (the products in torch's order, so an exact
// D_i = 0 at p < 1, or S = 0 at p > 1, gives NaN as autograd does):
//   d s_j = G c_{j-1} [j >= 1] - G c_j [j <= N-2], written to the element sorted to j;
//   d wu_k = sum_{i: s_i >= u_k} g_i, the reverse scan of g read at the start of u_k's tie
//   group (a forward max-scan of the group starts); d wv_k the same, negated.
// The backward recomputes the order.  Every scan and sum runs in a fixed order (a run of
// L = M / threads elements per thread, then the warps by shuffles, then the warp totals),
// nothing is atomic and nothing but the [R] distances and the four gradients touches
// global memory: bit-reproducible.
#pragma once
#include "common.cuh"

namespace ddsp {
namespace ws_ {

constexpr int kMaxSide = DDSP_B200_WASSERSTEIN_MAX_SIDE;  // elements per side
constexpr int kMinPadded = 64;
constexpr int kMaxThreads = 512;

// The padded sort length of N elements and the threads that run it (one compare-exchange
// per thread per stage up to 512 threads).
__host__ __device__ inline int padded(int n) {
  int m = kMinPadded;
  while (m < n) m <<= 1;
  return m;
}
__host__ __device__ inline int threads_for(int m) {
  return m / 2 < kMaxThreads ? m / 2 : kMaxThreads;
}
// keys (8 B) and three 4-byte arrays per padded element
__host__ inline size_t smem_bytes(int m) { return (size_t)m * (8 + 3 * 4); }

struct Params {
  const float* u;    // [R, Nu]
  const float* v;    // [R, Nv]
  const float* wu;   // [R, Nu]
  const float* wv;   // [R, Nv]
  int Nu, Nv;
  float p, inv_p;    // p and (float)(1 / p)
};

__device__ __forceinline__ uint32_t order_key(float x) {
  if (x == 0.f) x = 0.f;                   // -0 ties with +0
  if (x != x) x = __int_as_float(0x7fc00000);
  const uint32_t b = __float_as_uint(x);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ float key_value(uint64_t key) {
  const uint32_t h = (uint32_t)(key >> 32);
  return __uint_as_float((h & 0x80000000u) ? (h & 0x7fffffffu) : ~h);
}

// Stages the row: keys[i] for the concat order and w[i] = +wu / -wv; the padding gets the
// largest key and no weight.
__device__ __forceinline__ void stage(const Params& p, int64_t r, int m, uint64_t* keys,
                                      float* w) {
  const int n = p.Nu + p.Nv;
  const float* u = p.u + r * p.Nu;
  const float* v = p.v + r * p.Nv;
  const float* wu = p.wu + r * p.Nu;
  const float* wv = p.wv + r * p.Nv;
  for (int i = threadIdx.x; i < m; i += blockDim.x) {
    uint64_t key = ~0ull;
    float wi = 0.f;
    if (i < p.Nu) {
      key = ((uint64_t)order_key(u[i]) << 32) | (uint32_t)i;
      wi = wu[i];
    } else if (i < n) {
      key = ((uint64_t)order_key(v[i - p.Nu]) << 32) | (uint32_t)i;
      wi = -wv[i - p.Nu];
    }
    keys[i] = key;
    w[i] = wi;
  }
  __syncthreads();
}

__device__ __forceinline__ void bitonic_sort(uint64_t* keys, int m) {
  const int half = m >> 1;
  for (int k = 2; k <= m; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < half; i += blockDim.x) {
        const int lo = ((i & ~(j - 1)) << 1) | (i & (j - 1));
        const int hi = lo + j;
        const uint64_t a = keys[lo], b = keys[hi];
        if ((a > b) == ((lo & k) == 0)) {
          keys[lo] = b;
          keys[hi] = a;
        }
      }
      __syncthreads();
    }
  }
}

struct Sum {
  __device__ float operator()(float a, float b) const { return a + b; }
};
struct Min {
  __device__ int operator()(int a, int b) const { return a < b ? a : b; }
};
struct Max {
  __device__ int operator()(int a, int b) const { return a > b ? a : b; }
};

// Inclusive scan of x[0 .. m) in place (from the end when `rev`), in a fixed order:
// thread t scans its run of L = m / blockDim.x elements serially, the run totals are
// scanned by warp shuffles, the warp totals serially by one thread, and each run adds
// the exclusive prefix of the runs before it.  `tot` holds 32 values of T.
template <class T, class Op>
__device__ void block_scan(T* x, int m, bool rev, Op op, T identity, T* tot) {
  const int L = m / blockDim.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int base = threadIdx.x * L;
  T acc = identity;
  for (int k = 0; k < L; ++k) {
    const int e = rev ? m - 1 - (base + k) : base + k;
    acc = op(acc, x[e]);
    x[e] = acc;
  }
  T incl = acc;
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl = op(y, incl);
  }
  if (lane == 31) tot[warp] = incl;
  __syncthreads();
  if (threadIdx.x == 0) {
    const int nw = blockDim.x >> 5;
    for (int w = 1; w < nw; ++w) tot[w] = op(tot[w - 1], tot[w]);
  }
  __syncthreads();
  T prev = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) prev = identity;
  const T prefix = warp > 0 ? op(tot[warp - 1], prev) : prev;
  if (threadIdx.x > 0) {
    for (int k = 0; k < L; ++k) {
      const int e = rev ? m - 1 - (base + k) : base + k;
      x[e] = op(prefix, x[e]);
    }
  }
  __syncthreads();
}

// The sum of every thread's `part` in a fixed order (warp shuffles, then the warp totals
// serially), returned to every thread.
__device__ float block_sum(float part, float* tot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 16; o > 0; o >>= 1) part += __shfl_down_sync(0xffffffffu, part, o);
  if (lane == 0) tot[warp] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = tot[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) s += tot[w];
    tot[32] = s;
  }
  __syncthreads();
  const float s = tot[32];
  __syncthreads();
  return s;
}

__device__ __forceinline__ float abs_pow(float d, float p) {
  return p == 1.f ? fabsf(d) : powf(fabsf(d), p);
}

// The steps the forward and the backward share: stage, sort, and D at every sorted
// position j < N (in d[j]); `w` is left holding the sorted signed weights' scan and `idx`
// the tie-group ends.  Returns this thread's part of S: the sum over its run of
// delta_j |D_j|^p.
__device__ float row_terms(const Params& p, int64_t r, int m, uint64_t* keys, float* w,
                           float* d, int* idx, int* itot, float* ftot) {
  const int n = p.Nu + p.Nv;
  stage(p, r, m, keys, d);   // d holds the weights in concat order until gathered
  bitonic_sort(keys, m);
  for (int j = threadIdx.x; j < m; j += blockDim.x)
    w[j] = j < n ? d[(uint32_t)keys[j]] : 0.f;
  __syncthreads();
  block_scan(w, m, false, Sum(), 0.f, ftot);
  for (int j = threadIdx.x; j < m; j += blockDim.x) {
    const bool end = j >= n - 1 || (keys[j] >> 32) != (keys[j + 1] >> 32);
    idx[j] = end ? j : INT_MAX;
  }
  __syncthreads();
  block_scan(idx, m, true, Min(), INT_MAX, itot);
  for (int j = threadIdx.x; j < m; j += blockDim.x) d[j] = j < n ? w[idx[j]] : 0.f;
  __syncthreads();
  const int L = m / blockDim.x;
  float part = 0.f;
  for (int k = 0; k < L; ++k) {
    const int j = threadIdx.x * L + k;
    if (j < n - 1) part += (key_value(keys[j + 1]) - key_value(keys[j])) * abs_pow(d[j], p.p);
  }
  return part;
}

__global__ void __launch_bounds__(kMaxThreads)
wasserstein_kernel(Params p, float* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ float ftot[33];
  __shared__ int itot[32];
  const int m = padded(p.Nu + p.Nv);
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);
  float* w = reinterpret_cast<float*>(keys + m);
  float* d = w + m;
  int* idx = reinterpret_cast<int*>(d + m);
  const int64_t r = blockIdx.x;
  const float part = row_terms(p, r, m, keys, w, d, idx, itot, ftot);
  const float s = block_sum(part, ftot);
  if (threadIdx.x == 0) out[r] = powf(s, p.inv_p);
}

__global__ void __launch_bounds__(kMaxThreads)
wasserstein_backward_kernel(Params p, const float* __restrict__ grad, float* __restrict__ du,
                            float* __restrict__ dv, float* __restrict__ dwu,
                            float* __restrict__ dwv) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ float ftot[33];
  __shared__ int itot[32];
  const int n = p.Nu + p.Nv;
  const int m = padded(n);
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);
  float* w = reinterpret_cast<float*>(keys + m);
  float* d = w + m;
  int* idx = reinterpret_cast<int*>(d + m);
  const int64_t r = blockIdx.x;
  float* c = w;   // the scan of w is spent once D is in d
  const float part = row_terms(p, r, m, keys, w, d, idx, itot, ftot);
  const float s = block_sum(part, ftot);   // after this barrier w is free for c
  const float G = grad[r] * (p.inv_p * powf(s, p.inv_p - 1.f));
  for (int j = threadIdx.x; j < m; j += blockDim.x) c[j] = j < n - 1 ? abs_pow(d[j], p.p) : 0.f;
  __syncthreads();
  // value gradients through the permutation, and g_j in place of D_j
  for (int j = threadIdx.x; j < m; j += blockDim.x) {
    if (j < n) {
      const float lo = j >= 1 ? G * c[j - 1] : 0.f;
      const float hi = j <= n - 2 ? G * c[j] : 0.f;
      const float ds = lo + (-hi);
      const uint32_t i = (uint32_t)keys[j];
      if (i < (uint32_t)p.Nu) du[r * p.Nu + i] = ds;
      else dv[r * p.Nv + (i - p.Nu)] = ds;
    }
    float gj = 0.f;
    if (j < n - 1) {
      const float dj = d[j];
      const float delta = key_value(keys[j + 1]) - key_value(keys[j]);
      const float dpow = p.p == 1.f ? 1.f : p.p * powf(fabsf(dj), p.p - 1.f);
      const float sgn = dj > 0.f ? 1.f : (dj < 0.f ? -1.f : 0.f);   // torch's sgn: 0 at NaN
      gj = ((G * delta) * dpow) * sgn;
    }
    d[j] = gj;
    const bool head = j == 0 || (j < n && (keys[j] >> 32) != (keys[j - 1] >> 32));
    idx[j] = head ? j : 0;
  }
  __syncthreads();
  block_scan(idx, m, false, Max(), 0, itot);
  block_scan(d, m, true, Sum(), 0.f, ftot);
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const float rj = d[idx[j]];
    const uint32_t i = (uint32_t)keys[j];
    if (i < (uint32_t)p.Nu) dwu[r * p.Nu + i] = rj;
    else dwv[r * p.Nv + (i - p.Nu)] = -rj;
  }
}

}  // namespace ws_
}  // namespace ddsp
