// C ABI of the network layers' kernels: the GRU handle (gru.cuh), which owns the packed
// recurrent weights of one layer on one device, and its pack, forward and
// backward-through-time launches; the ResNet's fused normalize + ReLU and the dilated
// convolution stack's residual site (norm.cuh).
#include "capi.cuh"
#include "gru.cuh"
#include "norm.cuh"

using namespace ddsp;

struct ddsp_b200_gru {
  int device = -1;
  int H = 0;
  float* pack = nullptr;   // forward blocks, backward blocks, c: 6 H^2 + 3 H floats
  bool loaded = false;
  // clusters of each launch that fit on the device at once (0: it does not fit)
  int fwd_clusters[kGruMaxSlice] = {};
  int bwd_clusters[kGruMaxSlice] = {};
};

namespace {

template <int BS>
void* gru_kernel(int H, bool backward) {
  if (gru_chunks(H) == 4)
    return backward ? (void*)gru_backward_kernel<kGruRegRowsBwd, BS>
                    : (void*)gru_forward_kernel<kGruRegRowsFwd, BS>;
  return backward ? (void*)gru_backward_kernel<0, BS> : (void*)gru_forward_kernel<0, BS>;
}

void* gru_kernel(int H, int BS, bool backward) {
  switch (BS) {
    case 1: return gru_kernel<1>(H, backward);
    case 2: return gru_kernel<2>(H, backward);
    case 3: return gru_kernel<3>(H, backward);
    default: return gru_kernel<4>(H, backward);
  }
}

// How many clusters of the launch (H, BS, direction) the device runs at once, asked of
// the occupancy calculator; 0 when its shared memory does not fit.
int gru_max_clusters(int H, int BS, bool backward) {
  const size_t smem = gru_smem_bytes(H, BS, backward);
  if (smem > kGruMaxSmem) return 0;
  const void* kern = gru_kernel(H, BS, backward);
  // The calculator needs the reservation the launch will make, so this is the one place
  // outside launch() that sets it (launch() sets it again before every launch).
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
      cudaSuccess) {
    (void)cudaGetLastError();
    return 0;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(kGruCluster);
  cfg.blockDim = dim3(gru_chunks(H) * (H / kGruCluster));
  cfg.dynamicSmemBytes = smem;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) {
    (void)cudaGetLastError();
    return 0;
  }
  return n;
}

// Items per cluster for B items: the smallest slice whose clusters all run at once, or
// else the largest that fits (the clusters then run in waves).  0: nothing fits.
int gru_slice(const int* clusters, int B) {
  int best = 0;
  for (int bs = 1; bs <= kGruMaxSlice; ++bs) {
    if (clusters[bs - 1] <= 0) continue;
    best = bs;
    if ((B + bs - 1) / bs <= clusters[bs - 1]) return bs;
  }
  return best;
}

// The handle's own checks: not null, loaded, and on the current device.
int gru_check(const ddsp_b200_gru* gru, const char* fn) {
  DDSP_REQUIRE(gru != nullptr, DDSP_B200_E_INVALID, "%s: null handle", fn);
  int dev = 0;
  DDSP_CUDA_TRY(cudaGetDevice(&dev), fn);
  DDSP_REQUIRE(dev == gru->device, DDSP_B200_E_INVALID,
               "%s: the handle belongs to device %d, the current device is %d", fn,
               gru->device, dev);
  return 0;
}

template <int RR, int BS>
int launch_gru_forward(const ddsp_b200_gru* g, float* gates, float* states, int B, int T,
                       cudaStream_t st) {
  const int H = g->H;
  return launch("gru_forward", gru_forward_kernel<RR, BS>,
                dim3(kGruCluster * ((B + BS - 1) / BS)), dim3(gru_chunks(H) * (H / kGruCluster)),
                gru_smem_bytes(H, BS, false), st, (const float*)g->pack, gates, states, B, T, H);
}

template <int RR, int BS>
int launch_gru_backward(const ddsp_b200_gru* g, const float* gates, const float* states,
                        const float* grad_out, float* d_pre, float* d_rec, int B, int T,
                        cudaStream_t st) {
  const int H = g->H;
  return launch("gru_backward", gru_backward_kernel<RR, BS>,
                dim3(kGruCluster * ((B + BS - 1) / BS)), dim3(gru_chunks(H) * (H / kGruCluster)),
                gru_smem_bytes(H, BS, true), st, (const float*)g->pack, gates, states,
                grad_out, d_pre, d_rec, B, T, H);
}

template <int BS>
int gru_forward_bs(const ddsp_b200_gru* g, float* gates, float* states, int B, int T,
                   cudaStream_t st) {
  return gru_chunks(g->H) == 4
             ? launch_gru_forward<kGruRegRowsFwd, BS>(g, gates, states, B, T, st)
             : launch_gru_forward<0, BS>(g, gates, states, B, T, st);
}

template <int BS>
int gru_backward_bs(const ddsp_b200_gru* g, const float* gates, const float* states,
                    const float* grad_out, float* d_pre, float* d_rec, int B, int T,
                    cudaStream_t st) {
  return gru_chunks(g->H) == 4
             ? launch_gru_backward<kGruRegRowsBwd, BS>(g, gates, states, grad_out, d_pre,
                                                       d_rec, B, T, st)
             : launch_gru_backward<0, BS>(g, gates, states, grad_out, d_pre, d_rec, B, T, st);
}

}  // namespace

extern "C" {

int ddsp_b200_gru_takes(int units) { return units >= 32 && units <= 512 && units % 32 == 0; }

int ddsp_b200_gru_create(ddsp_b200_gru** out, int units) {
  const char* fn = "gru_create";
  DDSP_REQUIRE(out != nullptr, DDSP_B200_E_INVALID, "%s: null out", fn);
  *out = nullptr;
  DDSP_REQUIRE(ddsp_b200_gru_takes(units), DDSP_B200_E_UNSUPPORTED,
               "%s: units=%d; the GRU takes multiples of 32 from 32 to 512", fn, units);
  int dev = 0;
  DDSP_CUDA_TRY(cudaGetDevice(&dev), "gru_create: cudaGetDevice");
  ddsp_b200_gru* g = new ddsp_b200_gru();
  g->device = dev;
  g->H = units;
  const size_t n = 6 * (size_t)units * units + 3 * (size_t)units;
  cudaError_t e = cudaMalloc(&g->pack, n * sizeof(float));
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    delete g;
    set_error("%s: cudaMalloc(%zu B): %s", fn, n * sizeof(float), cudaGetErrorString(e));
    return DDSP_B200_E_CUDA;
  }
  for (int bs = 1; bs <= kGruMaxSlice; ++bs) {
    g->fwd_clusters[bs - 1] = gru_max_clusters(units, bs, false);
    g->bwd_clusters[bs - 1] = gru_max_clusters(units, bs, true);
  }
  *out = g;
  return 0;
}

int ddsp_b200_gru_destroy(ddsp_b200_gru* gru) {
  if (!gru) return 0;
  int cur = 0;
  cudaGetDevice(&cur);
  cudaSetDevice(gru->device);
  cudaFree(gru->pack);   // waits for the handle's queued launches to finish
  cudaSetDevice(cur);
  delete gru;
  return 0;
}

int ddsp_b200_gru_clusters(const ddsp_b200_gru* gru, int B, int backward) {
  if (!gru || B < 1) return 0;
  const int* c = backward ? gru->bwd_clusters : gru->fwd_clusters;
  const int bs = gru_slice(c, B);
  return bs ? c[bs - 1] : 0;
}

int ddsp_b200_gru_load(ddsp_b200_gru* gru, const float* recurrent_kernel,
                       const float* recurrent_bias, void* stream) {
  const char* fn = "gru_load";
  DDSP_REQUIRE(gru != nullptr, DDSP_B200_E_INVALID, "%s: null handle", fn);
  DDSP_REQUIRE(recurrent_kernel && recurrent_bias, DDSP_B200_E_INVALID, "%s: null pointer", fn);
  if (int rc = gru_check(gru, fn)) return rc;
  const int H = gru->H;
  if (int rc = check_overlap(fn, {DDSP_OUT(gru->pack, 6 * (size_t)H * H + 3 * H)},
                             {DDSP_IN(recurrent_kernel, 3 * (size_t)H * H),
                              DDSP_IN(recurrent_bias, 3 * H)}))
    return rc;
  const int64_t n = 6LL * H * H + 3 * H;
  int rc = launch("gru_pack", gru_pack_kernel, dim3(grid_for(n, 256)), dim3(256), 0,
                  (cudaStream_t)stream, recurrent_kernel, recurrent_bias, gru->pack, H);
  if (rc) return rc;
  gru->loaded = true;
  return 0;
}

int ddsp_b200_gru_forward(ddsp_b200_gru* gru, float* gates, float* states, int B, int T,
                          void* stream) {
  const char* fn = "gru_forward";
  DDSP_REQUIRE(gru != nullptr, DDSP_B200_E_INVALID, "%s: null handle", fn);
  DDSP_REQUIRE(B >= 0 && T >= 0, DDSP_B200_E_INVALID, "%s: bad shape B=%d T=%d", fn, B, T);
  if (B == 0 || T == 0) return 0;
  DDSP_REQUIRE(gates && states, DDSP_B200_E_INVALID, "%s: null pointer", fn);
  if (int rc = gru_check(gru, fn)) return rc;
  DDSP_REQUIRE(gru->loaded, DDSP_B200_E_INVALID,
               "%s: no recurrent weights: call ddsp_b200_gru_load first", fn);
  const int H = gru->H;
  if (int rc = check_overlap(fn, {DDSP_OUT(gates, extent(B, T, 4 * H))},
                             {DDSP_IN(states, extent(B, T + 1, H))}))
    return rc;
  const int bs = gru_slice(gru->fwd_clusters, B);
  DDSP_REQUIRE(bs > 0, DDSP_B200_E_UNSUPPORTED,
               "%s: no cluster of the H=%d recurrence fits on this device", fn, H);
  cudaStream_t st = (cudaStream_t)stream;
  switch (bs) {
    case 1: return gru_forward_bs<1>(gru, gates, states, B, T, st);
    case 2: return gru_forward_bs<2>(gru, gates, states, B, T, st);
    case 3: return gru_forward_bs<3>(gru, gates, states, B, T, st);
    default: return gru_forward_bs<4>(gru, gates, states, B, T, st);
  }
}

int ddsp_b200_gru_backward(ddsp_b200_gru* gru, const float* gates, const float* states,
                           const float* grad_out, float* d_pre, float* d_rec, int B, int T,
                           void* stream) {
  const char* fn = "gru_backward";
  DDSP_REQUIRE(gru != nullptr, DDSP_B200_E_INVALID, "%s: null handle", fn);
  DDSP_REQUIRE(B >= 0 && T >= 0, DDSP_B200_E_INVALID, "%s: bad shape B=%d T=%d", fn, B, T);
  if (B == 0 || T == 0) return 0;
  DDSP_REQUIRE(gates && states && grad_out && d_pre && d_rec, DDSP_B200_E_INVALID,
               "%s: null pointer", fn);
  if (int rc = gru_check(gru, fn)) return rc;
  DDSP_REQUIRE(gru->loaded, DDSP_B200_E_INVALID,
               "%s: no recurrent weights: call ddsp_b200_gru_load first", fn);
  const int H = gru->H;
  const size_t n_pre = extent(B, T, 3 * H), n_rec = extent(B, T + 1, 3 * H);
  DDSP_REQUIRE(!overlaps(d_pre, n_pre * sizeof(float), d_rec, n_rec * sizeof(float)),
               DDSP_B200_E_INVALID, "%s: d_pre must not overlap d_rec", fn);
  if (int rc = check_overlap(fn, {DDSP_OUT(d_pre, n_pre), DDSP_OUT(d_rec, n_rec)},
                             {DDSP_IN(gates, extent(B, T, 4 * H)),
                              DDSP_IN(states, extent(B, T + 1, H)),
                              DDSP_IN(grad_out, extent(B, T, H))}))
    return rc;
  const int bs = gru_slice(gru->bwd_clusters, B);
  DDSP_REQUIRE(bs > 0, DDSP_B200_E_UNSUPPORTED,
               "%s: no cluster of the H=%d recurrence fits on this device", fn, H);
  cudaStream_t st = (cudaStream_t)stream;
  switch (bs) {
    case 1: return gru_backward_bs<1>(gru, gates, states, grad_out, d_pre, d_rec, B, T, st);
    case 2: return gru_backward_bs<2>(gru, gates, states, grad_out, d_pre, d_rec, B, T, st);
    case 3: return gru_backward_bs<3>(gru, gates, states, grad_out, d_pre, d_rec, B, T, st);
    default: return gru_backward_bs<4>(gru, gates, states, grad_out, d_pre, d_rec, B, T, st);
  }
}

int ddsp_b200_norm_relu_takes(int C, int G) {
  return C >= 4 && C <= kNormMaxChannels && C % 4 == 0 && G >= 1 && C % G == 0;
}

}  // extern "C"

namespace {

// The checks both directions share: shape, takes-query and the float4 alignment of the
// [B, HW, C] operands.  Returns 0, or the status with the error set.
int norm_relu_check(const char* fn, int B, int HW, int C, int G,
                    std::initializer_list<const void*> rows) {
  DDSP_REQUIRE(B >= 0 && HW >= 0, DDSP_B200_E_INVALID, "%s: bad shape B=%d HW=%d", fn, B, HW);
  DDSP_REQUIRE(ddsp_b200_norm_relu_takes(C, G), DDSP_B200_E_UNSUPPORTED,
               "%s: C=%d channels in G=%d groups; the kernel takes C a multiple of 4 from 4 "
               "to %d, in groups that divide it", fn, C, G, kNormMaxChannels);
  for (const void* p : rows)
    DDSP_REQUIRE(((uintptr_t)p & 15) == 0, DDSP_B200_E_INVALID,
                 "%s: the [B, HW, C] operands must be 16-byte aligned", fn);
  return 0;
}

}  // namespace

extern "C" {

int ddsp_b200_norm_relu_forward(const float* x, const float* scale, const float* shift,
                                void* y_out, void* mean_out, void* rstd_out, int B, int HW,
                                int C, int G, float eps, void* stream) {
  const char* fn = "norm_relu_forward";
  float* y = static_cast<float*>(y_out);
  float* mean = static_cast<float*>(mean_out);
  float* rstd = static_cast<float*>(rstd_out);
  if (int rc = norm_relu_check(fn, B, HW, C, G, {x, y})) return rc;
  if (B == 0 || HW == 0) return 0;
  DDSP_REQUIRE(x && scale && shift && y && mean && rstd, DDSP_B200_E_INVALID,
               "%s: null pointer", fn);
  const size_t n = extent(B, HW, C);
  if (int rc = check_overlap(fn, {DDSP_OUT(y, n), DDSP_OUT(mean, extent(B, G)),
                                  DDSP_OUT(rstd, extent(B, G))},
                             {DDSP_IN(x, n), DDSP_IN(scale, C), DDSP_IN(shift, C)}))
    return rc;
  DDSP_REQUIRE(!overlaps(y, n * sizeof(float), mean, extent(B, G) * sizeof(float)) &&
                   !overlaps(y, n * sizeof(float), rstd, extent(B, G) * sizeof(float)) &&
                   !overlaps(mean, extent(B, G) * sizeof(float), rstd,
                             extent(B, G) * sizeof(float)),
               DDSP_B200_E_INVALID, "%s: y, mean and rstd must not overlap", fn);
  return launch("norm_relu_forward", norm_relu_forward_kernel, dim3(kNormCluster * B),
                dim3(kNormThreads), norm_smem_bytes(C, G, false), (cudaStream_t)stream, x,
                scale, shift, y, mean, rstd, HW, C, G, eps);
}

int ddsp_b200_norm_relu_backward(const float* x, const float* scale, const float* shift,
                                 const float* mean, const float* rstd, const float* dy,
                                 float* dx, float* dscale, float* dshift, void* workspace,
                                 size_t workspace_bytes, int B, int HW, int C, int G,
                                 void* stream) {
  const char* fn = "norm_relu_backward";
  if (int rc = norm_relu_check(fn, B, HW, C, G, {x, dy, dx})) return rc;
  if (B == 0 || HW == 0) return 0;
  DDSP_REQUIRE(x && scale && shift && mean && rstd && dy && dx && dscale && dshift &&
                   workspace, DDSP_B200_E_INVALID, "%s: null pointer", fn);
  const size_t n = extent(B, HW, C), np = extent(B, kNormCluster, 2 * C);
  DDSP_REQUIRE(workspace_bytes >= np * sizeof(float), DDSP_B200_E_INVALID,
               "%s: the workspace has %zu B, it needs %zu", fn, workspace_bytes,
               np * sizeof(float));
  float* partial = static_cast<float*>(workspace);
  if (int rc = check_overlap(fn, {DDSP_OUT(dx, n), DDSP_OUT(dscale, C), DDSP_OUT(dshift, C),
                                  DDSP_OUT(partial, np)},
                             {DDSP_IN(x, n), DDSP_IN(scale, C), DDSP_IN(shift, C),
                              DDSP_IN(mean, extent(B, G)), DDSP_IN(rstd, extent(B, G)),
                              DDSP_IN(dy, n)}))
    return rc;
  DDSP_REQUIRE(!overlaps(dx, n * sizeof(float), dscale, C * sizeof(float)) &&
                   !overlaps(dx, n * sizeof(float), dshift, C * sizeof(float)) &&
                   !overlaps(dscale, C * sizeof(float), dshift, C * sizeof(float)) &&
                   !overlaps(partial, np * sizeof(float), dx, n * sizeof(float)) &&
                   !overlaps(partial, np * sizeof(float), dscale, C * sizeof(float)) &&
                   !overlaps(partial, np * sizeof(float), dshift, C * sizeof(float)),
               DDSP_B200_E_INVALID, "%s: dx, dscale, dshift and the workspace must not "
               "overlap", fn);
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = launch("norm_relu_backward", norm_relu_backward_kernel, dim3(kNormCluster * B),
                      dim3(kNormThreads), norm_smem_bytes(C, G, true), st, x, scale, shift,
                      mean, rstd, dy, dx, partial, HW, C, G))
    return rc;
  return launch("norm_relu_param_grad", norm_relu_param_grad_kernel,
                dim3((2 * C + 255) / 256), dim3(256), 0, st, (const float*)partial, dscale,
                dshift, kNormCluster * B, C);
}

int ddsp_b200_norm_residual_takes(int C, int G) {
  return C >= 4 && C <= kNormMaxChannels && C % 4 == 0 && G >= 0 && (G == 0 || C % G == 0);
}

}  // extern "C"

namespace {

// Elements from the first to the last of B T rows of C at stride ld (ld = 0: C alone).
size_t row_extent(int B, int T, int C, int ld) {
  const size_t rows = extent(B, T);
  return ld == 0 ? (size_t)C : rows ? (rows - 1) * (size_t)ld + C : 0;
}

// Whether no two of the float ranges (first element, extent) share a byte.
bool pairwise_disjoint(std::initializer_list<std::pair<const void*, size_t>> ranges) {
  for (auto a = ranges.begin(); a != ranges.end(); ++a)
    for (auto b = a + 1; b != ranges.end(); ++b)
      if (overlaps(a->first, a->second * sizeof(float), b->first, b->second * sizeof(float)))
        return false;
  return true;
}

// The checks both directions of the residual site share: shape, takes-query, the row
// stride and the float4 alignment of every row operand.  Returns 0, or the status with
// the error set.
int norm_residual_check(const char* fn, int B, int T, int C, int G, int ld,
                        std::initializer_list<const void*> rows) {
  DDSP_REQUIRE(B >= 0 && T >= 0, DDSP_B200_E_INVALID, "%s: bad shape B=%d T=%d", fn, B, T);
  DDSP_REQUIRE(ddsp_b200_norm_residual_takes(C, G), DDSP_B200_E_UNSUPPORTED,
               "%s: C=%d channels in G=%d groups; the kernel takes C a multiple of 4 from 4 "
               "to %d, in groups that divide it, or G = 0 (no normalization)", fn, C, G,
               kNormMaxChannels);
  DDSP_REQUIRE(ld == 0 || (ld >= C && ld % 4 == 0), DDSP_B200_E_INVALID,
               "%s: row stride ld=%d; it is 0 (per-channel scale and shift) or a multiple of "
               "4 of at least C=%d", fn, ld, C);
  for (const void* p : rows)
    DDSP_REQUIRE(((uintptr_t)p & 15) == 0, DDSP_B200_E_INVALID,
                 "%s: the row operands must be 16-byte aligned", fn);
  return 0;
}

template <bool kNorm, bool kRow>
int launch_norm_residual_forward(const float* y, const float* x, const float* scale,
                                 const float* shift, int ld, float* x_next, float* r,
                                 float* mean, float* rstd, int B, int T, int C, int G,
                                 float eps, cudaStream_t st) {
  return launch("norm_residual_forward", norm_residual_forward_kernel<kNorm, kRow>,
                dim3(kNormCluster * B), dim3(kNormThreads),
                kNorm ? norm_smem_bytes(C, G, false) : 0, st, y, x, scale, shift, ld, x_next,
                r, mean, rstd, T, C, G, eps);
}

template <bool kNorm, bool kRow>
int launch_norm_residual_backward(const float* y, const float* scale, int ld,
                                  const float* x_next, const float* mean, const float* rstd,
                                  const float* gx, const float* gr, float* dy, float* dx,
                                  float* dscale, float* dshift, float* partial, int B, int T,
                                  int C, int G, cudaStream_t st) {
  const bool smem = kNorm || !kRow;
  return launch("norm_residual_backward", norm_residual_backward_kernel<kNorm, kRow>,
                dim3(kNormCluster * B), dim3(kNormThreads),
                smem ? norm_smem_bytes(C, kNorm ? G : 0, true) : 0, st, y, scale, ld, x_next,
                mean, rstd, gx, gr, dy, dx, dscale, dshift, partial, T, C, G);
}

}  // namespace

extern "C" {

int ddsp_b200_norm_residual_forward(const float* y, const float* x, const float* scale,
                                    const float* shift, int ld, void* x_next_out, void* r_out,
                                    void* mean_out, void* rstd_out, int B, int T, int C, int G,
                                    float eps, void* stream) {
  const char* fn = "norm_residual_forward";
  float* x_next = static_cast<float*>(x_next_out);
  float* r = static_cast<float*>(r_out);
  float* mean = static_cast<float*>(mean_out);
  float* rstd = static_cast<float*>(rstd_out);
  const bool row = ld > 0;
  if (int rc = norm_residual_check(fn, B, T, C, G, ld,
                                   {y, x, x_next, r, row ? scale : nullptr,
                                    row ? shift : nullptr}))
    return rc;
  if (B == 0 || T == 0) return 0;
  DDSP_REQUIRE(y && x && shift && x_next && (scale || row) && (G == 0 || (mean && rstd)),
               DDSP_B200_E_INVALID, "%s: null pointer", fn);
  const size_t n = extent(B, T, C), ns = row_extent(B, T, C, ld), nm = G ? extent(B, G) : 0;
  if (int rc = check_overlap(fn, {DDSP_OUT(x_next, n), DDSP_OUT(r, r ? n : 0),
                                  DDSP_OUT(mean, nm), DDSP_OUT(rstd, nm)},
                             {DDSP_IN(y, n), DDSP_IN(x, n), DDSP_IN(scale, scale ? ns : 0),
                              DDSP_IN(shift, ns)}))
    return rc;
  DDSP_REQUIRE(pairwise_disjoint({{x_next, n}, {r, r ? n : 0}, {mean, nm}, {rstd, nm}}),
               DDSP_B200_E_INVALID, "%s: x_next, r, mean and rstd must not overlap", fn);
  cudaStream_t st = (cudaStream_t)stream;
#define DDSP_NR_FWD(N, ROW) \
  launch_norm_residual_forward<N, ROW>(y, x, scale, shift, ld, x_next, r, mean, rstd, B, T, C, \
                                     G, eps, st)
  if (G > 0) return row ? DDSP_NR_FWD(true, true) : DDSP_NR_FWD(true, false);
  return row ? DDSP_NR_FWD(false, true) : DDSP_NR_FWD(false, false);
#undef DDSP_NR_FWD
}

int ddsp_b200_norm_residual_backward(const float* y, const float* scale, int ld,
                                     const float* x_next, const float* mean, const float* rstd,
                                     const float* gx, const float* gr, float* dy, float* dx,
                                     float* dscale, float* dshift, void* workspace,
                                     size_t workspace_bytes, int B, int T, int C, int G,
                                     void* stream) {
  const char* fn = "norm_residual_backward";
  const bool row = ld > 0;
  if (int rc = norm_residual_check(fn, B, T, C, G, ld,
                                   {y, x_next, gx, gr, dy, dx, row ? scale : nullptr,
                                    row ? dscale : nullptr, row ? dshift : nullptr}))
    return rc;
  if (B == 0 || T == 0) return 0;
  DDSP_REQUIRE(y && gx && dy && dx && dshift && (!gr || x_next) && (G == 0 || (mean && rstd)) &&
                   (row ? !scale == !dscale : scale && dscale && workspace),
               DDSP_B200_E_INVALID, "%s: null pointer", fn);
  if (row && dscale) {
    const ptrdiff_t gap = dshift > dscale ? dshift - dscale : dscale - dshift;
    DDSP_REQUIRE(gap >= C && gap <= ld - C, DDSP_B200_E_INVALID,
                 "%s: dscale and dshift must be disjoint column blocks of one row", fn);
  }
  const size_t n = extent(B, T, C), ns = row_extent(B, T, C, ld), nm = G ? extent(B, G) : 0;
  const size_t np = row ? 0 : extent(B, kNormCluster, 2 * C);
  DDSP_REQUIRE(workspace_bytes >= np * sizeof(float), DDSP_B200_E_INVALID,
               "%s: the workspace has %zu B, it needs %zu", fn, workspace_bytes,
               np * sizeof(float));
  float* partial = row ? nullptr : static_cast<float*>(workspace);
  if (int rc = check_overlap(fn, {DDSP_OUT(dy, n), DDSP_OUT(dx, n),
                                  DDSP_OUT(dscale, dscale ? ns : 0), DDSP_OUT(dshift, ns),
                                  DDSP_OUT(partial, np)},
                             {DDSP_IN(y, n), DDSP_IN(scale, scale ? ns : 0),
                              DDSP_IN(x_next, gr ? n : 0), DDSP_IN(mean, nm),
                              DDSP_IN(rstd, nm), DDSP_IN(gx, n), DDSP_IN(gr, gr ? n : 0)}))
    return rc;
  // Per row, dscale and dshift are column blocks of one buffer, checked above.
  const bool disjoint =
      row ? pairwise_disjoint({{dy, n}, {dx, n}, {dscale, dscale ? ns : 0}}) &&
                pairwise_disjoint({{dy, n}, {dx, n}, {dshift, ns}})
          : pairwise_disjoint({{dy, n}, {dx, n}, {dscale, ns}, {dshift, ns}, {partial, np}});
  DDSP_REQUIRE(disjoint, DDSP_B200_E_INVALID,
               "%s: dy, dx, dscale, dshift and the workspace must not overlap", fn);
  cudaStream_t st = (cudaStream_t)stream;
#define DDSP_NR_BWD(N, ROW)                                                                   \
  launch_norm_residual_backward<N, ROW>(y, scale, ld, x_next, mean, rstd, gx, gr, dy, dx,     \
                                      dscale, dshift, partial, B, T, C, G, st)
  const int rc = G > 0 ? (row ? DDSP_NR_BWD(true, true) : DDSP_NR_BWD(true, false))
                       : (row ? DDSP_NR_BWD(false, true) : DDSP_NR_BWD(false, false));
#undef DDSP_NR_BWD
  if (rc || row) return rc;
  return launch("norm_relu_param_grad", norm_relu_param_grad_kernel,
                dim3((2 * C + 255) / 256), dim3(256), 0, st, (const float*)partial, dscale,
                dshift, kNormCluster * B, C);
}

}  // extern "C"
