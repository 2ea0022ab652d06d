// Shared helpers for libpcb200 (sm_90a).  Not part of the public ABI.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include "../../include/pcb200.h"

namespace pcb {

void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;

inline int check_launch(const char* what) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("%s: %s", what, cudaGetErrorString(e)); return PCB_ERR_CUDA; }
  return PCB_OK;
}
#define PCB_CUDA(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { pcb::set_error("%s: %s", #call, cudaGetErrorString(e_)); return PCB_ERR_CUDA; } } while (0)
#define PCB_ARG(cond) do { if (!(cond)) { pcb::set_error("bad argument: %s (%s:%d)", #cond, __FILE__, __LINE__); return PCB_ERR_ARG; } } while (0)

inline unsigned blocks_for(int64_t n, int bs) { return (unsigned)((n + bs - 1) / bs); }
inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

// Workspace layouts.  Each entry point that takes `ws` has ONE layout function that takes its pieces from a Carve in order.  Run on a
// null base it only counts (the *_ws_bytes query returns `used`); run on the caller's ws it hands out the same pieces, each at a
// 256-byte aligned offset.  An entry point never touches a byte at or beyond `used`.
struct Carve {
  char* base;
  size_t used = 0;
  template <class T> T* take(int64_t count) {
    T* p = base ? reinterpret_cast<T*>(base + used) : nullptr;
    used += align_up((size_t)count * sizeof(T));
    return p;
  }
};
// the *_ws_bytes query of a layout function
template <class Layout, class... Args> size_t layout_bytes(Layout layout, Args... args) {
  Carve c{nullptr};
  layout(c, args...);
  return c.used;
}

constexpr uint64_t KEY_EMPTY = 0xFFFFFFFFFFFFFFFFull;
constexpr int COORD_BIAS = 32768;

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33; return k;
}

__device__ __forceinline__ int hash_lookup(const uint64_t* __restrict__ tk, const int32_t* __restrict__ tv,
                                           uint64_t mask, uint64_t key) {
  uint64_t slot = mix64(key) & mask;
  while (true) {
    uint64_t k = tk[slot];
    if (k == key) return tv[slot];
    if (k == KEY_EMPTY) return -1;
    slot = (slot + 1) & mask;
  }
}

// Optional per-launch timing (pcb_profile_*, unit.cu): CUDA events around every convolution / weight-gradient entry point.
void prof_begin(cudaStream_t st);
// kind: 0 conv forward / data gradient, 1 weight gradient, 2 BatchNorm forward pass(es) of a unit, 3 BatchNorm backward of a unit,
// 4 PointInfoNCE forward + backward, 5 SGD step, 6 weight re-tiling
void prof_end(cudaStream_t st, int kind);
struct ProfScope {
  cudaStream_t st; int kind;
  ProfScope(cudaStream_t s, int k) : st(s), kind(k) { prof_begin(st); }
  ~ProfScope() { prof_end(st, kind); }
};

// ---- functions one .cu file defines and another calls.  Declared only here, so each definition is checked against its callers.
// conv.cu: the tensor-core forward / data gradient of pcb_conv_forward_split_ordered, without its profile scope.  partials != NULL: the
// caller runs the reduction of an offset-split launch itself (bias and PCB_CONV_ACCUMULATE are then rejected: that pass applies them);
// *partials receives the planes P[*nsplit][n_out][Cout] in ws, or NULL when the convolution ran unsplit and wrote Y.
int conv_forward_split_impl(const uint16_t* Xhi, const uint16_t* Xlo, int lds, const int32_t* tbl, int64_t tbl_stride, const int32_t* kmap,
                            int K, const int32_t* perm, int64_t n_out, int Cin, int Cout, const void* w_tiles, const float* bias, float* Y, int ldy, void* ws,
                            size_t ws_bytes, int flags, cudaStream_t st, const float** partials, int* nsplit);
// conv_wgmma.cu: the wgmma kernels behind conv.cu's split-operand entry points
int launch_conv_wgmma(const uint16_t* Xhi, const uint16_t* Xlo, int lds, const void* wt, const int32_t* tbl, int64_t tbl_stride,
                      const int* kmap, int K, const int32_t* perm, int64_t n_out, int Cin, int Cout, const float* bias, float* Y, int ldy,
                      float* partial, int nsplit, int bn, int accumulate, cudaStream_t st, int x_fp16, int w_fp16);
int launch_wgrad_wgmma(const uint16_t* Ahi, const uint16_t* Alo, int lda, const uint16_t* Bhi, const uint16_t* Blo, int ldb,
                       const int32_t* tbl, int64_t tbl_stride, int K, int64_t n_out, int Ca, int Cb, int rows_per_split, int splits,
                       float* partial, int transpose_out, int tn, cudaStream_t st);
// conv.cu: the channel tile of the tensor-core kernels, the largest of {128, 96, 64, 32} dividing C (0 if none does)
int pick_tile(int C);
// bn.cu: the statistics passes of pcb_unit_forward -- eval mode, and fused into the reduction of an offset-split convolution
int bn_eval_stats_launch(const float* running_mean, const float* running_var, int C, float eps, float* mean, float* invstd, cudaStream_t st);
int bn_reduce_stats_launch(const float* P, int nsplit, float* Y, int ldy, int64_t n, int64_t n0, int C, float eps, float momentum,
                           float* mean, float* invstd, float* running_mean, float* running_var, void* ws, size_t ws_bytes, cudaStream_t st);
// loss.cu: the mean cross-entropy pass of pcb_ce_forward_backward, out[0] = sum of rowloss over the rows whose target is in [0, C) and
// != ignore, divided by their count (fp64, fixed order, rounded to fp32), out[1] = that count.  pcb_seg_metrics (metrics.cu) runs the
// same pass, so its evaluation loss is the training loss bit for bit.
int ce_mean_launch(const float* rowloss, const int64_t* target, int64_t n, int C, int64_t ignore, float* out, cudaStream_t st);
// nce_wgmma.cu: the tensor-core PointInfoNCE behind pcb_nce_forward_backward (loss.cu)
bool nce_tc_supported(int64_t n, int D);
size_t nce_tc_ws_bytes(int64_t n, int D);
int nce_tc_forward_backward(const float* q, const float* k, int64_t n, int D, float inv_T, float* loss, float* dq, float* dk, void* ws,
                            cudaStream_t st);

// Programmatic dependent launch: launch_kernel() launches every kernel with programmatic stream serialisation, and every kernel
// below starts with pdl_wait() -- it blocks until the preceding kernel of the stream has completed and its writes are visible --
// followed by pdl_trigger(), which lets the NEXT kernel's CTAs be scheduled as soon as all of this kernel's CTAs are running.  The
// launch latency and CTA ramp-up of a kernel then overlap the tail of its predecessor; ordering is unchanged (nothing precedes the
// wait).  In a kernel launched with <<<>>> (no attribute) both are no-ops.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... Exp, typename... Act>
inline void launch_kernel(void (*kernel)(Exp...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Act&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<Act&&>(args)...);       // errors surface through check_launch (cudaGetLastError)
}

// One warp's row statistics of a logit row x[0, C) (lanes stride over the columns): m = the row maximum (fmaxf: NaN-free), s =
// sum of expf(x - m).  The cross-entropy kernels (loss.cu) and the metric kernel (metrics.cu) both take lse = m + logf(s) from here.
__device__ __forceinline__ void warp_row_max_sumexp(const float* __restrict__ x, int C, int lane, float& m, float& s) {
  m = -INFINITY;
  for (int c = lane; c < C; c += 32) m = fmaxf(m, x[c]);
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  s = 0.f;
  for (int c = lane; c < C; c += 32) s += expf(x[c] - m);
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
}

// Order-preserving integer keys of floating-point values: key(a) < key(b) when a < b, -0.0 below +0.0, a NaN below -inf or above
// +inf by its sign bit.  Radix selection (det_data.cu) and atomic min / max of bounds (det_data.cu, det_prep.cu) work on these keys;
// add / sub / mul are the explicitly rounded operations of the type.
template <class T> struct Ord;
template <> struct Ord<float> {
  using K = uint32_t;
  static constexpr int BITS = 32;
  __device__ static K key(float v) { const uint32_t u = __float_as_uint(v); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
  __device__ static float val(K k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }
  __device__ static float add(float a, float b) { return __fadd_rn(a, b); }
  __device__ static float sub(float a, float b) { return __fsub_rn(a, b); }
  __device__ static float mul(float a, float b) { return __fmul_rn(a, b); }
};
template <> struct Ord<double> {
  using K = unsigned long long;
  static constexpr int BITS = 64;
  __device__ static K key(double v) {
    const K u = (K)__double_as_longlong(v);
    return (u >> 63) ? ~u : (u | (1ull << 63));
  }
  __device__ static double val(K k) { return __longlong_as_double((long long)((k >> 63) ? (k & ~(1ull << 63)) : ~k)); }
  __device__ static double add(double a, double b) { return __dadd_rn(a, b); }
  __device__ static double sub(double a, double b) { return __dsub_rn(a, b); }
  __device__ static double mul(double a, double b) { return __dmul_rn(a, b); }
};

inline int current_device() { int dev = 0; cudaGetDevice(&dev); return (dev >= 0 && dev < 64) ? dev : 0; }

inline int num_sms() {
  static int n[64] = {};
  const int dev = current_device();
  if (!n[dev]) { cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev); if (n[dev] <= 0) n[dev] = 132; }
  return n[dev];
}

}  // namespace pcb
