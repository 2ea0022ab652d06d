// Sparse convolution on a dense neighbour table: output-stationary gather-GEMM (no scatter, no atomics).
//
//   forward / data-gradient :  Y[j,:] = sum_k X[tbl[kmap[k]][j], :] . W[k]
//   weight-gradient         :  dW[k]  = sum_j A[tbl[k][j], :]^T . B[j, :]
//
// Replaces MinkowskiEngine 0.4.3 ConvolutionForwardGPU / ConvolutionBackwardGPU (+Transpose): per-offset
// gather -> SIMT matmul -> atomicAdd scatter, K launches per layer (reference call sites in include/pcb200.h).
//
// Numerics: the tensor-core entry points (pcb_conv_forward_split / pcb_conv_wgrad_split, kernels in conv_wgmma.cu) take their
// operands as 16-bit hi/lo planes (x = hi + lo) and run the contraction as a 3-term split:
//   x.w ~= hi.hi + lo.hi + hi.lo,  fp32 accumulate  ->  per-product relative error <= ~2^-16, i.e. fp32-class
// parity (tests: 1e-3 relative against the fp64 oracle after 63 layers).  The exact fp32 entry points (pcb_conv_forward /
// pcb_conv_wgrad) cover the channel counts the tensor-core tiling does not (Cin = 3, odd widths) and are the in-library
// cross-check of the tensor-core ones.
#include <algorithm>
#include <cuda_fp16.h>
#include "common.cuh"

using namespace pcb;

int pcb::pick_tile(int C) {
  if (C % 128 == 0) return 128;
  if (C % 96 == 0) return 96;
  if (C % 64 == 0) return 64;
  if (C % 32 == 0) return 32;
  return 0;
}

namespace {

struct KMap { int v[PCB_MAX_KERNEL_VOLUME]; };

constexpr int BM = 128;        // output rows per CTA tile of the tensor-core kernels (conv_wgmma.cu)
constexpr int BK = 32;         // input channels per pipeline step


// Y[row, c] = bias[c] + sum_z partial[z][row][c]   (fixed order: deterministic)
__global__ void conv_split_reduce_kernel(const float* __restrict__ partial, int nsplit, int64_t n_out, int Cout,
                                         const float* __restrict__ bias, float* __restrict__ Y, int ldy, int accumulate) {
  pdl_wait(); pdl_trigger();
  const int cv = Cout / 4;
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n_out * cv) return;
  int64_t row = i / cv;
  int c4 = (int)(i - row * cv);
  float4 s = bias ? reinterpret_cast<const float4*>(bias)[c4] : make_float4(0.f, 0.f, 0.f, 0.f);
  const int64_t plane = n_out * cv;
  for (int z = 0; z < nsplit; ++z) {
    float4 v = __ldg(reinterpret_cast<const float4*>(partial) + z * plane + i);
    s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
  }
  float4* dst = reinterpret_cast<float4*>(Y + row * ldy + c4 * 4);
  if (accumulate) { float4 o = *dst; s.x += o.x; s.y += o.y; s.z += o.z; s.w += o.w; }
  *dst = s;
}

// --------------------------------------------------------------------------------------------- pooling (table gather-sum)
// Y[j, :] = sum_k X[tbl[kmap[k]][j], :]  (cnt[j] = number of present neighbours): the kernel of MinkowskiSumPooling / AvgPooling /
// PoolingTranspose / AvgUnpooling and of their backward passes (the same sum over the transposed table) -- the sibling models'
// pooling layers (`model/resnet.py:63`, `model/modules/common.py:170-214`).  One thread per (row, 4 channels).
__global__ void gather_sum_kernel(const float* __restrict__ X, int ldx, const int32_t* __restrict__ tbl, int64_t tbl_stride, KMap kmap, int K,
                                  int64_t n_out, int C, float* __restrict__ Y, int ldy, float* __restrict__ cnt) {
  pdl_wait(); pdl_trigger();
  const int cv = C / 4;
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n_out * cv) return;
  const int64_t j = e / cv;
  const int c4 = (int)(e - j * cv);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  int present = 0;
  for (int k = 0; k < K; ++k) {
    const int idx = __ldg(tbl + (int64_t)kmap.v[k] * tbl_stride + j);
    if (idx < 0) continue;
    const float4 v = __ldg(reinterpret_cast<const float4*>(X + (int64_t)idx * ldx) + c4);
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    ++present;
  }
  *reinterpret_cast<float4*>(Y + j * ldy + c4 * 4) = acc;
  if (cnt && c4 == 0) cnt[j] = (float)present;
}

// --------------------------------------------------------------------------------------------- forward (exact fp32 SIMT)
__global__ void conv_simt_kernel(const float* __restrict__ X, int ldx, const int32_t* __restrict__ tbl, int64_t tbl_stride,
                                 KMap kmap, int K, int64_t n_out, int Cin, int Cout, const float* __restrict__ W,
                                 const float* __restrict__ bias, float* __restrict__ Y, int ldy) {
  pdl_wait(); pdl_trigger();
  // one thread per (row, cout); consecutive threads -> consecutive cout (W reads coalesced, X reads broadcast)
  int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n_out * Cout) return;
  int64_t j = e / Cout;
  int co = (int)(e - j * Cout);
  float acc = bias ? bias[co] : 0.f;
  for (int k = 0; k < K; ++k) {
    int idx = tbl[(int64_t)kmap.v[k] * tbl_stride + j];
    if (idx < 0) continue;
    const float* x = X + (int64_t)idx * ldx;
    const float* w = W + (int64_t)k * Cin * Cout + co;
    for (int ci = 0; ci < Cin; ++ci) acc = fmaf(x[ci], w[(int64_t)ci * Cout], acc);
  }
  Y[j * ldy + co] = acc;
}

// The stem layer (CIN = 3 -> 32 channels, exact fp32).  Thread = output row (consecutive threads -> consecutive rows: the table reads
// tbl[k][j] are coalesced), all 32 output channels of the row in registers, weights [K][CIN][32] broadcast from shared memory.
template <int CIN>
__global__ void __launch_bounds__(128) conv_stem_kernel(const float* __restrict__ X, int ldx, const int32_t* __restrict__ tbl,
                                                        int64_t tbl_stride, KMap kmap, int K, int64_t n_out, const float* __restrict__ W,
                                                        const float* __restrict__ bias, float* __restrict__ Y, int ldy) {
  pdl_wait(); pdl_trigger();
  __shared__ __align__(16) float s_w[PCB_MAX_KERNEL_VOLUME * CIN * 32];
  for (int e = threadIdx.x; e < K * CIN * 32; e += 128) s_w[e] = W[e];
  __syncthreads();
  const int64_t j = blockIdx.x * 128ll + threadIdx.x;
  if (j >= n_out) return;
  float acc[32];
#pragma unroll
  for (int co = 0; co < 32; ++co) acc[co] = bias ? bias[co] : 0.f;
  for (int k = 0; k < K; ++k) {
    const int idx = __ldg(tbl + (int64_t)kmap.v[k] * tbl_stride + j);
    if (idx < 0) continue;
    const float* xr = X + (int64_t)idx * ldx;
#pragma unroll
    for (int c = 0; c < CIN; ++c) {
      const float x = __ldg(xr + c);
      const float4* w = reinterpret_cast<const float4*>(s_w + (k * CIN + c) * 32);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 v = w[q];
        acc[q * 4 + 0] = fmaf(x, v.x, acc[q * 4 + 0]); acc[q * 4 + 1] = fmaf(x, v.y, acc[q * 4 + 1]);
        acc[q * 4 + 2] = fmaf(x, v.z, acc[q * 4 + 2]); acc[q * 4 + 3] = fmaf(x, v.w, acc[q * 4 + 3]);
      }
    }
  }
  float4* yo = reinterpret_cast<float4*>(Y + j * ldy);
#pragma unroll
  for (int q = 0; q < 8; ++q) yo[q] = make_float4(acc[q * 4], acc[q * 4 + 1], acc[q * 4 + 2], acc[q * 4 + 3]);
}

// --------------------------------------------------------------------------------------------- weight gradient (exact fp32)
struct WgradArgs {
  const float* A; int lda;      // gathered operand  [*, Ca]
  const float* B; int ldb;      // row-aligned operand [n_out, Cb]
  const int32_t* tbl; int64_t tbl_stride;
  int K; int64_t n_out; int Ca; int Cb;
  int rows_per_split;
  float* partial;               // [splits][K][Ca][Cb] (or transposed)
  int transpose_out;
};

// exact fp32 SIMT weight gradient: block = (k, split), threads stride over the Ca*Cb outputs
__global__ void wgrad_simt_kernel(const WgradArgs p) {
  const int k = blockIdx.x, split = blockIdx.y;
  const int64_t r_begin = (int64_t)split * p.rows_per_split;
  const int64_t r_end = min(p.n_out, r_begin + p.rows_per_split);
  const int32_t* trow = p.tbl + (int64_t)k * p.tbl_stride;
  float* out = p.partial + ((int64_t)split * p.K + k) * (int64_t)p.Ca * p.Cb;
  for (int e = threadIdx.x; e < p.Ca * p.Cb; e += blockDim.x) {
    int m = e / p.Cb, n = e - m * p.Cb;
    float acc = 0.f;
    for (int64_t r = r_begin; r < r_end; ++r) {
      int idx = trow[r];
      if (idx >= 0) acc = fmaf(p.A[(int64_t)idx * p.lda + m], p.B[r * p.ldb + n], acc);
    }
    if (!p.transpose_out) out[(int64_t)m * p.Cb + n] = acc; else out[(int64_t)n * p.Ca + m] = acc;
  }
}

// Stem layer (CA = 3 input channels -> 32), exact fp32, deterministic.  A CTA walks tiles of 64 table rows: the gathered inputs of
// the tile, xs[row][k][c] (table reads coalesced along the rows), and the 64 x 32 dY tile are staged in shared memory; thread
// (kc, co) then owns output dW[k][c][co] for ~K*CA/8 values of kc and accumulates over the tile's rows from shared memory
// (xs broadcast within a warp, dY conflict-free).  One partial tile [K*CA*32] per CTA, summed by wgrad_reduce_kernel.
template <int CA>
__global__ void __launch_bounds__(256) wgrad_stem_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb,
                                                         const int32_t* __restrict__ tbl, int64_t tbl_stride, int K, int64_t n_out,
                                                         int rows_per_block, float* __restrict__ partial) {
  pdl_wait(); pdl_trigger();
  constexpr int TR = 64, KC = PCB_MAX_KERNEL_VOLUME * CA, PER = (KC + 7) / 8;
  __shared__ float s_x[TR][KC + 1];
  __shared__ float s_dy[TR][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nkc = K * CA;
  float acc[PER];
#pragma unroll
  for (int i = 0; i < PER; ++i) acc[i] = 0.f;
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
  const int64_t r1 = min(n_out, r0 + rows_per_block);
  for (int64_t t0 = r0; t0 < r1; t0 += TR) {
    const int rows = (int)min((int64_t)TR, r1 - t0);
    __syncthreads();
    for (int e = threadIdx.x; e < K * TR; e += 256) {          // (k, row): consecutive threads -> consecutive rows of one table row
      const int k = e / TR, r = e - k * TR;
      int idx = -1;
      if (r < rows) idx = __ldg(tbl + (int64_t)k * tbl_stride + t0 + r);
      const float* ar = A + (int64_t)(idx >= 0 ? idx : 0) * lda;
#pragma unroll
      for (int c = 0; c < CA; ++c) s_x[r][k * CA + c] = idx >= 0 ? __ldg(ar + c) : 0.f;
    }
    for (int e = threadIdx.x; e < TR * 32; e += 256) {
      const int r = e >> 5, co = e & 31;
      s_dy[r][co] = r < rows ? __ldg(B + (t0 + r) * ldb + co) : 0.f;
    }
    __syncthreads();
    for (int r = 0; r < rows; ++r) {
      const float dy = s_dy[r][lane];
#pragma unroll
      for (int i = 0; i < PER; ++i) {
        const int kc = warp + 8 * i;
        if (kc < nkc) acc[i] = fmaf(s_x[r][kc], dy, acc[i]);
      }
    }
  }
  float* out = partial + (int64_t)blockIdx.x * nkc * 32;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int kc = warp + 8 * i;
    if (kc < nkc) out[kc * 32 + lane] = acc[i];
  }
}

__global__ void wgrad_reduce_kernel(const float* __restrict__ partial, int splits, int64_t n, float* __restrict__ dW, int accumulate) {
  pdl_wait(); pdl_trigger();
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int sp = 0; sp < splits; ++sp) s += partial[(int64_t)sp * n + i];
  dW[i] = accumulate ? dW[i] + s : s;
}

// Small levels (a few hundred rows at 256 channels) would otherwise be a handful of CTAs each walking 27 x Cin/32
// pipeline steps serially: split that loop over gridDim.z and reduce.
int conv_splits(int K, int64_t n_out, int Cin, int Cout) {
  int bn = pick_tile(Cout);
  int64_t base = ((n_out + BM - 1) / BM) * (Cout / bn);
  const int64_t one_wave = num_sms();          // the tensor-core kernel runs one CTA per SM
  if (base >= one_wave) return 1;
  const double waves = 0.5;         // CTAs to aim for on a small level, in units of one resident wave
  int64_t s = ((int64_t)(waves * one_wave) + base - 1) / base;
  int64_t T = (int64_t)K * (Cin / BK);
  if (s > T) s = T;
  if (s > 64) s = 64;
  return s < 2 ? 1 : (int)s;
}

int wgrad_splits(int K, int64_t n_out, int Ca, int Cb, int tm, int tn) {
  int64_t base = (int64_t)K * (tm ? Ca / tm : 1) * (tn ? Cb / tn : 1);
  int64_t target = 4ll * num_sms();
  int64_t s = (target + base - 1) / base;
  int64_t max_s = (n_out + 255) / 256;      // at least 256 rows per split
  if (s > max_s) s = max_s;
  if (s < 1) s = 1;
  if (s > 64) s = 64;
  return (int)s;
}

bool stem_shape(int Ca, int Cb) { return Ca == 3 && Cb == 32; }

// [partials][K][Ca][Cb]: one partial per CTA of the stem kernel (at most 2 x num_sms) or per row split of the generic kernel,
// enough for whichever of the two the call takes
float* wgrad_layout(Carve& c, int K, int64_t n_out, int Ca, int Cb) {
  const int64_t splits = wgrad_splits(K, n_out, Ca, Cb, 0, 0);
  return c.take<float>((stem_shape(Ca, Cb) ? std::max<int64_t>(2 * num_sms(), splits) : splits) * K * Ca * Cb);
}

}  // namespace

// Exact fp32 forward / data gradient: the stem kernel for the 3 -> 32 layer, the generic SIMT kernel for every other width.
extern "C" int pcb_conv_forward(const float* X, int ldx, const int32_t* tbl, int64_t tbl_stride, const int32_t* kmap, int K,
                                int64_t n_out, int Cin, int Cout, const float* W, const float* bias, float* Y, int ldy, void* stream) {
  PCB_ARG(K >= 1 && K <= PCB_MAX_KERNEL_VOLUME && n_out >= 0 && Cin >= 1 && Cout >= 1 && ldx >= Cin && ldy >= Cout);
  if (n_out == 0) return PCB_OK;
  PCB_ARG(X && tbl && W && Y && tbl_stride >= n_out);
  cudaStream_t st = (cudaStream_t)stream;
  ProfScope prof(st, 0);
  KMap km;
  for (int k = 0; k < K; ++k) { km.v[k] = kmap ? kmap[k] : k; PCB_ARG(km.v[k] >= 0 && km.v[k] < PCB_MAX_KERNEL_VOLUME); }
  if (Cin == 3 && Cout == 32) {         // the stem layer
    launch_kernel(conv_stem_kernel<3>, (unsigned)((n_out + 127) / 128), 128, 0, st, X, ldx, tbl, tbl_stride, km, K, n_out, W, bias, Y, ldy);
    return check_launch("conv_stem_kernel");
  }
  int64_t total = n_out * Cout;
  launch_kernel(conv_simt_kernel, (unsigned)((total + 255) / 256), 256, 0, st, X, ldx, tbl, tbl_stride, km, K, n_out, Cin, Cout,
                                                                    W, bias, Y, ldy);
  return check_launch("conv_simt_kernel");
}

extern "C" int pcb_gather_sum(const float* X, int ldx, const int32_t* tbl, int64_t tbl_stride, const int32_t* kmap, int K, int64_t n_out, int C,
                              float* Y, int ldy, float* cnt, void* stream) {
  PCB_ARG(K >= 1 && K <= PCB_MAX_KERNEL_VOLUME && n_out >= 0 && C >= 4 && C % 4 == 0 && ldx >= C && ldy >= C && ldx % 4 == 0 && ldy % 4 == 0);
  if (n_out == 0) return PCB_OK;
  PCB_ARG(X && tbl && Y && tbl_stride >= n_out);
  KMap km;
  for (int k = 0; k < K; ++k) { km.v[k] = kmap ? kmap[k] : k; PCB_ARG(km.v[k] >= 0 && km.v[k] < PCB_MAX_KERNEL_VOLUME); }
  const int64_t total = n_out * (C / 4);
  launch_kernel(gather_sum_kernel, (unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream, X, ldx, tbl, tbl_stride, km, K, n_out, C, Y, ldy,
                cnt);
  return check_launch("gather_sum_kernel");
}

extern "C" size_t pcb_conv_wgrad_ws_bytes(int K, int64_t n_out, int Ca, int Cb) {
  return layout_bytes(wgrad_layout, K, n_out, Ca, Cb);
}

// Exact fp32 weight gradient (the 3-channel stem layer, widths the tensor-core tiling does not cover, PCB_CONV_FORCE_SIMT cross-checks).
// Tensor-core shapes go through pcb_conv_wgrad_split on split (hi/lo) operands.
extern "C" int pcb_conv_wgrad(const float* A, int lda, const float* B, int ldb, const int32_t* tbl, int64_t tbl_stride, int K,
                              int64_t n_out, int Ca, int Cb, float* dW, int transpose_out, void* ws, size_t ws_bytes,
                              int flags, void* stream) {
  PCB_ARG(K >= 1 && K <= PCB_MAX_KERNEL_VOLUME && n_out >= 0 && Ca >= 1 && Cb >= 1 && dW && lda >= Ca && ldb >= Cb);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t nW = (int64_t)K * Ca * Cb;
  if (n_out == 0) {
    if (!(flags & PCB_CONV_ACCUMULATE)) PCB_CUDA(cudaMemsetAsync(dW, 0, nW * sizeof(float), st));
    return PCB_OK;
  }
  Carve c{(char*)ws};
  float* partial = wgrad_layout(c, K, n_out, Ca, Cb);
  PCB_ARG(A && B && tbl && ws && ws_bytes >= c.used && tbl_stride >= n_out);
  ProfScope prof(st, 1);
  if (stem_shape(Ca, Cb) && !transpose_out && !(flags & PCB_CONV_FORCE_SIMT)) {      // the stem layer: dedicated exact-fp32 kernel
    int nb = 2 * num_sms();
    int64_t rpb = (n_out + nb - 1) / nb;
    rpb = (rpb + 63) / 64 * 64;
    nb = (int)((n_out + rpb - 1) / rpb);
    launch_kernel(wgrad_stem_kernel<3>, nb, 256, 0, st, A, lda, B, ldb, tbl, tbl_stride, K, n_out, (int)rpb, partial);
    if (int e = check_launch("wgrad_stem_kernel")) return e;
    launch_kernel(wgrad_reduce_kernel, (unsigned)((nW + 255) / 256), 256, 0, st, (const float*)partial, nb, nW, dW, (flags & PCB_CONV_ACCUMULATE) ? 1 : 0);
    return check_launch("wgrad_reduce_kernel");
  }
  const int splits = wgrad_splits(K, n_out, Ca, Cb, 0, 0);
  WgradArgs a;
  a.A = A; a.lda = lda; a.B = B; a.ldb = ldb; a.tbl = tbl; a.tbl_stride = tbl_stride; a.K = K; a.n_out = n_out;
  a.Ca = Ca; a.Cb = Cb; a.partial = partial; a.transpose_out = transpose_out;
  a.rows_per_split = (int)((n_out + splits - 1) / splits);
  dim3 grid(K, splits);
  wgrad_simt_kernel<<<grid, 256, 0, st>>>(a);
  if (int e = check_launch("wgrad_simt_kernel")) return e;
  launch_kernel(wgrad_reduce_kernel, (unsigned)((nW + 255) / 256), 256, 0, st, (const float*)partial, splits, nW, dW,
                (flags & PCB_CONV_ACCUMULATE) ? 1 : 0);
  return check_launch("wgrad_reduce_kernel");
}


// ------------------------------------------------------------------------------------------------ split-operand entry points
// Weights as shared-memory images for the split conv kernel: per (offset k, 32-channel chunk kc, BN-column block nb) one blob
//   [hi plane | lo plane], plane = 4 k8-groups x (BN/8 core matrices x 128 B + 16 B pad)   (wgmma K-major, no swizzle)
// so that a pipeline stage's weight tile is ONE contiguous TMA bulk copy.
namespace {
__host__ __device__ inline int64_t tile_plane_bytes(int bn) { return 4ll * ((bn / 8) * 128 + 16); }

__device__ __forceinline__ uint32_t pack_bf16(float a, float b, float& ra, float& rb) {
  const __nv_bfloat16 ha = __float2bfloat16_rn(a), hb = __float2bfloat16_rn(b);
  ra = a - __bfloat162float(ha); rb = b - __bfloat162float(hb);
  return (uint32_t)__bfloat16_as_ushort(ha) | ((uint32_t)__bfloat16_as_ushort(hb) << 16);
}
__device__ __forceinline__ uint32_t pack_f16(float a, float b, float& ra, float& rb) {
  const __half ha = __float2half_rn(a), hb = __float2half_rn(b);
  ra = a - __half2float(ha); rb = b - __half2float(hb);
  return (uint32_t)__half_as_ushort(ha) | ((uint32_t)__half_as_ushort(hb) << 16);
}
template <bool F16>
__device__ __forceinline__ void split8(const float (&w)[8], uint4& hi, uint4& lo) {
  float v[8], r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = F16 ? fminf(fmaxf(w[j] * 1024.0f, -65000.f), 65000.f) : w[j];
  uint32_t h[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float d0, d1;
    h[j] = F16 ? pack_f16(v[2 * j], v[2 * j + 1], r[2 * j], r[2 * j + 1]) : pack_bf16(v[2 * j], v[2 * j + 1], r[2 * j], r[2 * j + 1]);
    l[j] = F16 ? pack_f16(r[2 * j], r[2 * j + 1], d0, d1) : pack_bf16(r[2 * j], r[2 * j + 1], d0, d1);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]); lo = make_uint4(l[0], l[1], l[2], l[3]);
}

// Chunk t of convolution d: one 16-byte chunk (8 contraction-direction elements of one tile row) of BOTH planes for each role, so the
// tile images are written with 128-bit stores that line up across a warp (an element per thread scatters 2-byte stores: 0.53 ms per
// step for the 38 M parameters).  Forward roles: 8 consecutive input channels of one output channel (threads along Cout: 8 coalesced
// 4-byte loads); data-gradient roles: 8 consecutive output channels of one input channel (threads along Cin: two 128-bit loads).
__device__ __forceinline__ void weight_tile_chunk(const pcb_tile_desc& d, int64_t t) {
  const int Cin = d.Cin, Cout = d.Cout;
  const float* __restrict__ W = d.W;
  {   // forward roles: N = Cout, contraction = Cin; chunk = input channels ci0 .. ci0 + 7 of output channel co
    const int co = (int)(t % Cout);
    const int64_t g = t / Cout;
    const int cig = (int)(g % (Cin / 8)), k = (int)(g / (Cin / 8));
    const int ci0 = cig * 8;
    float w[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) w[j] = __ldg(W + ((int64_t)k * Cin + ci0 + j) * Cout + co);
    const int bn = d.bn_f;
    const int64_t plane = tile_plane_bytes(bn);
    const int64_t blob = ((int64_t)(k * (Cin / 32) + ci0 / 32) * (Cout / bn) + co / bn) * 2 * plane;
    const int nn = co % bn, c = ci0 % 32;
    unsigned char* dst = (unsigned char*)d.fwd + blob + (c / 8) * (plane / 4) + (nn / 8) * 128 + (nn % 8) * 16;
    uint4 h, l;
    if (d.flags & PCB_PLANES_B_FP16) split8<true>(w, h, l); else split8<false>(w, h, l);
    *reinterpret_cast<uint4*>(dst) = h;
    *reinterpret_cast<uint4*>(dst + plane) = l;
  }
  {   // data-gradient roles: N = Cin, contraction = Cout; chunk = output channels co0 .. co0 + 7 of input channel ci
    const int ci = (int)(t % Cin);
    const int64_t g = t / Cin;
    const int cog = (int)(g % (Cout / 8)), k = (int)(g / (Cout / 8));
    const int co0 = cog * 8;
    const float4 a = __ldg(reinterpret_cast<const float4*>(W + ((int64_t)k * Cin + ci) * Cout + co0));
    const float4 b = __ldg(reinterpret_cast<const float4*>(W + ((int64_t)k * Cin + ci) * Cout + co0) + 1);
    const float w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    const int bn = d.bn_d;
    const int64_t plane = tile_plane_bytes(bn);
    const int64_t blob = ((int64_t)(k * (Cout / 32) + co0 / 32) * (Cin / bn) + ci / bn) * 2 * plane;
    const int nn = ci % bn, c = co0 % 32;
    unsigned char* dst = (unsigned char*)d.dgrad + blob + (c / 8) * (plane / 4) + (nn / 8) * 128 + (nn % 8) * 16;
    uint4 h, l;
    split8<false>(w, h, l);
    *reinterpret_cast<uint4*>(dst) = h;
    *reinterpret_cast<uint4*>(dst + plane) = l;
  }
}

// One convolution (pcb_weight_tile): d passed by value, `chunks` = K*Cin*Cout / 8.
__global__ void weight_tile_single_kernel(const pcb_tile_desc d, int64_t chunks) {
  pdl_wait(); pdl_trigger();
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t < chunks) weight_tile_chunk(d, t);
}

// All convolutions of a network in ONE launch (the fused executor re-tiles every kernel after each SGD step: 62 small launches
// otherwise).  descs: DEVICE array; `start` = prefix sum of K*Cin*Cout; a thread finds its convolution by binary search.
__global__ void weight_tile_batch_kernel(const pcb_tile_desc* __restrict__ descs, int n, int64_t total) {
  pdl_wait(); pdl_trigger();
  __shared__ int64_t s_start[257];
  for (int i = threadIdx.x; i <= n; i += blockDim.x) s_start[i] = i < n ? descs[i].start : total;
  __syncthreads();
  const int64_t t8 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;      // chunk index; every start is a multiple of 8 (channels % 32 == 0)
  if (t8 * 8 >= total) return;
  int lo_ = 0, hi_ = n - 1;
  while (lo_ < hi_) { const int mid = (lo_ + hi_ + 1) >> 1; if (s_start[mid] <= t8 * 8) lo_ = mid; else hi_ = mid - 1; }
  const pcb_tile_desc d = descs[lo_];
  weight_tile_chunk(d, t8 - d.start / 8);
}
}  // namespace

extern "C" int pcb_tile_desc_fill(pcb_tile_desc* d, const float* W, int K, int Cin, int Cout, void* fwd_tiles, void* dgrad_tiles, int flags,
                                  int64_t start) {
  PCB_ARG(d && W && fwd_tiles && dgrad_tiles && K >= 1 && Cin % 32 == 0 && Cout % 32 == 0 && Cin >= 32 && Cout >= 32);
  d->W = W; d->fwd = fwd_tiles; d->dgrad = dgrad_tiles; d->K = K; d->Cin = Cin; d->Cout = Cout; d->flags = flags;
  d->bn_f = pick_tile(Cout); d->bn_d = pick_tile(Cin); d->start = start;
  return PCB_OK;
}

extern "C" int pcb_weight_tile_batch(const pcb_tile_desc* descs_dev, int n, int64_t total, void* stream) {
  PCB_ARG(descs_dev && n >= 1 && n <= 256 && total >= 1);
  ProfScope prof((cudaStream_t)stream, 6);
  PCB_ARG(total % 8 == 0);
  launch_kernel(weight_tile_batch_kernel, (unsigned)((total / 8 + 255) / 256), 256, 0, (cudaStream_t)stream, descs_dev, n, total);
  return check_launch("weight_tile_batch_kernel");
}

extern "C" size_t pcb_weight_tile_bytes(int K, int Cin, int Cout, int dgrad_roles) {
  if (Cin % 32 || Cout % 32) return 0;
  const int N = dgrad_roles ? Cin : Cout, Kc = dgrad_roles ? Cout : Cin;
  const int bn = pick_tile(N);
  return (size_t)K * (Kc / 32) * (N / bn) * 2 * tile_plane_bytes(bn);
}

extern "C" int pcb_weight_tile(const float* W, int K, int Cin, int Cout, void* fwd_tiles, void* dgrad_tiles, int flags, void* stream) {
  pcb_tile_desc d;
  if (int e = pcb_tile_desc_fill(&d, W, K, Cin, Cout, fwd_tiles, dgrad_tiles, flags, 0)) return e;
  const int64_t chunks = (int64_t)K * Cin * Cout / 8;
  launch_kernel(weight_tile_single_kernel, (unsigned)((chunks + 255) / 256), 256, 0, (cudaStream_t)stream, d, chunks);
  return check_launch("weight_tile_single_kernel");
}

namespace pcb {
// the offset-split partial planes [nsplit][n_out][Cout]; none (NULL: the kernel writes Y directly) when the convolution runs unsplit
float* conv_split_layout(Carve& c, int nsplit, int64_t n_out, int Cout) { return nsplit > 1 ? c.take<float>(nsplit * n_out * Cout) : nullptr; }

int conv_forward_split_impl(const uint16_t* Xhi, const uint16_t* Xlo, int lds, const int32_t* tbl, int64_t tbl_stride, const int32_t* kmap,
                            int K, const int32_t* perm, int64_t n_out, int Cin, int Cout, const void* w_tiles, const float* bias, float* Y, int ldy, void* ws,
                            size_t ws_bytes, int flags, cudaStream_t st, const float** partials, int* nsplit_out) {
  PCB_ARG(K >= 1 && K <= PCB_MAX_KERNEL_VOLUME && n_out >= 0 && Cin % 32 == 0 && Cout % 32 == 0 && Cin >= 32 && Cout >= 32);
  PCB_ARG(lds >= Cin && lds % 8 == 0 && ldy >= Cout && ldy % 4 == 0);
  if (partials) *partials = nullptr;
  if (n_out == 0) return PCB_OK;
  PCB_ARG(Xhi && Xlo && tbl && Y && w_tiles && tbl_stride >= n_out);
  const int nsplit = conv_splits(K, n_out, Cin, Cout);
  Carve c{(char*)ws};
  float* partial = conv_split_layout(c, nsplit, n_out, Cout);
  PCB_ARG(c.used == 0 || (ws && ws_bytes >= c.used));
  int km[PCB_MAX_KERNEL_VOLUME];
  for (int k = 0; k < K; ++k) { km[k] = kmap ? kmap[k] : k; PCB_ARG(km[k] >= 0 && km[k] < PCB_MAX_KERNEL_VOLUME); }
  const int accumulate = (flags & PCB_CONV_ACCUMULATE) ? 1 : 0;
  PCB_ARG(!partials || (nsplit_out && !bias && !accumulate));
  PCB_ARG(n_out < (1ll << 31) || !perm);
  // An offset-split launch keeps the identity order: a tile's split boundaries fall within its own list of offsets, so another tile
  // composition would regroup each row's fp32 partial sums.
  if (int e = launch_conv_wgmma(Xhi, Xlo, lds, w_tiles, tbl, tbl_stride, km, K, nsplit == 1 ? perm : nullptr, n_out, Cin, Cout, bias, Y, ldy,
                                partial, nsplit, pick_tile(Cout), accumulate, st,
                                (flags & PCB_PLANES_A_FP16) ? 1 : 0, (flags & PCB_PLANES_B_FP16) ? 1 : 0)) return e;
  if (nsplit == 1) return PCB_OK;
  if (partials) {
    *partials = partial;
    *nsplit_out = nsplit;
    return PCB_OK;
  }
  int64_t n4 = n_out * (Cout / 4);
  launch_kernel(conv_split_reduce_kernel, (unsigned)((n4 + 255) / 256), 256, 0, st, (const float*)partial, nsplit, n_out, Cout, bias, Y, ldy, accumulate);
  return check_launch("conv_split_reduce_kernel");
}
}  // namespace pcb

extern "C" size_t pcb_conv_forward_split_ws_bytes(int K, int64_t n_out, int Cin, int Cout) {
  if (Cin % 32 || Cout % 32 || n_out <= 0) return 0;
  return layout_bytes(conv_split_layout, conv_splits(K, n_out, Cin, Cout), n_out, Cout);
}

extern "C" int pcb_conv_forward_split_ordered(const uint16_t* Xhi, const uint16_t* Xlo, int lds, const int32_t* tbl, int64_t tbl_stride,
                                              const int32_t* kmap, int K, const int32_t* perm, int64_t n_out, int Cin, int Cout,
                                              const void* w_tiles, const float* bias, float* Y, int ldy, void* ws, size_t ws_bytes,
                                              int flags, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  ProfScope prof(st, 0);
  return pcb::conv_forward_split_impl(Xhi, Xlo, lds, tbl, tbl_stride, kmap, K, perm, n_out, Cin, Cout, w_tiles, bias, Y, ldy, ws, ws_bytes,
                                      flags, st, nullptr, nullptr);
}

extern "C" int pcb_conv_forward_split(const uint16_t* Xhi, const uint16_t* Xlo, int lds, const int32_t* tbl, int64_t tbl_stride,
                                      const int32_t* kmap, int K, int64_t n_out, int Cin, int Cout, const void* w_tiles,
                                      const float* bias, float* Y, int ldy, void* ws, size_t ws_bytes,
                                      int flags, void* stream) {
  return pcb_conv_forward_split_ordered(Xhi, Xlo, lds, tbl, tbl_stride, kmap, K, nullptr, n_out, Cin, Cout, w_tiles, bias, Y, ldy, ws,
                                        ws_bytes, flags, stream);
}

namespace {
int wgrad_split_splits(int K, int64_t n_out, int Ca, int Cb) {
  int tn = pick_tile(Cb);
  // the row partition counts units of 2 offsets x 128 channels of A, whatever the kernel's tile: it fixes which rows each fp32 partial
  // sums, and so the result bits
  constexpr int UNIT_OFFSETS = 2, UNIT_CHANNELS = 128;
  int64_t base = (int64_t)((K + UNIT_OFFSETS - 1) / UNIT_OFFSETS) * ((Ca + UNIT_CHANNELS - 1) / UNIT_CHANNELS) * (Cb / tn);
  const double wwaves = 1.0;
  // heuristic, not tuned on H100: aim for 2 x num_sms units, never a nearly-empty extra wave; shorter row ranges per split
  // also keep each fp32 accumulator's sum short
  int64_t s = (int64_t)(wwaves * 2 * num_sms()) / base;
  int64_t max_s = (n_out + 63) / 64;          // small levels: rather many short CTAs than a few long serial ones
  if (s > max_s) s = max_s;
  if (s < 1) s = 1;
  if (s > 96) s = 96;
  return (int)s;
}

// [splits][K][Ca][Cb] partial weight gradients
float* wgrad_split_layout(Carve& c, int splits, int K, int Ca, int Cb) { return c.take<float>((int64_t)splits * K * Ca * Cb); }
}  // namespace

extern "C" size_t pcb_conv_wgrad_split_ws_bytes(int K, int64_t n_out, int Ca, int Cb) {
  if (Ca % 32 || Cb % 32 || n_out <= 0) return 0;
  return layout_bytes(wgrad_split_layout, wgrad_split_splits(K, n_out, Ca, Cb), K, Ca, Cb);
}

extern "C" int pcb_conv_wgrad_split(const uint16_t* Ahi, const uint16_t* Alo, int lda, const uint16_t* Bhi, const uint16_t* Blo, int ldb,
                                    const int32_t* tbl, int64_t tbl_stride, int K, int64_t n_out, int Ca, int Cb, float* dW,
                                    int transpose_out, void* ws, size_t ws_bytes, int flags, void* stream) {
  PCB_ARG(K >= 1 && K <= PCB_MAX_KERNEL_VOLUME && n_out >= 0 && Ca % 32 == 0 && Cb % 32 == 0 && Ca >= 32 && Cb >= 32 && dW);
  PCB_ARG(lda >= Ca && ldb >= Cb && lda % 8 == 0 && ldb % 8 == 0);
  PCB_ARG(!(flags & (PCB_PLANES_A_FP16 | PCB_PLANES_B_FP16)));       // the weight gradient reads bf16 hi/lo planes only
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t nW = (int64_t)K * Ca * Cb;
  if (n_out == 0) {
    if (!(flags & PCB_CONV_ACCUMULATE)) PCB_CUDA(cudaMemsetAsync(dW, 0, nW * sizeof(float), st));
    return PCB_OK;
  }
  const int splits = wgrad_split_splits(K, n_out, Ca, Cb);
  Carve c{(char*)ws};
  float* partial = wgrad_split_layout(c, splits, K, Ca, Cb);
  PCB_ARG(Ahi && Alo && Bhi && Blo && tbl && ws && ws_bytes >= c.used && tbl_stride >= n_out);
  ProfScope prof(st, 1);
  int64_t rps = (n_out + splits - 1) / splits;
  rps = (rps + 15) / 16 * 16;
  if (int e = launch_wgrad_wgmma(Ahi, Alo, lda, Bhi, Blo, ldb, tbl, tbl_stride, K, n_out, Ca, Cb, (int)rps, splits, partial,
                                 transpose_out, pick_tile(Cb), st)) return e;
  launch_kernel(wgrad_reduce_kernel, (unsigned)((nW + 255) / 256), 256, 0, st, (const float*)partial, splits, nW, dW,
                                                                    (flags & PCB_CONV_ACCUMULATE) ? 1 : 0);
  return check_launch("wgrad_reduce_kernel");
}
