// BatchNorm over the rows of a sparse tensor's feature matrix (training-mode statistics), with the
// affine-normalise (+ residual, + ReLU) fused into one elementwise pass.  HBM-bound: every kernel moves
// 16-byte vectors with consecutive threads on consecutive channels.
// Replaces MinkowskiBatchNorm == torch.nn.BatchNorm1d on .F (reference call sites in include/pcb200.h).
#include <cuda_fp16.h>
#include "common.cuh"

using namespace pcb;

namespace {


// fp32 x4 -> fp16 hi x4 + fp16 lo x4 (x ~= hi + lo to 2^-22 |x|, absolute floor 2^-25: fp16 subnormals): the operand format of the
// FORWARD convolutions.  Activations are O(1) after BatchNorm; |x| is clamped to the fp16 range (65504) so that hi stays finite.
__device__ __forceinline__ void store_split4_f16(const float4& v, void* hi, void* lo) {
  const float M = 65000.f;
  const float x = fminf(fmaxf(v.x, -M), M), y = fminf(fmaxf(v.y, -M), M), z = fminf(fmaxf(v.z, -M), M), w = fminf(fmaxf(v.w, -M), M);
  __half2 h0 = __floats2half2_rn(x, y), h1 = __floats2half2_rn(z, w);
  float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
  __half2 l0 = __floats2half2_rn(x - f0.x, y - f0.y), l1 = __floats2half2_rn(z - f1.x, w - f1.y);
  uint2 H, L;
  H.x = *reinterpret_cast<uint32_t*>(&h0); H.y = *reinterpret_cast<uint32_t*>(&h1);
  L.x = *reinterpret_cast<uint32_t*>(&l0); L.y = *reinterpret_cast<uint32_t*>(&l1);
  *reinterpret_cast<uint2*>(hi) = H;
  *reinterpret_cast<uint2*>(lo) = L;
}

// fp32 x4 -> bf16 hi x4 + bf16 lo x4 (x ~= hi + lo to 2^-17): the operand format of the tensor-core conv kernels
__device__ __forceinline__ void store_split4(const float4& v, __nv_bfloat16* hi, __nv_bfloat16* lo) {
  __nv_bfloat162 h0 = __floats2bfloat162_rn(v.x, v.y);
  __nv_bfloat162 h1 = __floats2bfloat162_rn(v.z, v.w);
  float2 f0 = __bfloat1622float2(h0), f1 = __bfloat1622float2(h1);
  __nv_bfloat162 l0 = __floats2bfloat162_rn(v.x - f0.x, v.y - f0.y);
  __nv_bfloat162 l1 = __floats2bfloat162_rn(v.z - f1.x, v.w - f1.y);
  uint2 H, L;
  H.x = *reinterpret_cast<uint32_t*>(&h0); H.y = *reinterpret_cast<uint32_t*>(&h1);
  L.x = *reinterpret_cast<uint32_t*>(&l0); L.y = *reinterpret_cast<uint32_t*>(&l1);
  *reinterpret_cast<uint2*>(hi) = H;
  *reinterpret_cast<uint2*>(lo) = L;
}

__global__ void split_rows_kernel(const float* __restrict__ X, int ldx, int64_t n4, int cv, __nv_bfloat16* __restrict__ hi,
                                  __nv_bfloat16* __restrict__ lo, int lds, int fp16) {
  pdl_wait(); pdl_trigger();
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n4) return;
  int c4 = (int)(i % cv);
  const int64_t row = i / cv;
  float4 x = __ldg(reinterpret_cast<const float4*>(X + row * ldx) + c4);
  if (fp16) store_split4_f16(x, hi + row * lds + c4 * 4, lo + row * lds + c4 * 4);
  else store_split4(x, hi + row * lds + c4 * 4, lo + row * lds + c4 * 4);
}

// partial[chunk][0][C] = sum(a), partial[chunk][1][C] = sum(a*b)    (b == a for the forward statistics)
// block: (C/4) channel-vectors x RP row lanes; grid: one CTA per chunk of rows.
// Strides: lda / ldb (floats), ldm (elements).  Mask (backward only): a is zeroed where the ReLU output is not positive (ReLU folded
// into the BN backward).
// Row segments: rows [0, n0) and [n0, n) are two independent BatchNorm batches (the two views of a pair stacked in one
// matrix); chunks never straddle the boundary: CTAs [0, chunks0) cover segment 0, the rest segment 1.  n0 == n: one segment.
// mean / invstd are [segments][C].
// ReLU mask from the 16-bit hi plane of the ReLU output: out > 0  <=>  hi > 0 (bf16 keeps fp32's exponent range; the only
// difference is an fp32 denormal below 2^-134 rounding to 0).  4 channels = 8 bytes.
__device__ __forceinline__ void mask4_bf16(const __nv_bfloat16* m, float4& a) {
  const uint2 b = __ldg(reinterpret_cast<const uint2*>(m));
  auto pos = [](uint32_t h) { return (h & 0x7FFFu) != 0u && !(h & 0x8000u); };
  a.x = pos(b.x & 0xFFFFu) ? a.x : 0.f; a.y = pos(b.x >> 16) ? a.y : 0.f;
  a.z = pos(b.y & 0xFFFFu) ? a.z : 0.f; a.w = pos(b.y >> 16) ? a.w : 0.f;
}

// ---- column reductions.  A CTA owns one CHUNK of R rows (R = chunk_rows(n): a power of two chosen so that a launch has a few
// hundred CTAs whatever the level size; chunks never straddle the view boundary n0: CTAs [0, chunks0) cover segment 0, the rest
// segment 1); block = (C/4) channel-vectors x RP row lanes, row loop unrolled for memory-level parallelism; one partial row
// [2][C] per chunk, combined in fp64 by the finalize kernels (fixed order: deterministic).
//   MODE 0  forward statistics of A:            partial = { sum(x), M2 = sum((x - chunk mean)^2) }, accumulated around a pivot
//           (the chunk's first row) so that |mean| >> std does not cancel; the finalize kernel merges chunks with Chan's formula
//   MODE 2  the same on A = sum_z P[z] (offset-split convolution partial planes), which is also written to Y
//   MODE 1  backward sums: a = dY (ReLU-masked), partial = { sum(a), sum(a * xhat) }
template <int MODE>
__global__ void __launch_bounds__(256) colstat_kernel(const float* __restrict__ A, int lda, const float* __restrict__ Bm, int ldb,
                                                      const __nv_bfloat16* __restrict__ Mask, int ldm, int nsplit, float* __restrict__ Y,
                                                      int ldy, int64_t n, int64_t n0, int chunks0, int R, int C,
                                                      const float* __restrict__ mean, const float* __restrict__ invstd,
                                                      float* __restrict__ partial) {
  pdl_wait(); pdl_trigger();
  extern __shared__ float sm[];      // [RP][2][C]
  const int cv = C / 4;
  const int rp = blockDim.x / cv;    // row lanes
  const int c4 = threadIdx.x % cv;
  const int rl = threadIdx.x / cv;
  const int seg = (int)blockIdx.x >= chunks0 ? 1 : 0;
  const int64_t r0 = seg ? n0 + (int64_t)((int)blockIdx.x - chunks0) * R : (int64_t)blockIdx.x * R;
  const int64_t r1 = min(seg ? n : n0, r0 + R);
  const int64_t plane = n * cv;
  auto load_a = [&](int64_t r) {
    if (MODE == 2) {
      float4 a = make_float4(0, 0, 0, 0);
#pragma unroll 4
      for (int z = 0; z < nsplit; ++z) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(A) + z * plane + r * cv + c4);
        a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
      }
      return a;
    }
    return __ldg(reinterpret_cast<const float4*>(A + r * lda) + c4);
  };
  float4 s1 = make_float4(0, 0, 0, 0), s2 = make_float4(0, 0, 0, 0);
  float4 mu = make_float4(0, 0, 0, 0), is = make_float4(1, 1, 1, 1), pv = make_float4(0, 0, 0, 0);
  if (rl < rp) {
    if (MODE == 1) {
      mu = reinterpret_cast<const float4*>(mean + seg * C)[c4];
      is = reinterpret_cast<const float4*>(invstd + seg * C)[c4];
    } else if (r0 < r1) {
      pv = load_a(r0);               // pivot: the chunk's first row (every row lane reads the same line)
    }
#pragma unroll 4
    for (int64_t r = r0 + rl; r < r1; r += rp) {
      float4 a = load_a(r);
      if (MODE == 2) *reinterpret_cast<float4*>(Y + r * ldy + c4 * 4) = a;
      if (MODE == 1) {
        if (Mask) mask4_bf16(Mask + r * ldm + c4 * 4, a);
        const float4 x = __ldg(reinterpret_cast<const float4*>(Bm + r * ldb) + c4);
        s1.x += a.x; s1.y += a.y; s1.z += a.z; s1.w += a.w;
        s2.x += a.x * ((x.x - mu.x) * is.x); s2.y += a.y * ((x.y - mu.y) * is.y);
        s2.z += a.z * ((x.z - mu.z) * is.z); s2.w += a.w * ((x.w - mu.w) * is.w);
      } else {
        a.x -= pv.x; a.y -= pv.y; a.z -= pv.z; a.w -= pv.w;
        s1.x += a.x; s1.y += a.y; s1.z += a.z; s1.w += a.w;
        s2.x += a.x * a.x; s2.y += a.y * a.y; s2.z += a.z * a.z; s2.w += a.w * a.w;
      }
    }
    float* d = sm + (int64_t)rl * 2 * C;
    reinterpret_cast<float4*>(d)[c4] = s1;
    reinterpret_cast<float4*>(d + C)[c4] = s2;
  }
  __syncthreads();
  const float m = (float)(r1 > r0 ? r1 - r0 : 1);
  for (int e = threadIdx.x; e < C; e += blockDim.x) {
    float t1 = 0.f, t2 = 0.f;
    for (int l = 0; l < rp; ++l) { t1 += sm[(int64_t)l * 2 * C + e]; t2 += sm[(int64_t)l * 2 * C + C + e]; }
    if (MODE != 1) {                 // shifted sums -> { sum(x), M2 about the chunk mean }
      const float p = MODE == 2 ? Y[r0 * ldy + e] : A[r0 * lda + e];
      const float M2 = t2 - t1 * t1 / m;
      t2 = M2 > 0.f ? M2 : 0.f;
      t1 = t1 + m * p;
    }
    partial[(int64_t)blockIdx.x * 2 * C + e] = t1;
    partial[(int64_t)blockIdx.x * 2 * C + C + e] = t2;
  }
}

// Forward statistics from the per-chunk { sum, M2 } partials (Chan et al. pairwise merge, fp64).  Segment s has chunks
// [s ? chunks0 : 0, ...) of R rows (the last one shorter) and n0 / n - n0 rows.  The running statistics see the segments one after
// the other, as two forward calls would (`ddp_trainer.py:290-297`: the model runs on view 0, then on view 1).
// One warp per channel.  A lane's share of the partials (both segments) is loaded into registers with independent loads BEFORE anything
// is reduced: the kernel is a single memory round trip plus shuffles instead of four dependent passes over the partial rows (it runs 62
// times per step on a few hundred KB: pure latency).
constexpr int FIN_PER_LANE = 12;          // 32 x 12 = 384 chunks per segment held in registers; beyond that a plain loop
// The prefetch of both finalize kernels: v1 / v2[seg][j] = entries 0 / 1 of channel c in chunk lane + 32 j of segment seg, all loads
// independent; 0 past the segment's chunks and for seg >= nseg.
__device__ __forceinline__ void load_partials(const float* partial, int chunks, int chunks0, int nseg, int C, int c, int lane,
                                              float (&v1)[2][FIN_PER_LANE], float (&v2)[2][FIN_PER_LANE]) {
#pragma unroll
  for (int seg = 0; seg < 2; ++seg) {
    const float* p = partial + (seg ? (int64_t)chunks0 * 2 * C : 0);
    const int ch = seg < nseg ? (seg ? chunks - chunks0 : chunks0) : 0;
#pragma unroll
    for (int j = 0; j < FIN_PER_LANE; ++j) {
      const int k = lane + 32 * j;
      v1[seg][j] = k < ch ? __ldg(p + (int64_t)k * 2 * C + c) : 0.f;
      v2[seg][j] = k < ch ? __ldg(p + (int64_t)k * 2 * C + C + c) : 0.f;
    }
  }
}

__global__ void bn_finalize_kernel(const float* __restrict__ partial, int chunks, int chunks0, int R, int64_t n, int64_t n0, int C, float eps,
                                   float momentum, float* __restrict__ mean, float* __restrict__ invstd, float* running_mean,
                                   float* running_var) {
  pdl_wait(); pdl_trigger();
  int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= C) return;
  const int lane = threadIdx.x & 31;
  const int nseg = n0 < n ? 2 : 1;
  float v1[2][FIN_PER_LANE], v2[2][FIN_PER_LANE];
  load_partials(partial, chunks, chunks0, nseg, C, c, lane, v1, v2);
#pragma unroll
  for (int seg = 0; seg < 2; ++seg) {
    if (seg >= nseg) break;
    const float* p = partial + (seg ? (int64_t)chunks0 * 2 * C : 0);
    const int ch = seg ? chunks - chunks0 : chunks0;
    const int64_t rows = seg ? n - n0 : n0;
    double s1 = 0.0;
#pragma unroll
    for (int j = 0; j < FIN_PER_LANE; ++j) s1 += (double)v1[seg][j];
    for (int k = lane + 32 * FIN_PER_LANE; k < ch; k += 32) s1 += p[(int64_t)k * 2 * C + c];
    for (int o = 16; o; o >>= 1) s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    const double m = s1 / (double)rows;
    const double invR = 1.0 / (double)R;
    double M2 = 0.0;
    auto term = [&](int k, float a1, float a2) {
      const int64_t left = rows - (int64_t)k * R;
      const double mk = (double)(left < R ? left : R);
      const double d = (left < R ? (double)a1 / mk : (double)a1 * invR) - m;
      return (double)a2 + mk * d * d;
    };
#pragma unroll
    for (int j = 0; j < FIN_PER_LANE; ++j) {
      const int k = lane + 32 * j;
      if (k < ch) M2 += term(k, v1[seg][j], v2[seg][j]);
    }
    for (int k = lane + 32 * FIN_PER_LANE; k < ch; k += 32) M2 += term(k, p[(int64_t)k * 2 * C + c], p[(int64_t)k * 2 * C + C + c]);
    for (int o = 16; o; o >>= 1) M2 += __shfl_xor_sync(0xffffffffu, M2, o);
    if (lane == 0) {
      double var = M2 / (double)rows;
      if (var < 0.0) var = 0.0;
      mean[seg * C + c] = (float)m;
      invstd[seg * C + c] = (float)(1.0 / sqrt(var + (double)eps));
      if (running_mean) running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)m;
      if (running_var) {
        double unb = rows > 1 ? var * ((double)rows / (double)(rows - 1)) : var;
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unb;
      }
    }
  }
}

__global__ void bn_apply_kernel(const float* __restrict__ X, int ldx, int64_t n4, int cv, const float* __restrict__ mean,
                                const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                                const float* __restrict__ residual, int ldr, int relu, float* __restrict__ Y, int ldy,
                                __nv_bfloat16* __restrict__ Yhi, __nv_bfloat16* __restrict__ Ylo, int lds, int64_t n0, int fp16,
                                __nv_bfloat16* __restrict__ Ybhi, __nv_bfloat16* __restrict__ Yblo) {
  pdl_wait(); pdl_trigger();
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n4) return;
  int c4 = (int)(i % cv);
  const int64_t row = i / cv;
  const int so = row >= n0 ? cv : 0;          // statistics of this row's segment ([segments][C], in float4 units)
  float4 x = __ldg(reinterpret_cast<const float4*>(X + row * ldx) + c4);
  float4 mu = reinterpret_cast<const float4*>(mean)[so + c4], is = reinterpret_cast<const float4*>(invstd)[so + c4];
  float4 g = reinterpret_cast<const float4*>(gamma)[c4], b = reinterpret_cast<const float4*>(beta)[c4];
  float4 y;
  y.x = (x.x - mu.x) * is.x * g.x + b.x; y.y = (x.y - mu.y) * is.y * g.y + b.y;
  y.z = (x.z - mu.z) * is.z * g.z + b.z; y.w = (x.w - mu.w) * is.w * g.w + b.w;
  if (residual) {
    float4 r = __ldg(reinterpret_cast<const float4*>(residual + row * ldr) + c4);
    y.x += r.x; y.y += r.y; y.z += r.z; y.w += r.w;
  }
  if (relu) { y.x = fmaxf(y.x, 0.f); y.y = fmaxf(y.y, 0.f); y.z = fmaxf(y.z, 0.f); y.w = fmaxf(y.w, 0.f); }
  if (Y) *reinterpret_cast<float4*>(Y + row * ldy + c4 * 4) = y;
  if (Yhi) {
    if (fp16) store_split4_f16(y, Yhi + row * lds + c4 * 4, Ylo + row * lds + c4 * 4);
    else store_split4(y, Yhi + row * lds + c4 * 4, Ylo + row * lds + c4 * 4);
  }
  if (Ybhi) store_split4(y, Ybhi + row * lds + c4 * 4, Yblo + row * lds + c4 * 4);
}

// dgamma = sum(dY*xhat), dbeta = sum(dY) over ALL rows (both segments: the parameters are shared);
// sums[seg][0][C] = that segment's dbeta, sums[seg][1][C] = its dgamma for the apply pass.
__global__ void bn_bwd_finalize_kernel(const float* __restrict__ partial, int chunks, int chunks0, int nseg, int C,
                                       float* __restrict__ dgamma, float* __restrict__ dbeta, int accumulate, float* __restrict__ sums) {
  pdl_wait(); pdl_trigger();
  int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= C) return;
  const int lane = threadIdx.x & 31;
  // both segments' partials of this lane in registers first (independent loads, one round trip), then the fp64 shuffle reductions
  float v1[2][FIN_PER_LANE], v2[2][FIN_PER_LANE];
  load_partials(partial, chunks, chunks0, nseg, C, c, lane, v1, v2);
  float tb = 0.f, tg = 0.f;
#pragma unroll
  for (int seg = 0; seg < 2; ++seg) {
    if (seg >= nseg) break;
    const float* p = partial + (seg ? (int64_t)chunks0 * 2 * C : 0);
    const int ch = seg ? chunks - chunks0 : chunks0;
    double s1 = 0.0, s2 = 0.0;
#pragma unroll
    for (int j = 0; j < FIN_PER_LANE; ++j) { s1 += (double)v1[seg][j]; s2 += (double)v2[seg][j]; }
    for (int k = lane + 32 * FIN_PER_LANE; k < ch; k += 32) { s1 += p[(int64_t)k * 2 * C + c]; s2 += p[(int64_t)k * 2 * C + C + c]; }
    for (int o = 16; o; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
    if (lane == 0) {
      sums[seg * 2 * C + c] = (float)s1;
      sums[seg * 2 * C + C + c] = (float)s2;
    }
    if (seg == 0) { tb = (float)s1; tg = (float)s2; }
    else { tb = (float)((double)tb + s1); tg = (float)((double)tg + s2); }
  }
  if (lane != 0) return;
  if (accumulate) { dbeta[c] += tb; dgamma[c] += tg; }
  else { dbeta[c] = tb; dgamma[c] = tg; }
}

// gout_mode: 0 none, 1 write, 2 accumulate -- the (ReLU-masked) incoming gradient, i.e. the gradient of the residual input
__global__ void bn_bwd_apply_kernel(const float* dY, int lddy, const float* __restrict__ X, int ldx,
                                    const __nv_bfloat16* __restrict__ Mask, int ldm, int64_t n4, int cv, int64_t n0, float inv_n0,
                                    float inv_n1, const float* __restrict__ mean, const float* __restrict__ invstd,
                                    const float* __restrict__ gamma, const float* __restrict__ sums, float* __restrict__ dX, int lddx,
                                    float* gout, int ldg, int gout_mode, __nv_bfloat16* __restrict__ dXhi,
                                    __nv_bfloat16* __restrict__ dXlo, int lds) {
  pdl_wait(); pdl_trigger();
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n4) return;
  int c4 = (int)(i % cv);
  const int64_t row = i / cv;
  float4 dy = *(reinterpret_cast<const float4*>(dY + row * lddy) + c4);
  if (Mask) mask4_bf16(Mask + row * ldm + c4 * 4, dy);
  if (gout_mode) {
    float4* gp = reinterpret_cast<float4*>(gout + row * ldg) + c4;
    float4 gv = dy;
    if (gout_mode == 2) { float4 o = *gp; gv.x += o.x; gv.y += o.y; gv.z += o.z; gv.w += o.w; }
    *gp = gv;
  }
  float4 x = __ldg(reinterpret_cast<const float4*>(X + row * ldx) + c4);
  const bool second = row >= n0;
  const int so = second ? cv : 0;
  const float inv_n = second ? inv_n1 : inv_n0;
  float4 mu = reinterpret_cast<const float4*>(mean)[so + c4], is = reinterpret_cast<const float4*>(invstd)[so + c4];
  float4 g = reinterpret_cast<const float4*>(gamma)[c4];
  // sums: [segment][dbeta | dgamma][C]
  float4 db = reinterpret_cast<const float4*>(sums)[2 * so + c4], dg = reinterpret_cast<const float4*>(sums)[2 * so + cv + c4];
  float4 o;
  o.x = g.x * is.x * (dy.x - db.x * inv_n - (x.x - mu.x) * is.x * dg.x * inv_n);
  o.y = g.y * is.y * (dy.y - db.y * inv_n - (x.y - mu.y) * is.y * dg.y * inv_n);
  o.z = g.z * is.z * (dy.z - db.z * inv_n - (x.z - mu.z) * is.z * dg.z * inv_n);
  o.w = g.w * is.w * (dy.w - db.w * inv_n - (x.w - mu.w) * is.w * dg.w * inv_n);
  if (dX) *reinterpret_cast<float4*>(dX + row * lddx + c4 * 4) = o;
  if (dXhi) store_split4(o, dXhi + row * lds + c4 * 4, dXlo + row * lds + c4 * 4);
}

// rows per chunk: a power of two in [16, 1024] near n / 512, so that every level launches a few hundred CTAs
inline int chunk_rows(int64_t n) {
  const int64_t t = n / 512;
  int R = 16;
  while (R < 1024 && (int64_t)R * 3 / 2 < t) R <<= 1;
  return R;
}
inline int chunks_of(int64_t rows, int R) { return (int)((rows + R - 1) / R); }
// A column-statistics launch over rows [0, n) with the segment boundary n0: one CTA per R-row chunk, chunks never straddle n0 (chunks0
// of them in segment 0); block = (C/4) channel-vectors x row lanes, <= 256 threads and at least one row lane; smem: [lanes][2][C].
struct Chunks { int R, chunks, chunks0, threads; size_t smem; };
Chunks chunk_geometry(int64_t n, int64_t n0, int C) {
  const int R = chunk_rows(n);
  const int chunks0 = chunks_of(n0 < n ? n0 : n, R);
  const int cv = C / 4;
  const int rp = 256 / cv < 1 ? 1 : 256 / cv;
  return {R, chunks0 + (n0 < n ? chunks_of(n - n0, R) : 0), chunks0, cv * rp, (size_t)rp * 2 * C * sizeof(float)};
}

// eval-mode BatchNorm: "statistics" = the running ones
__global__ void bn_eval_stats_kernel(const float* __restrict__ running_mean, const float* __restrict__ running_var, int C, float eps,
                                     float* __restrict__ mean, float* __restrict__ invstd) {
  pdl_wait(); pdl_trigger();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) { mean[c] = running_mean[c]; invstd[c] = 1.0f / sqrtf(running_var[c] + eps); }
}

// per-chunk partials [chunks][2][C] (at most one chunk more than n rows make: the two segments round up separately), then the
// backward pass's [2 segments][dbeta | dgamma][C]
struct BnWs { float* partial; float* sums; };
BnWs bn_layout(Carve& c, int64_t n, int C) { return {c.take<float>((int64_t)(chunks_of(n, chunk_rows(n)) + 1) * 2 * C), c.take<float>(2 * 2 * C)}; }

// Forward statistics: colstat_kernel<MODE> (0: of A; 2: of A = the sum of nsplit planes, also written to Y) -> per-chunk partials
// -> bn_finalize_kernel -> mean / invstd / running statistics.
template <int MODE>
int stats_launch(const float* A, int lda, int nsplit, float* Y, int ldy, int64_t n, int64_t n0, int C, float eps, float momentum,
                 float* mean, float* invstd, float* running_mean, float* running_var, void* ws, size_t ws_bytes, cudaStream_t st) {
  Carve c{(char*)ws};
  const BnWs w = bn_layout(c, n, C);
  PCB_ARG(ws_bytes >= c.used);
  const Chunks g = chunk_geometry(n, n0, C);
  launch_kernel(colstat_kernel<MODE>, g.chunks, g.threads, g.smem, st, A, lda, nullptr, 0, nullptr, 0, nsplit, Y, ldy, n, n0, g.chunks0, g.R, C,
                nullptr, nullptr, w.partial);
  if (int e = check_launch(MODE == 2 ? "colstat_kernel<reduce+stats>" : "colstat_kernel<fwd>")) return e;
  launch_kernel(bn_finalize_kernel, (C + 7) / 8, 256, 0, st, (const float*)w.partial, g.chunks, g.chunks0, g.R, n, n0, C, eps, momentum, mean,
                invstd, running_mean, running_var);
  return check_launch("bn_finalize_kernel");
}

}  // namespace

extern "C" size_t pcb_bn_ws_bytes(int64_t n, int C) {
  return layout_bytes(bn_layout, n < 1 ? 1 : n, C);
}

// n0: rows [0, n0) and [n0, n) are separate BatchNorm batches (n0 == n: one batch).  mean / invstd: [segments][C].
extern "C" int pcb_bn_stats_seg(const float* X, int ldx, int64_t n, int64_t n0, int C, float eps, float momentum, float* mean,
                                float* invstd, float* running_mean, float* running_var, void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(X && mean && invstd && ws && n >= 1 && n0 >= 1 && n0 <= n && C >= 4 && C % 4 == 0 && C <= 1024 && ldx >= C && ldx % 4 == 0);
  return stats_launch<0>(X, ldx, 0, nullptr, 0, n, n0, C, eps, momentum, mean, invstd, running_mean, running_var, ws, ws_bytes,
                         (cudaStream_t)stream);
}

extern "C" int pcb_split_rows(const float* X, int ldx, int64_t n, int C, uint16_t* hi, uint16_t* lo, int lds, int flags, void* stream) {
  PCB_ARG(n >= 0 && C >= 4 && C % 4 == 0 && ldx >= C && ldx % 4 == 0 && lds >= C && lds % 4 == 0);
  if (n == 0) return PCB_OK;
  PCB_ARG(X && hi && lo);
  int64_t n4 = n * (C / 4);
  launch_kernel(split_rows_kernel, (unsigned)((n4 + 255) / 256), 256, 0, (cudaStream_t)stream, X, ldx, n4, C / 4, (__nv_bfloat16*)hi,
                (__nv_bfloat16*)lo, lds, (flags & PCB_PLANES_A_FP16) ? 1 : 0);
  return check_launch("split_rows_kernel");
}

extern "C" int pcb_bn_apply_seg(const float* X, int ldx, int64_t n, int64_t n0, int C, const float* mean, const float* invstd,
                                const float* gamma, const float* beta, const float* residual, int ldr, int flags, float* Y, int ldy,
                                uint16_t* Yhi, uint16_t* Ylo, int lds, uint16_t* Ybhi, uint16_t* Yblo, void* stream) {
  const int relu = flags & PCB_BN_RELU;
  // n0 == 0 < n would normalise every row with mean[1] / invstd[1], which no statistics call writes (they require n0 >= 1)
  PCB_ARG(n >= 0 && (n0 >= 1 || n == 0) && n0 <= n && C >= 4 && C % 4 == 0 && ldx % 4 == 0 && ldx >= C && (!Y || (ldy % 4 == 0 && ldy >= C)));
  if (n == 0) return PCB_OK;
  PCB_ARG(X && (Y || Yhi) && mean && invstd && gamma && beta && (!residual || (ldr >= C && ldr % 4 == 0)));
  PCB_ARG(!Yhi || (Ylo && lds >= C && lds % 4 == 0));
  PCB_ARG(!Ybhi || (Yblo && Yhi));
  int64_t n4 = n * (C / 4);
  launch_kernel(bn_apply_kernel, (unsigned)((n4 + 255) / 256), 256, 0, (cudaStream_t)stream, X, ldx, n4, C / 4, mean, invstd, gamma, beta, residual,
                ldr, relu, Y, ldy, (__nv_bfloat16*)Yhi, (__nv_bfloat16*)Ylo, lds, n0, (flags & PCB_PLANES_A_FP16) ? 1 : 0,
                (__nv_bfloat16*)Ybhi, (__nv_bfloat16*)Yblo);
  return check_launch("bn_apply_kernel");
}

// relu_hi: the 16-bit hi plane of the ReLU output (row stride ldmh in elements); NULL: no ReLU
extern "C" int pcb_bn_backward_seg(const float* dY, int lddy, const float* X, int ldx, const uint16_t* relu_hi, int ldmh, int64_t n,
                                   int64_t n0, int C, const float* mean, const float* invstd, const float* gamma, float* dX, int lddx,
                                   float* dgamma, float* dbeta, int accumulate_param_grads, float* gout, int ldg, int gout_mode,
                                   uint16_t* dXhi, uint16_t* dXlo, int lds, void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(dY && X && mean && invstd && gamma && (dX || dXhi) && dgamma && dbeta && ws && n >= 1 && C >= 4 && C % 4 == 0 && C <= 1024);
  PCB_ARG(n0 >= 1 && n0 <= n);
  PCB_ARG(lddy >= C && ldx >= C && lddy % 4 == 0 && ldx % 4 == 0 && (!dX || (lddx >= C && lddx % 4 == 0)));
  PCB_ARG(!dXhi || (dXlo && lds >= C && lds % 4 == 0));
  PCB_ARG(!relu_hi || (ldmh >= C && ldmh % 4 == 0));
  PCB_ARG(gout_mode == 0 || (gout && ldg >= C && ldg % 4 == 0));
  Carve c{(char*)ws};
  const BnWs w = bn_layout(c, n, C);
  PCB_ARG(ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  const int nseg = n0 < n ? 2 : 1;
  const Chunks g = chunk_geometry(n, n0, C);
  launch_kernel(colstat_kernel<1>, g.chunks, g.threads, g.smem, st, dY, lddy, X, ldx, (const __nv_bfloat16*)relu_hi, ldmh, 0, nullptr, 0, n, n0,
                g.chunks0, g.R, C, mean, invstd, w.partial);
  if (int e = check_launch("colstat_kernel<bwd>")) return e;
  launch_kernel(bn_bwd_finalize_kernel, (C + 7) / 8, 256, 0, st, w.partial, g.chunks, g.chunks0, nseg, C, dgamma, dbeta, accumulate_param_grads,
                w.sums);
  if (int e = check_launch("bn_bwd_finalize_kernel")) return e;
  int64_t n4 = n * (C / 4);
  launch_kernel(bn_bwd_apply_kernel, (unsigned)((n4 + 255) / 256), 256, 0, st, dY, lddy, X, ldx, (const __nv_bfloat16*)relu_hi, ldmh, n4,
                                                                    C / 4, n0, 1.0f / (float)n0, nseg == 2 ? 1.0f / (float)(n - n0) : 0.f, mean,
                                                                    invstd, gamma, w.sums, dX, lddx, gout, ldg, gout_mode,
                                                                    (__nv_bfloat16*)dXhi, (__nv_bfloat16*)dXlo, lds);
  return check_launch("bn_bwd_apply_kernel");
}

namespace pcb {
int bn_eval_stats_launch(const float* running_mean, const float* running_var, int C, float eps, float* mean, float* invstd, cudaStream_t st) {
  PCB_ARG(running_mean && running_var && mean && invstd && C >= 1);
  launch_kernel(bn_eval_stats_kernel, (C + 127) / 128, 128, 0, st, running_mean, running_var, C, eps, mean, invstd);
  return check_launch("bn_eval_stats_kernel");
}

// Forward statistics fused into the reduction pass of an offset-split convolution: Y = sum of the nsplit partial planes
// P[z][n][C], BatchNorm statistics of Y (segments [0, n0) / [n0, n)) -> mean / invstd / running statistics.  ws: pcb_bn_ws_bytes(n, C).
int bn_reduce_stats_launch(const float* P, int nsplit, float* Y, int ldy, int64_t n, int64_t n0, int C, float eps, float momentum,
                           float* mean, float* invstd, float* running_mean, float* running_var, void* ws, size_t ws_bytes, cudaStream_t st) {
  PCB_ARG(P && Y && ws && nsplit >= 1 && n >= 1 && n0 >= 1 && n0 <= n && C % 4 == 0 && C <= 1024 && ldy >= C && ldy % 4 == 0);
  return stats_launch<2>(P, 0, nsplit, Y, ldy, n, n0, C, eps, momentum, mean, invstd, running_mean, running_var, ws, ws_bytes, st);
}
}  // namespace pcb
