// PointInfoNCE on the tensor cores, fused: the N x D . D x N feature-similarity contraction (`lib/ddp_trainer.py:420-426`,
// `lib/criterion.py:15-19`: logits = q k^T / T, cross-entropy against the diagonal) as wgmma tiles, the softmax statistics and both
// gradients computed straight from those tiles -- the n x n logits matrix (67 MB at n = 4096) is never written anywhere.
//
//   S[i][j] = q_i . k_j / T          loss = mean_i( lse_i - S[i][i] ),  lse_i = log sum_j exp S[i][j]
//   dq_i = ( sum_j P[i][j] k_j - k_i ) / (T n),   dk_j = ( sum_i P[i][j] q_i - q_j ) / (T n),   P[i][j] = exp(S[i][j] - lse_i)
//
// One kernel, three roles (template MODE), CTA = 128 rows of the "own" matrix X x a range of 128-row blocks of the "other" matrix Y:
//   X and Y rows are split fp32 -> fp16 hi/lo (|features| <= 1 after the L2 normalisation: 2^-22 per operand) and laid out as
//   K-major no-swizzle wgmma tiles; each of the two warpgroups issues 3 x D/16 MMAs (lo.hi + hi.lo + hi.hi, M64 x N128 x K16) for its
//   64 rows, and stores its accumulator fragments into a padded fp32 tile in shared memory; all 8 warps then read their rows'
//   16-column chunks back and
//     MODE_LSE : keep an online (max, sum exp) per row and pick up the diagonal logit      -> partial (m, l), S[i][i]
//     MODE_DX  : P = exp(S - lse_row);  acc[d] += P . Y[j][d]   (fp32 FMAs, Y rows broadcast from shared memory)   -> dq partials
//     MODE_DY  : the same with X = k, Y = q and lse indexed by COLUMN (the tile is S^T)                            -> dk partials
//   The column range is split over gridDim.y CTAs per row block so that ~one wave of SMs is busy; a small combine kernel merges the
//   partial statistics / partial gradients in a fixed order (deterministic).
// Exact-fp32 SIMT kernels (loss.cu) remain for feature widths other than 32 / 64.
#include <cuda_fp16.h>
#include "common.cuh"
#include "wgmma_ptx.cuh"

using namespace pcb;
using namespace pcb::hw;

namespace {

constexpr int XM = 128;          // rows of X per CTA (two warpgroups x M64)
constexpr int YN = 128;          // rows of Y per tile (= MMA N)
constexpr int S_LD = YN + 4;     // fp32 tile row stride: a warp reading 16 B per lane from 32 consecutive rows is conflict-free
constexpr int NTHR = 256;
enum { MODE_LSE = 0, MODE_DX = 1, MODE_DY = 2 };

struct NceArgs {
  const float* X; const float* Y;          // [n, D] row-major fp32 (X: own rows, Y: the other matrix)
  int64_t n; int D; float inv_T;
  const float* lse;                         // [n] (MODE_DX: indexed by X row, MODE_DY: by Y row)
  float* part_ml;                           // MODE_LSE: [splits][n][2] partial (max, sum exp)
  float* diag;                              // MODE_LSE: [n] S[i][i]
  float* part_d;                            // MODE_DX / MODE_DY: [splits][n][D] partial sums  sum_j P . Y[j]
  int tiles_per_split;
};

__device__ __forceinline__ void split_f16(float v, __half& h, __half& l) {
  h = __float2half_rn(v);
  l = __float2half_rn(v - __half2float(h));
}

// K-major, no-swizzle wgmma tile of `rows` x D fp16: core matrix = 8 rows x 16 B; k8-group stride LBO, 8-row-group stride 128 B
__device__ __forceinline__ uint32_t tile_off(int r, int c, int lbo) { return (c >> 3) * lbo + (r >> 3) * 128 + (r & 7) * 16 + (c & 7) * 2; }

template <int MODE, int D>
__global__ void __launch_bounds__(NTHR, 1) nce_wgmma_kernel(const NceArgs p) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2;
  constexpr int X_LBO = (XM / 8) * 128 + 16, Y_LBO = (YN / 8) * 128 + 16;
  constexpr int X_PLANE = (D / 8) * X_LBO, Y_PLANE = (D / 8) * Y_LBO;
  unsigned char* sXh = smem;                          // X tile hi / lo
  unsigned char* sXl = sXh + X_PLANE;
  unsigned char* sYh = sXl + X_PLANE;                 // Y tile hi / lo
  unsigned char* sYl = sYh + Y_PLANE;
  float* sS = reinterpret_cast<float*>(sYl + Y_PLANE);          // the S tile [XM][S_LD] in fp32 (unscaled)
  float* sYf = sS + XM * S_LD;                                  // Y tile in fp32 [YN][D] (MODE_DX / MODE_DY), column lse [YN] after it
  float* sLse = sYf + (MODE == MODE_LSE ? 0 : YN * D);
  float* sRed = sLse + YN;                                      // cross-half combine: [XM][D] (or [XM][2])
  const int64_t row0 = (int64_t)blockIdx.x * XM;
  const int ntiles = (int)((p.n + YN - 1) / YN);
  const int t0 = blockIdx.y * p.tiles_per_split, t1 = min(ntiles, t0 + p.tiles_per_split);

  pdl_wait(); pdl_trigger();
  // X tile: 128 rows x D, split to fp16 hi/lo (rows beyond n are zero)
  for (int e = tid; e < XM * D; e += NTHR) {
    const int r = e / D, c = e - r * D;
    const float v = row0 + r < p.n ? p.X[(row0 + r) * D + c] : 0.f;
    __half h, l; split_f16(v, h, l);
    const uint32_t o = tile_off(r, c, X_LBO);
    *reinterpret_cast<__half*>(sXh + o) = h; *reinterpret_cast<__half*>(sXl + o) = l;
  }

  const int q = warp & 3, half = warp >> 2;             // consumer view: row quarter, column half of the tile
  const int64_t my_row = row0 + q * 32 + lane;
  float lse_row = 0.f;
  if (MODE == MODE_DX && my_row < p.n) lse_row = p.lse[my_row];
  float m_run = -INFINITY, l_run = 0.f, diag = 0.f;     // MODE_LSE
  float acc[D];                                         // MODE_DX / MODE_DY: sum_j P[i][j] Y[j][0..D)
#pragma unroll
  for (int d = 0; d < D; ++d) acc[d] = 0.f;
  const float L2E = 1.4426950408889634f;

  for (int t = t0; t < t1; ++t) {
    const int64_t col0 = (int64_t)t * YN;
    // ---- stage the Y tile: fp16 hi/lo wgmma planes (+ fp32 copy and column lse for the gradient modes)
    for (int e = tid; e < YN * D; e += NTHR) {
      const int r = e / D, c = e - r * D;
      const float v = col0 + r < p.n ? p.Y[(col0 + r) * D + c] : 0.f;
      __half h, l; split_f16(v, h, l);
      const uint32_t o = tile_off(r, c, Y_LBO);
      *reinterpret_cast<__half*>(sYh + o) = h; *reinterpret_cast<__half*>(sYl + o) = l;
      if (MODE != MODE_LSE) sYf[e] = v;
    }
    if (MODE == MODE_DY)
      for (int e = tid; e < YN; e += NTHR) sLse[e] = col0 + e < p.n ? p.lse[col0 + e] : 0.f;
    fence_proxy_async();          // generic-proxy smem writes -> visible to the tensor cores (async proxy)
    __syncthreads();
    {
      // ---- this warpgroup's 64 rows x 128 columns of S, then its fragments -> the fp32 tile
      float s[YN / 2];
#pragma unroll
      for (int e = 0; e < YN / 2; ++e) s[e] = 0.f;
      fence_regs(s);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < D / 16; ++j) {
        const uint32_t xo = wg * 8 * 128 + j * 2 * X_LBO, yo = j * 2 * Y_LBO;
        const uint64_t dxh = make_desc(smem_u32(sXh) + xo, X_LBO, 128), dxl = make_desc(smem_u32(sXl) + xo, X_LBO, 128);
        const uint64_t dyh = make_desc(smem_u32(sYh) + yo, Y_LBO, 128), dyl = make_desc(smem_u32(sYl) + yo, Y_LBO, 128);
        wgmma<YN, true, 0, 0>(s, dxl, dyh, 1u);
        wgmma<YN, true, 0, 0>(s, dxh, dyl, 1u);
        wgmma<YN, true, 0, 0>(s, dxh, dyh, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float* dst = sS + (wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h) * S_LD + 2 * (lane & 3);
#pragma unroll
        for (int c = 0; c < YN / 8; ++c) *reinterpret_cast<float2*>(dst + 8 * c) = make_float2(s[4 * c + 2 * h], s[4 * c + 2 * h + 1]);
      }
    }
    __syncthreads();
    // ---- consume the tile: this thread's row, columns [half * 64, +64) in chunks of 16
#pragma unroll 1
    for (int c0 = 0; c0 < YN / 2; c0 += 16) {
      const int cb = half * (YN / 2) + c0;
      float r[16];
      const float4* src = reinterpret_cast<const float4*>(sS + (q * 32 + lane) * S_LD + cb);
#pragma unroll
      for (int e4 = 0; e4 < 4; ++e4) {
        const float4 x = src[e4];
        r[4 * e4] = x.x; r[4 * e4 + 1] = x.y; r[4 * e4 + 2] = x.z; r[4 * e4 + 3] = x.w;
      }
      if (MODE == MODE_LSE) {
        float cm = -INFINITY;
#pragma unroll
        for (int e = 0; e < 16; ++e) {
          const float sv = r[e] * p.inv_T;
          r[e] = sv;
          if (col0 + cb + e < p.n) cm = fmaxf(cm, sv);
          if (col0 + cb + e == my_row) diag = sv;
        }
        if (cm > -INFINITY) {
          const float mn = fmaxf(m_run, cm);
          float add = 0.f;
#pragma unroll
          for (int e = 0; e < 16; ++e)
            if (col0 + cb + e < p.n) add += exp2f((r[e] - mn) * L2E);
          l_run = l_run * exp2f((m_run - mn) * L2E) + add;
          m_run = mn;
        }
      } else {
#pragma unroll 4
        for (int e = 0; e < 16; ++e) {
          const int j = cb + e;
          const float ls = MODE == MODE_DX ? lse_row : sLse[j];
          const float pj = col0 + j < p.n ? exp2f((r[e] * p.inv_T - ls) * L2E) : 0.f;
          const float4* yr = reinterpret_cast<const float4*>(sYf + j * D);
#pragma unroll
          for (int d4 = 0; d4 < D / 4; ++d4) {
            const float4 y = yr[d4];
            acc[d4 * 4 + 0] = fmaf(pj, y.x, acc[d4 * 4 + 0]); acc[d4 * 4 + 1] = fmaf(pj, y.y, acc[d4 * 4 + 1]);
            acc[d4 * 4 + 2] = fmaf(pj, y.z, acc[d4 * 4 + 2]); acc[d4 * 4 + 3] = fmaf(pj, y.w, acc[d4 * 4 + 3]);
          }
        }
      }
    }
    __syncthreads();          // every warp is done with the S tile and the Y tile before the next tile overwrites them
  }

  // ---- combine the two column halves of each row (fixed order) and write this split's partial
  const int rr = q * 32 + lane;
  if (MODE == MODE_LSE) {
    if (half == 1) { sRed[rr * 2] = m_run; sRed[rr * 2 + 1] = l_run; }
    __syncthreads();
    if (half == 0 && my_row < p.n) {
      const float m2 = sRed[rr * 2], l2 = sRed[rr * 2 + 1];
      const float mn = fmaxf(m_run, m2);
      float l = 0.f;
      if (mn > -INFINITY) l = (m_run > -INFINITY ? l_run * exp2f((m_run - mn) * L2E) : 0.f) + (m2 > -INFINITY ? l2 * exp2f((m2 - mn) * L2E) : 0.f);
      float* o = p.part_ml + ((int64_t)blockIdx.y * p.n + my_row) * 2;
      o[0] = mn; o[1] = l;
    }
    // the diagonal logit lives in exactly one (split, half): whoever saw it writes it
    const int64_t dc = my_row;      // column index of the diagonal
    if (my_row < p.n && dc >= (int64_t)t0 * YN && dc < (int64_t)t1 * YN && ((dc % YN) >= YN / 2) == (half == 1)) p.diag[my_row] = diag;
  } else {
    if (half == 1) {
#pragma unroll
      for (int d = 0; d < D; ++d) sRed[rr * D + d] = acc[d];
    }
    __syncthreads();
    if (half == 0 && my_row < p.n) {
      float* o = p.part_d + ((int64_t)blockIdx.y * p.n + my_row) * D;
#pragma unroll
      for (int d = 0; d < D; ++d) o[d] = acc[d] + sRed[rr * D + d];
    }
  }
}

// lse_i from the per-split (max, sum) pairs; rowloss_i = lse_i - S[i][i]
__global__ void nce_lse_combine_kernel(const float* __restrict__ part_ml, const float* __restrict__ diag, int splits, int64_t n,
                                       float* __restrict__ lse, float* __restrict__ rowloss) {
  pdl_wait(); pdl_trigger();
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float m = -INFINITY;
  for (int s = 0; s < splits; ++s) m = fmaxf(m, part_ml[((int64_t)s * n + i) * 2]);
  float l = 0.f;
  for (int s = 0; s < splits; ++s) {
    const float ms = part_ml[((int64_t)s * n + i) * 2], ls = part_ml[((int64_t)s * n + i) * 2 + 1];
    if (ms > -INFINITY) l += ls * expf(ms - m);
  }
  const float v = m + logf(l);
  lse[i] = v;
  rowloss[i] = v - diag[i];
}

// d[i][:] = ( sum_s part[s][i][:] - partner[i][:] ) * scale
__global__ void nce_grad_combine_kernel(const float* __restrict__ part, const float* __restrict__ partner, int splits, int64_t n, int D,
                                        float scale, float* __restrict__ out) {
  pdl_wait(); pdl_trigger();
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n * D) return;
  float s = 0.f;
  for (int k = 0; k < splits; ++k) s += part[(int64_t)k * n * D + e];
  out[e] = (s - partner[e]) * scale;
}

__global__ void nce_mean_kernel(const float* __restrict__ v, int64_t n, float* __restrict__ out) {
  pdl_wait(); pdl_trigger();
  __shared__ double sm[32];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s += v[i];
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sm[w];
    *out = (float)(t / (double)n);
  }
}

size_t nce_smem_bytes(int D, int mode) {
  const int X_LBO = (XM / 8) * 128 + 16, Y_LBO = (YN / 8) * 128 + 16;
  size_t b = 2 * (size_t)(D / 8) * X_LBO + 2 * (size_t)(D / 8) * Y_LBO + (size_t)XM * S_LD * 4;
  b += (mode == MODE_LSE ? 0 : (size_t)YN * D * 4) + YN * 4 + (size_t)XM * (mode == MODE_LSE ? 2 : D) * 4 + 64;
  return b;
}

template <int MODE, int D>
int launch_nce_d(const NceArgs& a, int splits, cudaStream_t st) {
  const size_t smem = nce_smem_bytes(D, MODE);
  static bool attr_set[64] = {};          // per device: the opt-in is a per-device function attribute
  const int dev_ = current_device();
  if (!attr_set[dev_]) {
    PCB_CUDA(cudaFuncSetAttribute(nce_wgmma_kernel<MODE, D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set[dev_] = true;
  }
  dim3 grid((unsigned)((a.n + XM - 1) / XM), splits);
  launch_kernel(nce_wgmma_kernel<MODE, D>, grid, NTHR, smem, st, a);
  return check_launch("nce_wgmma_kernel");
}

template <int MODE>
int launch_nce(const NceArgs& a, int splits, cudaStream_t st) {
  return a.D == 32 ? launch_nce_d<MODE, 32>(a, splits, st) : launch_nce_d<MODE, 64>(a, splits, st);
}

// [part_ml: ntiles*n*2][diag: n][lse: n][rowloss: n][part_d: ntiles*n*D]  (splits <= ntiles)
struct NceTcWs { float* part_ml; float* diag; float* lse; float* rowloss; float* part_d; };
NceTcWs nce_tc_layout(Carve& c, int64_t n, int D) {
  const int64_t ntiles = (n + YN - 1) / YN;
  return {c.take<float>(ntiles * n * 2), c.take<float>(n), c.take<float>(n), c.take<float>(n), c.take<float>(ntiles * n * D)};
}

}  // namespace

namespace pcb {

bool nce_tc_supported(int64_t n, int D) { return (D == 32 || D == 64) && n >= 1; }

size_t nce_tc_ws_bytes(int64_t n, int D) {
  return layout_bytes(nce_tc_layout, n, D);
}

int nce_tc_forward_backward(const float* q, const float* k, int64_t n, int D, float inv_T, float* loss, float* dq, float* dk, void* ws,
                            cudaStream_t st) {
  const int rowblocks = (int)((n + XM - 1) / XM), ntiles = (int)((n + YN - 1) / YN);
  int splits = num_sms() / rowblocks;
  if (splits < 1) splits = 1;
  if (splits > ntiles) splits = ntiles;
  const int tps = (ntiles + splits - 1) / splits;
  splits = (ntiles + tps - 1) / tps;
  Carve c{(char*)ws};
  const auto [part_ml, diag, lse, rowloss, part_d] = nce_tc_layout(c, n, D);
  NceArgs a;
  a.X = q; a.Y = k; a.n = n; a.D = D; a.inv_T = inv_T; a.lse = nullptr; a.part_ml = part_ml; a.diag = diag; a.part_d = part_d; a.tiles_per_split = tps;
  if (int e = launch_nce<MODE_LSE>(a, splits, st)) return e;
  launch_kernel(nce_lse_combine_kernel, (unsigned)((n + 255) / 256), 256, 0, st, part_ml, diag, splits, n, lse, rowloss);
  if (int e = check_launch("nce_lse_combine_kernel")) return e;
  launch_kernel(nce_mean_kernel, 1, 1024, 0, st, rowloss, n, loss);
  if (int e = check_launch("nce_mean_kernel")) return e;
  const float scale = inv_T / (float)n;
  a.lse = lse;
  if (int e = launch_nce<MODE_DX>(a, splits, st)) return e;                      // dq: X = q, Y = k, lse by row
  launch_kernel(nce_grad_combine_kernel, (unsigned)((n * D + 255) / 256), 256, 0, st, part_d, k, splits, n, D, scale, dq);
  if (int e = check_launch("nce_grad_combine_kernel")) return e;
  a.X = k; a.Y = q;
  if (int e = launch_nce<MODE_DY>(a, splits, st)) return e;                      // dk: X = k, Y = q, lse by column
  launch_kernel(nce_grad_combine_kernel, (unsigned)((n * D + 255) / 256), 256, 0, st, part_d, q, splits, n, D, scale, dk);
  return check_launch("nce_grad_combine_kernel");
}

}  // namespace pcb
