// Hopper sparse convolution: the output-stationary gather-GEMM of conv.cu with the per-offset Cin x Cout contraction issued as
// wgmma.mma_async, fp32 accumulators in registers.  CTA = 128 output rows x BN channels = one producer warpgroup and two consumer
// warpgroups of M64.  The producer gathers the input, 16-bit hi/lo planes, per offset by cp.async (zero-filled where there is no
// neighbour) into the 64-byte swizzled K-major layout, and fetches the weights, pre-tiled as shared-memory images, by one TMA
// bulk copy per stage; both complete on the stage's mbarrier.  Per 32-channel step each consumer warpgroup issues 2 k16-steps x 3
// products (lo.hi + hi.lo + hi.hi).  Offsets without a neighbour in the tile are skipped; small levels split the steps over
// gridDim.z (partial planes + fixed-order reduce).  With a tile order `perm` (pcb_conv_tile_order), tile position i is output row
// perm[i]: rows with the same neighbour offsets share tiles, so the skip drops whole pipeline steps; every row still takes its own
// offsets in ascending order, and the steps it skips would have added exact zeros, so a direct launch computes the same bits.
#include "common.cuh"
#include "wgmma_ptx.cuh"

using namespace pcb;

namespace pcb {

namespace hw {

// Warpgroup 0 produces, warpgroups 1 and 2 consume.  Ring slot s has two mbarriers: full[s] (the producer's 128 threads arrive
// through cp.async.mbarrier.arrive.noinc, thread 0 once more with the weight tile's expect_tx) and empty[s] (lane 0 of each of the
// 8 consumer warps, once wgmma.wait_group shows that the MMAs reading the slot have retired).
constexpr int BM = 128, BK = 32, NPROD = 128, NCONS_WARPS = 8, NTHR = NPROD + 32 * NCONS_WARPS;
constexpr int SMEM_OPTIN = 227 * 1024, SMEM_PER_SM = 228 * 1024;      // sm_90: largest dynamic shared memory of one CTA, of one SM
// A tile plane: the 64-byte swizzled K-major layout of wgmma (SWIZZLE_64B): tile row r's 32 channels are the 64 bytes at 64 r, its
// 16-byte chunk c stored at chunk c ^ ((r >> 1) & 3).  The 8-row atoms (512 bytes) follow each other, and a k16 step starts 32 bytes
// into the row.  A quarter-warp's copy (two rows x four chunks) covers one 128-byte bank line.  The weight-gradient kernel (wg::)
// stores its MN-major atoms with the same byte pattern.
constexpr int A_ROW = BK * 2, A_ATOM = 8 * A_ROW;
constexpr int A_PLANE = BM * A_ROW;
__device__ __forceinline__ uint32_t a_chunk(int r, int c) { return r * A_ROW + ((c ^ ((r >> 1) & 3)) << 4); }
__device__ __forceinline__ uint64_t a_desc(uint32_t saddr) { return make_desc(saddr, 16, A_ATOM) | (2ull << 62); }   // layout type 2: 64B swizzle

struct Args {
  const __nv_bfloat16* Xhi; const __nv_bfloat16* Xlo; int lds;      // the input as 16-bit hi/lo planes
  const int32_t* tbl; int64_t tbl_stride;
  int kmap[PCB_MAX_KERNEL_VOLUME]; int K;
  const int32_t* perm;  // output row of each tile position, or NULL (identity)
  int64_t n_out; int Cin; int Cout;
  const unsigned char* wt;                                      // weights pre-tiled as shared-memory images
  const float* bias;
  float* Y; int ldy;
  float* partial;
  int accumulate;       // Y += result (direct mode only; the split mode accumulates in the reduce kernel)
  float out_scale;      // applied to the accumulators on the way out (2^-10 when the weight tiles hold fp16(W * 2^10))
};

// The ring takes every slot that fits beside the table slice in the CTA's share of shared memory.  BN = 128 runs one CTA per SM with
// 6 slots.  BN = 96, 64 and 32 run two CTAs per SM with 3, 4 and 4 slots each: on an H100 that beat one CTA with 7, 8 and 10 slots
// at the C1 training step's layer shapes (BN <= 64: up to 22 % less kernel time, 0.65 ms less per step; BN = 96: 1.3 ms less
// kernel time per step, DESIGN.md section 7).  While one CTA loads its table slice, fills its ring or writes its tile out, the
// other keeps the tensor cores busy.  BN = 128 stays at one CTA: its consumers need 90 registers, above the 85 of two CTAs.
template <int BN>
struct Smem {
  static constexpr int B_SBO = 128;
  static constexpr int B_LBO = (BN / 8) * 128 + 16;
  static constexpr int B_PLANE = (BK / 8) * B_LBO;
  static constexpr int STAGE = (2 * A_PLANE + 2 * B_PLANE + 511) / 512 * 512;   // A planes stay aligned to the 512-byte swizzle atom
  static constexpr int CTAS = BN <= 96 ? 2 : 1;                                  // resident CTAs per SM
  static constexpr int BUDGET = CTAS == 1 ? SMEM_OPTIN : SMEM_PER_SM / 2 - 1024;  // 1 KB per CTA is reserved by the system
  static constexpr int FIXED = PCB_MAX_KERNEL_VOLUME * BM * 4 + 72 * 4 + 16;
  static constexpr int NS = (BUDGET - FIXED) / (STAGE + 16);                      // + full and empty barrier per slot
  static constexpr int IDX_OFF = NS * STAGE;
  static constexpr int META_OFF = IDX_OFF + PCB_MAX_KERNEL_VOLUME * BM * 4;     // flags[32] klist[32] nk
  static constexpr int BAR_OFF = META_OFF + 72 * 4;                               // full[NS], empty[NS]
  static constexpr int TOTAL = BAR_OFF + 2 * NS * 8 + 16;
  static_assert(TOTAL <= BUDGET, "ring does not fit");
};

template <int BN, bool F16>
__global__ void __launch_bounds__(NTHR, Smem<BN>::CTAS) conv_wgmma_kernel(const Args p) {
  using S = Smem<BN>;
  constexpr int NS = S::NS;
  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2;
  const int64_t row0 = (int64_t)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  int* s_idx = reinterpret_cast<int*>(smem + S::IDX_OFF);
  int* s_flag = reinterpret_cast<int*>(smem + S::META_OFF);
  int* s_klist = s_flag + 32;
  int* s_nk = s_klist + 32;
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t full_bar = smem_base + S::BAR_OFF;          // "A rows and weight tile of slot s landed"
  const uint32_t empty_bar = full_bar + 8 * NS;              // "the MMAs reading slot s have retired"

  if (tid == 0) {
    for (int i = 0; i < NS; ++i) {
      mbar_init(full_bar + 8 * i, NPROD + 1);
      mbar_init(empty_bar + 8 * i, NCONS_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  pdl_wait(); pdl_trigger();        // no global memory touched before this
  {
    // this tile's slice of the neighbour table -> shared memory; all loads of a thread are issued before the first store.  A thread
    // loads the entries of one tile row (NTHR is a multiple of BM): offsets tid / BM, + NTHR / BM, ...
    static_assert(NTHR % BM == 0, "one tile row per thread");
    constexpr int FILL = (PCB_MAX_KERNEL_VOLUME * BM + NTHR - 1) / NTHR;
    const int64_t row = row0 + tid % BM;
    const int64_t orow = row < p.n_out ? (p.perm ? (int64_t)__ldg(p.perm + row) : row) : -1;
    int vals[FILL];
#pragma unroll
    for (int f = 0; f < FILL; ++f) {
      const int e = tid + f * NTHR;
      int v = -1;
      if (e < p.K * BM && orow >= 0) v = __ldg(p.tbl + (int64_t)p.kmap[e / BM] * p.tbl_stride + orow);
      vals[f] = v;
    }
#pragma unroll
    for (int f = 0; f < FILL; ++f) {
      const int e = tid + f * NTHR;
      if (e < p.K * BM) s_idx[e] = vals[f];
    }
  }
  __syncthreads();
  for (int k = warp; k < p.K; k += NTHR / 32) {
    unsigned any = 0;
#pragma unroll
    for (int s = 0; s < 4; ++s) any |= __ballot_sync(0xffffffffu, s_idx[k * BM + s * 32 + lane] >= 0);
    if (lane == 0) s_flag[k] = any ? 1 : 0;
  }
  __syncthreads();
  if (warp == 0) {                  // offsets with at least one neighbour in this tile, in order (K <= 27 < 32: one ballot)
    static_assert(PCB_MAX_KERNEL_VOLUME <= 32, "one ballot per tile");
    const int f = lane < p.K ? s_flag[lane] : 0;
    const unsigned m = __ballot_sync(0xffffffffu, f != 0);
    if (f) s_klist[__popc(m & ((1u << lane) - 1u))] = lane;
    if (lane == 0) *s_nk = __popc(m);
  }
  __syncthreads();
  const int nk = *s_nk;
  const int nkc = p.Cin / BK;
  const int T = nk * nkc;
  const int it0 = (int)((int64_t)T * blockIdx.z / gridDim.z);
  const int it1 = (int)((int64_t)T * (blockIdx.z + 1) / gridDim.z);
  const int n_it = it1 - it0;
  const int nblk = p.Cout / BN;
  constexpr uint32_t BLOB = 2 * S::B_PLANE;

  // ---- pipeline step i (relative to it0) uses slot i % NS, in its (i / NS)-th round
  if (wg == 0) {
    // producer: thread t copies the 16-byte k8-chunk t % 4 of rows t / 4 + 32 q (q < 4) of both planes, zero-filled where there
    // is no neighbour; thread 0 also issues the stage's weight tile, one TMA bulk copy of the pre-tiled image
    const int k8 = tid & 3, r0 = tid >> 2;
#pragma unroll 1
    for (int i = 0; i < n_it; ++i) {
      const int it = it0 + i, s = i % NS;
      const int k = s_klist[it / nkc], kc = it % nkc;
      const uint32_t sb = smem_base + s * S::STAGE;
      mbar_wait(empty_bar + 8 * s, (uint32_t)(((i / NS) & 1) ^ 1));    // round 0 passes at once
      if (tid == 0) {
        mbar_arrive_expect_tx(full_bar + 8 * s, BLOB);
        tma_bulk_load(sb + 2 * A_PLANE, p.wt + ((int64_t)(k * nkc + kc) * nblk + blockIdx.y) * BLOB, BLOB, full_bar + 8 * s);
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int r = r0 + 32 * q;
        const int idx = s_idx[k * BM + r];
        const int64_t off = (int64_t)(idx >= 0 ? idx : 0) * p.lds + kc * BK + k8 * 8;
        const uint32_t dst = sb + a_chunk(r, k8);
        cp_async16_zfill(dst, p.Xhi + off, idx >= 0 ? 16u : 0u);
        cp_async16_zfill(dst + A_PLANE, p.Xlo + off, idx >= 0 ? 16u : 0u);
      }
      cp_async_mbar_arrive_noinc(full_bar + 8 * s);
    }
    cp_async_commit();
    cp_async_wait<0>();         // no copy of this thread outlives it
    return;
  }

  // consumers: warpgroup 1 + h owns the rows 64 h .. 64 h + 63 of the tile
  const int h64 = wg - 1;
  float acc[BN / 2];
#pragma unroll
  for (int e = 0; e < BN / 2; ++e) acc[e] = 0.f;
  if (n_it > 0) {
    for (int i = 0; i < n_it; ++i) {
      const int s = i % NS;
      mbar_wait(full_bar + 8 * s, (uint32_t)((i / NS) & 1));
      fence_proxy_async();                             // generic-proxy smem writes (cp.async) -> visible to the tensor cores
      const uint32_t a_hi = smem_base + s * S::STAGE + h64 * 64 * A_ROW, a_lo = a_hi + A_PLANE;
      const uint32_t b_hi = smem_base + s * S::STAGE + 2 * A_PLANE, b_lo = b_hi + S::B_PLANE;
      fence_regs(acc);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < BK / 16; ++j) {
        const uint64_t dah = a_desc(a_hi + j * 32), dal = a_desc(a_lo + j * 32);
        const uint64_t dbh = make_desc(b_hi + j * 2 * S::B_LBO, S::B_LBO, S::B_SBO);
        const uint64_t dbl = make_desc(b_lo + j * 2 * S::B_LBO, S::B_LBO, S::B_SBO);
        wgmma<BN, F16, 0, 0>(acc, dal, dbh, 1u);
        wgmma<BN, F16, 0, 0>(acc, dah, dbl, 1u);
        wgmma<BN, F16, 0, 0>(acc, dah, dbh, 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();                                 // the MMAs of step i - 1 have retired: release its slot
      fence_regs(acc);
      if (i > 0 && lane == 0) mbar_arrive(empty_bar + 8 * ((i - 1) % NS));
    }
    wgmma_wait<0>();
    fence_regs(acc);
  }

  // ---- epilogue from the accumulator fragments: row 64 h64 + 16 (warp % 4) + lane / 4 (+ 8), columns 8 c + 2 (lane % 4) (+ 1)
  float* outp = p.partial ? p.partial + (int64_t)blockIdx.z * p.n_out * p.Cout : p.Y;
  const int ldo = p.partial ? p.Cout : p.ldy;
  const float* bias = p.partial ? nullptr : p.bias;
  // Every read of Y (PCB_CONV_ACCUMULATE) is issued before the first write: a store to dst followed by a load from dst would make each
  // load wait for the one before it, one memory round trip per 8 columns.
  float* dst[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t row = row0 + h64 * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    dst[h] = row < p.n_out ? outp + (p.perm ? (int64_t)__ldg(p.perm + row) : row) * ldo + n0 : nullptr;
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!dst[h]) continue;
#pragma unroll
    for (int c = 0; c < BN / 8; ++c) {
      const int col = c * 8 + 2 * (lane & 3);
      float& x = acc[4 * c + 2 * h];
      float& y = acc[4 * c + 2 * h + 1];
      x *= p.out_scale; y *= p.out_scale;
      if (bias) { x += bias[n0 + col]; y += bias[n0 + col + 1]; }
      if (p.accumulate && !p.partial) {
        const float2 old = *reinterpret_cast<const float2*>(dst[h] + col);
        x += old.x; y += old.y;
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!dst[h]) continue;
#pragma unroll
    for (int c = 0; c < BN / 8; ++c)
      *reinterpret_cast<float2*>(dst[h] + c * 8 + 2 * (lane & 3)) = make_float2(acc[4 * c + 2 * h], acc[4 * c + 2 * h + 1]);
  }
}

template <int BN, bool F16>
int launch_cfg(const Args& a, int nsplit, cudaStream_t st) {
  using S = Smem<BN>;
  static bool attr_set[64] = {};          // per device: the opt-in is a per-device function attribute
  const int dev_ = current_device();
  if (!attr_set[dev_]) {
    PCB_CUDA(cudaFuncSetAttribute(conv_wgmma_kernel<BN, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
    attr_set[dev_] = true;
  }
  dim3 grid((unsigned)((a.n_out + BM - 1) / BM), a.Cout / BN, nsplit);
  launch_kernel(conv_wgmma_kernel<BN, F16>, grid, NTHR, S::TOTAL, st, a);
  return check_launch("conv_wgmma_kernel");
}

template <int BN>
int launch(const Args& a, int nsplit, cudaStream_t st, int f16) {
  return f16 ? launch_cfg<BN, true>(a, nsplit, st) : launch_cfg<BN, false>(a, nsplit, st);
}

}  // namespace hw

// Called by conv_forward_split_impl (conv.cu).  wt: the weights of this call's roles pre-tiled by pcb_weight_tile[_batch].
int launch_conv_wgmma(const uint16_t* Xhi, const uint16_t* Xlo, int lds, const void* wt, const int32_t* tbl, int64_t tbl_stride,
                      const int* kmap, int K, const int32_t* perm, int64_t n_out, int Cin, int Cout, const float* bias, float* Y, int ldy,
                      float* partial, int nsplit, int bn, int accumulate, cudaStream_t st, int x_fp16, int w_fp16) {
  // wgmma takes ONE 16-bit format for both operands
  if (x_fp16 != w_fp16) { set_error("conv: fp16 and bf16 operand planes cannot be mixed"); return PCB_ERR_ARG; }
  hw::Args a;
  a.accumulate = accumulate;
  a.out_scale = w_fp16 ? 1.0f / 1024.0f : 1.0f;
  a.Xhi = (const __nv_bfloat16*)Xhi; a.Xlo = (const __nv_bfloat16*)Xlo; a.lds = lds;
  a.wt = (const unsigned char*)wt;
  a.tbl = tbl; a.tbl_stride = tbl_stride; a.K = K; a.n_out = n_out; a.Cin = Cin; a.Cout = Cout;
  for (int k = 0; k < K; ++k) a.kmap[k] = kmap[k];
  a.perm = perm;
  a.bias = bias; a.Y = Y; a.ldy = ldy;
  a.partial = partial;
  switch (bn) {
    case 128: return hw::launch<128>(a, nsplit, st, x_fp16);
    case 96: return hw::launch<96>(a, nsplit, st, x_fp16);
    case 64: return hw::launch<64>(a, nsplit, st, x_fp16);
    default: return hw::launch<32>(a, nsplit, st, x_fp16);
  }
}

// ------------------------------------------------------------------------------------------------ weight gradient
// dW[k] (Ca x Cb) = sum_j A[tbl[k][j], :]^T . B[j, :] on split (16-bit hi/lo) operands.
// A CTA owns a group of GK kernel offsets, a CB-channel block of A (CB = pick_tile(Ca)), a TN-channel block of B and one row split.
// The offsets are stacked along M: D[M = GK offsets x CB channels][N = TN] += A[M x 16 rows] . B[16 rows x N], so the row-aligned
// operand B is staged once per row step and shared by every offset of the group, and GK * CB fills whole M64 slices without padding.
// Both operands are MN-major (a matrix row is contiguous along channels) in wgmma's 64-byte swizzled layout: an atom is 8 rows (K) x
// 32 channels, row r's 64 bytes at 64 (r % 8) with its 16-byte chunk c at chunk c ^ ((r >> 1) & 3) (hw::a_chunk, the forward kernel's
// A-tile pattern); atoms follow each other along the channels (LBO = hw::A_ATOM), then along the rows (SBO = one 8-row group of atoms).
// The stacked A tile's atoms run (offset, channel).
// Warpgroup 0 produces: per 32-row stage, the zero-filling cp.async copies of B's rows (not read where no offset of the group has a
// neighbour) and of every offset's gathered A rows, completing on the slot's "full" mbarrier; the table entries they depend on are
// loaded TF stages earlier into registers.  Warpgroups 1 and 2 consume, each SL of the tile's M64 slices, and release a slot on its
// "empty" mbarrier once wgmma.wait_group shows that the MMAs reading it have retired.  Within a split, every accumulator element takes
// the k16 steps in ascending row order and per step the products lo.hi, hi.lo, hi.hi.
// grid: x = groups * mblocks * nblocks, y = row splits; partial tiles are reduced by wgrad_reduce_kernel (conv.cu).
namespace wg {

constexpr int WK = 16, NPROD = 128, NCONS_WARPS = 8, NTHR = NPROD + 32 * NCONS_WARPS, TF = 4;
// registers per thread after setmaxnreg: 128 x 40 + 256 x 232 <= 64 K; the consumers hold up to 3 x 64 accumulators (CB = 96, TN = 128)
constexpr int PROD_REGS = 40, CONS_REGS = 232;

struct Args {
  const __nv_bfloat16* Ahi; const __nv_bfloat16* Alo; int lda;      // gathered operand (elements)
  const __nv_bfloat16* Bhi; const __nv_bfloat16* Blo; int ldb;      // row-aligned operand
  const int32_t* tbl; int64_t tbl_stride;
  int K; int64_t n_out; int Ca; int Cb; int rows_per_split;
  float* partial; int transpose_out;
};

// MN-major 64-byte swizzled operand: LBO = the stride between atoms along M / N, SBO = the stride between 8-row groups along K;
// layout type 2: 64B swizzle
__device__ __forceinline__ uint64_t mn_desc(uint32_t saddr, uint32_t sbo) { return hw::make_desc(saddr, hw::A_ATOM, sbo) | (2ull << 62); }

// Stage = B hi, B lo, A hi, A lo planes of RS rows, each a multiple of 2 KB, so every atom stays 512-byte aligned; the ring takes
// every slot that fits.
template <int CB, int TN>
struct Smem {
  static constexpr int GK = CB % 64 == 0 ? 2 : 4;        // offsets per CTA: GK * CB is a multiple of 128 (two consumers x M64)
  static constexpr int MT = GK * CB;
  static constexpr int SL = MT / 128;                     // M64 slices per consumer warpgroup
  static constexpr int RS = 32;                           // rows per stage
  static constexpr int NQ = RS / 32;                      // rows per producer thread
  static constexpr int A_SBO = MT / 32 * hw::A_ATOM, B_SBO = TN / 32 * hw::A_ATOM;   // one 8-row group of atoms
  static constexpr int A_PLANE = RS / 8 * A_SBO, B_PLANE = RS / 8 * B_SBO;
  static constexpr int A_OFF = 2 * B_PLANE;
  static constexpr int STAGE = 2 * B_PLANE + 2 * A_PLANE;
  static constexpr int NS = (hw::SMEM_OPTIN - 16) / (STAGE + 16);    // + full and empty barrier per slot
  static constexpr int BAR_OFF = NS * STAGE;
  static constexpr int TOTAL = BAR_OFF + 2 * NS * 8;
  static_assert(MT % 128 == 0 && NS >= 3 && TOTAL <= hw::SMEM_OPTIN, "weight-gradient tile does not fit");
};

template <int CB, int TN>
__global__ void __launch_bounds__(NTHR, 1) wgrad_wgmma_kernel(const Args p) {
  using namespace hw;
  using S = Smem<CB, TN>;
  constexpr int GK = S::GK, NS = S::NS, RS = S::RS, NQ = S::NQ, ACH = CB / 8, BCH = TN / 8;
  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = warp >> 2;
  const int mblocks = p.Ca / CB, nblocks = p.Cb / TN;
  int bx = blockIdx.x;
  const int nb = bx % nblocks; bx /= nblocks;
  const int mb = bx % mblocks; bx /= mblocks;
  const int k0 = bx * GK;
  const int nk = min(GK, p.K - k0);                     // offsets of this group; the A rows of the others are zero-filled
  const int m0 = mb * CB, n0 = nb * TN;
  const int64_t r_begin = (int64_t)blockIdx.y * p.rows_per_split;
  const int64_t r_end = min(p.n_out, r_begin + p.rows_per_split);
  const int nst = r_end > r_begin ? (int)((r_end - r_begin + RS - 1) / RS) : 0;
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t full_bar = smem_base + S::BAR_OFF;     // "B and A rows of slot s landed"
  const uint32_t empty_bar = full_bar + 8 * NS;         // "the MMAs reading slot s have retired"
  if (tid == 0) {
    for (int i = 0; i < NS; ++i) {
      mbar_init(full_bar + 8 * i, NPROD);
      mbar_init(empty_bar + 8 * i, NCONS_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  pdl_wait(); pdl_trigger();
  __syncthreads();

  // ---- stage i (RS rows from r_begin + RS i) uses slot i % NS, in its (i / NS)-th round
  if (wgi == 0) {
    setmaxnreg_dec<PROD_REGS>();
    // thread: rows r + 32 q of every stage, 16-byte channel chunks c4 + 4 j of B and of each offset's A block.  A warp's copy covers
    // 8 rows x 64 contiguous bytes in global memory and one 8-row group of atoms in shared memory; a quarter-warp's (two rows x four
    // chunks) fills one 128-byte bank line.
    const int r = 8 * warp + (lane >> 2), c4 = lane & 3;
    const uint32_t dst = a_chunk(r & 7, c4);
    const uint32_t dst_b = dst + (r >> 3) * S::B_SBO, dst_a = S::A_OFF + dst + (r >> 3) * S::A_SBO;
    int tq[TF + 1][NQ][GK];                              // table entries of stages i .. i + TF
    auto fetch = [&](int (&d)[NQ][GK], int st) {
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int64_t row = r_begin + (int64_t)st * RS + r + 32 * q;
#pragma unroll
        for (int g = 0; g < GK; ++g)
          d[q][g] = (row < r_end && g < nk) ? __ldg(p.tbl + (int64_t)(k0 + g) * p.tbl_stride + row) : -1;
      }
    };
#pragma unroll
    for (int f = 0; f < TF; ++f) fetch(tq[f], f);
#pragma unroll 1
    for (int i = 0; i < nst; ++i) {
      fetch(tq[TF], i + TF);
      const int s = i % NS;
      mbar_wait(empty_bar + 8 * s, (uint32_t)(((i / NS) & 1) ^ 1));    // round 0 passes at once
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int64_t row = r_begin + (int64_t)i * RS + r + 32 * q;
        const uint32_t sb = smem_base + s * S::STAGE + q * 4 * S::B_SBO, sa = smem_base + s * S::STAGE + q * 4 * S::A_SBO;
        bool any = false;
#pragma unroll
        for (int g = 0; g < GK; ++g) any |= tq[0][q][g] >= 0;
        const int64_t boff = (any ? row : 0) * p.ldb + n0 + c4 * 8;
#pragma unroll
        for (int j = 0; j < BCH / 4; ++j) {
          cp_async16_zfill(sb + dst_b + j * A_ATOM, p.Bhi + boff + j * 32, any ? 16u : 0u);
          cp_async16_zfill(sb + S::B_PLANE + dst_b + j * A_ATOM, p.Blo + boff + j * 32, any ? 16u : 0u);
        }
#pragma unroll
        for (int g = 0; g < GK; ++g) {
          const int c = tq[0][q][g];
          const int64_t aoff = (int64_t)(c >= 0 ? c : 0) * p.lda + m0 + c4 * 8;
#pragma unroll
          for (int j = 0; j < ACH / 4; ++j) {
            const uint32_t d = sa + dst_a + (g * ACH / 4 + j) * A_ATOM;
            cp_async16_zfill(d, p.Ahi + aoff + j * 32, c >= 0 ? 16u : 0u);
            cp_async16_zfill(d + S::A_PLANE, p.Alo + aoff + j * 32, c >= 0 ? 16u : 0u);
          }
        }
      }
      cp_async_mbar_arrive_noinc(full_bar + 8 * s);
#pragma unroll
      for (int f = 0; f < TF; ++f) {
#pragma unroll
        for (int q = 0; q < NQ; ++q) {
#pragma unroll
          for (int g = 0; g < GK; ++g) tq[f][q][g] = tq[f + 1][q][g];
        }
      }
    }
    cp_async_commit();
    cp_async_wait<0>();         // no copy of this thread outlives it
    return;
  }

  // consumers: warpgroup 1 + h owns the M64 slices h SL .. h SL + SL - 1 of the stacked tile
  setmaxnreg_inc<CONS_REGS>();
  const int h = wgi - 1;
  float acc[S::SL][TN / 2];
#pragma unroll
  for (int sl = 0; sl < S::SL; ++sl) {
#pragma unroll
    for (int e = 0; e < TN / 2; ++e) acc[sl][e] = 0.f;
  }
  if (nst > 0) {
#pragma unroll 1
    for (int i = 0; i < nst; ++i) {
      const int s = i % NS;
      mbar_wait(full_bar + 8 * s, (uint32_t)((i / NS) & 1));
      fence_proxy_async();                             // generic-proxy smem writes (cp.async) -> visible to the tensor cores
      const uint32_t sb = smem_base + s * S::STAGE;
#pragma unroll
      for (int sl = 0; sl < S::SL; ++sl) fence_regs(acc[sl]);
      wgmma_fence();
      // issued unconditionally (branch-free, so the wgmma's stay asynchronous): rows past the split's end are zero-filled, and the
      // fragment rows of offsets past K are never read back
#pragma unroll
      for (int kk = 0; kk < RS / WK; ++kk) {
        // a k16 step is two 8-row groups; an M64 slice of A is two atoms
        const uint32_t b_hi = sb + kk * 2 * S::B_SBO;
        const uint64_t dbh = mn_desc(b_hi, S::B_SBO), dbl = mn_desc(b_hi + S::B_PLANE, S::B_SBO);
#pragma unroll
        for (int sl = 0; sl < S::SL; ++sl) {
          const uint32_t a_hi = sb + S::A_OFF + kk * 2 * S::A_SBO + (h * S::SL + sl) * 2 * A_ATOM;
          const uint64_t dah = mn_desc(a_hi, S::A_SBO), dal = mn_desc(a_hi + S::A_PLANE, S::A_SBO);
          wgmma<TN, false, 1, 1>(acc[sl], dal, dbh, 1u);
          wgmma<TN, false, 1, 1>(acc[sl], dah, dbl, 1u);
          wgmma<TN, false, 1, 1>(acc[sl], dah, dbh, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();                                 // the MMAs of stage i - 1 have retired: release its slot
#pragma unroll
      for (int sl = 0; sl < S::SL; ++sl) fence_regs(acc[sl]);
      if (i > 0 && lane == 0) mbar_arrive(empty_bar + 8 * ((i - 1) % NS));
    }
    wgmma_wait<0>();
#pragma unroll
    for (int sl = 0; sl < S::SL; ++sl) fence_regs(acc[sl]);
  }

  // ---- epilogue: fragment row m of the stacked tile = channel m0 + m % CB of offset k0 + m / CB, column n = channel of B
#pragma unroll
  for (int sl = 0; sl < S::SL; ++sl) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int m = (h * S::SL + sl) * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * hh;
      const int g = m / CB, ch = m0 + m % CB;
      if (g >= nk) continue;
      float* out = p.partial + ((int64_t)blockIdx.y * p.K + k0 + g) * (int64_t)p.Ca * p.Cb;
#pragma unroll
      for (int c = 0; c < TN / 8; ++c) {
        const int col = n0 + c * 8 + 2 * (lane & 3);
        const float x0 = acc[sl][4 * c + 2 * hh], x1 = acc[sl][4 * c + 2 * hh + 1];
        if (!p.transpose_out) {
          *reinterpret_cast<float2*>(out + (int64_t)ch * p.Cb + col) = make_float2(x0, x1);
        } else {
          out[(int64_t)col * p.Ca + ch] = x0;
          out[(int64_t)(col + 1) * p.Ca + ch] = x1;
        }
      }
    }
  }
}

template <int CB, int TN>
int launch_cfg(const Args& a, int splits, cudaStream_t st) {
  using S = Smem<CB, TN>;
  static bool attr_set[64] = {};          // per device: the opt-in is a per-device function attribute
  const int dev_ = current_device();
  if (!attr_set[dev_]) {
    PCB_CUDA(cudaFuncSetAttribute(wgrad_wgmma_kernel<CB, TN>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
    attr_set[dev_] = true;
  }
  const int groups = (a.K + S::GK - 1) / S::GK;
  dim3 grid((unsigned)(groups * (a.Ca / CB) * (a.Cb / TN)), splits);
  launch_kernel(wgrad_wgmma_kernel<CB, TN>, grid, NTHR, S::TOTAL, st, a);
  return check_launch("wgrad_wgmma_kernel");
}

template <int CB>
int launch(const Args& a, int splits, int tn, cudaStream_t st) {
  switch (tn) {
    case 128: return launch_cfg<CB, 128>(a, splits, st);
    case 96: return launch_cfg<CB, 96>(a, splits, st);
    case 64: return launch_cfg<CB, 64>(a, splits, st);
    default: return launch_cfg<CB, 32>(a, splits, st);
  }
}

}  // namespace wg

// Called by pcb_conv_wgrad_split (conv.cu): both operands as bf16 hi/lo planes.
int launch_wgrad_wgmma(const uint16_t* Ahi, const uint16_t* Alo, int lda, const uint16_t* Bhi, const uint16_t* Blo, int ldb,
                       const int32_t* tbl, int64_t tbl_stride, int K, int64_t n_out, int Ca, int Cb, int rows_per_split, int splits,
                       float* partial, int transpose_out, int tn, cudaStream_t st) {
  wg::Args a;
  a.Ahi = (const __nv_bfloat16*)Ahi; a.Alo = (const __nv_bfloat16*)Alo; a.lda = lda;
  a.Bhi = (const __nv_bfloat16*)Bhi; a.Blo = (const __nv_bfloat16*)Blo; a.ldb = ldb;
  a.tbl = tbl; a.tbl_stride = tbl_stride; a.K = K; a.n_out = n_out; a.Ca = Ca; a.Cb = Cb; a.rows_per_split = rows_per_split;
  a.partial = partial; a.transpose_out = transpose_out;
  switch (pick_tile(Ca)) {
    case 128: return wg::launch<128>(a, splits, tn, st);
    case 96: return wg::launch<96>(a, splits, tn, st);
    case 64: return wg::launch<64>(a, splits, tn, st);
    default: return wg::launch<32>(a, splits, tn, st);
  }
}

}  // namespace pcb
