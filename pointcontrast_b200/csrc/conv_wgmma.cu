// Hopper sparse convolution: the output-stationary gather-GEMM of conv.cu with the per-offset Cin x Cout contraction issued as
// wgmma.mma_async, fp32 accumulators in registers.  CTA = 128 output rows x BN channels = one producer warpgroup and two consumer
// warpgroups of M64.  The producer gathers the input, 16-bit hi/lo planes, per offset by cp.async (zero-filled where there is no
// neighbour) into the K-major no-swizzle core-matrix layout, and fetches the weights, pre-tiled as shared-memory images, by one TMA
// bulk copy per stage; both complete on the stage's mbarrier.  Per 32-channel step each consumer warpgroup issues 2 k16-steps x 3
// products (lo.hi + hi.lo + hi.hi).  Offsets without a neighbour in the tile are skipped; small levels split the steps over
// gridDim.z (partial planes + fixed-order reduce).
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
constexpr int A_SBO = 128;
// k8-chunk stride of the A tile: +32 bytes, so that the four 16-byte chunks (t & 3) x two rows (t >> 2) written by a quarter-warp of a
// 128-bit st.shared cover eight different 16-byte slots of a 128-byte bank line.
constexpr int A_LBO = (BM / 8) * 128 + 32;
constexpr int A_PLANE = (BK / 8) * A_LBO;

struct Args {
  const __nv_bfloat16* Xhi; const __nv_bfloat16* Xlo; int lds;      // the input as 16-bit hi/lo planes
  const int32_t* tbl; int64_t tbl_stride;
  int kmap[PCB_MAX_KERNEL_VOLUME]; int K;
  int64_t n_out; int Cin; int Cout;
  const unsigned char* wt;                                      // weights pre-tiled as shared-memory images
  const float* bias;
  float* Y; int ldy;
  float* partial;
  int accumulate;       // Y += result (direct mode only; the split mode accumulates in the reduce kernel)
  float out_scale;      // applied to the accumulators on the way out (2^-10 when the weight tiles hold fp16(W * 2^10))
};

// The ring takes every slot that fits beside the table slice in the CTA's share of shared memory.  BN = 128 and 96 run one CTA per
// SM, with 6 and 7 slots.  BN = 64 and 32 run two CTAs per SM with 4 slots each: on an H100 that beat one CTA with 8 and 10 slots
// at every BN <= 64 layer shape of the C1 training step (up to 22 % less kernel time, 0.65 ms less per step).
template <int BN>
struct Smem {
  static constexpr int B_SBO = 128;
  static constexpr int B_LBO = (BN / 8) * 128 + 16;
  static constexpr int B_PLANE = (BK / 8) * B_LBO;
  static constexpr int STAGE = 2 * A_PLANE + 2 * B_PLANE;
  static constexpr int CTAS = BN <= 64 ? 2 : 1;                                  // resident CTAs per SM
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
  extern __shared__ __align__(128) unsigned char smem[];
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
    // this tile's slice of the neighbour table -> shared memory; all loads of a thread are issued before the first store
    constexpr int FILL = (PCB_MAX_KERNEL_VOLUME * BM + NTHR - 1) / NTHR;
    int vals[FILL];
#pragma unroll
    for (int f = 0; f < FILL; ++f) {
      const int e = tid + f * NTHR;
      int v = -1;
      if (e < p.K * BM) {
        const int k = e / BM, r = e - k * BM;
        const int64_t row = row0 + r;
        if (row < p.n_out) v = __ldg(p.tbl + (int64_t)p.kmap[k] * p.tbl_stride + row);
      }
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
        const uint32_t dst = sb + k8 * A_LBO + (r >> 3) * A_SBO + (r & 7) * 16;
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
      const uint32_t a_hi = smem_base + s * S::STAGE + h64 * 8 * A_SBO, a_lo = a_hi + A_PLANE;
      const uint32_t b_hi = smem_base + s * S::STAGE + 2 * A_PLANE, b_lo = b_hi + S::B_PLANE;
      fence_regs(acc);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < BK / 16; ++j) {
        const uint64_t dah = make_desc(a_hi + j * 2 * A_LBO, A_LBO, A_SBO), dal = make_desc(a_lo + j * 2 * A_LBO, A_LBO, A_SBO);
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
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t row = row0 + h64 * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    if (row >= p.n_out) continue;
    float* dst = outp + row * ldo + n0;
#pragma unroll
    for (int c = 0; c < BN / 8; ++c) {
      const int col = c * 8 + 2 * (lane & 3);
      float2 o = make_float2(acc[4 * c + 2 * h] * p.out_scale, acc[4 * c + 2 * h + 1] * p.out_scale);
      if (bias) { o.x += bias[n0 + col]; o.y += bias[n0 + col + 1]; }
      if (p.accumulate && !p.partial) {
        const float2 old = *reinterpret_cast<const float2*>(dst + col);
        o.x += old.x; o.y += old.y;
      }
      *reinterpret_cast<float2*>(dst + col) = o;
    }
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
                      const int* kmap, int K, int64_t n_out, int Cin, int Cout, const float* bias, float* Y, int ldy,
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
// wgmma view: D_k[M = Ca-block (padded to 128)][N = Cb-block] += A_k[M x 16 rows] . B[16 rows x N]; both operands MN-major
// (a matrix row is contiguous along channels): core matrix = 8 rows (K) x 16 B (8 channels), channel-chunk stride SBO = 144 B,
// 8-row-group stride LBO.  Warpgroup g computes the channel rows 64g .. 64g + 63 of the block.
// A CTA owns a GROUP of WG_GROUP kernel offsets and a range of table rows: the row-aligned operand B is staged ONCE per 16-row step and
// shared by the gathered operands A_k, each accumulating into its own register accumulator.  Thread = (row, 16-byte channel chunk) of
// the step; its copies are cp.async (zero-filled where there is no neighbour), the table entries they depend on are fetched TF steps
// earlier into registers so that no dependent global-load latency sits on the per-step path.
// grid: x = groups * mblocks * nblocks, y = row splits; partial tiles are reduced by wgrad_reduce_kernel (conv.cu).
int wgrad_group() { return 2; }

namespace wg {

// NS-slot ring, loads PF = NS - 2 steps ahead: the slot written at step i was last read by the MMAs of step i - 2, which every
// warpgroup has waited for (wgmma.wait_group 1) before the barrier of step i - 1.
constexpr int WM = 128, WK = 16, GK = 2, NTHR = 256, NS = 4, PF = NS - 2, TF = 2;

struct Args {
  const __nv_bfloat16* Ahi; const __nv_bfloat16* Alo; int lda;      // gathered operand (elements)
  const __nv_bfloat16* Bhi; const __nv_bfloat16* Blo; int ldb;      // row-aligned operand
  const int32_t* tbl; int64_t tbl_stride;
  int K; int64_t n_out; int Ca; int Cb; int rows_per_split;
  float* partial; int transpose_out;
};

// channel-chunk (core-matrix) stride 144 B, not 128: the 16 threads of one row write 16 consecutive chunks, and a 128-byte stride
// would put them on the same shared-memory banks
constexpr int SBO = 144;
__host__ __device__ inline int a_lbo(int mrows) { return (mrows / 8) * SBO + 16; }
__host__ __device__ inline int b_lbo(int tn) { return (tn / 8) * SBO + 16; }
__host__ __device__ inline int stage_bytes(int mrows, int tn) { return 4 * b_lbo(tn) + GK * 4 * a_lbo(mrows); }

template <int TN>
__global__ void __launch_bounds__(NTHR, 1) wgrad_wgmma_kernel(const Args p) {
  using namespace hw;
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = warp >> 2;
  const int mblocks = (p.Ca + WM - 1) / WM, nblocks = p.Cb / TN;
  int bx = blockIdx.x;
  const int nb = bx % nblocks; bx /= nblocks;
  const int mb = bx % mblocks; bx /= mblocks;
  const int k0 = bx * GK;
  const int nk = min(GK, p.K - k0);
  const int m0 = mb * WM, n0 = nb * TN;
  const int mrows = min(WM, p.Ca - m0);                 // valid M rows of this block (multiple of 32)
  const int ach = mrows / 8;
  constexpr int BCH = TN / 8;
  const int A_LBO = a_lbo(mrows), B_LBO = b_lbo(TN);
  const int STAGE = stage_bytes(mrows, TN);
  const int64_t r_begin = (int64_t)blockIdx.y * p.rows_per_split;
  const int64_t r_end = min(p.n_out, r_begin + p.rows_per_split);
  const int nsteps = r_end > r_begin ? (int)((r_end - r_begin + WK - 1) / WK) : 0;
  const uint32_t smem_base = smem_u32(smem);
  pdl_wait(); pdl_trigger();

  const int r = tid >> 4, ch = tid & 15;                // row of the step, 16-byte channel chunk
  const bool a_on = ch < ach, b_on = ch < BCH;
  const uint32_t a_dst = (r >> 3) * A_LBO + ch * SBO + (r & 7) * 16;
  const uint32_t b_dst = (r >> 3) * B_LBO + ch * SBO + (r & 7) * 16;
  const int64_t a_col = m0 + ch * 8, b_col = n0 + ch * 8;
  const int32_t* trow = p.tbl + (int64_t)k0 * p.tbl_stride;
  int tq[TF + PF][GK];                                  // table entries of steps issued .. issued + TF + PF - 1
  auto fetch = [&](int (&d)[GK], int step) {
    const int64_t row = r_begin + (int64_t)step * WK + r;
    const bool live = step < nsteps && row < r_end;
#pragma unroll
    for (int g = 0; g < GK; ++g) d[g] = (live && g < nk) ? __ldg(trow + g * p.tbl_stride + row) : -1;
  };
  // copies of step i into slot i % NS (one cp.async group per call, possibly empty); consumes tq[0] and shifts the table ring
  int issued = 0;
  auto load = [&]() {
    if (issued < nsteps) {
      const int64_t row = r_begin + (int64_t)issued * WK + r;
      const uint32_t sb = smem_base + (issued % NS) * STAGE;
      bool any = false;
#pragma unroll
      for (int g = 0; g < GK; ++g) any |= tq[0][g] >= 0;
      if (b_on) {
        const int64_t off = (any ? row : 0) * p.ldb + b_col;
        cp_async16_zfill(sb + b_dst, p.Bhi + off, any ? 16u : 0u);
        cp_async16_zfill(sb + 2 * B_LBO + b_dst, p.Blo + off, any ? 16u : 0u);
      }
      if (a_on) {
#pragma unroll
        for (int g = 0; g < GK; ++g) {
          const int c = tq[0][g];
          const int64_t off = (int64_t)(c >= 0 ? c : 0) * p.lda + a_col;
          const uint32_t ab = sb + 4 * B_LBO + g * 4 * A_LBO + a_dst;
          cp_async16_zfill(ab, p.Ahi + off, c >= 0 ? 16u : 0u);
          cp_async16_zfill(ab + 2 * A_LBO, p.Alo + off, c >= 0 ? 16u : 0u);
        }
      }
    }
    cp_async_commit();
#pragma unroll
    for (int f = 0; f + 1 < TF + PF; ++f) {
#pragma unroll
      for (int g = 0; g < GK; ++g) tq[f][g] = tq[f + 1][g];
    }
    fetch(tq[TF + PF - 1], issued + TF + PF);
    ++issued;
  };

  float acc[GK][TN / 2];
#pragma unroll
  for (int g = 0; g < GK; ++g) {
#pragma unroll
    for (int e = 0; e < TN / 2; ++e) acc[g][e] = 0.f;
  }
  if (nsteps > 0) {
#pragma unroll
    for (int f = 0; f < TF + PF; ++f) fetch(tq[f], f);
#pragma unroll 1
    for (int i = 0; i < PF; ++i) load();
    for (int i = 0; i < nsteps; ++i) {
      const int s = i % NS;
      cp_async_wait<PF - 1>();
      fence_proxy_async();
      __syncthreads();
      // issued unconditionally (branch-free, so the wgmma's stay asynchronous): the A slots of a missing second offset are
      // zero-filled, and the fragment rows of an upper warpgroup beyond mrows are never read back
      const uint32_t sb = smem_base + s * STAGE;
      const uint64_t dbh = make_desc(sb, B_LBO, SBO), dbl = make_desc(sb + 2 * B_LBO, B_LBO, SBO);
#pragma unroll
      for (int g = 0; g < GK; ++g) fence_regs(acc[g]);
      wgmma_fence();
#pragma unroll
      for (int g = 0; g < GK; ++g) {
        const uint32_t ab = sb + 4 * B_LBO + g * 4 * A_LBO + wgi * 8 * SBO;
        const uint64_t dah = make_desc(ab, A_LBO, SBO), dal = make_desc(ab + 2 * A_LBO, A_LBO, SBO);
        wgmma<TN, false, 1, 1>(acc[g], dal, dbh, 1u);
        wgmma<TN, false, 1, 1>(acc[g], dah, dbl, 1u);
        wgmma<TN, false, 1, 1>(acc[g], dah, dbh, 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();
#pragma unroll
      for (int g = 0; g < GK; ++g) fence_regs(acc[g]);
      load();                 // step i + PF: its slot was last read by the MMAs of step i - 2
    }
    wgmma_wait<0>();
#pragma unroll
    for (int g = 0; g < GK; ++g) fence_regs(acc[g]);
  }

  // ---- epilogue: accumulator g, fragment row m (channel of A), column n (channel of B) -> partial tile of offset k0 + g
#pragma unroll
  for (int g = 0; g < GK; ++g) {
    if (g >= nk) break;
    float* out = p.partial + ((int64_t)blockIdx.y * p.K + k0 + g) * (int64_t)p.Ca * p.Cb;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = wgi * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
      if (m >= mrows) continue;
#pragma unroll
      for (int c = 0; c < TN / 8; ++c) {
        const int col = n0 + c * 8 + 2 * (lane & 3);
        const float x0 = acc[g][4 * c + 2 * h], x1 = acc[g][4 * c + 2 * h + 1];
        if (!p.transpose_out) {
          *reinterpret_cast<float2*>(out + (int64_t)(m0 + m) * p.Cb + col) = make_float2(x0, x1);
        } else {
          out[(int64_t)col * p.Ca + m0 + m] = x0;
          out[(int64_t)(col + 1) * p.Ca + m0 + m] = x1;
        }
      }
    }
  }
}

template <int TN>
int launch(const Args& a, int splits, cudaStream_t st) {
  static bool attr_set[64] = {};          // per device: the opt-in is a per-device function attribute
  const int mrows_max = a.Ca < WM ? a.Ca : WM;
  // + 4 KB: the M = 64 descriptor of the upper warpgroup of a 96-channel block reads (and ignores) a few hundred bytes past the
  // last staged chunk
  const size_t smem = (size_t)NS * stage_bytes(mrows_max, TN) + 4096;
  const int dev_ = current_device();
  if (!attr_set[dev_]) {
    PCB_CUDA(cudaFuncSetAttribute(wgrad_wgmma_kernel<TN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  NS * stage_bytes(WM, 128) + 4096));
    attr_set[dev_] = true;
  }
  const int groups = (a.K + GK - 1) / GK;
  dim3 grid((unsigned)(groups * ((a.Ca + WM - 1) / WM) * (a.Cb / TN)), splits);
  launch_kernel(wgrad_wgmma_kernel<TN>, grid, NTHR, smem, st, a);
  return check_launch("wgrad_wgmma_kernel");
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
  switch (tn) {
    case 128: return wg::launch<128>(a, splits, st);
    case 96: return wg::launch<96>(a, splits, st);
    case 64: return wg::launch<64>(a, splits, st);
    default: return wg::launch<32>(a, splits, st);
  }
}

}  // namespace pcb
