// wgmma / mbarrier / TMA / cp.async PTX wrappers shared by the Hopper tensor-core kernels (conv_wgmma.cu, nce_wgmma.cu).  sm_90a only.
#pragma once
#include "common.cuh"

namespace pcb {
namespace hw {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(dst), "l"(src));
}
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void* src, uint32_t src_bytes) {   // src_bytes 16 or 0
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar) : "memory");
}
// one arrival on bar once every cp.async this thread has issued so far has landed; .noinc: the arrival counts against the
// barrier's initial count
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];\n" ::"r"(bar) : "memory");
}
// TMA 1-D bulk copy global -> shared (async proxy), completion signalled on an mbarrier
__device__ __forceinline__ void tma_bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// wgmma shared-memory matrix descriptor, no swizzle: 8 x 16-byte core matrices.  K-major operand: LBO = byte stride between the two
// core matrices of one k16 step (K direction), SBO = byte stride between 8-row groups (M/N direction).  MN-major operand: LBO = byte
// stride between 8-row groups (K direction), SBO = byte stride between 8-element chunks (M/N direction).
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  const uint32_t lo = ((saddr >> 4) & 0x3FFFu) | (((lbo >> 4) & 0x3FFFu) << 16);
  const uint32_t hi = (sbo >> 4) & 0x3FFFu;
  return ((uint64_t)hi << 32) | lo;
}

// Per-thread register budget of the executing warpgroup (warp-specialised kernels: producer down, consumers up).
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(R)); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// Keeps the compiler from moving accumulator reads / writes across a wgmma.fence / wait (the registers are written asynchronously).
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] . B[16 x N], fp32 accumulators in the issuing warpgroup's registers.  TA / TB: 0 = K-major, 1 = MN-major.
// Fragment of thread t (warp w = t / 32 of the warpgroup, lane l): d[4i + 2h + e] = D[16w + l/4 + 8h][8i + 2(l%4) + e].
#define PCB_WG_D16 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}"
#define PCB_WG_C16(d) "+f"(d[0]),"+f"(d[1]),"+f"(d[2]),"+f"(d[3]),"+f"(d[4]),"+f"(d[5]),"+f"(d[6]),"+f"(d[7]),"+f"(d[8]),"+f"(d[9]),"+f"(d[10]),"+f"(d[11]),"+f"(d[12]),"+f"(d[13]),"+f"(d[14]),"+f"(d[15])
#define PCB_WG_D32 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}"
#define PCB_WG_C32(d) "+f"(d[0]),"+f"(d[1]),"+f"(d[2]),"+f"(d[3]),"+f"(d[4]),"+f"(d[5]),"+f"(d[6]),"+f"(d[7]),"+f"(d[8]),"+f"(d[9]),"+f"(d[10]),"+f"(d[11]),"+f"(d[12]),"+f"(d[13]),"+f"(d[14]),"+f"(d[15]),"+f"(d[16]),"+f"(d[17]),"+f"(d[18]),"+f"(d[19]),"+f"(d[20]),"+f"(d[21]),"+f"(d[22]),"+f"(d[23]),"+f"(d[24]),"+f"(d[25]),"+f"(d[26]),"+f"(d[27]),"+f"(d[28]),"+f"(d[29]),"+f"(d[30]),"+f"(d[31])
#define PCB_WG_D48 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}"
#define PCB_WG_C48(d) "+f"(d[0]),"+f"(d[1]),"+f"(d[2]),"+f"(d[3]),"+f"(d[4]),"+f"(d[5]),"+f"(d[6]),"+f"(d[7]),"+f"(d[8]),"+f"(d[9]),"+f"(d[10]),"+f"(d[11]),"+f"(d[12]),"+f"(d[13]),"+f"(d[14]),"+f"(d[15]),"+f"(d[16]),"+f"(d[17]),"+f"(d[18]),"+f"(d[19]),"+f"(d[20]),"+f"(d[21]),"+f"(d[22]),"+f"(d[23]),"+f"(d[24]),"+f"(d[25]),"+f"(d[26]),"+f"(d[27]),"+f"(d[28]),"+f"(d[29]),"+f"(d[30]),"+f"(d[31]),"+f"(d[32]),"+f"(d[33]),"+f"(d[34]),"+f"(d[35]),"+f"(d[36]),"+f"(d[37]),"+f"(d[38]),"+f"(d[39]),"+f"(d[40]),"+f"(d[41]),"+f"(d[42]),"+f"(d[43]),"+f"(d[44]),"+f"(d[45]),"+f"(d[46]),"+f"(d[47])
#define PCB_WG_D64 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}"
#define PCB_WG_C64(d) "+f"(d[0]),"+f"(d[1]),"+f"(d[2]),"+f"(d[3]),"+f"(d[4]),"+f"(d[5]),"+f"(d[6]),"+f"(d[7]),"+f"(d[8]),"+f"(d[9]),"+f"(d[10]),"+f"(d[11]),"+f"(d[12]),"+f"(d[13]),"+f"(d[14]),"+f"(d[15]),"+f"(d[16]),"+f"(d[17]),"+f"(d[18]),"+f"(d[19]),"+f"(d[20]),"+f"(d[21]),"+f"(d[22]),"+f"(d[23]),"+f"(d[24]),"+f"(d[25]),"+f"(d[26]),"+f"(d[27]),"+f"(d[28]),"+f"(d[29]),"+f"(d[30]),"+f"(d[31]),"+f"(d[32]),"+f"(d[33]),"+f"(d[34]),"+f"(d[35]),"+f"(d[36]),"+f"(d[37]),"+f"(d[38]),"+f"(d[39]),"+f"(d[40]),"+f"(d[41]),"+f"(d[42]),"+f"(d[43]),"+f"(d[44]),"+f"(d[45]),"+f"(d[46]),"+f"(d[47]),"+f"(d[48]),"+f"(d[49]),"+f"(d[50]),"+f"(d[51]),"+f"(d[52]),"+f"(d[53]),"+f"(d[54]),"+f"(d[55]),"+f"(d[56]),"+f"(d[57]),"+f"(d[58]),"+f"(d[59]),"+f"(d[60]),"+f"(d[61]),"+f"(d[62]),"+f"(d[63])
// one wrapper per (type, N): R = N / 2 accumulator registers, operands %R .. %R+4 follow them
#define PCB_WG_DEF(TY, N, R, A, B, S, TA_, TB_)                                                                      \
  template <int TA, int TB>                                                                                         \
  __device__ __forceinline__ void wgmma_##TY##_n##N(float (&d)[R], uint64_t a, uint64_t b, uint32_t accumulate) {   \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" S ", 0;\n\t"                                             \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." #TY "." #TY " " PCB_WG_D##R ", %" A ", %" B        \
                 ", p, 1, 1, %" TA_ ", %" TB_ ";\n\t}\n"                                                             \
                 : PCB_WG_C##R(d) : "l"(a), "l"(b), "r"(accumulate), "n"(TA), "n"(TB));                             \
  }
PCB_WG_DEF(f16, 32, 16, "16", "17", "18", "19", "20")
PCB_WG_DEF(f16, 64, 32, "32", "33", "34", "35", "36")
PCB_WG_DEF(f16, 96, 48, "48", "49", "50", "51", "52")
PCB_WG_DEF(f16, 128, 64, "64", "65", "66", "67", "68")
PCB_WG_DEF(bf16, 32, 16, "16", "17", "18", "19", "20")
PCB_WG_DEF(bf16, 64, 32, "32", "33", "34", "35", "36")
PCB_WG_DEF(bf16, 96, 48, "48", "49", "50", "51", "52")
PCB_WG_DEF(bf16, 128, 64, "64", "65", "66", "67", "68")

template <int N, bool F16, int TA, int TB>
__device__ __forceinline__ void wgmma(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (F16) {
    if constexpr (N == 32) wgmma_f16_n32<TA, TB>(d, a, b, accumulate);
    else if constexpr (N == 64) wgmma_f16_n64<TA, TB>(d, a, b, accumulate);
    else if constexpr (N == 96) wgmma_f16_n96<TA, TB>(d, a, b, accumulate);
    else wgmma_f16_n128<TA, TB>(d, a, b, accumulate);
  } else {
    if constexpr (N == 32) wgmma_bf16_n32<TA, TB>(d, a, b, accumulate);
    else if constexpr (N == 64) wgmma_bf16_n64<TA, TB>(d, a, b, accumulate);
    else if constexpr (N == 96) wgmma_bf16_n96<TA, TB>(d, a, b, accumulate);
    else wgmma_bf16_n128<TA, TB>(d, a, b, accumulate);
  }
}

}  // namespace hw
}  // namespace pcb
