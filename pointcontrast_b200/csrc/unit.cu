// Fused "units" of the Res16UNet graph: convolution -> BatchNorm -> (+ residual) -> (ReLU) issued from one C call, and the
// reverse sweep of the same unit (include/pcb200.h: pcb_unit).  Host-side sequencing only -- the kernels live in
// conv_wgmma.cu / conv.cu / bn.cu; what this file adds over calling them one by one from the host language:
//   * on small levels the BatchNorm statistics come from the convolution's offset-split reduction pass, so the separate
//     column-sum pass over z and its launch disappear;
//   * one boundary crossing per unit instead of three to five.
// Replaces the per-module call sequence of `model/modules/resnet_block.py:44-60` / `model/res16unet.py:206-268`.
#include "common.cuh"

using namespace pcb;

// ------------------------------------------------------------------------------------------------ per-launch timing
#include <vector>
namespace {
struct ProfRec { cudaEvent_t e0, e1; int kind; };
bool g_prof_on = false;
std::vector<ProfRec> g_prof;
std::vector<cudaEvent_t> g_prof_pool;
cudaEvent_t g_prof_open = nullptr;
cudaEvent_t prof_event() {
  if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}
}  // namespace
namespace pcb {
void prof_begin(cudaStream_t st) {
  if (!g_prof_on) return;
  g_prof_open = prof_event();
  cudaEventRecord(g_prof_open, st);
}
void prof_end(cudaStream_t st, int kind) {
  if (!g_prof_on || !g_prof_open) return;
  cudaEvent_t e1 = prof_event();
  cudaEventRecord(e1, st);
  g_prof.push_back({g_prof_open, e1, kind});
  g_prof_open = nullptr;
}
}  // namespace pcb

extern "C" int pcb_profile_enable(int on) {
  g_prof_on = on != 0;
  return PCB_OK;
}

extern "C" int pcb_profile_read(float* ms, int32_t* kinds, int max_records, int* count) {
  PCB_ARG(count && (max_records == 0 || (ms && kinds)));
  int n = 0;
  for (auto& r : g_prof) {
    PCB_CUDA(cudaEventSynchronize(r.e1));
    if (n < max_records) {
      float t = 0.f;
      PCB_CUDA(cudaEventElapsedTime(&t, r.e0, r.e1));
      ms[n] = t; kinds[n] = r.kind;
    }
    ++n;
    g_prof_pool.push_back(r.e0); g_prof_pool.push_back(r.e1);
  }
  g_prof.clear();
  *count = n;
  return PCB_OK;
}

namespace {
inline bool tensor_core_shape(int Cin, int Cout) { return Cin % 32 == 0 && Cout % 32 == 0; }

// convolution scratch: the largest of forward / data gradient / weight gradient
size_t conv_part_bytes(int K, int64_t n_in, int64_t n_out, int Cin, int Cout) {
  size_t a = pcb_conv_forward_split_ws_bytes(K, n_out, Cin, Cout), b = pcb_conv_forward_split_ws_bytes(K, n_in, Cout, Cin);
  size_t c = tensor_core_shape(Cin, Cout) ? pcb_conv_wgrad_split_ws_bytes(K, n_out > n_in ? n_out : n_in, Cin, Cout)
                                          : pcb_conv_wgrad_ws_bytes(K, n_out > n_in ? n_out : n_in, Cin, Cout);
  size_t d = tensor_core_shape(Cin, Cout) ? pcb_conv_wgrad_split_ws_bytes(K, n_out > n_in ? n_out : n_in, Cout, Cin) : 0;
  size_t m = a > b ? a : b;
  if (c > m) m = c;
  if (d > m) m = d;
  return m;
}

// [convolution scratch | BatchNorm scratch]
struct UnitWs { void* conv; size_t conv_bytes; void* bn; size_t bn_bytes; };
UnitWs unit_layout(Carve& c, int K, int64_t n_in, int64_t n_out, int Cin, int Cout) {
  const size_t conv = conv_part_bytes(K, n_in, n_out, Cin, Cout), bn = pcb_bn_ws_bytes(n_out, Cout);
  return {c.take<char>(conv), conv, c.take<char>(bn), bn};
}
}  // namespace

extern "C" size_t pcb_unit_ws_bytes(int K, int64_t n_in, int64_t n_out, int Cin, int Cout) {
  return layout_bytes(unit_layout, K, n_in, n_out, Cin, Cout);
}

extern "C" int pcb_unit_forward(const pcb_unit* u, void* stream) {
  PCB_ARG(u && u->K >= 1 && u->K <= PCB_MAX_KERNEL_VOLUME && u->n_out >= 1 && u->n_in >= 1 && u->n0 >= 1 && u->n0 <= u->n_out);
  PCB_ARG(u->fwd_tbl && u->z_p && u->out_hi && u->out_lo && u->mean && u->invstd && u->gamma && u->beta && u->ws);
  PCB_ARG(!(u->flags & PCB_UNIT_FP16_FORWARD) || (u->flags & PCB_UNIT_EVAL) || (u->out_bhi && u->out_blo));
  PCB_ARG(!(u->flags & PCB_UNIT_EVAL) || (u->n0 == u->n_out && u->running_mean && u->running_var));
  Carve c{(char*)u->ws};
  const UnitWs w = unit_layout(c, u->K, u->n_in, u->n_out, u->Cin, u->Cout);
  PCB_ARG(u->ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  const bool f16 = (u->flags & PCB_UNIT_FP16_FORWARD) != 0;      // activations (x, out planes) and forward weight tiles are fp16 hi/lo
  // An offset-split convolution (small levels) leaves its partial planes to one pass that sums them into z and takes the BatchNorm
  // statistics: one read of the planes instead of a reduction plus a column-sum pass over z.  Unsplit, the statistics are a separate
  // pass (in the epilogue each thread holds scattered fragment rows; the separate pass reads z once, coalesced).
  const float* partials = nullptr;
  int nsplit = 0;
  if (tensor_core_shape(u->Cin, u->Cout)) {
    PCB_ARG(u->x_hi && u->x_lo && u->wt_fwd);
    const bool fuse = !(u->flags & (PCB_UNIT_SEPARATE_STATS | PCB_UNIT_EVAL));
    ProfScope prof(st, 0);                   // the convolution, and the reduction + statistics pass when it has one
    if (int e = conv_forward_split_impl(u->x_hi, u->x_lo, u->x_lds, u->fwd_tbl, u->fwd_stride, u->fwd_kmap, u->K, u->fwd_perm, u->n_out, u->Cin, u->Cout,
                                        u->wt_fwd, nullptr, u->z_p, u->z_ld, w.conv, w.conv_bytes, f16 ? (PCB_PLANES_A_FP16 | PCB_PLANES_B_FP16) : 0,
                                        st, fuse ? &partials : nullptr, &nsplit)) return e;
    if (partials) {
      if (int e = bn_reduce_stats_launch(partials, nsplit, u->z_p, u->z_ld, u->n_out, u->n0, u->Cout, u->eps, u->momentum, u->mean, u->invstd,
                                         u->running_mean, u->running_var, w.bn, w.bn_bytes, st)) return e;
    }
  } else {
    PCB_ARG(u->x_p && u->W);
    if (int e = pcb_conv_forward(u->x_p, u->x_ld, u->fwd_tbl, u->fwd_stride, u->fwd_kmap, u->K, u->n_out, u->Cin, u->Cout, u->W,
                                 nullptr, u->z_p, u->z_ld, stream)) return e;
  }
  ProfScope prof(st, 2);                     // BatchNorm forward: statistics (unless fused into the split reduction) + normalise / residual / ReLU / planes
  if (u->flags & PCB_UNIT_EVAL) {            // eval-mode BatchNorm (`downstream/semseg/lib/test.py:95-117`): normalise with the running statistics
    if (int e = bn_eval_stats_launch(u->running_mean, u->running_var, u->Cout, u->eps, u->mean, u->invstd, st)) return e;
  } else if (!partials) {
    if (int e = pcb_bn_stats_seg(u->z_p, u->z_ld, u->n_out, u->n0, u->Cout, u->eps, u->momentum, u->mean, u->invstd, u->running_mean,
                                 u->running_var, w.bn, w.bn_bytes, stream)) return e;
  }
  return pcb_bn_apply_seg(u->z_p, u->z_ld, u->n_out, u->n0, u->Cout, u->mean, u->invstd, u->gamma, u->beta, u->res_p, u->res_ld,
                          (u->relu ? PCB_BN_RELU : 0) | (f16 ? PCB_PLANES_A_FP16 : 0), u->out_p, u->out_ld, u->out_hi, u->out_lo, u->out_lds,
                          f16 ? u->out_bhi : nullptr, f16 ? u->out_blo : nullptr, stream);
}

extern "C" int pcb_unit_backward(const pcb_unit* u, void* stream) {
  PCB_ARG(u && u->K >= 1 && u->K <= PCB_MAX_KERNEL_VOLUME && u->n_out >= 1 && u->n_in >= 1 && u->n0 >= 1 && u->n0 <= u->n_out);
  PCB_ARG(u->g_p && u->z_p && u->mean && u->invstd && u->gamma && u->dgamma && u->dbeta && u->dW && u->wg_tbl && u->ws);
  Carve c{(char*)u->ws};
  const UnitWs w = unit_layout(c, u->K, u->n_in, u->n_out, u->Cin, u->Cout);
  PCB_ARG(u->ws_bytes >= c.used);
  const bool tc = tensor_core_shape(u->Cin, u->Cout);
  const bool f16 = (u->flags & PCB_UNIT_FP16_FORWARD) != 0;
  PCB_ARG(tc ? (u->dz_hi && u->dz_lo && u->x_hi && u->x_lo) : (u->dz_p && u->x_p));
  PCB_ARG(tc || u->gin_mode == 0);               // only the 3-channel stem is not tensor-core shaped: its input wants no gradient
  // the activation operand of the weight gradient as bf16 hi/lo planes (its fp16 planes serve the forward pass only): both MMA operands
  // share one format
  const uint16_t* xh = f16 ? u->x_bhi : u->x_hi;
  const uint16_t* xl = f16 ? u->x_blo : u->x_lo;
  PCB_ARG(!tc || (xh && xl));
  PCB_ARG(tc || u->wg_gather_x);
  PCB_ARG(u->gin_mode == 0 || (u->gin_p && u->dg_tbl && u->wt_dg));
  // every argument is checked above: a rejected call leaves dz, dgamma / dbeta, gres, dW and gin as they were
  cudaStream_t st = (cudaStream_t)stream;
  // 1. g * (out > 0) -> BatchNorm backward -> dz (split planes), residual-gradient fan-out, dgamma / dbeta accumulated
  prof_begin(st);
  if (int e = pcb_bn_backward_seg(u->g_p, u->g_ld, u->z_p, u->z_ld, u->relu ? u->out_hi : nullptr, u->out_lds, u->n_out, u->n0, u->Cout,
                                  u->mean, u->invstd, u->gamma, u->dz_p, u->dz_ld, u->dgamma, u->dbeta, 1, u->gres_p, u->gres_ld, u->gres_mode,
                                  u->dz_hi, u->dz_lo, u->dz_ld, w.bn, w.bn_bytes, stream)) return e;
  prof_end(st, 3);
  // 2. weight gradient, accumulated into dW (the flat parameter-gradient buffer)
  if (tc) {
    const uint16_t *Ahi, *Alo, *Bhi, *Blo; int lda, ldb, Ca, Cb, tr; int64_t rows;
    if (u->wg_gather_x) { Ahi = xh; Alo = xl; lda = u->x_lds; Bhi = u->dz_hi; Blo = u->dz_lo; ldb = u->dz_ld; Ca = u->Cin; Cb = u->Cout; tr = 0; rows = u->n_out; }
    else { Ahi = u->dz_hi; Alo = u->dz_lo; lda = u->dz_ld; Bhi = xh; Blo = xl; ldb = u->x_lds; Ca = u->Cout; Cb = u->Cin; tr = 1; rows = u->n_in; }
    if (int e = pcb_conv_wgrad_split(Ahi, Alo, lda, Bhi, Blo, ldb, u->wg_tbl, u->wg_stride, u->K, rows, Ca, Cb, u->dW, tr, w.conv, w.conv_bytes,
                                     PCB_CONV_ACCUMULATE, stream)) return e;
  } else {
    if (int e = pcb_conv_wgrad(u->x_p, u->x_ld, u->dz_p, u->dz_ld, u->wg_tbl, u->wg_stride, u->K, u->n_out, u->Cin, u->Cout, u->dW, 0, w.conv,
                               w.conv_bytes, PCB_CONV_ACCUMULATE, stream)) return e;
  }
  // 3. data gradient: the forward kernel on the data-gradient weight tiles and the opposite-offset table
  if (u->gin_mode) {
    if (int e = pcb_conv_forward_split(u->dz_hi, u->dz_lo, u->dz_ld, u->dg_tbl, u->dg_stride, u->dg_kmap, u->K, u->n_in, u->Cout, u->Cin, u->wt_dg,
                                       nullptr, u->gin_p, u->gin_ld, w.conv, w.conv_bytes, u->gin_mode == 2 ? PCB_CONV_ACCUMULATE : 0, stream)) return e;
  }
  return PCB_OK;
}
