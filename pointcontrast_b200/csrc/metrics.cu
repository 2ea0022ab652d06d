// Semantic-segmentation evaluation (`downstream/semseg/lib/test.py:62-196`, `lib/utils.py:117-138`) on the device, accumulated across
// batches without a host round trip:
//   * pcb_seg_metrics: one warp per logit row -- argmax, softmax, the row's cross-entropy -- then the batch's mean loss (the pass of
//     pcb_ce_forward_backward), precision@1 and the confusion histogram added to device accumulators
//   * pcb_average_precision: sklearn's uninterpolated average precision of every class column at once, from ONE radix sort of
//     (class, descending score) keys over all n * C entries (sort.cuh), head flags and scans.
// Integer counts use integer atomics (order-free); every fp64 sum runs in a fixed order, so results are bit-reproducible.
#include <cub/cub.cuh>
#include "sort.cuh"

using namespace pcb;

namespace {

// ------------------------------------------------------------------------------------------------ per-voxel metrics
// One warp per row.  pred: the first index among the maximal values, a NaN counting as maximal (torch `output.max(1)[1]`).
// rowloss: lse - x[t] on rows whose target is in [0, C) and != ignore, else 0 (ce_rows_kernel's value).  hist[t * C + pred] += 1 for
// 0 <= t < C (`fast_hist`); counts[0] += rows with t != 255 and counts[1] += those with pred == t (`precision_at_one`).
__global__ void seg_rows_kernel(const float* __restrict__ X, const int64_t* __restrict__ target, int64_t n, int C, int64_t ignore,
                                int32_t* __restrict__ pred, float* __restrict__ prob, float* __restrict__ rowloss,
                                unsigned long long* __restrict__ hist, unsigned long long* __restrict__ counts) {
  pdl_wait(); pdl_trigger();
  __shared__ unsigned int s_cnt[2];
  if (threadIdx.x == 0) { s_cnt[0] = 0; s_cnt[1] = 0; }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t row = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row < n) {
    const float* x = X + row * C;
    const int64_t t = target[row];
    float m, s;
    warp_row_max_sumexp(x, C, lane, m, s);
    float bv = 0.f;
    int bi = C;                                                   // C: nothing seen yet
    for (int c = lane; c < C; c += 32) {                          // ascending c per lane: a tie keeps the earlier index
      const float v = x[c];
      if (bi == C || v > bv || (isnan(v) && !isnan(bv))) { bv = v; bi = c; }
    }
    for (int o = 16; o; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      bool take;
      if (oi == C) take = false;
      else if (bi == C) take = true;
      else if (isnan(ov) != isnan(bv)) take = isnan(ov);
      else if (isnan(ov) || ov == bv) take = oi < bi;
      else take = ov > bv;
      if (take) { bv = ov; bi = oi; }
    }
    if (prob)
      for (int c = lane; c < C; c += 32) prob[row * C + c] = expf(x[c] - m) / s;
    if (lane == 0) {
      const float lse = m + logf(s);
      rowloss[row] = (t == ignore || t < 0 || t >= C) ? 0.f : lse - x[t];
      pred[row] = bi;
      if (t >= 0 && t < C) atomicAdd(hist + t * C + bi, 1ull);
      if (t != 255) {
        atomicAdd(&s_cnt[0], 1u);
        if (t == bi) atomicAdd(&s_cnt[1], 1u);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_cnt[0]) {
    atomicAdd(counts, (unsigned long long)s_cnt[0]);
    if (s_cnt[1]) atomicAdd(counts + 1, (unsigned long long)s_cnt[1]);
  }
}

// stats += (batch CE * n, precision@1 * n, n).  precision@1 as `precision_at_one` computes it: fp32 sum of the hits times fp32(100 / rows)
__global__ void seg_stats_kernel(const float* __restrict__ ce, const unsigned long long* __restrict__ counts, int64_t n,
                                 double* __restrict__ stats) {
  pdl_wait(); pdl_trigger();
  const double rows = (double)counts[0];
  const double score = counts[0] ? (double)((float)counts[1] * (float)(100.0 / rows)) : (double)NAN;
  stats[0] += (double)ce[0] * (double)n;
  stats[1] += score * (double)n;
  stats[2] += (double)n;
}

// rowloss, the mean CE pass's (loss, count), the two precision@1 counts
struct SegWs { float* rowloss; float* ce; unsigned long long* counts; };
SegWs seg_layout(Carve& c, int64_t n) { return {c.take<float>(n), c.take<float>(2), c.take<unsigned long long>(2)}; }

// ------------------------------------------------------------------------------------------------ average precision
// Key of entry (row i, class c): class in bits [32, ...), below it the score's bits in DESCENDING order (-0.0 taken as +0.0, as sklearn
// ties them); payload: the label bit (target == c).  A NaN score marks its class.
__global__ void ap_key_kernel(const float* __restrict__ S, const int64_t* __restrict__ target, int64_t n, int C, uint64_t* __restrict__ keys,
                              int32_t* __restrict__ label, int32_t* __restrict__ nan_flag) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= n * C) return;
  const int64_t i = e / C;
  const int c = (int)(e - i * C);
  float v = S[e];
  if (v == 0.f) v = 0.f;
  if (isnan(v)) atomicOr(nan_flag + c, 1);
  const uint32_t u = __float_as_uint(v);
  const uint32_t asc = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  keys[e] = ((uint64_t)c << 32) | (uint64_t)(~asc);
  label[e] = target[i] == (int64_t)c ? 1 : 0;
}

// After the sort class c holds sorted positions [c n, (c+1) n); run j = rank - 1 is one tie group (same class and score).  tp: the
// inclusive scan of the sorted label bits.  Per run: start_tp = positives of its class ranked before it, end_tp = up to and including
// it, end_rank = the 1-based rank of its last entry within the class.
__global__ void ap_runs_kernel(const int32_t* __restrict__ flag, const int32_t* __restrict__ rank, const int32_t* __restrict__ tp, int64_t n,
                               int64_t total, int32_t* __restrict__ start_tp, int32_t* __restrict__ end_tp, int32_t* __restrict__ end_rank) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int64_t c0 = (i / n) * n;
  const int32_t base = c0 ? tp[c0 - 1] : 0;
  const int32_t run = rank[i] - 1;
  if (flag[i]) start_tp[run] = (i == c0) ? 0 : tp[i - 1] - base;
  if (i + 1 == total || flag[i + 1]) { end_tp[run] = tp[i] - base; end_rank[run] = (int32_t)(i - c0 + 1); }
}

// One block per class: AP_c = sum over its runs of (end_tp - start_tp) * end_tp / end_rank, divided by the class's positives T_c, in a
// fixed order.  A class without a positive leaves its accumulators alone; a NaN score makes the batch's AP NaN.
constexpr int AP_THREADS = 256;
__global__ void __launch_bounds__(AP_THREADS) ap_class_kernel(const int32_t* __restrict__ rank, const int32_t* __restrict__ tp,
                                                              const int32_t* __restrict__ start_tp, const int32_t* __restrict__ end_tp,
                                                              const int32_t* __restrict__ end_rank, const int32_t* __restrict__ nan_flag,
                                                              int64_t n, double* __restrict__ ap_sum, int64_t* __restrict__ ap_cnt) {
  __shared__ double red[AP_THREADS];
  const int c = blockIdx.x;
  const int64_t c0 = (int64_t)c * n, c1 = c0 + n;
  const int32_t T = tp[c1 - 1] - (c0 ? tp[c0 - 1] : 0);
  if (T == 0) return;
  const int32_t r0 = rank[c0] - 1, r1 = rank[c1 - 1];
  double acc = 0.0;
  for (int32_t j = r0 + threadIdx.x; j < r1; j += AP_THREADS)
    acc += (double)(end_tp[j] - start_tp[j]) * (double)end_tp[j] / (double)end_rank[j];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int h = AP_THREADS / 2; h; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    ap_sum[c] += nan_flag[c] ? (double)NAN : red[0] / (double)T;
    ap_cnt[c] += 1;
  }
}

// The sort pipeline's buffers over n * C entries, then the per-class NaN flags.  Once the sort has run, its input keys / payloads and
// its sorted keys are dead and hold the per-run arrays and the label scan.
struct ApWs { SortWs s; int32_t* nan_flag; };
ApWs ap_layout(Carve& c, int64_t total, int C) { return {sort_layout(c, total), c.take<int32_t>(C)}; }

int class_bits(int C) { int b = 0; while ((1 << b) < C) ++b; return b; }

}  // namespace

extern "C" size_t pcb_seg_metrics_ws_bytes(int64_t n) {
  return layout_bytes(seg_layout, n);
}

extern "C" int pcb_seg_metrics(const float* logits, const int64_t* target, int64_t n, int C, int64_t ignore_index, int32_t* pred, float* prob,
                               int64_t* hist, double* stats, void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(logits && target && pred && hist && stats && ws && n >= 1 && C >= 1 && C <= 1024);
  Carve c{(char*)ws};
  const auto [rowloss, ce, counts] = seg_layout(c, n);
  PCB_ARG(ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  PCB_CUDA(cudaMemsetAsync(counts, 0, 2 * sizeof(unsigned long long), st));
  launch_kernel(seg_rows_kernel, (unsigned)((n + 7) / 8), 256, 0, st, logits, target, n, C, ignore_index, pred, prob, rowloss,
                (unsigned long long*)hist, counts);
  if (int e = check_launch("seg_rows_kernel")) return e;
  if (int e = ce_mean_launch(rowloss, target, n, C, ignore_index, ce, st)) return e;
  launch_kernel(seg_stats_kernel, 1, 1, 0, st, (const float*)ce, (const unsigned long long*)counts, n, stats);
  return check_launch("seg_stats_kernel");
}

extern "C" size_t pcb_average_precision_ws_bytes(int64_t n, int C) {
  if (n < 1 || C < 1) return 0;
  return layout_bytes(ap_layout, n * C, C);
}

extern "C" int pcb_average_precision(const float* score, const int64_t* target, int64_t n, int C, double* ap_sum, int64_t* ap_cnt, void* ws,
                                     size_t ws_bytes, void* stream) {
  PCB_ARG(score && target && ap_sum && ap_cnt && ws && n >= 1 && C >= 1 && C <= 1024 && n * C < ((int64_t)1 << 31));
  const int64_t total = n * C;
  Carve c{(char*)ws};
  const auto [w, nan_flag] = ap_layout(c, total, C);
  PCB_ARG(ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  PCB_CUDA(cudaMemsetAsync(nan_flag, 0, C * sizeof(int32_t), st));
  ap_key_kernel<<<blocks_for(total, 256), 256, 0, st>>>(score, target, n, C, w.k, w.idx, nan_flag);
  if (int e = check_launch("ap_key_kernel")) return e;
  if (int e = sort_runs(total, w, 32 + class_bits(C), st)) return e;          // sk / sidx: sorted keys / labels; flag, rank: the runs
  int32_t* tp = (int32_t*)w.sk;                                                  // the sorted keys are dead after the head flags
  size_t cb = w.cub_bytes;
  PCB_CUDA(cub::DeviceScan::InclusiveSum(w.cub, cb, w.sidx, tp, (int)total, st));
  g_launches.fetch_add(1);
  int32_t* end_tp = (int32_t*)w.k;                                               // the input keys / labels are dead after the sort
  int32_t* end_rank = end_tp + total;
  int32_t* start_tp = w.idx;
  ap_runs_kernel<<<blocks_for(total, 256), 256, 0, st>>>(w.flag, w.rank, tp, n, total, start_tp, end_tp, end_rank);
  if (int e = check_launch("ap_runs_kernel")) return e;
  ap_class_kernel<<<C, AP_THREADS, 0, st>>>(w.rank, tp, start_tp, end_tp, end_rank, nan_flag, n, ap_sum, ap_cnt);
  return check_launch("ap_class_kernel");
}
