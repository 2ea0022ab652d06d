// Semantic segmentation on the original point cloud (SURVEY.md 8f-6): the hot part of the reference's `test_pointcloud`
// (`downstream/semseg/lib/datasets/scannet.py:131-172`, `stanford.py:41-84`), which builds a scipy KD-tree over the predicted voxel
// centres, queries it once per original point, maps the labels in Python loops and bins them with `fast_hist` (`lib/utils.py:131-133`):
//   * the nearest centre of every original point, exact in fp64, ties to the smallest index                  -> pcb_nearest
//   * the label it transfers, and the confusion histogram of the mapped labels                              -> pcb_label_transfer
// The grid is the sort-and-unique pipeline and the run table of sort.cuh, as in pcb_frame_overlap.  Results do not depend on the cell
// size, the launch shape or the workspace size (tests/test_gpu_semseg_fulleval.py: index-equal to oracle/semseg_fulleval_cpu.py).
#include <climits>
#include <cmath>
#include "sort.cuh"

using namespace pcb;

namespace {

constexpr int NN_SHELLS = 8;         // Chebyshev shells searched on the grid before a query goes to the brute-force pass
constexpr int NN_THREADS = 128;      // grid search: one query per thread
constexpr int BF_THREADS = 256;      // brute force: one query per CTA
constexpr int LT_THREADS = 256;
constexpr int LT_SMEM_BINS = 4096;   // label transfer: a CTA bins in shared memory up to 64 x 64 classes

// ((dx dx + dy dy) + dz dz) without FMA contraction: the expression of pcb_frame_overlap
__device__ __forceinline__ double dist2(const double* __restrict__ a, double px, double py, double pz) {
  const double ex = __dsub_rn(a[0], px), ey = __dsub_rn(a[1], py), ez = __dsub_rn(a[2], pz);
  return __dadd_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)), __dmul_rn(ez, ez));
}

// the total order of candidates: smaller d2 first, then the smaller reference index (NaN never wins)
__device__ __forceinline__ void take_min(double d2, int32_t j, double& best, int32_t& bj) {
  if (d2 < best || (d2 == best && j < bj)) { best = d2; bj = j; }
}

__global__ void nn_key_kernel(const double* __restrict__ ref, int64_t m, double cell_size, uint64_t* __restrict__ keys,
                              int32_t* __restrict__ idx, int32_t* status) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= m) return;
  int cx, cy, cz;
  if (!grid_cell(ref + 3 * i, cell_size, cx, cy, cz)) atomicOr(status, PCB_NEAREST_RANGE);
  keys[i] = cell_key(cx, cy, cz);
  idx[i] = (int32_t)i;
}

// the references in cell order, so that a run is read contiguously
__global__ void nn_gather_kernel(const double* __restrict__ ref, int64_t m, const int32_t* __restrict__ sidx, double* __restrict__ sxyz) {
  const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (s >= m) return;
  const int64_t j = sidx[s];
  for (int k = 0; k < 3; ++k) sxyz[3 * s + k] = ref[3 * j + k];
}

// One thread per query: its own cell, then the Chebyshev shells r = 1, 2, ... around it.  After shell r every reference not yet seen
// lies in a cell at least r + 1 away along some axis, so its coordinate differs from the query's by more than (r - 2^-32) cells (the
// cell divisions are rounded once, |x / cell| < 2^20), and its computed d2 exceeds (r cell)^2 (1 - 2^-30).  The search stops once the
// best d2 is below (r cell)^2 (1 - 2^-16): no unseen reference can then reach it, not even as a tie.  A query still open after
// NN_SHELLS shells joins the brute-force list.
__global__ void __launch_bounds__(NN_THREADS) nn_grid_kernel(
    const double* __restrict__ query, int64_t n, double cell_size, const uint64_t* __restrict__ tk, const int32_t* __restrict__ tv,
    uint64_t mask, const int32_t* __restrict__ run_start, const int32_t* __restrict__ run_end, const double* __restrict__ sxyz,
    const int32_t* __restrict__ sidx, int32_t* __restrict__ idx, int32_t* __restrict__ fb_list, int32_t* __restrict__ fb_count,
    int32_t* status) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* q = query + 3 * i;
  const double px = q[0], py = q[1], pz = q[2];
  int cx, cy, cz;
  if (!grid_cell(q, cell_size, cx, cy, cz)) { atomicOr(status, PCB_NEAREST_RANGE); idx[i] = -1; return; }
  double best = INFINITY;
  int32_t bj = INT_MAX;
  for (int r = 0; r <= NN_SHELLS; ++r) {
    for (int dx = -r; dx <= r; ++dx) {
      const int x = cx + dx;
      if (abs(x) >= VB) continue;
      for (int dy = -r; dy <= r; ++dy) {
        const int y = cy + dy;
        if (abs(y) >= VB) continue;
        const int step = (abs(dx) == r || abs(dy) == r) ? 1 : 2 * r;       // inside the shell's x-y square only its two z faces
        for (int dz = -r; dz <= r; dz += step) {
          const int z = cz + dz;
          if (abs(z) >= VB) continue;
          const int run = hash_lookup(tk, tv, mask, cell_key(x, y, z));
          if (run < 0) continue;
          for (int32_t s = run_start[run]; s < run_end[run]; ++s) take_min(dist2(sxyz + 3 * s, px, py, pz), sidx[s], best, bj);
        }
      }
    }
    const double g = (double)r * cell_size;
    if (best < __dmul_rn(__dmul_rn(g, g), 1.0 - 0x1p-16)) { idx[i] = bj; return; }
  }
  fb_list[atomicAdd(fb_count, 1)] = (int32_t)i;
}

// One CTA per listed query: every reference in index order, then the CTA's minimum under the same total order.
__global__ void __launch_bounds__(BF_THREADS) nn_brute_kernel(const double* __restrict__ ref, int64_t m, const double* __restrict__ query,
                                                              const int32_t* __restrict__ fb_list, const int32_t* __restrict__ fb_count,
                                                              int32_t* __restrict__ idx) {
  __shared__ double sd[BF_THREADS / 32];
  __shared__ int32_t sj[BF_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int f = blockIdx.x; f < *fb_count; f += gridDim.x) {
    const int64_t i = fb_list[f];
    const double px = query[3 * i], py = query[3 * i + 1], pz = query[3 * i + 2];
    double best = INFINITY;
    int32_t bj = INT_MAX;
    for (int64_t j = threadIdx.x; j < m; j += BF_THREADS) take_min(dist2(ref + 3 * j, px, py, pz), (int32_t)j, best, bj);
    for (int o = 16; o; o >>= 1) take_min(__shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bj, o), best, bj);
    if (lane == 0) { sd[warp] = best; sj[warp] = bj; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < BF_THREADS / 32; ++w) take_min(sd[w], sj[w], best, bj);
      idx[i] = bj == INT_MAX ? -1 : bj;                     // no finite candidate: only with non-finite references (status set)
    }
    __syncthreads();
  }
}

// the cell sort of the references, its runs and their table, the references in cell order, the brute-force list and its length
struct NearestWs { SortWs s; RunsWs r; double* sxyz; int32_t* fb_list; int32_t* fb_count; };
NearestWs nearest_layout(Carve& c, int64_t m, int64_t n) {
  NearestWs w{sort_layout(c, m), runs_layout(c, m, true), nullptr, nullptr, nullptr};
  w.sxyz = c.take<double>(3 * m);
  w.fb_list = c.take<int32_t>(n);
  w.fb_count = c.take<int32_t>(1);
  return w;
}

bool sizes_ok(int64_t m, int64_t n) { return m >= 0 && n >= 0 && m < INT_MAX && n < INT_MAX; }

// the label of a row through the lookup table; -1 when it lies outside the table or the table has no entry for it
__device__ __forceinline__ int32_t lut_map(const int32_t* __restrict__ lut, int lut_n, int32_t v) {
  return (v >= 0 && v < lut_n) ? lut[v] : -1;
}

// One thread per query row.  With smem_bins the CTA bins into shared memory and adds its nonzero bins to hist once.
__global__ void __launch_bounds__(LT_THREADS) label_transfer_kernel(
    const int32_t* __restrict__ idx, const int32_t* __restrict__ ref_label, int64_t m, const int32_t* __restrict__ query_label, int64_t n,
    const int32_t* __restrict__ lut, int lut_n, int C, int32_t* __restrict__ point_label, unsigned long long* __restrict__ hist,
    int32_t* status, int smem_bins) {
  extern __shared__ uint32_t bins[];
  const int CC = C * C;
  if (smem_bins) {
    for (int t = threadIdx.x; t < CC; t += blockDim.x) bins[t] = 0;
    __syncthreads();
  }
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) {
    int32_t j = idx[i];
    if (j < 0 || j >= m) { atomicOr(status, PCB_NEAREST_RANGE); j = -1; }
    const int32_t p = j >= 0 ? ref_label[j] : -1;
    point_label[i] = p;
    if (query_label && j >= 0) {
      const int32_t gm = lut_map(lut, lut_n, query_label[i]), pm = lut_map(lut, lut_n, p);
      if (gm < 0 || pm < 0) {
        atomicOr(status, PCB_LABEL_RANGE);
      } else if (gm < C) {                                  // fast_hist: only rows with 0 <= gt < C count
        if (pm >= C) atomicOr(status, PCB_LABEL_RANGE);
        else if (smem_bins) atomicAdd(&bins[gm * C + pm], 1u);
        else atomicAdd(&hist[(int64_t)gm * C + pm], 1ull);
      }
    }
  }
  if (smem_bins) {
    __syncthreads();
    for (int t = threadIdx.x; t < CC; t += blockDim.x)
      if (const uint32_t v = bins[t]) atomicAdd(&hist[t], (unsigned long long)v);
  }
}

}  // namespace

extern "C" size_t pcb_nearest_ws_bytes(int64_t m, int64_t n) {
  if (!sizes_ok(m, n)) return 0;
  return layout_bytes(nearest_layout, m < 1 ? 1 : m, n < 1 ? 1 : n);
}

extern "C" int pcb_nearest(const double* ref, int64_t m, const double* query, int64_t n, double cell_size, int32_t* idx, int32_t* status,
                           void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(sizes_ok(m, n) && cell_size > 0.0 && cell_size < INFINITY);
  if (n == 0) return PCB_OK;
  PCB_ARG(m > 0);
  Carve c{(char*)ws};
  const NearestWs w = nearest_layout(c, m, n);
  PCB_ARG(ref && query && idx && status && ws && ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  PCB_CUDA(cudaMemsetAsync(w.fb_count, 0, sizeof(int32_t), st));
  nn_key_kernel<<<blocks_for(m, 256), 256, 0, st>>>(ref, m, cell_size, w.s.k, w.s.idx, status);
  if (int e = check_launch("nn_key_kernel")) return e;
  if (int e = sort_runs(m, w.s, 63, st)) return e;
  if (int e = find_runs(m, w.s, w.r, st)) return e;
  nn_gather_kernel<<<blocks_for(m, 256), 256, 0, st>>>(ref, m, w.s.sidx, w.sxyz);
  if (int e = check_launch("nn_gather_kernel")) return e;
  nn_grid_kernel<<<blocks_for(n, NN_THREADS), NN_THREADS, 0, st>>>(query, n, cell_size, w.r.tk, w.r.tv, (uint64_t)w.r.tcap - 1, w.r.start,
                                                                   w.r.end, w.sxyz, w.s.sidx, idx, w.fb_list, w.fb_count, status);
  if (int e = check_launch("nn_grid_kernel")) return e;
  // the list's length stays on the device: a fixed grid strides over it (empty in the common case)
  const int64_t grid = n < 4 * (int64_t)num_sms() ? n : 4 * (int64_t)num_sms();
  nn_brute_kernel<<<(unsigned)grid, BF_THREADS, 0, st>>>(ref, m, query, w.fb_list, w.fb_count, idx);
  return check_launch("nn_brute_kernel");
}

extern "C" int pcb_label_transfer(const int32_t* idx, const int32_t* ref_label, int64_t m, const int32_t* query_label, int64_t n,
                                  const int32_t* lut, int lut_n, int C, int32_t* point_label, int64_t* hist, int32_t* status, void* stream) {
  PCB_ARG(sizes_ok(m, n));
  PCB_ARG(!query_label || (C >= 1 && C <= 46340 && lut_n >= 1 && lut && hist));
  if (n == 0) return PCB_OK;
  PCB_ARG(idx && ref_label && point_label && status);
  cudaStream_t st = (cudaStream_t)stream;
  const int smem_bins = query_label && C * C <= LT_SMEM_BINS;
  const size_t smem = smem_bins ? (size_t)C * C * sizeof(uint32_t) : 0;
  label_transfer_kernel<<<blocks_for(n, LT_THREADS), LT_THREADS, smem, st>>>(idx, ref_label, m, query_label, n, lut, lut_n, query_label ? C : 0,
                                                                             point_label, (unsigned long long*)hist, status, smem_bins);
  return check_launch("label_transfer_kernel");
}
