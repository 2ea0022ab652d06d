// The pretraining pair list of a scan (SURVEY.md 8f-10): the two compute stages of the reference's
// `pretrain/data_preprocess/scannet_pair/compute_full_overlapping.py`, for all frames of a scene in one call each:
//   * open3d `PointCloud.voxel_down_sample` of every frame (`:15-26`, `:59-63`)                      -> pcb_voxel_down_sample
//   * for every ordered pair of frames (i, j) the number of points of frame j with a point of frame i within the radius, which
//     the reference gets from one open3d KD-tree radius query per point (`get_matching_indices(pcd_j, tree_i, r, K=1)`,
//     `:39-47`, `:67-74`)                                                                             -> pcb_frame_overlap
// Both are integer work on the sort-and-unique pipeline and the run table of sort.cuh, in fp64 like the npz frames and open3d.
// Results are exact and independent of the launch shape (tests/test_gpu_pair_list.py: bit-equal to oracle/pair_list_cpu.py).
// The stage before them, `point_cloud_extractor.py:47-75` (depth frames back-projected into world points), is pcb_depth_to_points.
#include <cmath>
#include <vector>
#include <cub/cub.cuh>
#include "sort.cuh"

using namespace pcb;

namespace {

constexpr int MAX_FRAMES = 4096;
constexpr int DB = 17;                      // down-sampling key: frame (12 bits) | x | y | z, 17 bits per voxel index
constexpr int OV_WARPS = 8;                 // pcb_frame_overlap: warps per CTA, one query point per warp at a time
constexpr int OV_ROWS = 256;                // query rows per CTA

// the frame of a row: the last f with off[f] <= row (off non-decreasing; clamped to [0, F))
__device__ __forceinline__ int frame_of(const int64_t* __restrict__ off, int F, int64_t row) {
  int lo = 0, hi = F - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= row) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// frame f's bounds break the contract: offsets non-decreasing from 0 to n
__device__ __forceinline__ bool offsets_bad(const int64_t* __restrict__ off, int F, int64_t n, int f) {
  const int64_t a = off[f], b = off[f + 1];
  return b < a || a < 0 || b > n || (f == 0 && a != 0) || (f == F - 1 && b != n);
}

__global__ void offsets_check_kernel(const int64_t* __restrict__ off, int F, int64_t n, int32_t* status) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < F && offsets_bad(off, F, n, f)) atomicOr(status, PCB_FRAMES_OFFSETS);
}

// one CTA per frame: lo[f] = min(points) - voxel_size * 0.5 per axis (open3d `voxel_min_bound`); flags non-finite coordinates and
// offsets that do not run from 0 to n without decreasing
__global__ void frame_lo_kernel(const double* __restrict__ xyz, int64_t n, const int64_t* __restrict__ off, int F, double half,
                                double* __restrict__ lo, int32_t* status) {
  const int f = blockIdx.x;
  const int64_t a = off[f], b = off[f + 1];
  if (threadIdx.x == 0 && offsets_bad(off, F, n, f)) atomicOr(status, PCB_FRAMES_OFFSETS);
  double m[3] = {INFINITY, INFINITY, INFINITY};
  bool finite = true;
  for (int64_t i = max(a, (int64_t)0) + threadIdx.x; i < min(b, n); i += blockDim.x)
    for (int k = 0; k < 3; ++k) {
      const double v = xyz[3 * i + k];
      finite &= isfinite(v);
      m[k] = fmin(m[k], v);
    }
  if (!finite) atomicOr(status, PCB_FRAMES_RANGE);
  __shared__ double part[3][32];
  for (int k = 0; k < 3; ++k) {
    for (int o = 16; o; o >>= 1) m[k] = fmin(m[k], __shfl_xor_sync(0xffffffffu, m[k], o));
    if ((threadIdx.x & 31) == 0) part[k][threadIdx.x >> 5] = m[k];
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    double v = INFINITY;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) v = fmin(v, part[threadIdx.x][w]);
    lo[3 * f + threadIdx.x] = __dsub_rn(v, half);
  }
}

// key = (frame, floor((p - lo) / voxel_size) per axis), one rounding per operation as open3d's Eigen expression
__global__ void down_key_kernel(const double* __restrict__ xyz, int64_t n, const int64_t* __restrict__ off, int F, const double* __restrict__ lo,
                                double voxel_size, uint64_t* __restrict__ keys, int32_t* __restrict__ idx, int32_t* status) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int f = frame_of(off, F, i);
  uint64_t key = (uint64_t)f << (3 * DB);
  for (int k = 0; k < 3; ++k) {
    double t = floor(__ddiv_rn(__dsub_rn(xyz[3 * i + k], lo[3 * f + k]), voxel_size));
    if (!(t >= 0.0 && t < (double)(1 << DB))) { atomicOr(status, PCB_FRAMES_RANGE); t = 0.0; }     // also NaN
    key |= (uint64_t)t << (DB * (2 - k));
  }
  keys[i] = key;
  idx[i] = (int32_t)i;
}

// one thread per voxel: the fp64 sum of its points in ascending input index (the stable sort keeps them so; open3d `AddPoint`),
// divided by their number (`GetAveragePoint`)
__global__ void down_write_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ sidx, const int32_t* __restrict__ start,
                                  const int32_t* __restrict__ end, const int64_t* __restrict__ n_runs, double* __restrict__ out) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= *n_runs) return;
  double s[3] = {0.0, 0.0, 0.0};
  for (int32_t p = start[r]; p < end[r]; ++p) {
    const int64_t j = sidx[p];
    for (int k = 0; k < 3; ++k) s[k] = __dadd_rn(s[k], xyz[3 * j + k]);
  }
  const double c = (double)(end[r] - start[r]);
  for (int k = 0; k < 3; ++k) out[3 * r + k] = __ddiv_rn(s[k], c);
}

// offsets[f] = the number of voxels of frames < f: the first run whose key is at least (f << 51)
__global__ void down_offsets_kernel(const uint64_t* __restrict__ run_key, const int64_t* __restrict__ n_runs, int F, int64_t* __restrict__ offsets,
                                    int64_t* __restrict__ stage) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > F) return;
  const uint64_t k = (uint64_t)f << (3 * DB);
  int64_t lo = 0, hi = *n_runs;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (run_key[mid] < k) lo = mid + 1; else hi = mid;
  }
  offsets[f] = lo;
  stage[f] = lo;
}

// the sort pipeline over the points, the runs, lo [F, 3], stage[F + 2]: the output offsets and the status, one copy to the host
struct DownWs { SortWs s; RunsWs r; double* lo; int64_t* stage; };
DownWs down_layout(Carve& c, int64_t n, int64_t F) {
  DownWs w{sort_layout(c, n), runs_layout(c, n, false), nullptr, nullptr};
  w.lo = c.take<double>(3 * F);
  w.stage = c.take<int64_t>(F + 2);
  w.s.status = (int32_t*)(w.stage + F + 1);
  return w;
}

__global__ void overlap_key_kernel(const double* __restrict__ xyz, int64_t n, double cell_size, uint64_t* __restrict__ keys,
                                   int32_t* __restrict__ idx, int32_t* status) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int cx, cy, cz;
  if (!grid_cell(xyz + 3 * i, cell_size, cx, cy, cz)) atomicOr(status, PCB_FRAMES_RANGE);
  keys[i] = cell_key(cx, cy, cz);
  idx[i] = (int32_t)i;
}

// the points in cell order with their frames, so that a run is read contiguously
__global__ void overlap_gather_kernel(const double* __restrict__ xyz, int64_t n, const int64_t* __restrict__ off, int F,
                                      const int32_t* __restrict__ sidx, double* __restrict__ sxyz, int32_t* __restrict__ sframe) {
  const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (s >= n) return;
  const int64_t j = sidx[s];
  for (int k = 0; k < 3; ++k) sxyz[3 * s + k] = xyz[3 * j + k];
  sframe[s] = frame_of(off, F, j);
}

// A CTA takes OV_ROWS consecutive query rows, frame segment by frame segment.  A warp takes one query q (frame j) at a time: its
// lanes stride over the points of the 27 cells around q and mark, in the warp's bitmask, each frame i != j with a point within the
// radius; then each marked frame adds one to the CTA's count row.  At the end of a segment the row goes to counts[i * F + j] with
// integer atomics (exact, so the result does not depend on the launch shape).  smem: F count words, then OV_WARPS masks of
// ceil(F / 32) words.
__global__ void __launch_bounds__(OV_WARPS * 32, 4) overlap_kernel(
    const double* __restrict__ xyz, int64_t n, const int64_t* __restrict__ off, int F, double cell_size, double r2,
    const uint64_t* __restrict__ tk, const int32_t* __restrict__ tv, uint64_t mask, const int32_t* __restrict__ run_start,
    const int32_t* __restrict__ run_end, const double* __restrict__ sxyz, const int32_t* __restrict__ sframe,
    unsigned long long* __restrict__ counts) {
  extern __shared__ uint32_t smem[];
  const int words = (F + 31) >> 5, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t* row = smem;
  uint32_t* bits = smem + F + warp * words;
  for (int t = threadIdx.x; t < F + OV_WARPS * words; t += blockDim.x) smem[t] = 0;
  __syncthreads();
  const int64_t a = blockIdx.x * (int64_t)OV_ROWS, b = min(n, a + OV_ROWS);
  for (int j = frame_of(off, F, a); j < F && off[j] < b; ++j) {
    const int64_t lo = max(a, off[j]), hi = min(b, off[j + 1]);
    if (lo >= hi) continue;                                   // the same for every thread of the CTA
    for (int64_t q = lo + warp; q < hi; q += OV_WARPS) {
      const double px = xyz[3 * q], py = xyz[3 * q + 1], pz = xyz[3 * q + 2];
      int cx, cy, cz;
      if (!grid_cell(xyz + 3 * q, cell_size, cx, cy, cz)) continue;
      for (int d = 0; d < 27; ++d) {
        const int qx = cx + d / 9 - 1, qy = cy + (d / 3) % 3 - 1, qz = cz + d % 3 - 1;
        if (abs(qx) >= VB || abs(qy) >= VB || abs(qz) >= VB) continue;
        const int run = hash_lookup(tk, tv, mask, cell_key(qx, qy, qz));
        if (run < 0) continue;
        for (int s = run_start[run] + lane; s < run_end[run]; s += 32) {
          const int i = sframe[s];
          if (i == j || ((bits[i >> 5] >> (i & 31)) & 1u)) continue;          // the mask read only saves work
          const double ex = __dsub_rn(sxyz[3 * s], px), ey = __dsub_rn(sxyz[3 * s + 1], py), ez = __dsub_rn(sxyz[3 * s + 2], pz);
          // ((dx dx + dy dy) + dz dz) < r^2, no FMA contraction
          if (__dadd_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)), __dmul_rn(ez, ez)) < r2) atomicOr(&bits[i >> 5], 1u << (i & 31));
        }
      }
      __syncwarp();
      for (int w = lane; w < words; w += 32) {
        uint32_t m = bits[w];
        if (!m) continue;
        bits[w] = 0;
        for (; m; m &= m - 1) atomicAdd(&row[32 * w + __ffs(m) - 1], 1u);
      }
      __syncwarp();
    }
    __syncthreads();
    for (int i = threadIdx.x; i < F; i += blockDim.x)
      if (const uint32_t v = row[i]) { atomicAdd(&counts[(int64_t)i * F + j], (unsigned long long)v); row[i] = 0; }
    __syncthreads();
  }
}

// the cell sort of all frames' points, its runs and their table, the points in cell order and their frames
struct OverlapWs { SortWs s; RunsWs r; double* sxyz; int32_t* sframe; };
OverlapWs overlap_layout(Carve& c, int64_t n) {
  OverlapWs w{sort_layout(c, n), runs_layout(c, n, true), nullptr, nullptr};
  w.sxyz = c.take<double>(3 * n);
  w.sframe = c.take<int32_t>(n);
  return w;
}

bool frames_ok(int64_t n, int64_t F) { return n >= 0 && n < (1ll << 31) && F >= 1 && F <= MAX_FRAMES; }

// pcb_depth_to_points: a CTA takes one tile of DP_TILE consecutive pixels of one frame (grid: tiles x frames); a thread takes
// DP_ITEMS consecutive pixels of the tile, so a block-wide exclusive scan over the threads in order ranks the valid pixels in
// row-major order (a stable compaction).
constexpr int DP_THREADS = 256;
constexpr int DP_ITEMS = 4;
constexpr int DP_TILE = DP_THREADS * DP_ITEMS;
constexpr int64_t DP_MAX_SIDE = 1 << 15;
using DpScan = cub::BlockScan<int, DP_THREADS>;

// tile_count[f * T + t] = the number of nonzero pixels of tile t of frame f
__global__ void __launch_bounds__(DP_THREADS) depth_count_kernel(const uint16_t* __restrict__ depth, int64_t P, int T,
                                                                   int64_t* __restrict__ tile_count) {
  using Reduce = cub::BlockReduce<int, DP_THREADS>;
  __shared__ typename Reduce::TempStorage tmp;
  const int f = blockIdx.y, t = blockIdx.x;
  const uint16_t* d = depth + f * P;
  const int64_t p0 = (int64_t)t * DP_TILE + threadIdx.x * DP_ITEMS;
  int c = 0;
  for (int k = 0; k < DP_ITEMS; ++k) c += (p0 + k < P && d[p0 + k] != 0);
  c = Reduce(tmp).Sum(c);
  if (threadIdx.x == 0) tile_count[(int64_t)f * T + t] = c;
}

// The reference's arithmetic (`point_cloud_extractor.py:51-75`), one rounding per operation:
//   d = depth / 1000, X = ((u - cx) d) / fx + bx, Y = ((v - cy) d) / fy + by, Z = d,
//   w_r = ((X P[r,0] + Y P[r,1]) + Z P[r,2]) + P[r,3]        (np.dot(points, pose.T) with the homogeneous 1 of `points`)
// Pixel p goes to row tile_off[f * T + t] + (its rank among the tile's valid pixels).  A NaN coordinate sets the frame's flag.
__global__ void __launch_bounds__(DP_THREADS) depth_write_kernel(const uint16_t* __restrict__ depth, int64_t W, int64_t P, int T,
                                                                   double fx, double fy, double cx, double cy, double bx, double by,
                                                                   const double* __restrict__ poses, const int64_t* __restrict__ tile_off,
                                                                   double* __restrict__ out, unsigned long long* __restrict__ nan_flag) {
  __shared__ typename DpScan::TempStorage tmp;
  __shared__ double pose[12];
  const int f = blockIdx.y, t = blockIdx.x;
  if (threadIdx.x < 12) pose[threadIdx.x] = poses[(int64_t)f * 16 + threadIdx.x];
  const uint16_t* d = depth + f * P;
  const int64_t p0 = (int64_t)t * DP_TILE + threadIdx.x * DP_ITEMS;
  uint16_t z[DP_ITEMS];
  int valid[DP_ITEMS], rank[DP_ITEMS];
  for (int k = 0; k < DP_ITEMS; ++k) {
    z[k] = p0 + k < P ? d[p0 + k] : (uint16_t)0;
    valid[k] = z[k] != 0;
  }
  DpScan(tmp).ExclusiveSum(valid, rank);
  __syncthreads();                                            // the pose in shared memory
  const int64_t base = tile_off[(int64_t)f * T + t];
  bool nan = false;
  for (int k = 0; k < DP_ITEMS; ++k) {
    if (!valid[k]) continue;
    const int64_t p = p0 + k;
    const double u = (double)(p % W), v = (double)(p / W);
    const double Z = __ddiv_rn((double)z[k], 1000.0);
    const double X = __dadd_rn(__ddiv_rn(__dmul_rn(__dsub_rn(u, cx), Z), fx), bx);
    const double Y = __dadd_rn(__ddiv_rn(__dmul_rn(__dsub_rn(v, cy), Z), fy), by);
    double* o = out + 3 * (base + rank[k]);
    for (int r = 0; r < 3; ++r) {
      const double* P4 = pose + 4 * r;
      const double w = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(X, P4[0]), __dmul_rn(Y, P4[1])), __dmul_rn(Z, P4[2])), P4[3]);
      nan |= isnan(w);
      o[r] = w;
    }
  }
  if (__syncthreads_or(nan) && threadIdx.x == 0) atomicOr(&nan_flag[f], 1ull);
}

// offsets[f] = tile_off[f * T] for f <= F, to the device output and the host stage
__global__ void depth_offsets_kernel(const int64_t* __restrict__ tile_off, int F, int T, int64_t* __restrict__ offsets,
                                     int64_t* __restrict__ stage) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > F) return;
  offsets[f] = stage[f] = tile_off[(int64_t)f * T];
}

// tile counts and their exclusive scan (F T + 1 entries: the last count is 0, so its offset is the total), the scan's temporary
// storage, stage[2 F + 1]: the offsets, then the per-frame NaN flags, one copy to the host
struct DepthWs { int64_t* count; int64_t* off; void* cub; size_t cub_bytes; int64_t* stage; };
DepthWs depth_layout(Carve& c, int64_t F, int64_t T) {
  const int64_t m = F * T + 1;
  size_t cub_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, (int64_t*)nullptr, (int64_t*)nullptr, (int)m);
  DepthWs w{c.take<int64_t>(m), c.take<int64_t>(m), nullptr, cub_bytes, nullptr};
  w.cub = c.take<char>(cub_bytes);
  w.stage = c.take<int64_t>(2 * F + 1);
  return w;
}

int64_t depth_tiles(int64_t H, int64_t W) { return (H * W + DP_TILE - 1) / DP_TILE; }
bool depth_shape_ok(int64_t F, int64_t H, int64_t W) {
  return F >= 1 && F <= MAX_FRAMES && H >= 1 && H <= DP_MAX_SIDE && W >= 1 && W <= DP_MAX_SIDE && F * depth_tiles(H, W) < (1ll << 31) - 1;
}

}  // namespace

extern "C" size_t pcb_voxel_down_sample_ws_bytes(int64_t n, int64_t F) {
  if (!frames_ok(n, F)) return 0;
  return layout_bytes(down_layout, n < 1 ? 1 : n, F);
}

extern "C" int pcb_voxel_down_sample(const double* xyz, int64_t n, const int64_t* offsets, int64_t F, double voxel_size, double* out,
                                     int64_t* out_offsets, int64_t* out_offsets_host, void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(frames_ok(n, F) && voxel_size > 0.0 && voxel_size < INFINITY);
  Carve c{(char*)ws};
  const DownWs w = down_layout(c, n < 1 ? 1 : n, F);
  PCB_ARG((n == 0 || (xyz && out)) && offsets && out_offsets && out_offsets_host && ws && ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  PCB_CUDA(cudaMemsetAsync(w.stage + F + 1, 0, sizeof(int64_t), st));
  PCB_CUDA(cudaMemsetAsync(w.s.count, 0, sizeof(int64_t), st));
  frame_lo_kernel<<<(unsigned)F, 256, 0, st>>>(xyz, n, offsets, (int)F, voxel_size * 0.5, w.lo, w.s.status);
  if (int e = check_launch("frame_lo_kernel")) return e;
  if (n > 0) {
    down_key_kernel<<<blocks_for(n, 256), 256, 0, st>>>(xyz, n, offsets, (int)F, w.lo, voxel_size, w.s.k, w.s.idx, w.s.status);
    if (int e = check_launch("down_key_kernel")) return e;
    if (int e = sort_runs(n, w.s, 12 + 3 * DB, st)) return e;
    if (int e = find_runs(n, w.s, w.r, st)) return e;
    down_write_kernel<<<blocks_for(n, 256), 256, 0, st>>>(xyz, w.s.sidx, w.r.start, w.r.end, w.s.count, out);
    if (int e = check_launch("down_write_kernel")) return e;
  }
  down_offsets_kernel<<<blocks_for(F + 1, 256), 256, 0, st>>>(w.r.key, w.s.count, (int)F, out_offsets, w.stage);
  if (int e = check_launch("down_offsets_kernel")) return e;
  std::vector<int64_t> host((size_t)F + 2);
  PCB_CUDA(cudaMemcpyAsync(host.data(), w.stage, (F + 2) * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  PCB_CUDA(cudaStreamSynchronize(st));
  const int32_t status = (int32_t)host[F + 1];
  if (status & PCB_FRAMES_OFFSETS) { set_error("pcb_voxel_down_sample: offsets must run from 0 to n without decreasing"); return PCB_ERR_ARG; }
  if (status & PCB_FRAMES_RANGE) { set_error("pcb_voxel_down_sample: a coordinate is not finite or a voxel index exceeds 2^17"); return PCB_ERR_RANGE; }
  std::copy(host.begin(), host.begin() + F + 1, out_offsets_host);
  return PCB_OK;
}

extern "C" size_t pcb_frame_overlap_ws_bytes(int64_t n, int64_t F) {
  if (!frames_ok(n, F)) return 0;
  return layout_bytes(overlap_layout, n < 1 ? 1 : n);
}

extern "C" int pcb_frame_overlap(const double* xyz, int64_t n, const int64_t* offsets, int64_t F, double radius, int64_t* counts, int32_t* status,
                                 void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(frames_ok(n, F) && radius > 0.0 && radius < INFINITY);
  Carve c{(char*)ws};
  const OverlapWs w = overlap_layout(c, n < 1 ? 1 : n);
  PCB_ARG((n == 0 || xyz) && offsets && counts && status && ws && ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  PCB_CUDA(cudaMemsetAsync(counts, 0, (size_t)(F * F) * sizeof(int64_t), st));
  offsets_check_kernel<<<blocks_for(F, 256), 256, 0, st>>>(offsets, (int)F, n, status);
  if (int e = check_launch("offsets_check_kernel")) return e;
  if (n == 0) return PCB_OK;
  // Two points within the radius lie in neighbouring cells: with cells of r (1 + 2^-20), |x_p / c - x_q / c| <= 1 - 2^-21 even after
  // the roundings of the distance test and of the divisions (|x / c| < 2^20), so the floors differ by at most one.
  const double cell_size = radius * (1.0 + 0x1p-20);
  overlap_key_kernel<<<blocks_for(n, 256), 256, 0, st>>>(xyz, n, cell_size, w.s.k, w.s.idx, status);
  if (int e = check_launch("overlap_key_kernel")) return e;
  if (int e = sort_runs(n, w.s, 63, st)) return e;
  if (int e = find_runs(n, w.s, w.r, st)) return e;
  overlap_gather_kernel<<<blocks_for(n, 256), 256, 0, st>>>(xyz, n, offsets, (int)F, w.s.sidx, w.sxyz, w.sframe);
  if (int e = check_launch("overlap_gather_kernel")) return e;
  const int words = (int)((F + 31) / 32);
  const size_t smem = (size_t)(F + OV_WARPS * words) * sizeof(uint32_t);
  overlap_kernel<<<blocks_for(n, OV_ROWS), OV_WARPS * 32, smem, st>>>(xyz, n, offsets, (int)F, cell_size, radius * radius, w.r.tk, w.r.tv,
                                                                      (uint64_t)w.r.tcap - 1, w.r.start, w.r.end, w.sxyz, w.sframe,
                                                                      (unsigned long long*)counts);
  return check_launch("overlap_kernel");
}

extern "C" size_t pcb_depth_to_points_ws_bytes(int64_t F, int64_t H, int64_t W) {
  if (!depth_shape_ok(F, H, W)) return 0;
  return layout_bytes(depth_layout, F, depth_tiles(H, W));
}

extern "C" int pcb_depth_to_points(const uint16_t* depth, int64_t F, int64_t H, int64_t W, double fx, double fy, double cx, double cy,
                                   double bx, double by, const double* poses, double* out, int64_t* out_offsets, int64_t* out_offsets_host,
                                   int32_t* nan_host, void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(depth_shape_ok(F, H, W));
  const int64_t T = depth_tiles(H, W), P = H * W;
  Carve c{(char*)ws};
  const DepthWs w = depth_layout(c, F, T);
  PCB_ARG(depth && poses && out && out_offsets && out_offsets_host && nan_host && ws && ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  PCB_CUDA(cudaMemsetAsync(w.count + F * T, 0, sizeof(int64_t), st));
  PCB_CUDA(cudaMemsetAsync(w.stage + F + 1, 0, F * sizeof(int64_t), st));
  const dim3 grid((unsigned)T, (unsigned)F);
  depth_count_kernel<<<grid, DP_THREADS, 0, st>>>(depth, P, (int)T, w.count);
  if (int e = check_launch("depth_count_kernel")) return e;
  size_t cb = w.cub_bytes;
  PCB_CUDA(cub::DeviceScan::ExclusiveSum(w.cub, cb, w.count, w.off, (int)(F * T + 1), st));
  depth_write_kernel<<<grid, DP_THREADS, 0, st>>>(depth, W, P, (int)T, fx, fy, cx, cy, bx, by, poses, w.off, out,
                                                  (unsigned long long*)(w.stage + F + 1));
  if (int e = check_launch("depth_write_kernel")) return e;
  depth_offsets_kernel<<<blocks_for(F + 1, 256), 256, 0, st>>>(w.off, (int)F, (int)T, out_offsets, w.stage);
  if (int e = check_launch("depth_offsets_kernel")) return e;
  std::vector<int64_t> host((size_t)(2 * F + 1));
  PCB_CUDA(cudaMemcpyAsync(host.data(), w.stage, (2 * F + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  PCB_CUDA(cudaStreamSynchronize(st));
  std::copy(host.begin(), host.begin() + F + 1, out_offsets_host);
  for (int64_t f = 0; f < F; ++f) nan_host[f] = (int32_t)host[F + 1 + f];
  return PCB_OK;
}
