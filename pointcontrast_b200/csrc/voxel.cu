// GPU voxelisation and correspondence search -- the per-sample work of the reference's data loader
// (`pretrain/pointcontrast/lib/ddp_data_loaders.py:196-265`), which today runs on CPU workers:
//   * `ME.utils.sparse_quantize(xyz / voxel_size, return_index=True)` (`:228-241`; semseg: `lib/voxelizer.py:113-148`):
//     one point per occupied voxel                                                          -> pcb_voxelize
//   * the same per scene of a collated VoteNet batch, the scene index in the key (`downstream/votenet_det_new/models/backbone/
//     sparseconv/voxelized_dataset.py:33-65`): rows scene-major, ascending first index        -> pcb_voxelize_scenes
//   * its label variant on integer coordinates (semseg `lib/voxelizer.py:145-146`): a voxel keeps the label its points share,
//     else ignore_label                                                                     -> pcb_voxelize_labels
//   * `get_matching_indices` (`:36-49`): an open3d KD-tree radius search PER POINT, radius 1.5 voxels   -> pcb_radius_pairs
// Both are integer / hashing work on the same primitives as the coordinate manager (radix sort + head flags + scan, the
// open-addressing hash table of common.cuh); results are exact (tests/test_gpu_voxel.py: vs numpy / scipy cKDTree).
#include <algorithm>
#include <vector>
#include <cub/cub.cuh>
#include "sort.cuh"

using namespace pcb;

namespace {

__device__ __forceinline__ bool cell_of(float x, float y, float z, float inv_unused, float size, int& cx, int& cy, int& cz) {
  // floor(v / size) in fp32, exactly what numpy does on float32 input (IEEE division, then floor)
  const float fx = floorf(x / size), fy = floorf(y / size), fz = floorf(z / size);
  cx = (int)fx; cy = (int)fy; cz = (int)fz;
  return fabsf(fx) < (float)VB && fabsf(fy) < (float)VB && fabsf(fz) < (float)VB;
}

__global__ void point_key_kernel(const float* __restrict__ xyz, int64_t n, float size, uint64_t* __restrict__ keys, int32_t* __restrict__ idx,
                                 int32_t* status) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int cx, cy, cz;
  if (!cell_of(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], 0.f, size, cx, cy, cz)) { atomicOr(status, PCB_ERR_RANGE); cx = cy = cz = 0; }
  keys[i] = cell_key(cx, cy, cz);
  idx[i] = (int32_t)i;
}

__global__ void head_kernel(const uint64_t* __restrict__ sk, int64_t n, int32_t* __restrict__ flag) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) flag[i] = (i == 0 || sk[i] != sk[i - 1]) ? 1 : 0;
}

// voxelisation output: one row per run of equal keys; the radix sort is stable, so the first element of a run is the point with the
// smallest original index (np.unique(..., return_index=True))
__global__ void voxel_write_kernel(const uint64_t* __restrict__ sk, const int32_t* __restrict__ sidx, const int32_t* __restrict__ rank,
                                   int64_t n, int32_t* __restrict__ coords, int32_t* __restrict__ sel, int64_t* m_out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (i == 0 || sk[i] != sk[i - 1]) {
    const int r = rank[i] - 1;
    const uint64_t k = sk[i];
    coords[3 * r] = (int)(k >> 42) - VB; coords[3 * r + 1] = (int)((k >> 21) & 0x1FFFFF) - VB; coords[3 * r + 2] = (int)(k & 0x1FFFFF) - VB;
    sel[r] = sidx[i];
  }
  if (i == n - 1) *m_out = rank[i];
}

// radius search: runs of the cell-sorted target points -> run start/end, hash (cell key -> run)
__global__ void run_bounds_kernel(const uint64_t* __restrict__ sk, const int32_t* __restrict__ rank, int64_t n, uint64_t* __restrict__ run_key,
                                  int32_t* __restrict__ run_start, int32_t* __restrict__ run_end, int64_t* n_runs) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = rank[i] - 1;
  if (i == 0 || sk[i] != sk[i - 1]) { run_key[r] = sk[i]; run_start[r] = (int32_t)i; }
  if (i == n - 1 || sk[i] != sk[i + 1]) run_end[r] = (int32_t)i + 1;
  if (i == n - 1) *n_runs = rank[i];
}

__global__ void run_insert_kernel(const uint64_t* __restrict__ run_key, const int64_t* __restrict__ n_runs, uint64_t* tk, int32_t* tv, uint64_t mask) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= *n_runs) return;
  const uint64_t key = run_key[i];
  uint64_t slot = mix64(key) & mask;
  while (true) {
    const unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long*>(tk + slot), (unsigned long long)KEY_EMPTY, (unsigned long long)key);
    if (prev == KEY_EMPTY) { tv[slot] = (int32_t)i; return; }
    slot = (slot + 1) & mask;
  }
}

// FILL = false: cnt[i] = number of targets within the radius of source i;  FILL = true: writes them at pairs[off[i] ...], ascending j
template <bool FILL>
__global__ void radius_kernel(const float* __restrict__ src, int64_t ns, const float* __restrict__ dst, float radius, const uint64_t* __restrict__ tk,
                              const int32_t* __restrict__ tv, uint64_t mask, const int32_t* __restrict__ run_start,
                              const int32_t* __restrict__ run_end, const int32_t* __restrict__ sidx, int32_t* __restrict__ cnt,
                              const int64_t* __restrict__ off, int32_t* __restrict__ pairs, int64_t cap) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= ns) return;
  const float px = src[3 * i], py = src[3 * i + 1], pz = src[3 * i + 2];
  int cx, cy, cz;
  int found = 0;
  const int64_t base = FILL ? off[i] : 0;
  if (cell_of(px, py, pz, 0.f, radius, cx, cy, cz)) {
    const float r2 = __fmul_rn(radius, radius);
    for (int dx = -1; dx <= 1; ++dx)
      for (int dy = -1; dy <= 1; ++dy)
        for (int dz = -1; dz <= 1; ++dz) {
          const int qx = cx + dx, qy = cy + dy, qz = cz + dz;
          if (abs(qx) >= VB || abs(qy) >= VB || abs(qz) >= VB) continue;
          const int run = hash_lookup(tk, tv, mask, cell_key(qx, qy, qz));
          if (run < 0) continue;
          for (int s = run_start[run]; s < run_end[run]; ++s) {
            const int j = sidx[s];
            const float ex = dst[3 * j] - px, ey = dst[3 * j + 1] - py, ez = dst[3 * j + 2] - pz;
            if (__fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez)) < r2) {      // no FMA contraction: reproducible on the host
              if (FILL && base + found < cap) { pairs[2 * (base + found)] = (int32_t)i; pairs[2 * (base + found) + 1] = j; }
              ++found;
            }
          }
        }
  }
  if (!FILL) { cnt[i] = found; return; }
  // ascending j within the row (a handful of entries): insertion sort in place
  const int64_t m = min((int64_t)found, cap - base > 0 ? cap - base : 0);
  for (int64_t a = 1; a < m; ++a) {
    const int32_t v = pairs[2 * (base + a) + 1];
    int64_t b = a - 1;
    while (b >= 0 && pairs[2 * (base + b) + 1] > v) { pairs[2 * (base + b + 1) + 1] = pairs[2 * (base + b) + 1]; --b; }
    pairs[2 * (base + b + 1) + 1] = v;
  }
}

size_t sort_scan_bytes(int64_t n) {
  size_t a = 0, b = 0, c = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, a, (uint64_t*)nullptr, (uint64_t*)nullptr, (int32_t*)nullptr, (int32_t*)nullptr, (int)n);
  cub::DeviceScan::InclusiveSum(nullptr, b, (int32_t*)nullptr, (int32_t*)nullptr, (int)n);
  cub::DeviceScan::ExclusiveSum(nullptr, c, (int32_t*)nullptr, (int64_t*)nullptr, (int)n);
  size_t m = a > b ? a : b;
  return m > c ? m : c;
}

}  // namespace

namespace pcb {

SortWs sort_layout(Carve& c, int64_t n) {
  const size_t cub_bytes = sort_scan_bytes(n);
  return {c.take<uint64_t>(n), c.take<uint64_t>(n), c.take<int32_t>(n), c.take<int32_t>(n), c.take<int32_t>(n), c.take<int32_t>(n),
          c.take<int64_t>(1), c.take<int32_t>(1), c.take<char>(cub_bytes), cub_bytes};
}

int sort_keys(int64_t n, const SortWs& w, int end_bit, cudaStream_t st) {
  size_t cb = w.cub_bytes;
  PCB_CUDA(cub::DeviceRadixSort::SortPairs(w.cub, cb, w.k, w.sk, w.idx, w.sidx, (int)n, 0, end_bit, st));
  g_launches.fetch_add(8);
  return PCB_OK;
}

int sort_runs(int64_t n, const SortWs& w, int end_bit, cudaStream_t st) {
  if (int e = sort_keys(n, w, end_bit, st)) return e;
  head_kernel<<<blocks_for(n, 256), 256, 0, st>>>(w.sk, n, w.flag);
  if (int e = check_launch("head_kernel")) return e;
  size_t cb = w.cub_bytes;
  PCB_CUDA(cub::DeviceScan::InclusiveSum(w.cub, cb, w.flag, w.rank, (int)n, st));
  g_launches.fetch_add(2);
  return PCB_OK;
}

RunsWs runs_layout(Carve& c, int64_t n, bool hashed) {
  RunsWs r{c.take<uint64_t>(n), c.take<int32_t>(n), c.take<int32_t>(n), 0, nullptr, nullptr};
  if (hashed) {
    r.tcap = 16;
    while (r.tcap < 2 * n) r.tcap <<= 1;
    r.tk = c.take<uint64_t>(r.tcap);
    r.tv = c.take<int32_t>(r.tcap);
  }
  return r;
}

int find_runs(int64_t n, const SortWs& w, const RunsWs& r, cudaStream_t st) {
  run_bounds_kernel<<<blocks_for(n, 256), 256, 0, st>>>(w.sk, w.rank, n, r.key, r.start, r.end, w.count);
  if (int e = check_launch("run_bounds_kernel")) return e;
  if (!r.tk) return PCB_OK;
  PCB_CUDA(cudaMemsetAsync(r.tk, 0xFF, (size_t)r.tcap * 8, st));
  run_insert_kernel<<<blocks_for(n, 256), 256, 0, st>>>(r.key, w.count, r.tk, r.tv, (uint64_t)r.tcap - 1);
  return check_launch("run_insert_kernel");
}

}  // namespace pcb

namespace {

int point_keys(const float* xyz, int64_t n, float size, const SortWs& w, cudaStream_t st) {
  PCB_CUDA(cudaMemsetAsync(w.status, 0, sizeof(int32_t), st));
  point_key_kernel<<<blocks_for(n, 256), 256, 0, st>>>(xyz, n, size, w.k, w.idx, w.status);
  return check_launch("point_key_kernel");
}

// keys of the points' cells -> sort_runs
int sort_cells(const float* xyz, int64_t n, float size, const SortWs& w, cudaStream_t st) {
  if (int e = point_keys(xyz, n, size, w, st)) return e;
  return sort_runs(n, w, 63, st);
}

// Batched voxelisation.  After the stable sort by cell key alone, a run of equal keys lists its points in ascending GLOBAL index, i.e.
// grouped by scene (scenes are contiguous in the input) and ascending within each scene; so a (scene, cell) voxel starts where the key
// or the scene changes, and its first element is the scene's smallest index in that cell.  The flag goes back to the head's ORIGINAL
// position, so one exclusive scan over the input order numbers the voxels scene-major, ascending first index within a scene.
__global__ void scene_head_kernel(const uint64_t* __restrict__ sk, const int32_t* __restrict__ sidx, int64_t n, int64_t N,
                                  int32_t* __restrict__ flag) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  flag[sidx[i]] = (i == 0 || sk[i] != sk[i - 1] || sidx[i] / N != sidx[i - 1] / N) ? 1 : 0;
}

// row = exclusive scan of the flags at the head's position; offsets[b] = the scan at b * N, offsets[B] = M (also into stage[])
__global__ void scene_write_kernel(const uint64_t* __restrict__ k, const int32_t* __restrict__ flag, const int64_t* __restrict__ row,
                                   int64_t n, int64_t N, int32_t* __restrict__ coords, int32_t* __restrict__ inds, int64_t* __restrict__ offsets,
                                   int64_t* __restrict__ stage) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t b = i / N;
  if (i - b * N == 0) { offsets[b] = row[i]; stage[b] = row[i]; }
  if (i == n - 1) { offsets[b + 1] = row[i] + flag[i]; stage[b + 1] = row[i] + flag[i]; }
  if (!flag[i]) return;
  const int64_t r = row[i];
  const uint64_t key = k[i];
  coords[4 * r] = (int32_t)b;
  coords[4 * r + 1] = (int)(key >> 42) - VB; coords[4 * r + 2] = (int)((key >> 21) & 0x1FFFFF) - VB; coords[4 * r + 3] = (int)(key & 0x1FFFFF) - VB;
  inds[r] = (int32_t)(i - b * N);
}

__global__ void int_key_kernel(const int32_t* __restrict__ c, int64_t n, uint64_t* __restrict__ keys, int32_t* __restrict__ idx, int32_t* status) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int x = c[3 * i], y = c[3 * i + 1], z = c[3 * i + 2];
  if (x <= -VB || x >= VB || y <= -VB || y >= VB || z <= -VB || z >= VB) { atomicOr(status, PCB_ERR_RANGE); x = y = z = 0; }
  keys[i] = cell_key(x, y, z);
  idx[i] = (int32_t)i;
}

// label-aware voxelisation output: one thread per run head writes the voxel and scans its run (the stable sort keeps the points of a
// voxel in ascending index order) for the smallest and largest label; the voxel keeps its label only if the two agree
__global__ void voxel_label_write_kernel(const uint64_t* __restrict__ sk, const int32_t* __restrict__ sidx, const int32_t* __restrict__ rank,
                                         const int32_t* __restrict__ labels, int64_t n, int32_t ignore_label, int32_t* __restrict__ coords,
                                         int32_t* __restrict__ sel, int32_t* __restrict__ out_labels, int64_t* m_out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (i == n - 1) *m_out = rank[i];
  const uint64_t k = sk[i];
  if (i > 0 && sk[i - 1] == k) return;
  const int r = rank[i] - 1;
  coords[3 * r] = (int)(k >> 42) - VB; coords[3 * r + 1] = (int)((k >> 21) & 0x1FFFFF) - VB; coords[3 * r + 2] = (int)(k & 0x1FFFFF) - VB;
  sel[r] = sidx[i];
  int32_t lo = labels[sidx[i]], hi = lo;
  for (int64_t j = i + 1; j < n && sk[j] == k; ++j) {
    const int32_t l = labels[sidx[j]];
    lo = min(lo, l); hi = max(hi, l);
  }
  out_labels[r] = lo == hi ? lo : ignore_label;
}

// the sort pipeline, then stage[B + 2]: offsets[0..B] and the range status, one copy back to the host
SortWs scenes_layout(Carve& c, int64_t B, int64_t N, int64_t*& stage) {
  SortWs w = sort_layout(c, B * N);
  stage = c.take<int64_t>(B + 2);
  w.status = (int32_t*)(stage + B + 1);
  return w;
}

// the cell sort of the targets, their runs and the hash table of the runs, per-source counts / offsets
struct PairsWs { SortWs s; RunsWs r; int32_t* cnt; int64_t* off; void* cub; size_t cub_bytes; };
PairsWs pairs_layout(Carve& c, int64_t ns, int64_t nd) {
  const size_t cub_bytes = sort_scan_bytes(ns);
  return {sort_layout(c, nd), runs_layout(c, nd, true), c.take<int32_t>(ns), c.take<int64_t>(ns), c.take<char>(cub_bytes), cub_bytes};
}

}  // namespace

extern "C" size_t pcb_voxelize_ws_bytes(int64_t n) {
  return layout_bytes(sort_layout, n < 1 ? 1 : n);
}

extern "C" int pcb_voxelize(const float* xyz, int64_t n, float voxel_size, int32_t* out_coords, int32_t* sel, int64_t* m_out, void* ws,
                            size_t ws_bytes, void* stream) {
  PCB_ARG(n >= 0 && n < (1ll << 31) && voxel_size > 0.f && m_out);
  *m_out = 0;
  if (n == 0) return PCB_OK;
  Carve c{(char*)ws};
  const SortWs w = sort_layout(c, n);
  PCB_ARG(xyz && out_coords && sel && ws && ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  if (int e = sort_cells(xyz, n, voxel_size, w, st)) return e;
  voxel_write_kernel<<<blocks_for(n, 256), 256, 0, st>>>(w.sk, w.sidx, w.rank, n, out_coords, sel, w.count);
  if (int e = check_launch("voxel_write_kernel")) return e;
  int32_t status = 0;
  PCB_CUDA(cudaMemcpyAsync(m_out, w.count, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  PCB_CUDA(cudaMemcpyAsync(&status, w.status, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  PCB_CUDA(cudaStreamSynchronize(st));
  if (status) { set_error("pcb_voxelize: a point lies outside +-2^20 voxels"); return PCB_ERR_RANGE; }
  return PCB_OK;
}

extern "C" size_t pcb_voxelize_scenes_ws_bytes(int64_t B, int64_t N) {
  if (B < 1 || N < 1 || B * N >= (1ll << 31)) return 0;
  Carve c{nullptr};
  int64_t* stage;
  scenes_layout(c, B, N, stage);
  return c.used;
}

extern "C" int pcb_voxelize_scenes(const float* xyz, int64_t B, int64_t N, float voxel_size, int32_t* out_coords, int32_t* inds, int64_t* offsets,
                                   int64_t* offsets_host, void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(B >= 1 && N >= 1 && B * N < (1ll << 31) && voxel_size > 0.f);
  Carve c{(char*)ws};
  int64_t* stage;
  const SortWs w = scenes_layout(c, B, N, stage);
  PCB_ARG(xyz && out_coords && inds && offsets && offsets_host && ws && ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n = B * N;
  PCB_CUDA(cudaMemsetAsync(stage + B + 1, 0, sizeof(int64_t), st));
  if (int e = point_keys(xyz, n, voxel_size, w, st)) return e;
  if (int e = sort_keys(n, w, 63, st)) return e;
  scene_head_kernel<<<blocks_for(n, 256), 256, 0, st>>>(w.sk, w.sidx, n, N, w.flag);
  if (int e = check_launch("scene_head_kernel")) return e;
  int64_t* row = (int64_t*)w.sk;                   // the sorted keys are dead after the head flags
  size_t cb = w.cub_bytes;
  PCB_CUDA(cub::DeviceScan::ExclusiveSum(w.cub, cb, w.flag, row, (int)n, st));
  g_launches.fetch_add(2);
  scene_write_kernel<<<blocks_for(n, 256), 256, 0, st>>>(w.k, w.flag, row, n, N, out_coords, inds, offsets, stage);
  if (int e = check_launch("scene_write_kernel")) return e;
  std::vector<int64_t> host((size_t)B + 2);
  PCB_CUDA(cudaMemcpyAsync(host.data(), stage, (B + 2) * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  PCB_CUDA(cudaStreamSynchronize(st));
  if ((int32_t)host[B + 1]) { set_error("pcb_voxelize_scenes: a point lies outside +-2^20 voxels"); return PCB_ERR_RANGE; }
  std::copy(host.begin(), host.begin() + B + 1, offsets_host);
  return PCB_OK;
}

extern "C" size_t pcb_voxelize_labels_ws_bytes(int64_t n) {
  return layout_bytes(sort_layout, n < 1 ? 1 : n);
}

extern "C" int pcb_voxelize_labels(const int32_t* coords, const int32_t* labels, int64_t n, int32_t ignore_label, int32_t* out_coords,
                                   int32_t* sel, int32_t* out_labels, int64_t* m_out, void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(n >= 0 && n < (1ll << 31) && m_out);
  *m_out = 0;
  if (n == 0) return PCB_OK;
  Carve c{(char*)ws};
  const SortWs w = sort_layout(c, n);
  PCB_ARG(coords && labels && out_coords && sel && out_labels && ws && ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  PCB_CUDA(cudaMemsetAsync(w.status, 0, sizeof(int32_t), st));
  int_key_kernel<<<blocks_for(n, 256), 256, 0, st>>>(coords, n, w.k, w.idx, w.status);
  if (int e = check_launch("int_key_kernel")) return e;
  if (int e = sort_runs(n, w, 63, st)) return e;
  voxel_label_write_kernel<<<blocks_for(n, 256), 256, 0, st>>>(w.sk, w.sidx, w.rank, labels, n, ignore_label, out_coords, sel, out_labels,
                                                               w.count);
  if (int e = check_launch("voxel_label_write_kernel")) return e;
  int32_t status = 0;
  PCB_CUDA(cudaMemcpyAsync(m_out, w.count, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  PCB_CUDA(cudaMemcpyAsync(&status, w.status, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  PCB_CUDA(cudaStreamSynchronize(st));
  if (status) { set_error("pcb_voxelize_labels: a coordinate lies outside +-2^20"); return PCB_ERR_RANGE; }
  return PCB_OK;
}

extern "C" size_t pcb_radius_pairs_ws_bytes(int64_t ns, int64_t nd) {
  return layout_bytes(pairs_layout, ns < 1 ? 1 : ns, nd < 1 ? 1 : nd);
}

// pairs == NULL / cap == 0: only counts (*n_pairs = total).  Otherwise writes min(total, cap) pairs (i ascending, j ascending within i).
extern "C" int pcb_radius_pairs(const float* src, int64_t ns, const float* dst, int64_t nd, float radius, int32_t* pairs, int64_t cap,
                                int64_t* n_pairs, void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(ns >= 0 && nd >= 0 && ns < (1ll << 31) && nd < (1ll << 31) && radius > 0.f && n_pairs);
  *n_pairs = 0;
  if (ns == 0 || nd == 0) return PCB_OK;
  Carve c{(char*)ws};
  const PairsWs w = pairs_layout(c, ns, nd);
  PCB_ARG(src && dst && ws && ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  if (int e = sort_cells(dst, nd, radius, w.s, st)) return e;
  if (int e = find_runs(nd, w.s, w.r, st)) return e;
  const uint64_t mask = (uint64_t)w.r.tcap - 1;
  radius_kernel<false><<<blocks_for(ns, 128), 128, 0, st>>>(src, ns, dst, radius, w.r.tk, w.r.tv, mask, w.r.start, w.r.end, w.s.sidx, w.cnt,
                                                            nullptr, nullptr, 0);
  if (int e = check_launch("radius_kernel<count>")) return e;
  size_t cb = w.cub_bytes;
  PCB_CUDA(cub::DeviceScan::ExclusiveSum(w.cub, cb, w.cnt, w.off, (int)ns, st));
  g_launches.fetch_add(2);
  int64_t last_off = 0; int32_t last_cnt = 0;
  PCB_CUDA(cudaMemcpyAsync(&last_off, w.off + ns - 1, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  PCB_CUDA(cudaMemcpyAsync(&last_cnt, w.cnt + ns - 1, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  PCB_CUDA(cudaStreamSynchronize(st));
  *n_pairs = last_off + last_cnt;
  if (!pairs || cap <= 0) return PCB_OK;
  radius_kernel<true><<<blocks_for(ns, 128), 128, 0, st>>>(src, ns, dst, radius, w.r.tk, w.r.tv, mask, w.r.start, w.r.end, w.s.sidx, w.cnt,
                                                           w.off, pairs, cap);
  return check_launch("radius_kernel<fill>");
}
