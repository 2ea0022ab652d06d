// Coordinate manager kernels: key packing, hash table, stride (sort + unique), neighbour-table kernel maps.
// Replaces MinkowskiEngine 0.4.3's CPU CoordsManager (see include/pcb200.h for the reference call sites).
// Integer-only: results are bit-exact against oracle/me_cpu.py (tests/test_gpu_coords.py).
#include <stdarg.h>
#include "sort.cuh"

namespace pcb {
static thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};
void set_error(const char* fmt, ...) {
  va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
}
}  // namespace pcb

using namespace pcb;

extern "C" const char* pcb_last_error(void) { return pcb::g_err; }
extern "C" const char* pcb_version(void) { return "pcb200 0.1 sm_90a"; }
extern "C" uint64_t pcb_launch_count(void) { return pcb::g_launches.load(); }
extern "C" int pcb_set_device(int device) { PCB_CUDA(cudaSetDevice(device)); return PCB_OK; }

namespace {

__global__ void pack_kernel(const int32_t* __restrict__ c, int64_t n, uint64_t* __restrict__ keys, int32_t* status) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int4 v = reinterpret_cast<const int4*>(c)[i];
  bool ok = v.x >= 0 && v.x < 65535 && v.y >= -COORD_BIAS && v.y < COORD_BIAS && v.z >= -COORD_BIAS && v.z < COORD_BIAS &&
            v.w >= -COORD_BIAS && v.w < COORD_BIAS;
  if (!ok) { atomicOr(status, PCB_ERR_RANGE); keys[i] = KEY_EMPTY - 1 - (uint64_t)i; return; }
  keys[i] = ((uint64_t)v.x << 48) | ((uint64_t)(v.y + COORD_BIAS) << 32) | ((uint64_t)(v.z + COORD_BIAS) << 16) |
            (uint64_t)(v.w + COORD_BIAS);
}

__global__ void unpack_kernel(const uint64_t* __restrict__ keys, int64_t n, int32_t* __restrict__ c) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t k = keys[i];
  int4 v;
  v.x = (int)(k >> 48);
  v.y = (int)((k >> 32) & 0xFFFF) - COORD_BIAS;
  v.z = (int)((k >> 16) & 0xFFFF) - COORD_BIAS;
  v.w = (int)(k & 0xFFFF) - COORD_BIAS;
  reinterpret_cast<int4*>(c)[i] = v;
}

__global__ void hash_insert_kernel(const uint64_t* __restrict__ keys, int64_t n, uint64_t* tk, int32_t* tv,
                                   uint64_t mask, int32_t* status) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t key = keys[i];
  uint64_t slot = mix64(key) & mask;
  while (true) {
    unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long*>(tk + slot),
                                        (unsigned long long)KEY_EMPTY, (unsigned long long)key);
    if (prev == KEY_EMPTY) { tv[slot] = (int32_t)i; return; }
    if (prev == key) { atomicOr(status, PCB_ERR_DUPLICATE); return; }
    slot = (slot + 1) & mask;
  }
}

__device__ __forceinline__ int floor_to(int x, int ts) {
  int q = (x >= 0) ? (x / ts) : -((-x + ts - 1) / ts);
  return q * ts;
}

__global__ void coarse_key_kernel(const uint64_t* __restrict__ keys, int64_t n, int ts, uint64_t* __restrict__ ck,
                                  int32_t* __restrict__ idx) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t k = keys[i];
  int x = floor_to((int)((k >> 32) & 0xFFFF) - COORD_BIAS, ts);
  int y = floor_to((int)((k >> 16) & 0xFFFF) - COORD_BIAS, ts);
  int z = floor_to((int)(k & 0xFFFF) - COORD_BIAS, ts);
  // floor can only move towards -inf by < ts; -32768 is a multiple of every power-of-two ts; clamp for safety
  x = max(x, -COORD_BIAS); y = max(y, -COORD_BIAS); z = max(z, -COORD_BIAS);
  ck[i] = (k & 0xFFFF000000000000ull) | ((uint64_t)(x + COORD_BIAS) << 32) | ((uint64_t)(y + COORD_BIAS) << 16) |
          (uint64_t)(z + COORD_BIAS);
  idx[i] = (int32_t)i;
}

__global__ void unique_write_kernel(const uint64_t* __restrict__ sk, const int32_t* __restrict__ sidx,
                                    const int32_t* __restrict__ rank, int64_t n, uint64_t* __restrict__ out_keys,
                                    int32_t* __restrict__ parent, int64_t* n_out) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int r = rank[i] - 1;
  if (i == 0 || sk[i] != sk[i - 1]) out_keys[r] = sk[i];
  if (parent) parent[sidx[i]] = r;
  if (i == n - 1) *n_out = r + 1;
}

struct Offsets { int v[PCB_MAX_KERNEL_VOLUME][3]; };

__global__ void kernel_map_kernel(const uint64_t* __restrict__ out_keys, int64_t n_out, const uint64_t* __restrict__ tk,
                                  const int32_t* __restrict__ tv, uint64_t mask, Offsets offs, int32_t* __restrict__ tbl) {
  int k = blockIdx.y;
  int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (j >= n_out) return;
  uint64_t key = out_keys[j];
  int x = (int)((key >> 32) & 0xFFFF) + offs.v[k][0];
  int y = (int)((key >> 16) & 0xFFFF) + offs.v[k][1];
  int z = (int)(key & 0xFFFF) + offs.v[k][2];
  int r = -1;
  if ((unsigned)x < 65536u && (unsigned)y < 65536u && (unsigned)z < 65536u) {
    uint64_t q = (key & 0xFFFF000000000000ull) | ((uint64_t)x << 32) | ((uint64_t)y << 16) | (uint64_t)z;
    r = hash_lookup(tk, tv, mask, q);
  }
  tbl[(int64_t)k * n_out + j] = r;
}

__global__ void map_count_kernel(const int32_t* __restrict__ tbl, int64_t n_out, unsigned long long* counts) {
  int k = blockIdx.y;
  int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  bool hit = (j < n_out) && tbl[(int64_t)k * n_out + j] >= 0;
  unsigned b = __ballot_sync(0xffffffffu, hit);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(counts + k, (unsigned long long)__popc(b));
}

// key[row] = (row / window) << 32 | mask, bit k of mask = (tbl[k][row] >= 0); payload = row
__global__ void tile_order_key_kernel(const int32_t* __restrict__ tbl, int64_t tbl_stride, int K, int64_t n_out, int64_t window,
                                      uint64_t* __restrict__ keys, int32_t* __restrict__ idx) {
  const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (j >= n_out) return;
  uint32_t mask = 0;
  for (int k = 0; k < K; ++k) mask |= (tbl[(int64_t)k * tbl_stride + j] >= 0 ? 1u : 0u) << k;
  keys[j] = ((uint64_t)(j / window) << 32) | mask;
  idx[j] = (int32_t)j;
}

}  // namespace

extern "C" int pcb_coords_pack(const int32_t* coords, int64_t n, uint64_t* keys, int32_t* status, void* stream) {
  PCB_ARG(n >= 0 && n < (1ll << 31));
  if (n == 0) return PCB_OK;
  PCB_ARG(coords && keys && status);
  pack_kernel<<<blocks_for(n, 256), 256, 0, (cudaStream_t)stream>>>(coords, n, keys, status);
  return check_launch("pack_kernel");
}

extern "C" int pcb_coords_unpack(const uint64_t* keys, int64_t n, int32_t* coords, void* stream) {
  PCB_ARG(n >= 0);
  if (n == 0) return PCB_OK;
  PCB_ARG(coords && keys);
  unpack_kernel<<<blocks_for(n, 256), 256, 0, (cudaStream_t)stream>>>(keys, n, coords);
  return check_launch("unpack_kernel");
}

extern "C" int pcb_hash_build(const uint64_t* keys, int64_t n, uint64_t* table_keys, int32_t* table_vals,
                              int64_t capacity, int32_t* status, void* stream) {
  PCB_ARG(capacity > 0 && (capacity & (capacity - 1)) == 0 && capacity >= 2 * n && table_keys && table_vals && status);
  cudaStream_t st = (cudaStream_t)stream;
  PCB_CUDA(cudaMemsetAsync(table_keys, 0xFF, (size_t)capacity * sizeof(uint64_t), st));
  if (n == 0) return PCB_OK;
  hash_insert_kernel<<<blocks_for(n, 256), 256, 0, st>>>(keys, n, table_keys, table_vals, (uint64_t)capacity - 1, status);
  return check_launch("hash_insert_kernel");
}

extern "C" size_t pcb_coords_stride_ws_bytes(int64_t n) {
  return layout_bytes(sort_layout, n < 1 ? 1 : n);
}

extern "C" int pcb_coords_stride(const uint64_t* keys, int64_t n, int32_t new_ts, uint64_t* out_keys, int32_t* parent,
                                 int64_t* n_out, void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(n >= 0 && n < (1ll << 31) && new_ts >= 1 && n_out);
  *n_out = 0;
  if (n == 0) return PCB_OK;
  Carve c{(char*)ws};
  const SortWs w = sort_layout(c, n);
  PCB_ARG(keys && out_keys && ws && ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  coarse_key_kernel<<<blocks_for(n, 256), 256, 0, st>>>(keys, n, new_ts, w.k, w.idx);
  if (int e = check_launch("coarse_key_kernel")) return e;
  if (int e = sort_runs(n, w, 64, st)) return e;      // all 64 bits: the batch index is the top 16
  unique_write_kernel<<<blocks_for(n, 256), 256, 0, st>>>(w.sk, w.sidx, w.rank, n, out_keys, parent, w.count);
  if (int e = check_launch("unique_write_kernel")) return e;
  PCB_CUDA(cudaMemcpyAsync(n_out, w.count, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  PCB_CUDA(cudaStreamSynchronize(st));
  return PCB_OK;
}

extern "C" int pcb_kernel_map(const uint64_t* out_keys, int64_t n_out, const uint64_t* table_keys,
                              const int32_t* table_vals, int64_t capacity, const int32_t* offsets, int K, int32_t* tbl,
                              void* stream) {
  PCB_ARG(K >= 1 && K <= PCB_MAX_KERNEL_VOLUME && offsets && n_out >= 0);
  PCB_ARG(capacity > 0 && (capacity & (capacity - 1)) == 0);
  if (n_out == 0) return PCB_OK;
  PCB_ARG(out_keys && table_keys && table_vals && tbl);
  Offsets o;
  for (int k = 0; k < K; ++k) for (int d = 0; d < 3; ++d) o.v[k][d] = offsets[k * 3 + d];
  dim3 grid(blocks_for(n_out, 256), K);
  kernel_map_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(out_keys, n_out, table_keys, table_vals, (uint64_t)capacity - 1, o, tbl);
  return check_launch("kernel_map_kernel");
}

extern "C" int pcb_kernel_map_count(const int32_t* tbl, int K, int64_t n_out, int64_t* counts, void* stream) {
  PCB_ARG(K >= 1 && counts);
  cudaStream_t st = (cudaStream_t)stream;
  PCB_CUDA(cudaMemsetAsync(counts, 0, K * sizeof(int64_t), st));
  if (n_out == 0) return PCB_OK;
  dim3 grid(blocks_for(n_out, 256), K);
  map_count_kernel<<<grid, 256, 0, st>>>(tbl, n_out, (unsigned long long*)counts);
  return check_launch("map_count_kernel");
}

extern "C" size_t pcb_conv_tile_order_ws_bytes(int64_t n_out) {
  return layout_bytes(sort_layout, n_out < 1 ? 1 : n_out);
}

extern "C" int pcb_conv_tile_order(const int32_t* tbl, int64_t tbl_stride, int K, int64_t n_out, int64_t window, int32_t* perm, void* ws,
                                   size_t ws_bytes, void* stream) {
  PCB_ARG(K >= 1 && K <= PCB_MAX_KERNEL_VOLUME && n_out >= 0 && n_out < (1ll << 31) && window >= 128 && window % 128 == 0);
  if (n_out == 0) return PCB_OK;
  Carve c{(char*)ws};
  SortWs w = sort_layout(c, n_out);
  PCB_ARG(tbl && perm && tbl_stride >= n_out && ws && ws_bytes >= c.used);
  w.sidx = perm;                                   // the sorted payloads are the order
  cudaStream_t st = (cudaStream_t)stream;
  tile_order_key_kernel<<<blocks_for(n_out, 256), 256, 0, st>>>(tbl, tbl_stride, K, n_out, window, w.k, w.idx);
  if (int e = check_launch("tile_order_key_kernel")) return e;
  int end_bit = 32;                                // the mask bits and as many window bits as there are windows
  while (end_bit < 64 && ((n_out - 1) / window) >> (end_bit - 32)) ++end_bit;
  return sort_keys(n_out, w, end_bit, st);
}
