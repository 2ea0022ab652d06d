// PointNet++ operators of the VoteNet detection downstream (`downstream/votenet_det_new/models/backbone/pointnet2/_ext_src`):
// furthest-point sampling, ball query, three-NN, the gathers (gather_points / group_points), three_interpolate and the adjoints of
// the last three.  Shapes follow `_ext`: xyz fp32 [B, N, 3], features fp32 [B, C, N] (channels first), indices int32.
//
// Distance arithmetic is written with __fmul_rn / __fadd_rn / __fsub_rn in the reference's operand order (no FMA contraction), so every
// index result is reproducible bit for bit in numpy fp32 (oracle/pointnet2_cpu.py) and by the reference kernels compiled with
// --fmad=false.  The backward passes gather through a per-scene CSR transpose of the index tensor (stable radix sort: each source
// point's readers in ascending output position) and sum in that fixed order in fp64: no atomics, run-to-run bit-identical.
#include <algorithm>
#include <cub/cub.cuh>
#include "common.cuh"

using namespace pcb;

namespace {

constexpr int64_t LIM = 1ll << 31;

__device__ __forceinline__ float dist2_rn(float ax, float ay, float az, float bx, float by, float bz) {
  const float dx = __fsub_rn(ax, bx), dy = __fsub_rn(ay, by), dz = __fsub_rn(az, bz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// ------------------------------------------------------------------------------------------------ furthest-point sampling
// One thread-block cluster per scene.  CTA r of the cluster owns points [r*per_cta, (r+1)*per_cta); the first FPS_SMEM_PTS of them
// live in shared memory as (x, y, z, running min-distance), the rest (scenes above the on-chip capacity) are read from xyz with their
// running distance in the workspace.  Per iteration every CTA finds its best point as the maximum of the 64-bit key
// (float bits of d) << 32 | (0xFFFFFFFF - k) -- largest distance, then smallest index, whatever the launch shape -- and publishes
// (key, x, y, z) into every peer's shared memory (st.shared::cluster, parity-double-buffered slots); after one cluster barrier each CTA
// reduces the <= 8 candidates itself.  A running distance < 0 marks a point that is never a candidate (|p|^2 <= 1e-3).
constexpr int FPS_THREADS = 512;
constexpr int FPS_MAX_CLUSTER = 8;
constexpr int FPS_PTS_PER_CTA = 1024;   // cluster size = ceil(N / this), at most FPS_MAX_CLUSTER
constexpr int FPS_SMEM_PTS = 12288;     // 192 KB of (x, y, z, d) per CTA
constexpr float FPS_INIT = 1e10f;       // `sampling.cpp:80`

struct __align__(16) FpsSlot { uint32_t klo, khi; float x, y, z, pad[3]; };

__device__ __forceinline__ uint32_t cluster_rank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void st_peer(const void* local, uint32_t peer, uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t e) {
  uint32_t addr = (uint32_t)__cvta_generic_to_shared(local), remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(addr), "r"(peer));
  asm volatile("st.shared::cluster.v4.u32 [%0], {%1, %2, %3, %4};" :: "r"(remote), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
  asm volatile("st.shared::cluster.u32 [%0], %1;" :: "r"(remote + 16), "r"(e) : "memory");
}
__device__ __forceinline__ unsigned long long fps_key(float d, int64_t k) {
  return ((unsigned long long)__float_as_uint(d) << 32) | (0xFFFFFFFFu - (uint32_t)k);
}

// Scene b is rows [offsets[b], offsets[b+1]) of xyz (ragged batches) or, with offsets == NULL, rows [b*N, (b+1)*N).  Indices are
// scene-local.  The selection does not depend on the cluster shape (per-point running distances, index-unique keys), so a ragged
// launch sized for its largest scene returns, for every scene, what a launch for that scene alone returns.  A ragged scene that is
// empty, ends past `total` rows or exceeds the cluster's capacity cs * per_cta gets -1 in every slot.
__global__ void __launch_bounds__(FPS_THREADS, 1) fps_kernel(const float* __restrict__ xyz, const int64_t* __restrict__ offsets, int64_t N,
                                                             int64_t total, int64_t npoint, int cs, int64_t per_cta, float* __restrict__ temp,
                                                             int32_t* __restrict__ out) {
  extern __shared__ float4 sp[];
  __shared__ FpsSlot slots[2][FPS_MAX_CLUSTER];
  __shared__ unsigned long long wbest[FPS_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t rank = cluster_rank();
  const int64_t b = blockIdx.x / cs;
  out += b * npoint;
  int64_t begin = b * N;
  if (offsets) {                                   // uniform over the cluster: either every CTA returns here or none does
    begin = offsets[b];
    N = offsets[b + 1] - begin;
    if (begin < 0 || N < 1 || begin + N > total || N > cs * per_cta) {
      if (rank == 0)
        for (int64_t j = tid; j < npoint; j += FPS_THREADS) out[j] = -1;
      return;
    }
  }
  xyz += begin * 3;
  const int64_t lo = rank * per_cta, n_loc = max((int64_t)0, min(N, lo + per_cta) - lo), n_sm = min(n_loc, (int64_t)FPS_SMEM_PTS);
  float* tg = temp ? temp + begin + lo : nullptr;
  for (int64_t i = tid; i < n_loc; i += FPS_THREADS) {
    const float x = xyz[3 * (lo + i)], y = xyz[3 * (lo + i) + 1], z = xyz[3 * (lo + i) + 2];
    const float mag = __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
    const float d = ((double)mag <= 1e-3) ? -1.f : FPS_INIT;      // float against the double 1e-3, as the reference compares
    if (i < n_sm) sp[i] = make_float4(x, y, z, d); else tg[i - n_sm] = d;
  }
  float sx = xyz[0], sy = xyz[1], sz = xyz[2];
  if (rank == 0 && tid == 0) out[0] = 0;
  cluster_sync_all();                              // every peer's shared memory is live before the first remote store
  for (int64_t j = 1; j < npoint; ++j) {
    unsigned long long best = 0;
    for (int64_t i = tid; i < n_sm; i += FPS_THREADS) {
      const float4 p = sp[i];
      if (p.w < 0.f) continue;
      const float d = fminf(dist2_rn(p.x, p.y, p.z, sx, sy, sz), p.w);
      sp[i].w = d;
      best = max(best, fps_key(d, lo + i));
    }
    for (int64_t i = n_sm + tid; i < n_loc; i += FPS_THREADS) {
      const float t = tg[i - n_sm];
      if (t < 0.f) continue;
      const float d = fminf(dist2_rn(xyz[3 * (lo + i)], xyz[3 * (lo + i) + 1], xyz[3 * (lo + i) + 2], sx, sy, sz), t);
      tg[i - n_sm] = d;
      best = max(best, fps_key(d, lo + i));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) best = max(best, __shfl_xor_sync(0xFFFFFFFFu, best, o));
    if (lane == 0) wbest[warp] = best;
    __syncthreads();
    FpsSlot* slot = &slots[j & 1][rank];
    if (warp == 0) {
      unsigned long long v = lane < FPS_THREADS / 32 ? wbest[lane] : 0ull;
#pragma unroll
      for (int o = 16; o; o >>= 1) v = max(v, __shfl_xor_sync(0xFFFFFFFFu, v, o));
      if (lane < cs) {
        float cx = 0.f, cy = 0.f, cz = 0.f;
        if (v) {
          const int64_t k = (int64_t)(0xFFFFFFFFu - (uint32_t)v) - lo;
          if (k < n_sm) { const float4 p = sp[k]; cx = p.x; cy = p.y; cz = p.z; }
          else { cx = xyz[3 * (lo + k)]; cy = xyz[3 * (lo + k) + 1]; cz = xyz[3 * (lo + k) + 2]; }
        }
        st_peer(slot, lane, (uint32_t)v, (uint32_t)(v >> 32), __float_as_uint(cx), __float_as_uint(cy), __float_as_uint(cz));
      }
    }
    cluster_sync_all();
    unsigned long long w = 0;
    for (int r = 0; r < cs; ++r) {
      const FpsSlot& s = slots[j & 1][r];
      const unsigned long long k = ((unsigned long long)s.khi << 32) | s.klo;
      if (k > w) { w = k; sx = s.x; sy = s.y; sz = s.z; }
    }
    int32_t sel = 0;                                 // no candidate left anywhere: the reference's besti stays 0
    if (w) sel = (int32_t)(0xFFFFFFFFu - (uint32_t)w);
    else { sx = xyz[0]; sy = xyz[1]; sz = xyz[2]; }
    if (rank == 0 && tid == 0) out[j] = sel;
  }
}

int fps_cluster(int64_t N) { return (int)std::min<int64_t>(FPS_MAX_CLUSTER, std::max<int64_t>(1, (N + FPS_PTS_PER_CTA - 1) / FPS_PTS_PER_CTA)); }
bool fps_overflows(int64_t N) { const int cs = fps_cluster(N); return (N + cs - 1) / cs > FPS_SMEM_PTS; }

// ------------------------------------------------------------------------------------------------ ball query
// One warp per query, 8 queries (of one scene) per CTA sharing shared-memory tiles of xyz.  Candidates are tested 32 at a time in
// ascending k; a ballot + popc prefix places the hits in order, and the warp stops at nsample hits.
constexpr int BQ_WARPS = 8;
constexpr int BQ_TILE = 2048;

__global__ void __launch_bounds__(BQ_WARPS * 32) ball_query_kernel(const float* __restrict__ new_xyz, const float* __restrict__ xyz, int64_t M,
                                                                   int64_t N, int64_t qblocks, float r2, int nsample, int32_t* __restrict__ idx) {
  __shared__ float tile[BQ_TILE * 3];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t b = blockIdx.x / qblocks, q = (blockIdx.x % qblocks) * BQ_WARPS + warp;
  const bool active = q < M;
  xyz += b * N * 3;
  float qx = 0.f, qy = 0.f, qz = 0.f;
  if (active) { const float* p = new_xyz + (b * M + q) * 3; qx = p[0]; qy = p[1]; qz = p[2]; }
  int32_t* row = idx + (b * M + q) * nsample;
  int cnt = 0, first = 0;
  bool done = !active;
  for (int64_t base = 0; base < N; base += BQ_TILE) {
    if (!__syncthreads_or(!done)) break;           // also: everyone is done reading the previous tile
    const int nt = (int)min((int64_t)BQ_TILE, N - base);
    const float* src = xyz + 3 * base;
    for (int i = tid; i < 3 * nt; i += BQ_WARPS * 32) tile[i] = src[i];
    __syncthreads();
    if (done) continue;
    for (int t = 0; t < nt; t += 32) {
      const int k = t + lane;
      const bool hit = k < nt && dist2_rn(qx, qy, qz, tile[3 * k], tile[3 * k + 1], tile[3 * k + 2]) < r2;   // d from new - p
      const unsigned m = __ballot_sync(0xFFFFFFFFu, hit);
      if (!m) continue;
      if (cnt == 0) first = (int)(base + t) + __ffs(m) - 1;
      const int pos = cnt + __popc(m & ((1u << lane) - 1));
      if (hit && pos < nsample) row[pos] = (int32_t)(base + k);
      cnt += __popc(m);
      if (cnt >= nsample) { done = true; break; }
    }
  }
  if (active)
    for (int s = min(cnt, nsample) + lane; s < nsample; s += 32) row[s] = first;   // no hit: first stays 0 (`ball_query.cpp:25` zeros)
}

// ------------------------------------------------------------------------------------------------ three-NN
// One thread per unknown point, known points tiled in shared memory, scanned in ascending k with strict < insertion.
constexpr int TN_THREADS = 256;
constexpr int TN_TILE = 2048;

__global__ void __launch_bounds__(TN_THREADS) three_nn_kernel(const float* __restrict__ unknown, const float* __restrict__ known, int64_t n, int64_t m,
                                                              int64_t nblocks, float* __restrict__ dist2, int32_t* __restrict__ idx) {
  __shared__ float tile[TN_TILE * 3];
  const int tid = threadIdx.x;
  const int64_t b = blockIdx.x / nblocks, j = (blockIdx.x % nblocks) * TN_THREADS + tid;
  const bool active = j < n;
  known += b * m * 3;
  float ux = 0.f, uy = 0.f, uz = 0.f;
  if (active) { const float* p = unknown + (b * n + j) * 3; ux = p[0]; uy = p[1]; uz = p[2]; }
  float b1 = INFINITY, b2 = INFINITY, b3 = INFINITY;   // the reference's double 1e40, stored as float: inf
  int32_t i1 = 0, i2 = 0, i3 = 0;
  for (int64_t base = 0; base < m; base += TN_TILE) {
    const int nt = (int)min((int64_t)TN_TILE, m - base);
    __syncthreads();
    for (int i = tid; i < 3 * nt; i += TN_THREADS) tile[i] = known[3 * base + i];
    __syncthreads();
    if (!active) continue;
    for (int t = 0; t < nt; ++t) {
      const float d = dist2_rn(ux, uy, uz, tile[3 * t], tile[3 * t + 1], tile[3 * t + 2]);
      const int32_t k = (int32_t)(base + t);
      if (d < b1) { b3 = b2; i3 = i2; b2 = b1; i2 = i1; b1 = d; i1 = k; }
      else if (d < b2) { b3 = b2; i3 = i2; b2 = d; i2 = k; }
      else if (d < b3) { b3 = d; i3 = k; }
    }
  }
  if (!active) return;
  float* d = dist2 + (b * n + j) * 3;
  int32_t* o = idx + (b * n + j) * 3;
  d[0] = b1; d[1] = b2; d[2] = b3;
  o[0] = i1; o[1] = i2; o[2] = i3;
}

// ------------------------------------------------------------------------------------------------ gathers
// Thread per (scene, output position), CH channels per thread: index (and weights) read once, writes coalesced along the position.
// An index outside [0, N) reads as 0.
constexpr int G_THREADS = 256;
constexpr int G_CH = 8;

__global__ void __launch_bounds__(G_THREADS) gather_kernel(const float* __restrict__ f, const int32_t* __restrict__ idx, int64_t B, int64_t C, int64_t N,
                                                           int64_t L, float* __restrict__ out) {
  const int64_t p = blockIdx.x * (int64_t)G_THREADS + threadIdx.x;
  if (p >= L) return;
  const int64_t c0 = (int64_t)blockIdx.y * G_CH;
  for (int64_t b = blockIdx.z; b < B; b += gridDim.z) {
    const int32_t a = idx[b * L + p];
    const bool ok = a >= 0 && a < N;
#pragma unroll
    for (int cc = 0; cc < G_CH; ++cc) {
      const int64_t c = c0 + cc;
      if (c < C) out[(b * C + c) * L + p] = ok ? f[(b * C + c) * N + a] : 0.f;
    }
  }
}

__global__ void __launch_bounds__(G_THREADS) interp_kernel(const float* __restrict__ f, const int32_t* __restrict__ idx, const float* __restrict__ w,
                                                           int64_t B, int64_t C, int64_t m, int64_t n, float* __restrict__ out) {
  const int64_t j = blockIdx.x * (int64_t)G_THREADS + threadIdx.x;
  if (j >= n) return;
  const int64_t c0 = (int64_t)blockIdx.y * G_CH;
  for (int64_t b = blockIdx.z; b < B; b += gridDim.z) {
    const int32_t* ip = idx + (b * n + j) * 3;
    const float* wp = w + (b * n + j) * 3;
    const int32_t a1 = ip[0], a2 = ip[1], a3 = ip[2];
    const float w1 = wp[0], w2 = wp[1], w3 = wp[2];
    const bool ok1 = a1 >= 0 && a1 < m, ok2 = a2 >= 0 && a2 < m, ok3 = a3 >= 0 && a3 < m;
#pragma unroll
    for (int cc = 0; cc < G_CH; ++cc) {
      const int64_t c = c0 + cc;
      if (c >= C) break;
      const float* row = f + (b * C + c) * m;
      const float v1 = ok1 ? row[a1] : 0.f, v2 = ok2 ? row[a2] : 0.f, v3 = ok3 ? row[a3] : 0.f;
      out[(b * C + c) * n + j] = __fadd_rn(__fadd_rn(__fmul_rn(v1, w1), __fmul_rn(v2, w2)), __fmul_rn(v3, w3));   // `interpolate_gpu.cu:103`
    }
  }
}

// ------------------------------------------------------------------------------------------------ adjoints (CSR transpose)
// Readers: position p in [0, L) of scene b reads source point idx[b, p].  key = b * N + idx (B * N for an index outside [0, N): read by
// nobody), value = p; a stable radix sort by key lists every source point's readers in ascending p.
__global__ void csr_key_kernel(const int32_t* __restrict__ idx, int64_t N, int64_t L, int64_t total, uint32_t sentinel, uint32_t* __restrict__ keys,
                               int32_t* __restrict__ vals) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int64_t b = i / L;
  const int32_t a = idx[i];
  keys[i] = (a >= 0 && a < N) ? (uint32_t)(b * N + a) : sentinel;
  vals[i] = (int32_t)(i - b * L);
}

// off[t] = first sorted position with key >= t, t in [0, B*N]
__global__ void csr_offsets_kernel(const uint32_t* __restrict__ skeys, int64_t total, int64_t rows, int32_t* __restrict__ off) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t > rows) return;
  int64_t lo = 0, hi = total;
  while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (skeys[mid] < (uint32_t)t) lo = mid + 1; else hi = mid; }
  off[t] = (int32_t)lo;
}

// grad_f[b, c, a] = sum over the readers p of a, ascending: grad_out[b, c, p / R] (* w[b, p]), accumulated in fp64
template <int R>
__global__ void __launch_bounds__(G_THREADS) csr_sum_kernel(const float* __restrict__ g, const float* __restrict__ w, const int32_t* __restrict__ off,
                                                            const int32_t* __restrict__ svals, int64_t B, int64_t C, int64_t N, int64_t L,
                                                            float* __restrict__ grad) {
  const int64_t a = blockIdx.x * (int64_t)G_THREADS + threadIdx.x;
  if (a >= N) return;
  const int64_t c0 = (int64_t)blockIdx.y * G_CH, Lg = L / R;
  for (int64_t b = blockIdx.z; b < B; b += gridDim.z) {
    double acc[G_CH];
#pragma unroll
    for (int cc = 0; cc < G_CH; ++cc) acc[cc] = 0.0;
    const int32_t r0 = off[b * N + a], r1 = off[b * N + a + 1];
    for (int32_t r = r0; r < r1; ++r) {
      const int64_t p = svals[r];
      const double wt = R == 1 ? 1.0 : (double)w[b * L + p];
#pragma unroll
      for (int cc = 0; cc < G_CH; ++cc)
        if (c0 + cc < C) acc[cc] += (double)g[(b * C + c0 + cc) * Lg + p / R] * wt;
    }
#pragma unroll
    for (int cc = 0; cc < G_CH; ++cc)
      if (c0 + cc < C) grad[(b * C + c0 + cc) * N + a] = (float)acc[cc];
  }
}

size_t cub_sort_bytes(int64_t total) {
  size_t s = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, s, (uint32_t*)nullptr, (uint32_t*)nullptr, (int32_t*)nullptr, (int32_t*)nullptr, (int)total);
  return s;
}

dim3 gather_grid(int64_t cols, int64_t C, int64_t B) {
  return dim3((unsigned)((cols + G_THREADS - 1) / G_THREADS), (unsigned)((C + G_CH - 1) / G_CH), (unsigned)std::min<int64_t>(B, 65535));
}

// the CSR transpose of B * L readers of B * N source points: sort keys / values before and after the sort, the offsets, CUB storage
struct CsrWs { uint32_t* keys; uint32_t* skeys; int32_t* vals; int32_t* svals; int32_t* off; void* cub; size_t cub_bytes; };
CsrWs csr_layout(Carve& c, int64_t B, int64_t N, int64_t L) {
  const int64_t total = B * L;
  const size_t cub_bytes = cub_sort_bytes(total);
  return {c.take<uint32_t>(total), c.take<uint32_t>(total), c.take<int32_t>(total), c.take<int32_t>(total), c.take<int32_t>(B * N + 1),
          c.take<char>(cub_bytes), cub_bytes};
}

// readers of every source point: w.off [B*N + 1], w.svals (reader positions, ascending within a source point)
int csr_build(const int32_t* idx, int64_t B, int64_t N, int64_t L, const CsrWs& w, cudaStream_t st) {
  const int64_t total = B * L, rows = B * N;
  size_t cb = w.cub_bytes;
  int end_bit = 1;
  while (end_bit < 32 && ((uint64_t)1 << end_bit) <= (uint64_t)rows) ++end_bit;     // keys are <= rows (the sentinel)
  if (total > 0) {
    csr_key_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(idx, N, L, total, (uint32_t)rows, w.keys, w.vals);
    if (int e = check_launch("csr_key_kernel")) return e;
    PCB_CUDA(cub::DeviceRadixSort::SortPairs(w.cub, cb, w.keys, w.skeys, w.vals, w.svals, (int)total, 0, end_bit, st));
    g_launches.fetch_add(4);
  }
  csr_offsets_kernel<<<(unsigned)((rows + 1 + 255) / 256), 256, 0, st>>>(w.skeys, total, rows, w.off);
  return check_launch("csr_offsets_kernel");
}

// row-major adjoint of a row gather: grad[a, c] = sum over the readers p of row a, ascending p, of g[p, c], in fp64
__global__ void __launch_bounds__(G_THREADS) rows_sum_kernel(const float* __restrict__ g, const int32_t* __restrict__ off,
                                                             const int32_t* __restrict__ svals, int64_t C, int64_t M, float* __restrict__ grad) {
  const int64_t t = blockIdx.x * (int64_t)G_THREADS + threadIdx.x;
  if (t >= M * C) return;
  const int64_t a = t / C, c = t - a * C;
  double acc = 0.0;
  for (int32_t r = off[a]; r < off[a + 1]; ++r) acc += (double)g[(int64_t)svals[r] * C + c];
  grad[t] = (float)acc;
}

int points_grad(const float* g, const int32_t* idx, const float* w, int R, int64_t B, int64_t C, int64_t N, int64_t L, float* grad,
                const CsrWs& ws, cudaStream_t st) {
  if (int e = csr_build(idx, B, N, L, ws, st)) return e;
  if (R == 1) csr_sum_kernel<1><<<gather_grid(N, C, B), G_THREADS, 0, st>>>(g, w, ws.off, ws.svals, B, C, N, L, grad);
  else csr_sum_kernel<3><<<gather_grid(N, C, B), G_THREADS, 0, st>>>(g, w, ws.off, ws.svals, B, C, N, L, grad);
  return check_launch("csr_sum_kernel");
}

}  // namespace

extern "C" size_t pcb_furthest_point_sampling_ws_bytes(int64_t B, int64_t N) {
  return (B > 0 && N > 0 && fps_overflows(N)) ? (size_t)(B * N * 4) : 0;
}

// one cluster per scene, its size chosen from max_n (the scene size, or an upper bound on it for ragged batches)
int fps_launch(const float* xyz, const int64_t* offsets, int64_t B, int64_t N, int64_t total, int64_t max_n, int64_t npoint, int32_t* idx,
               void* ws, cudaStream_t st) {
  const int cs = fps_cluster(max_n);
  const int64_t per_cta = (max_n + cs - 1) / cs;
  const size_t smem = (size_t)std::min<int64_t>(per_cta, FPS_SMEM_PTS) * sizeof(float4);
  PCB_ARG(B * cs < LIM);
  static bool attr_set[64] = {};
  const int dev = current_device();
  if (!attr_set[dev]) {
    PCB_CUDA(cudaFuncSetAttribute(fps_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FPS_SMEM_PTS * (int)sizeof(float4)));
    attr_set[dev] = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(B * cs)); cfg.blockDim = dim3(FPS_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, fps_kernel, xyz, offsets, N, total, npoint, cs, per_cta, fps_overflows(max_n) ? (float*)ws : (float*)nullptr, idx);
  return check_launch("fps_kernel");
}

extern "C" int pcb_furthest_point_sampling(const float* xyz, int64_t B, int64_t N, int64_t npoint, int32_t* idx, void* ws, size_t ws_bytes,
                                           void* stream) {
  PCB_ARG(B >= 0 && B < LIM && N >= 1 && N < LIM && npoint >= 1 && npoint < LIM && B * N < LIM && B * npoint < LIM);
  if (B == 0) return PCB_OK;
  PCB_ARG(xyz && idx && ws_bytes >= pcb_furthest_point_sampling_ws_bytes(B, N) && (ws || !fps_overflows(N)));
  return fps_launch(xyz, nullptr, B, N, B * N, N, npoint, idx, ws, (cudaStream_t)stream);
}

// max_n: an upper bound on every scene's size; no scene is larger than M, so a larger bound counts as M
extern "C" size_t pcb_furthest_point_sampling_ragged_ws_bytes(int64_t B, int64_t M, int64_t max_n) {
  return (B > 0 && M > 0 && max_n > 0 && M < LIM && fps_overflows(std::min(max_n, M))) ? (size_t)(M * 4) : 0;
}

extern "C" int pcb_furthest_point_sampling_ragged(const float* xyz, const int64_t* offsets, int64_t B, int64_t M, int64_t max_n, int64_t npoint,
                                                  int32_t* idx, void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(B >= 1 && B < LIM && M >= B && M < LIM && max_n >= 1 && npoint >= 1 && npoint < LIM && B * npoint < LIM);
  max_n = std::min(max_n, M);
  PCB_ARG(xyz && offsets && idx && ws_bytes >= pcb_furthest_point_sampling_ragged_ws_bytes(B, M, max_n) && (ws || !fps_overflows(max_n)));
  return fps_launch(xyz, offsets, B, 0, M, max_n, npoint, idx, ws, (cudaStream_t)stream);
}

extern "C" int pcb_ball_query(const float* new_xyz, const float* xyz, int64_t B, int64_t M, int64_t N, float radius, int nsample, int32_t* idx,
                              void* stream) {
  PCB_ARG(B >= 0 && M >= 0 && N >= 0 && B < LIM && M < LIM && N < LIM && nsample >= 1 && radius > 0.f);
  const int64_t qblocks = (M + BQ_WARPS - 1) / BQ_WARPS;
  PCB_ARG(B * N < LIM && B * qblocks < LIM);
  if (B == 0 || M == 0) return PCB_OK;
  PCB_ARG(new_xyz && idx && (xyz || N == 0));
  ball_query_kernel<<<(unsigned)(B * qblocks), BQ_WARPS * 32, 0, (cudaStream_t)stream>>>(new_xyz, xyz, M, N, qblocks, radius * radius,
                                                                                          nsample, idx);
  return check_launch("ball_query_kernel");
}

extern "C" int pcb_three_nn(const float* unknown, const float* known, int64_t B, int64_t n, int64_t m, float* dist2, int32_t* idx, void* stream) {
  PCB_ARG(B >= 0 && n >= 0 && m >= 0 && B < LIM && n < LIM && m < LIM && B * n < LIM && B * m < LIM);
  if (B == 0 || n == 0) return PCB_OK;
  PCB_ARG(unknown && dist2 && idx && (known || m == 0));
  const int64_t nblocks = (n + TN_THREADS - 1) / TN_THREADS;
  three_nn_kernel<<<(unsigned)(B * nblocks), TN_THREADS, 0, (cudaStream_t)stream>>>(unknown, known, n, m, nblocks, dist2, idx);
  return check_launch("three_nn_kernel");
}

extern "C" int pcb_gather_points(const float* features, const int32_t* idx, int64_t B, int64_t C, int64_t N, int64_t L, float* out, void* stream) {
  PCB_ARG(B >= 0 && C >= 0 && N >= 0 && L >= 0 && B < LIM && C < LIM && N < LIM && L < LIM && B * L < LIM);
  if (B == 0 || C == 0 || L == 0) return PCB_OK;
  PCB_ARG(idx && out && (features || N == 0));
  gather_kernel<<<gather_grid(L, C, B), G_THREADS, 0, (cudaStream_t)stream>>>(features, idx, B, C, N, L, out);
  return check_launch("gather_kernel");
}

extern "C" int pcb_three_interpolate(const float* features, const int32_t* idx, const float* weight, int64_t B, int64_t C, int64_t m, int64_t n,
                                     float* out, void* stream) {
  PCB_ARG(B >= 0 && C >= 0 && m >= 0 && n >= 0 && B < LIM && C < LIM && m < LIM && n < LIM && B * n * 3 < LIM);
  if (B == 0 || C == 0 || n == 0) return PCB_OK;
  PCB_ARG(idx && weight && out && (features || m == 0));
  interp_kernel<<<gather_grid(n, C, B), G_THREADS, 0, (cudaStream_t)stream>>>(features, idx, weight, B, C, m, n, out);
  return check_launch("interp_kernel");
}

extern "C" size_t pcb_points_grad_ws_bytes(int64_t B, int64_t N, int64_t L) {
  if (B < 0 || N < 0 || L < 0 || B * L >= LIM || B * N >= LIM) return 0;
  return layout_bytes(csr_layout, B, N, L);
}

extern "C" int pcb_gather_points_grad(const float* grad_out, const int32_t* idx, int64_t B, int64_t C, int64_t N, int64_t L, float* grad_features,
                                      void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(B >= 0 && C >= 0 && N >= 0 && L >= 0 && B < LIM && C < LIM && N < LIM && L < LIM && B * L < LIM && B * N < LIM);
  if (B == 0 || C == 0 || N == 0) return PCB_OK;
  Carve c{(char*)ws};
  const CsrWs w = csr_layout(c, B, N, L);
  PCB_ARG(grad_features && ws && ws_bytes >= c.used && ((grad_out && idx) || L == 0));
  return points_grad(grad_out, idx, nullptr, 1, B, C, N, L, grad_features, w, (cudaStream_t)stream);
}

extern "C" int pcb_gather_rows_grad(const float* grad_out, const int32_t* idx, int64_t L, int64_t C, int64_t M, float* grad_rows, void* ws,
                                    size_t ws_bytes, void* stream) {
  PCB_ARG(L >= 0 && C >= 0 && M >= 0 && L < LIM && C < LIM && M < LIM && M * C < (1ll << 40));
  if (C == 0 || M == 0) return PCB_OK;
  Carve c{(char*)ws};
  const CsrWs w = csr_layout(c, 1, M, L);
  PCB_ARG(grad_rows && ws && ws_bytes >= c.used && ((grad_out && idx) || L == 0));
  cudaStream_t st = (cudaStream_t)stream;
  if (int e = csr_build(idx, 1, M, L, w, st)) return e;
  rows_sum_kernel<<<(unsigned)((M * C + G_THREADS - 1) / G_THREADS), G_THREADS, 0, st>>>(grad_out, w.off, w.svals, C, M, grad_rows);
  return check_launch("rows_sum_kernel");
}

extern "C" int pcb_three_interpolate_grad(const float* grad_out, const int32_t* idx, const float* weight, int64_t B, int64_t C, int64_t n, int64_t m,
                                          float* grad_features, void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(B >= 0 && C >= 0 && n >= 0 && m >= 0 && B < LIM && C < LIM && n < LIM && m < LIM && B * n * 3 < LIM && B * m < LIM);
  if (B == 0 || C == 0 || m == 0) return PCB_OK;
  Carve c{(char*)ws};
  const CsrWs w = csr_layout(c, B, m, 3 * n);
  PCB_ARG(grad_features && ws && ws_bytes >= c.used && ((grad_out && idx && weight) || n == 0));
  return points_grad(grad_out, idx, weight, 3, B, C, m, 3 * n, grad_features, w, (cudaStream_t)stream);
}
