// Sort-and-unique pipeline for 64-bit integer keys (voxel.cu), shared by the coordinate manager and the voxelisation entry points:
// stable radix sort of (key, int32 payload) -> head flag where the key changes -> inclusive scan.  After sort_runs, rank[i] - 1 is
// the run (unique key) that sorted position i belongs to.  Not part of the public ABI.
#pragma once
#include "common.cuh"

namespace pcb {

// k / idx: keys and payloads in input order (the caller fills them); sk / sidx: sorted; count / status: one int64 / int32 for the
// caller; cub: temporary storage for the sort and the scans over n items
struct SortWs { uint64_t* k; uint64_t* sk; int32_t* idx; int32_t* sidx; int32_t* flag; int32_t* rank; int64_t* count; int32_t* status;
                void* cub; size_t cub_bytes; };
SortWs sort_layout(Carve& c, int64_t n);

// stable sort of bits [0, end_bit) of the keys
int sort_keys(int64_t n, const SortWs& w, int end_bit, cudaStream_t st);
// sort_keys -> head flags -> inclusive scan (rank)
int sort_runs(int64_t n, const SortWs& w, int end_bit, cudaStream_t st);

// The runs of sort_runs as a lookup structure: run r is sorted positions [start[r], end[r]) with key key[r]; with `hashed`, an
// open-addressing table (common.cuh hash_lookup) maps a key to its run, tcap slots (a power of two >= 2 n, at least 16).
struct RunsWs { uint64_t* key; int32_t* start; int32_t* end; int64_t tcap; uint64_t* tk; int32_t* tv; };
RunsWs runs_layout(Carve& c, int64_t n, bool hashed);
// after sort_runs over n >= 1 keys: the run bounds, *w.count = the number of runs, and the table if r.tk is set
int find_runs(int64_t n, const SortWs& w, const RunsWs& r, cudaStream_t st);

// Integer cells of a uniform grid, |index| < VB per axis, packed 21 bits per axis so that unsigned key order is (x, y, z) order.
constexpr int VB = 1 << 20;
__host__ __device__ __forceinline__ uint64_t cell_key(int cx, int cy, int cz) {
  return ((uint64_t)(cx + VB) << 42) | ((uint64_t)(cy + VB) << 21) | (uint64_t)(cz + VB);
}

}  // namespace pcb
