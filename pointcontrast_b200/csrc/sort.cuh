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

}  // namespace pcb
