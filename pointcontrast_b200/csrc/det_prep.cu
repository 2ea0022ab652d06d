// VoteNet detection preprocessing on the GPU (include/pcb200.h "VoteNet detection preprocessing"): the per-vertex work of one ScanNet
// scene (`load_scannet_data.py` `export`) and the ground-truth votes of a batch of SUN RGB-D scenes (`sunrgbd_data.py`
// `extract_sunrgbd_data`).  Every arithmetic operation the original does in numpy is one explicitly rounded operation here.
#include "common.cuh"
#include "sort.cuh"

using namespace pcb;

namespace {

constexpr int THREADS = 256;
constexpr uint64_t SIGN = 1ull << 63;

// ---------------------------------------------------------------------------------------------------------------- ScanNet

struct ScannetWs {
  SortWs sort;                  // the vertices' segment ids, sorted with their vertex index
  RunsWs runs;                  // distinct segments (runs) and the hashed segment id -> run table
  int32_t* lab_ord;             // per run: the last label write to it (ordinal), -1 if none
  int32_t* ins_ord;             // per run: the last instance write to it, -1 if none
  uint32_t* lo;                 // per bounds slot and axis: Ord<float> keys of the minimum / maximum, and a NaN flag
  uint32_t* hi;
  uint32_t* nan;
  int32_t* count;               // per bounds slot: vertices
  int32_t* row_owner;           // per box row: the last object (dict index) that writes it
};

ScannetWs scannet_layout(Carve& c, int64_t V, int64_t n_obj, int64_t n_rows) {
  ScannetWs w;
  w.sort = sort_layout(c, V);
  w.runs = runs_layout(c, V, true);
  w.lab_ord = c.take<int32_t>(V);
  w.ins_ord = c.take<int32_t>(V);
  w.lo = c.take<uint32_t>((n_obj + 1) * 3);
  w.hi = c.take<uint32_t>((n_obj + 1) * 3);
  w.nan = c.take<uint32_t>((n_obj + 1) * 3);
  w.count = c.take<int32_t>(n_obj + 1);
  w.row_owner = c.take<int32_t>(n_rows);
  return w;
}

// int64 segment ids as unsigned keys in the same order (sign bit flipped); the host rejects INT64_MAX, whose key is KEY_EMPTY
__device__ __forceinline__ uint64_t seg_key(int64_t s) { return (uint64_t)s ^ SIGN; }

__global__ void seg_keys_kernel(const int64_t* __restrict__ seg, int64_t V, uint64_t* __restrict__ k, int32_t* __restrict__ idx) {
  pdl_wait();
  pdl_trigger();
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= V) return;
  k[i] = seg_key(seg[i]);
  idx[i] = (int32_t)i;
}

// Label writes are ordinals [0, n_lab), instance writes [n_lab, n_lab + n_ins); the last write to a segment wins (`label_ids[verts] =
// label_id` in list order).  A write to a segment no vertex has is the original's KeyError: status[0] = its lowest ordinal.
__global__ void seg_writes_kernel(const int64_t* __restrict__ lab_seg, int64_t n_lab, const int64_t* __restrict__ ins_seg, int64_t n_ins,
                                  const uint64_t* __restrict__ tk, const int32_t* __restrict__ tv, uint64_t mask, int32_t* lab_ord,
                                  int32_t* ins_ord, int32_t* status) {
  pdl_wait();
  pdl_trigger();
  const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (k >= n_lab + n_ins) return;
  const bool lab = k < n_lab;
  const int64_t s = lab ? lab_seg[k] : ins_seg[k - n_lab];
  const int run = hash_lookup(tk, tv, mask, seg_key(s));
  if (run < 0) { atomicMin(status, (int32_t)k); return; }
  if (lab) atomicMax(lab_ord + run, (int32_t)k);
  else atomicMax(ins_ord + run, (int32_t)(k - n_lab));
}

// One thread per sorted vertex: the labels of its segment, the aligned vertex and its instance's bounds.  Alignment is `np.dot([x y z 1],
// M^T)` with one rounding per operation in k order; the fp32 store rounds once more.  Bounds slot 0 collects the vertices of instance id 0
// (unannotated, and an object whose id is 0), slot d + 1 those of object d.
__global__ void scannet_vertex_kernel(const float* __restrict__ vin, const double* __restrict__ M, int64_t V, const int32_t* __restrict__ sidx,
                                      const int32_t* __restrict__ rank, const int32_t* __restrict__ lab_ord, const int32_t* __restrict__ ins_ord,
                                      const uint32_t* __restrict__ lab_val, const int32_t* __restrict__ ins_obj,
                                      const uint32_t* __restrict__ obj_id, float* __restrict__ vout, uint32_t* __restrict__ sem,
                                      uint32_t* __restrict__ ins, uint32_t* lo, uint32_t* hi, uint32_t* nan, int32_t* count) {
  pdl_wait();
  pdl_trigger();
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= V) return;
  const int64_t v = sidx[i];
  const int run = rank[i] - 1;
  const int lo_k = lab_ord[run], io_k = ins_ord[run];
  sem[v] = lo_k >= 0 ? lab_val[lo_k] : 0u;
  const int d = io_k >= 0 ? ins_obj[io_k] : -1;
  const uint32_t id = d >= 0 ? obj_id[d] : 0u;
  ins[v] = id;
  const int slot = id == 0u ? 0 : d + 1;
  const double p[3] = {(double)vin[v * 6 + 0], (double)vin[v * 6 + 1], (double)vin[v * 6 + 2]};
  float a[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    double acc = __dmul_rn(p[0], M[r * 4 + 0]);
    acc = __dadd_rn(acc, __dmul_rn(p[1], M[r * 4 + 1]));
    acc = __dadd_rn(acc, __dmul_rn(p[2], M[r * 4 + 2]));
    acc = __dadd_rn(acc, M[r * 4 + 3]);                     // 1.0 * M[r][3] is exact
    a[r] = __double2float_rn(acc);
    vout[v * 6 + r] = a[r];
    if (isnan(a[r])) atomicOr(nan + slot * 3 + r, 1u);
    else {
      atomicMin(lo + slot * 3 + r, Ord<float>::key(a[r]));
      atomicMax(hi + slot * 3 + r, Ord<float>::key(a[r]));
    }
  }
#pragma unroll
  for (int c = 3; c < 6; ++c) vout[v * 6 + c] = vin[v * 6 + c];
  atomicAdd(count + slot, 1);
}

// One thread per object (dict index d): an object with vertices claims its box row (the last such object in dict order owns it), or, with no row (`obj_id - 1` outside the box array), sets status[1].
__global__ void scannet_object_kernel(const int64_t* __restrict__ first_seg, const uint32_t* __restrict__ obj_id,
                                      const int32_t* __restrict__ obj_row, int64_t n_obj, const uint64_t* __restrict__ tk,
                                      const int32_t* __restrict__ tv, uint64_t mask, const int32_t* __restrict__ count,
                                      int32_t* row_owner, int32_t* status) {
  pdl_wait();
  pdl_trigger();
  const int64_t d = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (d >= n_obj) return;
  if (hash_lookup(tk, tv, mask, seg_key(first_seg[d])) < 0) return;       // an unknown segment: status[0] is set
  const int slot = obj_id[d] == 0u ? 0 : (int)d + 1;
  if (count[slot] == 0) return;
  if (obj_row[d] < 0) { atomicMin(status + 1, (int32_t)d); return; }
  atomicMax(row_owner + obj_row[d], (int32_t)d);
}

// One thread per box row: (min + max) / 2 and max - min in fp32, then `object_id_to_label_id` = sem at the lowest vertex of the owner's
// first segment; a row no object owns stays zero.
__global__ void scannet_box_kernel(const int32_t* __restrict__ row_owner, int64_t n_rows, const int64_t* __restrict__ first_seg,
                                   const uint32_t* __restrict__ obj_id, const uint64_t* __restrict__ tk, const int32_t* __restrict__ tv,
                                   uint64_t mask, const int32_t* __restrict__ run_start, const int32_t* __restrict__ sidx,
                                   const uint32_t* __restrict__ sem, const uint32_t* __restrict__ lo, const uint32_t* __restrict__ hi,
                                   const uint32_t* __restrict__ nan, double* __restrict__ bbox) {
  pdl_wait();
  pdl_trigger();
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  double* out = bbox + r * 7;
  const int d = row_owner[r];
  if (d < 0) {
    for (int c = 0; c < 7; ++c) out[c] = 0.0;
    return;
  }
  const int slot = obj_id[d] == 0u ? 0 : d + 1;
  for (int c = 0; c < 3; ++c) {
    float mn = Ord<float>::val(lo[slot * 3 + c]), mx = Ord<float>::val(hi[slot * 3 + c]);
    if (nan[slot * 3 + c]) mn = mx = __uint_as_float(0x7fc00000u);
    out[c] = (double)__fdiv_rn(__fadd_rn(mn, mx), 2.f);
    out[3 + c] = (double)__fsub_rn(mx, mn);
  }
  const int run = hash_lookup(tk, tv, mask, seg_key(first_seg[d]));
  out[6] = (double)sem[sidx[run_start[run]]];
}

int scannet_checks(const float* vin, const double* M, int64_t V, const int64_t* seg, int64_t n_lab, int64_t n_ins, int64_t n_obj,
                   int64_t n_rows, float* vout, uint32_t* sem, uint32_t* ins, int32_t* status) {
  PCB_ARG(V >= 1 && V < (1ll << 31) && n_lab >= 0 && n_ins >= 0 && n_lab + n_ins < (1ll << 30) && n_obj >= 0 && n_obj < (1ll << 30));
  PCB_ARG(n_rows >= 0 && n_rows < (1ll << 31));
  PCB_ARG(vin && M && seg && vout && sem && ins && status);
  return PCB_OK;
}

// ---------------------------------------------------------------------------------------------------------------- SUN RGB-D

// One thread per point, its scene's boxes in file order.  Not det_eval.cu's points_in_box_kernel: that one counts fp32 points in
// full-size boxes rotated by roty in camera coordinates; this one needs fp64 upright-depth points, half sizes, rotz and the vote slots, and
// a shared kernel would branch on its caller throughout.
//
// box row: cx, cy, cz, l, w, h, c, s with c = cos(-heading), s = sin(-heading) (numpy's, from the host).  Inside is |u| <= (l, w, h) for
// u = rotz(-heading)^T (p - centroid): u_x = c dx + s dy, u_y = c dy - s dx, u_z = dz, each product and sum rounded once.  A box whose
// l, w or h is not > 0, or with a non-finite value, is skipped (Qhull raises on it; the original's except skips it).
__global__ void sunrgbd_votes_kernel(const double* __restrict__ pts, int ld, const int64_t* __restrict__ pt_off,
                                     const double* __restrict__ boxes, const int64_t* __restrict__ box_off, int64_t B, int64_t N,
                                     double* __restrict__ votes) {
  pdl_wait();
  pdl_trigger();
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= N) return;
  int64_t lo = 0, hi = B;                                  // scene b: pt_off[b] <= i < pt_off[b + 1]
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (pt_off[mid] <= i) lo = mid; else hi = mid;
  }
  const double px = pts[i * ld], py = pts[i * ld + 1], pz = pts[i * ld + 2];
  double v[10];
#pragma unroll
  for (int c = 0; c < 10; ++c) v[c] = 0.0;
  int idx = 0;
  for (int64_t k = box_off[lo]; k < box_off[lo + 1]; ++k) {
    const double* b = boxes + k * 8;
    bool ok = b[3] > 0.0 && b[4] > 0.0 && b[5] > 0.0;
#pragma unroll
    for (int c = 0; c < 8; ++c) ok = ok && isfinite(b[c]);
    if (!ok) continue;
    const double dx = __dsub_rn(px, b[0]), dy = __dsub_rn(py, b[1]), dz = __dsub_rn(pz, b[2]);
    const double ux = __dadd_rn(__dmul_rn(b[6], dx), __dmul_rn(b[7], dy));
    const double uy = __dsub_rn(__dmul_rn(b[6], dy), __dmul_rn(b[7], dx));
    if (!(fabs(ux) <= b[3] && fabs(uy) <= b[4] && fabs(dz) <= b[5])) continue;
    const double vx = __dsub_rn(b[0], px), vy = __dsub_rn(b[1], py), vz = __dsub_rn(b[2], pz);
    v[0] = 1.0;
#pragma unroll
    for (int s = 0; s < 3; ++s)                            // slot idx; the first box also fills slots 1 and 2
      if (s == idx || idx == 0) { v[1 + 3 * s] = vx; v[2 + 3 * s] = vy; v[3 + 3 * s] = vz; }
    idx = min(2, idx + 1);
  }
#pragma unroll
  for (int c = 0; c < 10; ++c) votes[i * 10 + c] = v[c];
}

}  // namespace

extern "C" {

size_t pcb_scannet_annotate_ws_bytes(int64_t V, int64_t n_obj, int64_t n_rows) {
  return layout_bytes(scannet_layout, V, n_obj, n_rows);
}

int pcb_scannet_annotate(const float* vin, const double* align, int64_t V, const int64_t* seg, const int64_t* lab_seg,
                         const uint32_t* lab_val, int64_t n_lab, const int64_t* ins_seg, const int32_t* ins_obj, int64_t n_ins,
                         const uint32_t* obj_id, const int64_t* first_seg, const int32_t* obj_row, int64_t n_obj, int64_t n_rows,
                         float* vout, uint32_t* sem, uint32_t* ins, double* bbox, int32_t* status, void* ws, size_t ws_bytes,
                         void* stream) {
  if (int e = scannet_checks(vin, align, V, seg, n_lab, n_ins, n_obj, n_rows, vout, sem, ins, status)) return e;
  PCB_ARG((n_lab == 0 || (lab_seg && lab_val)) && (n_ins == 0 || (ins_seg && ins_obj)) && (n_obj == 0 || (obj_id && first_seg && obj_row)));
  PCB_ARG(n_rows == 0 || bbox);
  PCB_ARG(ws && ws_bytes >= pcb_scannet_annotate_ws_bytes(V, n_obj, n_rows));
  cudaStream_t st = (cudaStream_t)stream;
  Carve c{(char*)ws};
  const ScannetWs w = scannet_layout(c, V, n_obj, n_rows);
  const uint64_t mask = (uint64_t)w.runs.tcap - 1;
  PCB_CUDA(cudaMemsetAsync(status, 0x7f, 2 * sizeof(int32_t), st));     // 0x7f7f7f7f: none
  PCB_CUDA(cudaMemsetAsync(w.lab_ord, 0xFF, (size_t)V * sizeof(int32_t), st));
  PCB_CUDA(cudaMemsetAsync(w.ins_ord, 0xFF, (size_t)V * sizeof(int32_t), st));
  PCB_CUDA(cudaMemsetAsync(w.lo, 0xFF, (size_t)(n_obj + 1) * 3 * sizeof(uint32_t), st));
  PCB_CUDA(cudaMemsetAsync(w.hi, 0, (size_t)(n_obj + 1) * 3 * sizeof(uint32_t), st));
  PCB_CUDA(cudaMemsetAsync(w.nan, 0, (size_t)(n_obj + 1) * 3 * sizeof(uint32_t), st));
  PCB_CUDA(cudaMemsetAsync(w.count, 0, (size_t)(n_obj + 1) * sizeof(int32_t), st));
  if (n_rows) PCB_CUDA(cudaMemsetAsync(w.row_owner, 0xFF, (size_t)n_rows * sizeof(int32_t), st));
  seg_keys_kernel<<<blocks_for(V, THREADS), THREADS, 0, st>>>(seg, V, w.sort.k, w.sort.idx);
  if (int e = check_launch("seg_keys_kernel")) return e;
  if (int e = sort_runs(V, w.sort, 64, st)) return e;
  if (int e = find_runs(V, w.sort, w.runs, st)) return e;
  if (n_lab + n_ins) {
    launch_kernel(seg_writes_kernel, blocks_for(n_lab + n_ins, THREADS), THREADS, 0, st, lab_seg, n_lab, ins_seg, n_ins,
                  (const uint64_t*)w.runs.tk, (const int32_t*)w.runs.tv, mask, w.lab_ord, w.ins_ord, status);
    if (int e = check_launch("seg_writes_kernel")) return e;
  }
  launch_kernel(scannet_vertex_kernel, blocks_for(V, THREADS), THREADS, 0, st, vin, align, V, (const int32_t*)w.sort.sidx,
                (const int32_t*)w.sort.rank, (const int32_t*)w.lab_ord, (const int32_t*)w.ins_ord, lab_val, ins_obj, obj_id, vout, sem, ins,
                w.lo, w.hi, w.nan, w.count);
  if (int e = check_launch("scannet_vertex_kernel")) return e;
  if (n_obj) {
    launch_kernel(scannet_object_kernel, blocks_for(n_obj, THREADS), THREADS, 0, st, first_seg, obj_id, obj_row, n_obj,
                  (const uint64_t*)w.runs.tk, (const int32_t*)w.runs.tv, mask, (const int32_t*)w.count, w.row_owner, status);
    if (int e = check_launch("scannet_object_kernel")) return e;
  }
  if (n_rows) {
    launch_kernel(scannet_box_kernel, blocks_for(n_rows, THREADS), THREADS, 0, st, (const int32_t*)w.row_owner, n_rows, first_seg, obj_id,
                  (const uint64_t*)w.runs.tk, (const int32_t*)w.runs.tv, mask, (const int32_t*)w.runs.start, (const int32_t*)w.sort.sidx,
                  (const uint32_t*)sem, (const uint32_t*)w.lo, (const uint32_t*)w.hi, (const uint32_t*)w.nan, bbox);
    if (int e = check_launch("scannet_box_kernel")) return e;
  }
  return PCB_OK;
}

int pcb_sunrgbd_votes(const double* pts, int32_t ld, const int64_t* pt_off_host, const int64_t* pt_off, const double* boxes,
                      const int64_t* box_off_host, const int64_t* box_off, int64_t B, double* votes, void* stream) {
  PCB_ARG(B >= 1 && ld >= 3 && pt_off_host && box_off_host && pt_off && box_off);
  PCB_ARG(pt_off_host[0] == 0 && box_off_host[0] == 0);
  for (int64_t b = 0; b < B; ++b) PCB_ARG(pt_off_host[b + 1] >= pt_off_host[b] && box_off_host[b + 1] >= box_off_host[b]);
  const int64_t N = pt_off_host[B];
  PCB_ARG(N < (1ll << 40) && (N == 0 || (pts && votes)) && (box_off_host[B] == 0 || boxes));
  if (N == 0) return PCB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  launch_kernel(sunrgbd_votes_kernel, blocks_for(N, THREADS), THREADS, 0, st, pts, (int)ld, pt_off, boxes, box_off, B, N, votes);
  return check_launch("sunrgbd_votes_kernel");
}

}  // extern "C"
