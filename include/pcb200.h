/*
 * pcb200.h -- C ABI of libpcb200.so: the H100 (sm_90a) replacement for the native half of the
 * MinkowskiEngine v0.4.3 operator library on PointContrast's Res16UNet34C hot path.
 *
 * What each entry point replaces (reference call sites are relative to the original PointContrast repository; the ME
 * native sources are an external, un-vendored dependency pinned at README.md:24,34):
 *
 *   pcb_coords_* / pcb_hash_* / pcb_kernel_map*   ME CoordsManager (CPU hash map): initialize, stride, getKernelMap.
 *        Reached implicitly from every `ME.SparseTensor(F, coords=C)` (pretrain/pointcontrast/lib/ddp_trainer.py:290-297,392-398)
 *        and every strided / 3x3x3 convolution (pretrain/pointcontrast/model/res16unet.py:47-190).
 *   pcb_conv_forward[_split] / pcb_conv_wgrad[_split] / pcb_weight_tile
 *        ME ConvolutionForwardGPU / ConvolutionBackwardGPU (and the Transpose variants), bound in ME's python as
 *        MinkowskiConvolutionFunction.apply(input_features, kernel, tensor_stride, stride, kernel_size, dilation,
 *        region_type, region_offset, in_coords_key, out_coords_key, coords_manager) -- signature evidenced by
 *        downstream/votenet_det_new/models/backbone/sparseconv/models/conditional_random_fields.py:135-137;
 *        constructed at pretrain/pointcontrast/model/modules/common.py:130-138,159-167.
 *   pcb_bn_*      MinkowskiBatchNorm == torch.nn.BatchNorm1d on .F (model/modules/common.py:21, model/resnet.py:95-97).
 *   pcb_nce_*     PointInfoNCE (lib/ddp_trainer.py:420-426 + lib/criterion.py:15-19).
 *   pcb_pdist_rowmin   pdist + min(1) of the hardest-contrastive loss (lib/ddp_trainer.py:182-184,215-219).
 *   pcb_sgd_step  optim.SGD(momentum, weight_decay) step (lib/ddp_trainer.py:107-111,319,435).
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on failure; pcb_last_error() returns the message
 *     of the last failure on the calling thread.  Nothing throws across this boundary.
 *   - all data pointers are CALLER-OWNED DEVICE memory (16-byte aligned); the library never allocates
 *     device memory.  Workspaces: an entry point that takes `ws` accepts any ws_bytes >= its *_ws_bytes query for the
 *     same arguments; with less it returns PCB_ERR_ARG before any CUDA call or launch (a call with nothing to compute,
 *     e.g. n == 0, may return earlier without looking at ws).  It touches no byte of ws at or beyond the query, and its
 *     results do not depend on how much larger ws is.
 *   - `stream` is a cudaStream_t passed as void*; every call is asynchronous on it unless stated.
 *   - feature matrices are fp32 row-major [rows, channels]; coordinates int32 [rows, 4] = (batch, x, y, z).
 *   - a kernel map is a dense neighbour table  tbl[K][n_out]  (int32): tbl[k][j] = input row feeding output
 *     row j through kernel offset k, or -1.  The ME per-offset (in,out) pair lists are exactly the
 *     non-negative entries of row k, in ascending j.
 */
#ifndef PCB200_H_
#define PCB200_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PCB_OK 0
#define PCB_ERR_CUDA 1
#define PCB_ERR_ARG 2
#define PCB_ERR_RANGE 3      /* coordinate outside the packable range */
#define PCB_ERR_DUPLICATE 4  /* duplicate coordinates in a SparseTensor */
#define PCB_MAX_KERNEL_VOLUME 27

const char* pcb_last_error(void);
/* "pcb200 <version> sm_90a" */
const char* pcb_version(void);
/* Number of kernels this library has launched on this process since load (bench.py's gpu_launches). */
uint64_t pcb_launch_count(void);
/* The library links its own (static) CUDA runtime: select the device the caller's pointers/streams live on. */
int pcb_set_device(int device);
/* Measurement aid (bench.py's roofline): while enabled, every convolution / weight-gradient entry point (including the ones
 * issued inside pcb_unit_*) is bracketed by CUDA events on its stream.  pcb_profile_read synchronises with them, returns the
 * elapsed ms and kind (0 = convolution forward / data gradient, 1 = weight gradient) of up to max_records records in issue
 * order, *count = records taken since the last read, and clears the list.  Not thread-safe; off by default. */
int pcb_profile_enable(int on);
int pcb_profile_read(float* ms, int32_t* kinds, int max_records, int* count);

/* ----------------------------------------------------------------------------------------------- coordinates */
/* (b,x,y,z) -> 64-bit keys whose unsigned order is lexicographic (b,x,y,z).  b in [0,65535), |x|,|y|,|z| < 32768.
 * `status` (device int32, caller-zeroed) receives PCB_ERR_RANGE bits on violation. */
int pcb_coords_pack(const int32_t* coords, int64_t n, uint64_t* keys, int32_t* status, void* stream);
int pcb_coords_unpack(const uint64_t* keys, int64_t n, int32_t* coords, void* stream);

/* Open-addressing hash table key -> row.  capacity must be a power of two >= 2n.  `status` gets
 * PCB_ERR_DUPLICATE if a key occurs twice. */
int pcb_hash_build(const uint64_t* keys, int64_t n, uint64_t* table_keys, int32_t* table_vals,
                   int64_t capacity, int32_t* status, void* stream);

/* Stride a level: coarse = floor(c / new_ts) * new_ts, unique, rows ordered by key (canonical order).
 * Writes out_keys[0..*n_out) and parent[i] = coarse row of fine row i.
 * SYNCHRONISES the stream once to return *n_out on the host. */
size_t pcb_coords_stride_ws_bytes(int64_t n);
int pcb_coords_stride(const uint64_t* keys, int64_t n, int32_t new_ts, uint64_t* out_keys, int32_t* parent,
                      int64_t* n_out, void* ws, size_t ws_bytes, void* stream);

/* tbl[k][j] = row of (out_coord[j] + offsets[k]) in the hashed level, or -1.  offsets: HOST int32 [K][3]. */
int pcb_kernel_map(const uint64_t* out_keys, int64_t n_out, const uint64_t* table_keys,
                   const int32_t* table_vals, int64_t capacity, const int32_t* offsets, int K, int32_t* tbl,
                   void* stream);
/* counts[k] = number of non-negative entries of row k (device int64 [K]). */
int pcb_kernel_map_count(const int32_t* tbl, int K, int64_t n_out, int64_t* counts, void* stream);
/* Tile order of a neighbour table for pcb_conv_forward_split_ordered: perm[i] (device int32 [n_out]) = the output row at tile
 * position i.  Rows are stably sorted by (row / window, mask), bit k of mask = (tbl[k][row] >= 0): rows with the same neighbour
 * offsets share the kernel's 128-row tiles, so a tile stages fewer offsets, while every tile stays inside one window of `window`
 * consecutive rows (a multiple of 128; >= n_out: one window), which bounds how far apart in the input a tile's gathers land.
 * The order depends on the table only, so it serves every kmap over the table.  n_out < 2^31.  ws: pcb_conv_tile_order_ws_bytes. */
size_t pcb_conv_tile_order_ws_bytes(int64_t n_out);
int pcb_conv_tile_order(const int32_t* tbl, int64_t tbl_stride, int K, int64_t n_out, int64_t window, int32_t* perm, void* ws,
                        size_t ws_bytes, void* stream);

/* ----------------------------------------------------------------------------------------------- data preparation (SURVEY.md 8f-2) */
/* One point per occupied voxel: voxel index = floor(xyz / voxel_size) per axis (fp32, |index| < 2^20).  Writes the M occupied voxels'
 * indices (int32 [M,3], sorted by (x,y,z)) and sel[M] = the smallest index of a point in each voxel -- np.unique(return_index=True) /
 * `ME.utils.sparse_quantize(xyz / voxel_size, return_index=True)` of `pretrain/pointcontrast/lib/ddp_data_loaders.py:228-241`.
 * out_coords / sel hold up to n rows.  SYNCHRONISES the stream once to return *m_out. */
size_t pcb_voxelize_ws_bytes(int64_t n);
int pcb_voxelize(const float* xyz, int64_t n, float voxel_size, int32_t* out_coords, int32_t* sel, int64_t* m_out, void* ws,
                 size_t ws_bytes, void* stream);
/* All (i, j) with |src_i - dst_j| < radius (fp32, strict), i ascending, j ascending within i -- `get_matching_indices`
 * (`ddp_data_loaders.py:36-49`: an open3d KD-tree radius search per source point; radius = 1.5 voxels) on a hashed uniform grid of
 * cell size `radius`.  *n_pairs = total number of pairs (SYNCHRONISES once); at most `cap` of them are written ([cap,2] int32;
 * pairs == NULL: count only). */
size_t pcb_radius_pairs_ws_bytes(int64_t ns, int64_t nd);
int pcb_radius_pairs(const float* src, int64_t ns, const float* dst, int64_t nd, float radius, int32_t* pairs, int64_t cap,
                     int64_t* n_pairs, void* ws, size_t ws_bytes, void* stream);
/* The pretraining pair list of a scan (`pretrain/data_preprocess/scannet_pair/compute_full_overlapping.py`, SURVEY.md 8f-10).  A scene
 * is one ragged batch of F frames, 1 <= F <= 4096: xyz fp64 [n, 3], frame f is rows [offsets[f], offsets[f+1]) (device int64 [F + 1],
 * non-decreasing from 0 to n).
 *
 * pcb_voxel_down_sample: open3d `PointCloud.voxel_down_sample` of every frame (`:15-26`, `:59-63`).  Per frame lo = min(points) -
 * voxel_size * 0.5 per axis, voxel index floor((p - lo) / voxel_size) (fp64, one rounding per operation, < 2^17 per axis); one output
 * point per occupied voxel, the fp64 sum of its points in ascending input index divided by their number.  Rows frame-major, ascending
 * (x, y, z) voxel index within a frame; out holds up to n rows.  out_offsets (device [F + 1]) delimit the frames of the output; SYNCHRONISES
 * once and copies them to out_offsets_host (host, F + 1 entries).  A non-finite coordinate or a voxel index >= 2^17 returns PCB_ERR_RANGE;
 * offsets that do not run from 0 to n return PCB_ERR_ARG (both found after the launches).  An empty frame has no output rows.
 *
 * pcb_frame_overlap: counts[i * F + j] (int64 [F, F], written in full, diagonal 0) = the number of points q of frame j with at least one
 * point p of frame i != j at ((dx dx + dy dy) + dz dz) < radius * radius in fp64 without FMA contraction -- the length of
 * `get_matching_indices(pcd_j, tree_i, radius, K=1)` (`:39-47`, `:67-74`).  One hashed grid of cell size radius (1 + 2^-20) over all
 * frames.  status (device int32, caller-zeroed) receives bits: PCB_FRAMES_RANGE if a point's cell index lies outside +-2^20 (or it is
 * not finite; that point matches nothing), PCB_FRAMES_OFFSETS if the offsets do not run from 0 to n without decreasing (the counts are
 * then meaningless, though nothing outside the arrays is read).  Does not synchronise.
 *
 * Both: n < 0, F outside [1, 4096], voxel_size / radius not positive and finite, NULL pointers (xyz / out may be NULL when n == 0) and
 * a short workspace return PCB_ERR_ARG before anything is launched. */
#define PCB_FRAMES_RANGE 1
#define PCB_FRAMES_OFFSETS 2
size_t pcb_voxel_down_sample_ws_bytes(int64_t n, int64_t F);
int pcb_voxel_down_sample(const double* xyz, int64_t n, const int64_t* offsets, int64_t F, double voxel_size, double* out, int64_t* out_offsets,
                          int64_t* out_offsets_host, void* ws, size_t ws_bytes, void* stream);
size_t pcb_frame_overlap_ws_bytes(int64_t n, int64_t F);
int pcb_frame_overlap(const double* xyz, int64_t n, const int64_t* offsets, int64_t F, double radius, int64_t* counts, int32_t* status,
                      void* ws, size_t ws_bytes, void* stream);

/* pcb_depth_to_points: `point_cloud_extractor.py:47-75` for a batch of F depth frames (device uint16 [F, H, W], millimetres) with
 * the depth intrinsics fx, fy, cx, cy, bx, by and the camera-to-world poses (device fp64 [F, 4, 4], row-major).  Every pixel (u, v)
 * with nonzero depth becomes one fp64 world point, one rounding per operation and no FMA:
 *   d = depth / 1000, X = ((u - cx) d) / fx + bx, Y = ((v - cy) d) / fy + by, Z = d,
 *   out[r] = ((X P[r][0] + Y P[r][1]) + Z P[r][2]) + P[r][3]      (r = 0, 1, 2)
 * Rows frame-major, within a frame in row-major pixel order (the order of np.where on the flattened image); out holds up to
 * F H W rows.  out_offsets (device int64 [F + 1]) delimit the frames; SYNCHRONISES once and copies them to out_offsets_host (host,
 * F + 1 entries) and to nan_host (host int32 [F]) a flag per frame that is 1 when any of its coordinates is NaN.  F outside
 * [1, 4096], H or W outside [1, 32768], F ceil(H W / 1024) >= 2^31 - 1, NULL pointers and a short workspace return PCB_ERR_ARG before
 * anything is launched. */
size_t pcb_depth_to_points_ws_bytes(int64_t F, int64_t H, int64_t W);
int pcb_depth_to_points(const uint16_t* depth, int64_t F, int64_t H, int64_t W, double fx, double fy, double cx, double cy, double bx,
                        double by, const double* poses, double* out, int64_t* out_offsets, int64_t* out_offsets_host, int32_t* nan_host,
                        void* ws, size_t ws_bytes, void* stream);

/* ----------------------------------------------------------------------------------------------- semseg on the original point cloud */
/* The label transfer of `test_pointcloud` (`downstream/semseg/lib/datasets/scannet.py:131-172`, `stanford.py:41-84`): a scipy KD-tree
 * query of every original point against the predicted voxel centres, then `fast_hist` (`lib/utils.py:131-133`).
 *
 * pcb_nearest: idx[i] (int32 [n]) = the smallest j in [0, m) whose d2 = ((dx dx + dy dy) + dz dz) (fp64, no FMA contraction) between
 * ref[j] and query[i] (fp64 [m, 3], [n, 3]) is the minimum over all j.  A hashed grid of cell size cell_size over the references, searched
 * in Chebyshev shells around the query's cell with an exact stop rule; a query not settled within 8 shells is compared with every
 * reference.  The result does not depend on cell_size (which only sets the speed), the launch shape or ws_bytes.  status (device int32,
 * caller-zeroed) receives PCB_NEAREST_RANGE if a coordinate is not finite or its cell lies outside +-2^20 (that query gets idx -1; the
 * other results are then meaningless).  Does not synchronise.  n == 0 returns at once; m == 0 < n, m or n >= 2^31 - 1, cell_size not
 * positive and finite, NULL pointers and a short workspace return PCB_ERR_ARG before anything is launched.
 *
 * pcb_label_transfer: point_label[i] = ref_label[idx[i]] (int32 [n]; ref_label int32 [m]).  With query_label (int32 [n], may be NULL): gt = lut[query_label[i]],
 * pred = lut[point_label[i]] (lut: device int32 [lut_n], original -> masked label, -1 for no entry), and for 0 <= gt < C
 * hist[gt * C + pred] += 1 (int64 [C, C], accumulated; the caller zeroes it).  status receives PCB_LABEL_RANGE if a label lies outside
 * the table, has no entry, or a counted pred lies outside [0, C) (the reference's KeyError / IndexError), PCB_NEAREST_RANGE if an idx
 * lies outside [0, m) (that row gets point_label -1 and is not counted).  Does not synchronise.  m or n outside [0, 2^31 - 1), and with
 * query_label C outside [1, 46340], lut_n < 1 or NULL lut / hist, return PCB_ERR_ARG before the launch. */
#define PCB_NEAREST_RANGE 1
#define PCB_LABEL_RANGE 2
size_t pcb_nearest_ws_bytes(int64_t m, int64_t n);
int pcb_nearest(const double* ref, int64_t m, const double* query, int64_t n, double cell_size, int32_t* idx, int32_t* status, void* ws,
                size_t ws_bytes, void* stream);
int pcb_label_transfer(const int32_t* idx, const int32_t* ref_label, int64_t m, const int32_t* query_label, int64_t n, const int32_t* lut,
                       int lut_n, int C, int32_t* point_label, int64_t* hist, int32_t* status, void* stream);

/* ----------------------------------------------------------------------------------------------- S3DIS preprocessing (8f-14) */
/* One room of `downstream/semseg/lib/datasets/preprocessing/stanford.py` `convert_to_ply`: its annotation files' bytes concatenated in
 * `text` (device, 16-byte aligned, readable up to nbytes rounded up to 16), file f = bytes [file_off[f], file_off[f+1]) (device int64
 * [nfiles + 1], non-decreasing from 0 to nbytes; a file may be empty).
 *
 * pcb_text_lines: the lines of Python's text-mode iteration of each file (universal newlines: "\n", "\r\n" and a lone "\r" end a line; a
 * last line without one counts; no line crosses a file; an empty file has none).  chunk_off (device int64 [ceil(nbytes / 16) + 1]) receives
 * the first line index of every 16-byte chunk, flags (device int32 [nfiles]) PCB_TEXT_NONASCII for every file holding a byte >= 0x80,
 * *n_lines (host) the number of lines.  SYNCHRONISES.
 *
 * pcb_s3dis_parse (after pcb_text_lines, same text / file_off / chunk_off / flags): line_start (int64 [n_lines + 1]) = each line's first
 * byte, then nbytes; per line j, `[float(t) for t in line.split()]` (`stanford.py:47-64`) decided on the device where it is exact --
 * status[j] (uint8):
 *   PCB_LINE_KEPT      6 tokens: xyz = float32(float()) (fp32 [n_lines, 3]), rgb = uint8(float32(float())) (uint8 [n_lines, 3]),
 *                      cell = floor(float64(xyz) / 0.01) in true fp64 division (int32 [n_lines, 3]; clamped to +-2^30)
 *   PCB_LINE_SKIPPED   a token float() rejects (the original's except branch)
 *   PCB_LINE_HOST      not decided here: a token outside [0-9+-.eE] that float() may accept (inf, nan, '_'), more than 19
 *                      significant digits, a value not exact by Clinger's fast path, an rgb value whose float32 lies outside [0, 256),
 *                      a line longer than 512 bytes, or any line of a PCB_TEXT_NONASCII file
 *   PCB_LINE_ERROR     only exact tokens, but not 6 of them (a blank line included): the original raises
 * label[j] = file_label[file of j] (int32 [n_lines]).  Values of lines not KEPT are unspecified.  Does not synchronise.
 *
 * pcb_ply_rows: rows[i] (16 bytes, of a 16-byte aligned buffer [m, 16]) = x, y, z <f4 of xyz[sel[i]], red, green, blue of rgb[sel[i]],
 * labels[i] & 0xff -- the PLY body `lib/pc_utils.py:41-70` writes for `sel` / `labels` of pcb_voxelize_labels.  Does not synchronise. */
#define PCB_TEXT_NONASCII 1
#define PCB_LINE_KEPT 0
#define PCB_LINE_SKIPPED 1
#define PCB_LINE_HOST 2
#define PCB_LINE_ERROR 3
size_t pcb_text_lines_ws_bytes(int64_t nbytes);
int pcb_text_lines(const uint8_t* text, int64_t nbytes, const int64_t* file_off, int32_t nfiles, int64_t* chunk_off, int32_t* flags,
                   int64_t* n_lines, void* ws, size_t ws_bytes, void* stream);
int pcb_s3dis_parse(const uint8_t* text, int64_t nbytes, const int64_t* file_off, const int32_t* file_label, int32_t nfiles,
                    const int64_t* chunk_off, int32_t* flags, int64_t n_lines, int64_t* line_start, float* xyz, uint8_t* rgb, int32_t* label,
                    int32_t* cell, uint8_t* status, void* stream);
int pcb_ply_rows(const float* xyz, const uint8_t* rgb, const int32_t* sel, const int32_t* labels, int64_t m, uint8_t* rows, void* stream);

/* ----------------------------------------------------------------------------------------------- VoteNet detection preprocessing (8f-15) */
/* pcb_scannet_annotate: the per-vertex work of one scene of `lib/datasets/scannet/load_scannet_data.py` `export`.  vin (device fp32 [V, 6]:
 * x y z r g b), align (device fp64 [16], the row-major `axisAlignment` matrix M), seg (device int64 [V], `segIndices`, each < INT64_MAX).
 * The host restates `read_aggregation` as two write lists in the original's loop order: label writes (lab_seg int64, lab_val uint32)
 * [n_lab] and instance writes (ins_seg int64, ins_obj int32 = the object's dict index) [n_ins]; per object d < n_obj (dict order):
 * obj_id[d] (uint32, the instance id), first_seg[d] (its first segment) and obj_row[d] (its box row, `obj_id - 1` wrapped as numpy
 * indexes, or -1 outside [0, n_rows)).  Outputs (device): vout fp32 [V, 6] (xyz = fp32 of fp64 [x y z 1] . M^T, one rounding per
 * operation in k order; rgb copied), sem / ins uint32 [V] (the last write to the vertex's segment wins, 0 where none), bbox fp64
 * [n_rows, 7] (per object with vertices: fp32 (min + max) / 2, max - min of its aligned xyz, then the label at the lowest vertex of its
 * first segment; a row no such object owns is zero; -0.0 is the minimum and +0.0 the maximum when both occur; a NaN coordinate makes
 * both bounds of its axis NaN), status int32 [2]: [0] the lowest write ordinal (label writes first, then instance writes) whose
 * segment no vertex has, [1] the lowest object with vertices and obj_row -1; 0x7f7f7f7f where none.  Does not synchronise. */
size_t pcb_scannet_annotate_ws_bytes(int64_t V, int64_t n_obj, int64_t n_rows);
int pcb_scannet_annotate(const float* vin, const double* align, int64_t V, const int64_t* seg, const int64_t* lab_seg,
                         const uint32_t* lab_val, int64_t n_lab, const int64_t* ins_seg, const int32_t* ins_obj, int64_t n_ins,
                         const uint32_t* obj_id, const int64_t* first_seg, const int32_t* obj_row, int64_t n_obj, int64_t n_rows,
                         float* vout, uint32_t* sem, uint32_t* ins, double* bbox, int32_t* status, void* ws, size_t ws_bytes,
                         void* stream);
/* pcb_sunrgbd_votes: the ground-truth votes of `lib/datasets/sunrgbd/sunrgbd_data.py` `extract_sunrgbd_data` for B scenes in one launch.
 * pts (device fp64 [N, ld], ld >= 3, xyz first), scene b = rows [pt_off[b], pt_off[b+1]); boxes (device fp64 [K, 8]: cx, cy, cz, l, w, h,
 * cos(-heading), sin(-heading)), scene b's boxes = rows [box_off[b], box_off[b+1]) in file order; offsets as int64 [B + 1] on both the
 * host and the device.  votes (device fp64 [N, 10]): column 0 = 1 if the point is in a box, then three votes centroid - p; the point's
 * k-th box writes slot min(k, 2), its first box all three.  Inside: |u| <= (l, w, h) for u = rotz(-heading)^T (p - centroid).  Boxes
 * with l, w or h not > 0, or a non-finite value, are skipped.  Does not synchronise. */
int pcb_sunrgbd_votes(const double* pts, int32_t ld, const int64_t* pt_off_host, const int64_t* pt_off, const double* boxes,
                      const int64_t* box_off_host, const int64_t* box_off, int64_t B, double* votes, void* stream);

/* ----------------------------------------------------------------------------------------------- semseg training data (8f-6) */
/* Label-aware voxelisation of integer coordinates (int32 [N,3], |c| < 2^20): the M occupied voxels in ascending (x,y,z) order
 * (out_coords int32 [M,3]), sel[M] = the smallest index of a point in the voxel, out_labels[M] = the label all of the voxel's points
 * share, else ignore_label -- `ME.utils.sparse_quantize(coords, feats, labels=, ignore_label=)` (ME 0.4.3 `quantize_label`) of
 * `downstream/semseg/lib/voxelizer.py:145-146`.  Outputs hold up to n rows.  SYNCHRONISES once to return *m_out. */
size_t pcb_voxelize_labels_ws_bytes(int64_t n);
int pcb_voxelize_labels(const int32_t* coords, const int32_t* labels, int64_t n, int32_t ignore_label, int32_t* out_coords, int32_t* sel,
                        int32_t* out_labels, int64_t* m_out, void* ws, size_t ws_bytes, void* stream);
/* Per-axis minimum (lo[3]) and maximum (hi[3]) of fp32 points [N,3], N >= 1; lo / hi are host pointers.  SYNCHRONISES. */
size_t pcb_point_bounds_ws_bytes(void);
int pcb_point_bounds(const float* xyz, int64_t n, float* lo, float* hi, void* ws, size_t ws_bytes, void* stream);
/* Elastic distortion (`downstream/semseg/lib/transforms.py:187-217`).  noise: the drawn fp32 grid [gx,gy,gz,3] (device, in place: on
 * return it holds the grid after two rounds of the x, y, z 3-tap box filters, scipy.ndimage.convolve's float64 accumulation, zero
 * outside).  axes: device fp64 [gx + gy + gz], the grid positions per axis (strictly ascending).  Then per point, in place:
 * xyz += RegularGridInterpolator(axes, grid, fill_value=0)(xyz) * magnitude, in fp64, rounded to fp32.  Bit-exact vs scipy. */
size_t pcb_elastic_distort_ws_bytes(int gx, int gy, int gz);
int pcb_elastic_distort(float* xyz, int64_t n, float* noise, int gx, int gy, int gz, const double* axes, double magnitude, void* ws,
                        size_t ws_bytes, void* stream);
/* out[i] = floor(homo(xyz_i) @ T[:3,:].T) - min_i(...) per axis (int32 [N,3]), min_out[3] (host) = that minimum
 * (`downstream/semseg/lib/voxelizer.py:134-142`).  T: host fp64 row-major 4x4 (rows 0-2 read); each value is
 * ((x T[j,0] + y T[j,1]) + z T[j,2]) + T[j,3] in fp64.  PCB_ERR_RANGE if a floor lies outside +-2^20.  SYNCHRONISES. */
size_t pcb_affine_floor_ws_bytes(void);
int pcb_affine_floor(const float* xyz, int64_t n, const double* T, int32_t* out, int32_t* min_out, void* ws, size_t ws_bytes, void* stream);
/* The semseg input transforms after dropout, in place on voxels coords int32 [N,3] / colours fp32 [N,3], in the loader's order
 * (`downstream/semseg/lib/dataset.py:344-350`, `lib/transforms.py:23-179`), with the per-scene draws as arguments (coords may be
 * NULL when flip_mask == 0):
 *   RandomHorizontalFlip    bit k of flip_mask: coords[:,k] = max(coords[:,k]) - coords[:,k]
 *   ChromaticAutoContrast   contrast != 0: fp32 (lo, hi, scale = 255 / (hi - lo)), blended with the fp64 factor `blend`;
 *                           PCB_ERR_RANGE if the largest colour is <= 1 (the reference's assert) -- SYNCHRONISES in that case
 *   ChromaticTranslation    translation (host fp64 [3]) or NULL: clip(translation + colour, 0, 255) in fp64, stored fp32
 *   ChromaticJitter         jitter_noise (device fp64 [N,3], standard normal) or NULL: clip(noise * jitter_scale + colour, 0, 255)
 *   normalize != 0          colour / 255 - 0.5 in fp32 (`downstream/semseg/lib/train.py:114`) */
size_t pcb_semseg_input_transform_ws_bytes(void);
int pcb_semseg_input_transform(int32_t* coords, float* feats, int64_t n, int flip_mask, int contrast, double blend,
                               const double* translation, const double* jitter_noise, double jitter_scale, int normalize, void* ws,
                               size_t ws_bytes, void* stream);

/* ----------------------------------------------------------------------------------------------- convolution */
/* Y[j, :] = bias + sum_k X[tbl[kmap[k]][j], :] . W[k]      (j < n_out)      -- EXACT fp32, any channel counts
 *   X  : [*, Cin] row stride ldx (floats);  Y: [n_out, Cout] row stride ldy;  W: fp32 [K][Cin][Cout];  bias: [Cout] or NULL.
 *   kmap : HOST int32 [K] table row used by weight k (NULL = identity).
 * The 3 -> 32 stem layer runs a dedicated kernel, every other width a generic SIMT kernel.  The tensor-core forward / data gradient is
 * pcb_conv_forward_split on split operands. */
int pcb_conv_forward(const float* X, int ldx, const int32_t* tbl, int64_t tbl_stride, const int32_t* kmap, int K,
                     int64_t n_out, int Cin, int Cout, const float* W, const float* bias, float* Y, int ldy, void* stream);
#define PCB_CONV_FORCE_SIMT 1  /* pcb_conv_wgrad: the generic exact kernel also for the stem layer (a cross-check of the stem kernel) */
#define PCB_CONV_ACCUMULATE 4  /* Y += result (pcb_conv_forward_split) / dW += result (weight gradients) */
#define PCB_PLANES_A_FP16 8    /* split-operand calls: the GATHERED operand's planes are fp16 hi/lo (default: bf16 hi/lo) */
#define PCB_PLANES_B_FP16 16   /* pcb_conv_forward_split: the weight tiles are fp16 x 2^10 (pcb_weight_tile with this flag).  Both
                                  operands of a call must use the same format (wgmma takes one 16-bit format for both operands): set
                                  both flags or neither.  pcb_conv_wgrad_split reads bf16 planes only and rejects either flag. */

/* Y[j, :] = sum_k X[tbl[kmap[k]][j], :];  cnt[j] (optional) = number of neighbours present.  The sum / average pooling and unpooling
 * layers of the sibling models (MinkowskiSumPooling / AvgPooling / PoolingTranspose / AvgUnpooling, `model/modules/common.py:170-214`,
 * `model/resnet.py:63`) and their backward passes (the same sum over the transposed table).  C % 4 == 0. */
int pcb_gather_sum(const float* X, int ldx, const int32_t* tbl, int64_t tbl_stride, const int32_t* kmap, int K, int64_t n_out, int C,
                   float* Y, int ldy, float* cnt, void* stream);

/* dW[k] = sum_j A[tbl[k][j], :]^T . B[j, :]       A: gathered [*, Ca] (lda), B: contiguous rows [n_out, Cb] (ldb).
 *   transpose_out = 0: dW is [K][Ca][Cb];  1: dW is [K][Cb][Ca].
 * pcb_conv_wgrad: EXACT fp32 kernels on fp32 operands (the 3-channel stem layer, widths the tensor-core tiling does not cover, cross-checks);
 * the tensor-core weight gradient is pcb_conv_wgrad_split on split operands. */
size_t pcb_conv_wgrad_ws_bytes(int K, int64_t n_out, int Ca, int Cb);
int pcb_conv_wgrad(const float* A, int lda, const float* B, int ldb, const int32_t* tbl, int64_t tbl_stride, int K,
                   int64_t n_out, int Ca, int Cb, float* dW, int transpose_out, void* ws, size_t ws_bytes,
                   int flags, void* stream);

/* Split-operand variants (tensor-core path; Cin, Cout multiples of 32): the gathered / row-aligned operands are 16-bit hi/lo planes
 * (see pcb_split_rows), row strides lds/lda/ldb in ELEMENTS (multiples of 8), and the convolution's weights are pre-tiled by
 * pcb_weight_tile[_batch].  Same semantics as pcb_conv_forward / pcb_conv_wgrad; the kernels' operand staging is then a pure
 * asynchronous copy (cp.async, zero-filled where a neighbour is missing, and one TMA bulk copy per weight tile). */
/* pcb_weight_tile: fp32 W[K][Cin][Cout] -> split weights pre-tiled as the shared-memory images of the split conv kernel (one
 * contiguous blob per (offset, 32-channel chunk, column block), fetched by ONE TMA bulk copy per pipeline stage):
 * `fwd_tiles` for the forward roles, `dgrad_tiles` for the data-gradient roles (Cin/Cout swapped).  flags & PCB_PLANES_B_FP16:
 * the FORWARD tiles hold fp16 hi/lo of W * 2^10 (|W| < 60; the kernel rescales its output), the data-gradient tiles stay bf16. */
size_t pcb_weight_tile_bytes(int K, int Cin, int Cout, int dgrad_roles);
int pcb_weight_tile(const float* W, int K, int Cin, int Cout, void* fwd_tiles, void* dgrad_tiles, int flags, void* stream);
/* The same for every convolution of a network in ONE launch: fill a HOST array of descriptors with pcb_tile_desc_fill (start = running
 * sum of K*Cin*Cout), copy it to the device, call pcb_weight_tile_batch(device array, n <= 256, total elements) after every optimiser step. */
typedef struct pcb_tile_desc {
  const float* W; void* fwd; void* dgrad;
  int32_t K, Cin, Cout, flags, bn_f, bn_d;
  int64_t start;
} pcb_tile_desc;
int pcb_tile_desc_fill(pcb_tile_desc* d, const float* W, int K, int Cin, int Cout, void* fwd_tiles, void* dgrad_tiles, int flags, int64_t start);
int pcb_weight_tile_batch(const pcb_tile_desc* descs_dev, int n, int64_t total, void* stream);
/* Small levels split the (offset, channel-chunk) loop of pcb_conv_forward_split over extra CTAs and reduce through `ws`
 * (deterministic). */
size_t pcb_conv_forward_split_ws_bytes(int K, int64_t n_out, int Cin, int Cout);
int pcb_conv_forward_split(const uint16_t* Xhi, const uint16_t* Xlo, int lds, const int32_t* tbl, int64_t tbl_stride,
                           const int32_t* kmap, int K, int64_t n_out, int Cin, int Cout, const void* w_tiles,
                           const float* bias, float* Y, int ldy, void* ws, size_t ws_bytes, int flags, void* stream);
/* The same with the output rows taken in the tile order `perm` of pcb_conv_tile_order on `tbl` (NULL: identity, which is
 * pcb_conv_forward_split).  Same bits as the identity order; an offset-split launch (small levels) runs in the identity order. */
int pcb_conv_forward_split_ordered(const uint16_t* Xhi, const uint16_t* Xlo, int lds, const int32_t* tbl, int64_t tbl_stride,
                                   const int32_t* kmap, int K, const int32_t* perm, int64_t n_out, int Cin, int Cout,
                                   const void* w_tiles, const float* bias, float* Y, int ldy, void* ws, size_t ws_bytes, int flags,
                                   void* stream);
/* pcb_conv_wgrad_split: both operands as bf16 hi/lo planes; flags: PCB_CONV_ACCUMULATE only (PCB_ERR_ARG if a PCB_PLANES_* flag
 * is set). */
size_t pcb_conv_wgrad_split_ws_bytes(int K, int64_t n_out, int Ca, int Cb);
int pcb_conv_wgrad_split(const uint16_t* Ahi, const uint16_t* Alo, int lda, const uint16_t* Bhi, const uint16_t* Blo, int ldb,
                         const int32_t* tbl, int64_t tbl_stride, int K, int64_t n_out, int Ca, int Cb, float* dW,
                         int transpose_out, void* ws, size_t ws_bytes, int flags, void* stream);

/* ----------------------------------------------------------------------------------------------- batch norm */
/* Training-mode BatchNorm on row-segmented matrices: rows [0, n0) and [n0, n) are two independent BatchNorm batches -- the two views
 * of a scene pair stacked in one feature matrix, each normalised with its own statistics exactly as the reference's two forward calls
 * do (`lib/ddp_trainer.py:290-297,392-398`); n0 == n is one batch (MinkowskiBatchNorm on the modular surface).  All ld* are row strides
 * in floats (>= C, multiples of 4), so inputs/outputs may be column slices of wider (concatenated) buffers.
 *   stats   : mean[seg][C], invstd[seg][C] = 1/sqrt(var_biased + eps); if running_* non-NULL:
 *             running = (1-momentum)*running + momentum*{mean, var_unbiased}, with segment 0 and then with segment 1.
 *             ws: pcb_bn_ws_bytes(n, C).
 *   apply   : Y = [relu]( (X-mean)*invstd*gamma+beta [+ residual] ), as fp32 (Y, may be NULL) and/or split planes (Yhi/Ylo);
 *             flags: PCB_BN_RELU, PCB_PLANES_A_FP16 (Yhi/Ylo are fp16 hi/lo instead of bf16 hi/lo; Ybhi/Yblo, if non-NULL, then
 *             receive the bf16 hi/lo planes as well)
 *   backward: g = dY * (relu > 0) if relu_hi else dY, where relu_hi is the 16-bit hi plane of the ReLU output (Yhi of the apply
 *             pass; row stride ldmh in elements) and relu > 0 <=> its sign bit is clear and it is not zero;
 *             dgamma/dbeta (+)= sum(g*xhat) / sum(g), summed over both segments;
 *             dX = gamma*invstd*(g - mean(g) - xhat*mean(g*xhat));   gout (=|+=) g  (gout_mode 0 none, 1 write, 2 add)
 *             -- gout is the gradient of the residual input of the forward unit; it may alias dY. */
#define PCB_BN_RELU 1
size_t pcb_bn_ws_bytes(int64_t n, int C);
int pcb_bn_stats_seg(const float* X, int ldx, int64_t n, int64_t n0, int C, float eps, float momentum, float* mean, float* invstd,
                     float* running_mean, float* running_var, void* ws, size_t ws_bytes, void* stream);
int pcb_bn_apply_seg(const float* X, int ldx, int64_t n, int64_t n0, int C, const float* mean, const float* invstd,
                     const float* gamma, const float* beta, const float* residual, int ldr, int flags, float* Y, int ldy,
                     uint16_t* Yhi, uint16_t* Ylo, int lds, uint16_t* Ybhi, uint16_t* Yblo, void* stream);
int pcb_bn_backward_seg(const float* dY, int lddy, const float* X, int ldx, const uint16_t* relu_hi, int ldmh, int64_t n, int64_t n0,
                        int C, const float* mean, const float* invstd, const float* gamma, float* dX, int lddx, float* dgamma,
                        float* dbeta, int accumulate_param_grads, float* gout, int ldg, int gout_mode, uint16_t* dXhi,
                        uint16_t* dXlo, int lds, void* ws, size_t ws_bytes, void* stream);
/* "Split" operand format of the tensor-core conv kernels: an fp32 matrix stored as two 16-bit planes, x ~= hi + lo: bf16 planes
 * (2^-17 relative, fp32's exponent range: gradients) or, with PCB_PLANES_A_FP16, fp16 planes (2^-22 relative, |x| < 65504: the
 * activations gathered by the FORWARD convolutions -- the forward pass sets the whole-network gradient error);
 * row stride lds in ELEMENTS.  The elementwise producers above can emit it directly (Yhi/Ylo, dXhi/dXlo; NULL = off; dX may
 * then be NULL), so the conv kernels' gather becomes a pure asynchronous copy.  pcb_split_rows converts an fp32 matrix. */
int pcb_split_rows(const float* X, int ldx, int64_t n, int C, uint16_t* hi, uint16_t* lo, int lds, int flags, void* stream);

/* ----------------------------------------------------------------------------------------------- fused units */
/* One "unit" of the Res16UNet graph = convolution -> BatchNorm (training statistics) -> [+ residual] -> [ReLU]
 * (`model/res16unet.py:206-268`, `model/modules/resnet_block.py:44-60`: a BasicBlock is two units).  pcb_unit_forward issues the whole
 * unit from ONE call -- on the small levels, where the convolution runs offset-split, its reduction pass also produces the BatchNorm
 * column statistics (no separate pass over z) --
 * and pcb_unit_backward issues its reverse: ReLU mask + BatchNorm backward + residual-gradient fan-out in one elementwise
 * pass, then the weight gradient (accumulated into dW) and the data gradient (written or accumulated into gin).
 * The caller (pointcontrast_b200/fused.py; a C++ host would do the same) owns every buffer; the struct is plain data.
 *
 * Matrices: fp32 pointer `*_p` (row stride `*_ld` floats) and/or bf16 split planes `*_hi`/`*_lo` (row stride `*_lds` elements).
 *   x    : unit input  [n_in, Cin]   (split planes when Cin % 32 == 0, else fp32: the 3-channel stem)
 *   z    : convolution output [n_out, Cout], fp32 (kept for the backward pass)
 *   out  : unit output [n_out, Cout]: split planes (always) and fp32 (only if out_p != NULL: it feeds a residual add)
 *   res  : residual input, fp32 (or NULL);  rows [0, n0) / [n0, n_out) are the two views of a stacked pair (n0 == n_out: one)
 *   g    : gradient of `out` (fp32, complete when pcb_unit_backward is called)
 *   dz   : scratch for the gradient of z: split planes [n_out, Cout] (+ fp32 `dz_p` when Cout or Cin is not a multiple of 32)
 *   gin  : gradient of x (fp32) -- written (gin_mode 1) or accumulated (2); 0: not wanted (network input)
 *   gres : gradient of the residual input -- written (1) / accumulated (2) / none (0)
 * Tables (device int32 [K][stride]) and kmaps (HOST int32 [K] or NULL) as for pcb_conv_forward / pcb_conv_wgrad.
 * ws: pcb_unit_ws_bytes(K, n_in, n_out, Cin, Cout) bytes of scratch. */
typedef struct pcb_unit {
  int64_t n_in, n_out, n0;
  int32_t K, Cin, Cout, relu;
  const int32_t* fwd_tbl; int64_t fwd_stride; const int32_t* fwd_kmap;
  const int32_t* dg_tbl; int64_t dg_stride; const int32_t* dg_kmap;
  const int32_t* fwd_perm;                          /* tile order (pcb_conv_tile_order) of fwd_tbl, or NULL (identity) */
  const int32_t* wg_tbl; int64_t wg_stride; int32_t wg_gather_x;
  const float* W; const void* wt_fwd; const void* wt_dg; float* dW;
  const float* gamma; const float* beta; float* running_mean; float* running_var; float* dgamma; float* dbeta;
  float eps, momentum;
  float* mean; float* invstd;                       /* [segments][Cout], written by forward, read by backward */
  const float* x_p; int32_t x_ld; const uint16_t* x_hi; const uint16_t* x_lo; int32_t x_lds;
  const uint16_t* x_bhi; const uint16_t* x_blo;     /* PCB_UNIT_FP16_FORWARD: x once more as bf16 hi/lo planes (the weight gradient pairs it
                                                       with the bf16 gradient planes: wgmma takes ONE format for both operands) */
  float* z_p; int32_t z_ld;
  float* out_p; int32_t out_ld; uint16_t* out_hi; uint16_t* out_lo; int32_t out_lds;
  uint16_t* out_bhi; uint16_t* out_blo;             /* PCB_UNIT_FP16_FORWARD: bf16 hi/lo copy of `out` (row stride out_lds) */
  const float* res_p; int32_t res_ld;
  const float* g_p; int32_t g_ld;
  float* dz_p; uint16_t* dz_hi; uint16_t* dz_lo; int32_t dz_ld;
  float* gin_p; int32_t gin_ld; int32_t gin_mode;
  float* gres_p; int32_t gres_ld; int32_t gres_mode;
  void* ws; size_t ws_bytes;
  int32_t flags;                                    /* PCB_UNIT_* */
} pcb_unit;
#define PCB_UNIT_SEPARATE_STATS 1   /* forward: BatchNorm statistics always by a separate pass over z (cross-check of the fused reduce+statistics pass) */
#define PCB_UNIT_FP16_FORWARD 2     /* activations are gathered by the forward convolutions as fp16 hi/lo planes (x_hi/x_lo, out_hi/out_lo)
                                       against fp16 weight tiles (pcb_weight_tile with PCB_PLANES_B_FP16): 2^-22 products in the
                                       forward pass.  Gradients (dz) and the data-gradient tiles stay bf16 hi/lo (fp32's exponent
                                       range); wgmma takes one 16-bit format for both operands, so every activation also carries bf16 hi/lo planes
                                       (x_bhi/x_blo, out_bhi/out_blo) for the weight gradient. */
#define PCB_UNIT_EVAL 4             /* forward only, eval-mode BatchNorm: normalise with running_mean / running_var (not updated) */
size_t pcb_unit_ws_bytes(int K, int64_t n_in, int64_t n_out, int Cin, int Cout);
int pcb_unit_forward(const pcb_unit* u, void* stream);
int pcb_unit_backward(const pcb_unit* u, void* stream);

/* ----------------------------------------------------------------------------------------------- losses */
/* PointInfoNCE on gathered rows q,k [n, D]: loss = mean_i(logsumexp_j(q_i.k_j/T) - q_i.k_i/T).
 * Writes loss (device float), dq, dk (= d loss / d q, d k).  ws: pcb_nce_ws_bytes(n).
 * D = 32 or 64: fused wgmma kernels (nce_wgmma.cu) -- q k^T tiles on the tensor cores from fp16 hi/lo operands (|q|,|k| <= ~1: the
 * L2-normalised features), softmax statistics and both gradients straight from the tiles, the n x n logits never stored.
 * Other widths: exact fp32 SIMT kernels that materialise the logits in ws. */
size_t pcb_nce_ws_bytes(int64_t n);
int pcb_nce_forward_backward(const float* q, const float* k, int64_t n, int D, float inv_T, float* loss, float* dq,
                             float* dk, void* ws, size_t ws_bytes, void* stream);
/* nn.CrossEntropyLoss(ignore_index) on logits [n, C] with int64 targets (`downstream/semseg/lib/train.py:68,120`): writes the mean loss
 * over the non-ignored rows (device float) and dlogits = grad_scale * d loss / d logits.  ws: pcb_ce_ws_bytes(n).  n >= 1, 1 <= C <= 1024.
 * A row counts when its target t is in [0, C) and != ignore_index.  A target outside [0, C) is treated as ignored (torch raises): its
 * logit x[t] is never read, and the row adds nothing to the loss or the count and gets a zero gradient.  With no counted row the loss is
 * NaN (0 / 0, as torch) and dlogits is all zero.  A NaN logit in a counted row makes the loss NaN and that row's gradient NaN (as
 * torch); in a row that does not count it changes nothing (torch's backward gives that row NaN times a zero incoming gradient). */
size_t pcb_ce_ws_bytes(int64_t n);
int pcb_ce_forward_backward(const float* logits, const int64_t* target, int64_t n, int C, int64_t ignore_index, float grad_scale,
                            float* loss, float* dlogits, void* ws, size_t ws_bytes, void* stream);
/* Semantic-segmentation evaluation (`downstream/semseg/lib/test.py:62-196`), accumulated on the device across calls (the caller zeroes
 * the accumulators once); nothing synchronises.  n >= 1, 1 <= C <= 1024.
 *
 * pcb_seg_metrics: one pass over logits [n, C]: pred[n] = argmax, the first index among the maximal values with a NaN counting as
 * maximal (torch `output.max(1)[1]`); prob[n, C] = exp(x - max) / sum exp(x - max), or NULL to skip it.  Then
 *   hist[t * C + pred] += 1 (int64 [C, C]) for the rows with 0 <= t < C (`lib/utils.py:131-133` fast_hist);
 *   stats[0] += loss * n, where loss is the mean cross-entropy over the rows with t in [0, C) and t != ignore_index -- the same bits
 *               pcb_ce_forward_backward returns on these logits (NaN when there is no such row);
 *   stats[1] += score * n, score = 100 * hits / rows with t != 255 in fp32 (`lib/utils.py:117-128` precision_at_one hard-codes 255);
 *   stats[2] += n                                                            (stats: fp64 [3], the AverageMeter sums of `test.py:138-139`)
 * ws: pcb_seg_metrics_ws_bytes(n).
 *
 * pcb_average_precision: per class c, sklearn's uninterpolated average precision of score[:, c] (fp32 [n, C]) against target == c (a
 * target outside [0, C) is a negative for every class: `label_binarize` of `test.py:55-59`), sum over tie groups g of
 * (R_g - R_{g-1}) * P_g in fp64.  A class with a positive in the batch adds its AP to ap_sum[c] (fp64) and 1 to ap_cnt[c] (int64); a
 * class without one changes neither (its AP is NaN, left out of the reference's np.nanmean); a NaN in a column with a positive adds
 * NaN.  n * C >= 2^31 returns PCB_ERR_ARG.  ws: pcb_average_precision_ws_bytes(n, C). */
size_t pcb_seg_metrics_ws_bytes(int64_t n);
int pcb_seg_metrics(const float* logits, const int64_t* target, int64_t n, int C, int64_t ignore_index, int32_t* pred, float* prob,
                    int64_t* hist, double* stats, void* ws, size_t ws_bytes, void* stream);
size_t pcb_average_precision_ws_bytes(int64_t n, int C);
int pcb_average_precision(const float* score, const int64_t* target, int64_t n, int C, double* ap_sum, int64_t* ap_cnt, void* ws,
                          size_t ws_bytes, void* stream);

/* VoteNet detection evaluation (`downstream/votenet_det_new/models/ap_helper.py`, `lib/utils/{nms,eval_det,box_util}.py`).  Nothing
 * synchronises.  Boxes are 8 corners fp64 [.., 8, 3] in upright-camera coordinates, built as `get_3d_box` builds them with one rounding
 * per operation; box params fp64 [.., 8] = (center (camera), l, w, h, cos, sin).  heading_rule 0: `class2angle` returns 0 (ScanNet);
 * 1: cls * 2 pi / H + residual, minus 2 pi above pi (SUN RGB-D).  mean_size: fp64 [S, 3] (device).
 *
 * pcb_det_decode_pred: per proposal of [B, K]: torch.argmax (first maximal index, NaN maximal) of heading_scores [B,K,H], size_scores
 *   [B,K,S] and sem_cls_scores [B,K,C] (C <= 1024), the chosen residuals of heading_residuals [B,K,H] / size_residuals [B,K,S,3], the
 *   corners and params from center [B,K,3] (depth coordinates); sem_cls int32 [B,K]; the reference's numpy fp32 softmax (fp32 exp of
 *   x - max, numpy's pairwise row sum, one division) of sem_cls_scores -> sem_prob fp32 [B,K,C] and of objectness_scores [B,K,2] ->
 *   obj_prob fp32 [B,K] (class 1).
 * pcb_det_decode_gt: corners and params of labels [B, K]: center fp32 [B,K,3], heading_class int64 [B,K], heading_residual fp32 [B,K],
 *   size_class int64 [B,K], size_residual fp32 [B,K,3].  A size class outside [0, S) (or heading class outside [0, H) under rule 1)
 *   ORs PCB_ERR_RANGE into status (device int32, caller-zeroed) and leaves that box unwritten.
 * pcb_det_points_in_box: counts int32 [B, K] = the points of points fp32 [B, N, ld] (xyz in the first 3 of ld channels, depth
 *   coordinates) inside each box of box params [B, K, 8] (|local coordinate| <= half size, fp64; a point within 1e-9 of a face is
 *   unpinned).  Zeroes counts itself.  ceil(N / 4096) > 65535 returns PCB_ERR_ARG.
 * pcb_det_nms: pred_mask int32 [B, K] = 1 on the proposals greedy NMS keeps among those with counts >= min_points (all when counts is
 *   NULL), scores fp32 [B, K], in the order of descending score, ties larger proposal index first.  mode 0: `nms_2d_faster` (camera x /
 *   z extents of the corners), 1: `nms_3d_faster`, 2: `nms_3d_faster_samecls` (sem_cls int32 [B, K]); old_type: overlap over the
 *   other box's area.  Overlaps are fp64 in the reference's expression order; a NaN overlap never suppresses.  A NaN score ranks above
 *   every number (np.argsort sorts it last, so it is picked first); -0.0 ties +0.0.  K <= 1024.
 * pcb_det_box_iou: iou fp64 [n] = `box3d_iou(corners1[i], corners2[i])[0]`, the IoU pcb_det_ap uses (see below), n >= 1.
 * pcb_det_ap: VOC average precision (`eval_det_cls`, `voc_ap`) for T <= 64 IoU thresholds (host fp64 [T]) at once.  Detections d < D:
 *   proposal row det_row (into prop_corners [P, 8, 3]), class det_cls, score det_score (fp32), scan det_scan; a class outside [0, C)
 *   marks a slot that is not a detection.  Ground truth g < G: gt_corners [G, 8, 3], gt_scan, gt_cls (outside [0, C): ignored).  Within
 *   a class detections rank by descending score, ties in input order (a stable sort); ground truth of one (scan, class) keeps input
 *   order for the first-maximal-j rule.  IoU is `box3d_iou` (Sutherland-Hodgman, convex-hull area, degenerate clips area 0), a NaN IoU
 *   never matching.  out fp64 [T, C, 4] = (AP, final recall, npos, ndet): AP and recall NaN for a class with detections but no ground
 *   truth, 0 for one with ground truth but no detections.  D, G, P, C >= 1, C <= 1024.  ws: pcb_det_ap_ws_bytes(D, G, C, T). */
int pcb_det_decode_pred(const float* center, const float* heading_scores, const float* heading_residuals, const float* size_scores,
                        const float* size_residuals, const float* sem_cls_scores, const float* objectness_scores, int64_t B, int64_t K,
                        int H, int S, int C, const double* mean_size, int heading_rule, double* corners, double* box, int32_t* sem_cls,
                        float* obj_prob, float* sem_prob, void* stream);
int pcb_det_decode_gt(const float* center, const int64_t* heading_class, const float* heading_residual, const int64_t* size_class,
                      const float* size_residual, int64_t B, int64_t K, int H, int S, const double* mean_size, int heading_rule,
                      double* corners, double* box, int32_t* status, void* stream);
int pcb_det_points_in_box(const float* points, int64_t B, int64_t N, int ld, const double* box, int64_t K, int32_t* counts, void* stream);
int pcb_det_nms(const double* corners, const float* score, const int32_t* sem_cls, const int32_t* counts, int min_points, int64_t B,
                int64_t K, int mode, int old_type, double nms_iou, int32_t* pred_mask, void* stream);
int pcb_det_box_iou(const double* corners1, const double* corners2, int64_t n, double* iou, void* stream);
size_t pcb_det_ap_ws_bytes(int64_t D, int64_t G, int C, int T);
int pcb_det_ap(const double* prop_corners, int64_t P, const int32_t* det_row, const int32_t* det_cls, const float* det_score,
               const int32_t* det_scan, int64_t D, const double* gt_corners, const int32_t* gt_scan, const int32_t* gt_cls, int64_t G, int C,
               const double* thresholds, int T, double* out, void* ws, size_t ws_bytes, void* stream);

/* VoteNet's training loss (`downstream/votenet_det_new/models/loss_helper.py::get_loss` with `lib/utils/nn_distance.py`, DESIGN.md
 * 8f-12).  Nothing synchronises; no floating-point atomics: every batch sum is fp64 in a fixed order, rounded once, so two calls give
 * the same bits.  Per-element arithmetic is fp32 with one rounding per operation, as the original's torch ops round:
 *   vote:        gt_j = vote_label[seed_inds] (j < 3) + seed_xyz; per GT vote the min over the V predicted votes of (|dx| + |dy|) + |dz|,
 *                then the min over j (ties: smallest index, predicted vote first); sum(dist mask) / (sum(mask) + 1e-6).
 *   assignment:  object_assignment = argmin_j ((dx dx + dy dy) + dz dz) from aggregated_vote_xyz to center_label[:, j, 0:3] over all K2
 *                slots, padded zero slots included; e = sqrtf(d + 1e-6); objectness_label = e < 0.3, objectness_mask = label | e > 0.6.
 *   objectness:  cross-entropy (row maximum subtracted) weighted [0.2, 0.8], masked mean.
 *   center:      nn_distance(center, center_label) both ways: dist1 weighted by objectness_label, dist2 by box_label_mask.
 *   heading / size / semantic: labels gathered through object_assignment; cross-entropy; Huber (delta 1) of the chosen residual minus
 *                heading_residual_label * heading_scale, and of the chosen size residual minus size_residual_label / mean_size (mean of
 *                the 3); each averaged over objectness_label.
 * out fp32 [13] = (vote_loss, objectness_loss, center_loss, heading_cls_loss, heading_reg_loss, size_cls_loss, size_reg_loss,
 * sem_cls_loss, box_loss, loss (x10), pos_ratio, neg_ratio, obj_acc).  A seed index outside [0, N) or a gathered heading, size or
 * semantic class outside its range (where torch raises a device assert) reads nothing out of bounds and makes the affected terms NaN.
 *
 * Inputs, described once by pcb_det_loss_args: seed_xyz fp32 [B,S,3], seed_inds int32 or int64 (seed_inds_i64) [B,S], vote_xyz fp32
 * [B,S*V,3], vote_label fp32 [B,N,9], vote_label_mask int64 [B,N], aggregated_vote_xyz fp32 [B,K,3] (all contiguous); the proposal head's
 * outputs through their element strides (`decode_scores` slices them from one [B, X, K] tensor): center [B,K,3], objectness_scores
 * [B,K,2], heading_scores / heading_residuals_normalized [B,K,NH], size_scores [B,K,NS], size_residuals_normalized [B,K,NS,3],
 * sem_cls_scores [B,K,C]; labels center_label fp32 [B,K2,center_label_ld >= 3], heading_class_label / size_class_label /
 * sem_cls_label int64 [B,K2], heading_residual_label fp32 [B,K2], size_residual_label fp32 [B,K2,3], box_label_mask fp32 [B,K2];
 * mean_size HOST fp32 [NS, 3] (NS <= 64, copied into the launch); heading_scale = 1 / fp32(pi / NH), which is how torch divides an fp32
 * tensor by a Python float on the GPU.
 *
 * pcb_det_loss_forward: out, objectness_label int64 [B,K], objectness_mask fp32 [B,K], object_assignment int64 [B,K], and `state`
 * (pcb_det_loss_state_bytes: the argmins and denominators the backward reads; keep it until then).  Two launches.
 * pcb_det_loss_backward: grad fp32 [13] = d/d out (box_loss and loss fold into the eight terms by their coefficients; the statistics
 * carry none), with the forward's objectness_label, objectness_mask, object_assignment and state.  Writes dense fp32 gradients, each in
 * full and each skipped when NULL: d_vote_xyz [B,S*V,3], d_seed_xyz [B,S,3], d_center [B,K,3], d_objectness_scores [B,K,2],
 * d_heading_scores / d_heading_residuals_normalized [B,K,NH], d_size_scores [B,K,NS], d_size_residuals_normalized [B,K,NS,3],
 * d_sem_cls_scores [B,K,C].  A min passes its gradient to the index it returned only, |x|' = 0 at 0, and the dist2 gradients of several
 * ground-truth boxes on one proposal sum in ascending box order.  One launch.
 * Both: a size below 1, B > 65535, NS > 64, center_label_ld < 3, B * max(S V, K, N) >= 2^31, NULL pointers and short ws / state
 * return PCB_ERR_ARG before anything is launched.  ws: pcb_det_loss_ws_bytes (forward only). */
typedef struct pcb_strided {
  const float* p;
  int64_t sb, sk, sc, sx;                    /* element strides of (scene, proposal, channel, xyz); sx only for size residuals */
} pcb_strided;
typedef struct pcb_det_loss_args {
  int64_t B, S, V, N, K, K2;
  int32_t NH, NS, C, seed_inds_i64;
  float heading_scale;
  const float* mean_size;
  const float* seed_xyz; const void* seed_inds; const float* vote_xyz; const float* vote_label; const int64_t* vote_label_mask;
  const float* aggregated_vote_xyz;
  pcb_strided center, objectness_scores, heading_scores, heading_residuals_normalized, size_scores, size_residuals_normalized,
      sem_cls_scores;
  const float* center_label; int64_t center_label_ld;
  const int64_t* heading_class_label; const float* heading_residual_label; const int64_t* size_class_label;
  const float* size_residual_label; const int64_t* sem_cls_label; const float* box_label_mask;
} pcb_det_loss_args;
size_t pcb_det_loss_ws_bytes(int64_t B, int64_t S, int64_t K, int64_t K2);
size_t pcb_det_loss_state_bytes(int64_t B, int64_t S, int64_t K, int64_t K2);
int pcb_det_loss_forward(const pcb_det_loss_args* args, float* out, int64_t* objectness_label, float* objectness_mask,
                         int64_t* object_assignment, void* state, size_t state_bytes, void* ws, size_t ws_bytes, void* stream);
int pcb_det_loss_backward(const pcb_det_loss_args* args, const float* grad, const int64_t* objectness_label, const float* objectness_mask,
                          const int64_t* object_assignment, const void* state, size_t state_bytes, float* d_vote_xyz, float* d_seed_xyz,
                          float* d_center, float* d_objectness_scores, float* d_heading_scores, float* d_heading_residuals_normalized,
                          float* d_size_scores, float* d_size_residuals_normalized, float* d_sem_cls_scores, void* stream);

/* ----------------------------------------------------------------------------------------------- VoteNet detection data (det_data.cu)
 * A batch of B ScanNet or SUN RGB-D detection scenes (`lib/datasets/{scannet,sunrgbd}/*_detection_dataset.py` `__getitem__`) as ragged
 * rows: scene b's source points are rows [offsets[b], offsets[b+1]) of the concatenated arrays (every scene non-empty), its boxes rows
 * [box_offsets[b], box_offsets[b+1]) of `boxes` (at most PCB_DET_MAX_OBJ).  Offsets are given twice, on the host (checked: start at 0,
 * monotone, end at M / the box count) and on the device (read by the kernels).  Arithmetic is the original's: fp32 where numpy's is fp32,
 * fp64 where it is fp64, one rounding per operation and no contraction; its 3-term dot products sum in index order.
 *
 * pcb_det_floor_height: floor[b] = np.percentile(z of scene b, 0.99) with numpy's `linear` rule (virtual index (n-1) q in the data's type,
 * a + (b-a) t, or b - (b-a)(1-t) where t >= 0.5), z read at element stride `stride` from fp32 (f64 = 0) or fp64 (f64 = 1) rows; the
 * result is exact in fp64.  Two order statistics by radix selection, one CTA per scene, one launch.
 * pcb_det_choices: out [B, k] int64 scene-local indices, `np.random.choice(n_b, k, replace=n_b < k)`: the first k of a random order of
 * the scene (sorted random 64-bit keys, the scene's bits on top) when n_b >= k, else k iid uniform indices; from a Philox4x32-10 stream
 * keyed by (seed, offset), so equal generator states give equal sets.  ws: pcb_det_choices_ws_bytes(M).
 * pcb_det_points: the sampled rows' point_clouds fp32 [B, k, C], vote_label fp32 [B, k, 9], vote_label_mask int64 [B, k] and, ScanNet,
 * pcl_color fp32 [B, k, 3].  ScanNet: flips, z-rotation (fp64, rounded to fp32) and the floor height column; then the instance votes:
 * per (scene, instance id) the fp32 min / max of the sampled rows (order-independent atomics), applied when the semantic label of the
 * instance's first sampled row is in nyu40ids.  SUN RGB-D: flip, rotation of points and vote end points, colour, scale, all fp64.
 * A choice outside [0, n_b) reads nothing out of bounds: its row takes the scene's first point and NaN coordinates.
 * ws: pcb_det_points_ws_bytes(B, k).
 * pcb_det_boxes: the box labels of every scene in fp64, one launch: center_label fp32 [B,64,3], heading_class_label int64 [B,64],
 * heading_residual_label fp32 [B,64], size_class_label int64 [B,64], size_residual_label fp32 [B,64,3], sem_cls_label int64 [B,64],
 * box_label_mask fp32 [B,64] and, SUN RGB-D, max_gt_bboxes fp64 [B,64,8].
 * Sizes below 1, B * k >= 2^31, M >= 2^31, bad offsets, a scene with more than 64 boxes, NULL pointers and short ws return PCB_ERR_ARG
 * before anything is launched. */
#define PCB_DET_MAX_OBJ 64
#define PCB_DET_SCANNET 0
#define PCB_DET_SUNRGBD 1
#define PCB_DET_HEIGHT 1          /* pcb_det_batch.flags: a floor-height column */
#define PCB_DET_COLOR 2           /* colour columns (SUN RGB-D only) */
#define PCB_DET_AUGMENT 4         /* apply the per-scene draws in `params` */
#define PCB_DET_NPARAM 11         /* params per scene: flip_x, flip_y, cos, sin of the rotation, scale, brightness[3], shift[3] */
typedef struct pcb_det_batch {
  int64_t B, M, num_points;                  /* scenes, source rows in all, sampled rows per scene (k) */
  int32_t dataset, flags;                    /* PCB_DET_SCANNET / PCB_DET_SUNRGBD, PCB_DET_* flags */
  const int64_t* offsets_host; const int64_t* offsets;              /* [B + 1] */
  const int64_t* box_offsets_host; const int64_t* box_offsets;      /* [B + 1] */
  const double* params;                      /* [B, PCB_DET_NPARAM] */
  const double* floor;                       /* [B] pcb_det_floor_height (PCB_DET_HEIGHT) */
  const int64_t* choices;                    /* [B, k] pcb_det_choices */
  const float* vert; const uint32_t* sem; const uint32_t* ins;      /* ScanNet: [M, 6], [M], [M] */
  const double* pc; const double* votes;     /* SUN RGB-D: [M, 6], [M, 10] */
  const double* jitter; const double* dropout;                      /* SUN RGB-D colour draws [M] (PCB_DET_COLOR with augmentation) */
  const double* boxes;                       /* [box count, 7] (ScanNet) or [box count, 8] (SUN RGB-D) */
  const double* headings;                    /* SUN RGB-D [box count, 3]: augmented heading, cos and sin of minus it (numpy's values) */
  const int64_t* nyu40ids; int32_t n_ids;    /* ScanNet: the detected nyu40 ids */
  int32_t num_heading_bin;
  const double* mean_size; int32_t n_size;   /* [n_size, 3] */
  int32_t pad_;
  float* point_clouds; float* pcl_color; float* vote_label; int64_t* vote_label_mask;
  float* center_label; int64_t* heading_class_label; float* heading_residual_label; int64_t* size_class_label;
  float* size_residual_label; int64_t* sem_cls_label; float* box_label_mask; double* max_gt_bboxes;
} pcb_det_batch;
int pcb_det_floor_height(const void* z, int64_t stride, int32_t f64, const int64_t* offsets_host, const int64_t* offsets, int64_t B,
                         double* floor, void* stream);
size_t pcb_det_choices_ws_bytes(int64_t M);
int pcb_det_choices(const int64_t* offsets_host, const int64_t* offsets, int64_t B, int64_t k, uint64_t seed, uint64_t offset, int64_t* out,
                    void* ws, size_t ws_bytes, void* stream);
size_t pcb_det_points_ws_bytes(int64_t B, int64_t k);
int pcb_det_points(const pcb_det_batch* a, void* ws, size_t ws_bytes, void* stream);
int pcb_det_boxes(const pcb_det_batch* a, void* stream);
/* Row-wise L2 normalisation of the output features, y = x / ||x||_2 with no epsilon (`model/res16unet.py:262-266`), and its
 * backward dx = (dy - y (y.dy)) / ||x||.  inv_norm: [n] scratch written by forward, read by backward.
 * Without an epsilon a row whose fp32 sum of squares is 0 -- a zero row, or one whose squares all underflow -- gets inv_norm = +inf
 * and y = x * inf (NaN at its zeros, +-inf elsewhere); a row whose sum of squares overflows gets inv_norm = 0 and y = +-0.  These are
 * the bits of x / torch.norm(x, p=2, dim=1, keepdim=True) in fp32 on CUDA for C >= 2 (at C = 1 torch's norm is |x|, so its
 * expression gives +-1 where this gives x / sqrt(x^2) with the same edges). */
int pcb_l2norm_forward(const float* X, int64_t n, int C, float* Y, float* inv_norm, void* stream);
int pcb_l2norm_backward(const float* dY, const float* Y, const float* inv_norm, int64_t n, int C, float* dX, void* stream);
/* minval[i] = min_j sqrt(sum_d (A[i,d]-B[j,d])^2 + 1e-7), argmin[i] = smallest such j.   packed: u64 scratch [P]. */
int pcb_pdist_rowmin(const float* A, int64_t P, const float* B, int64_t S, int D, float* minval, int32_t* argmin,
                     uint64_t* packed, void* stream);

/* ----------------------------------------------------------------------------------------------- PointNet++ operators (DESIGN.md 8f-5) */
/* The native operators of VoteNet's PointNet++ backbone and heads (`downstream/votenet_det_new/models/backbone/pointnet2/_ext_src`),
 * with their shapes: xyz fp32 [B, N, 3], features fp32 [B, C, N] (channels first), indices int32.  Distances are fp32 with one
 * rounding per operation, d = ((dx*dx + dy*dy) + dz*dz): index results are bit-reproducible on the host.  Sizes >= 2^31, npoint < 1,
 * nsample < 1 and radius <= 0 return PCB_ERR_ARG before anything is launched.
 *
 * Furthest-point sampling: idx [B, npoint]; idx[0] = 0, running min-distance from 1e10, points with |p|^2 <= 1e-3 never chosen (index 0
 * when nothing is left); ties go to the SMALLEST index.  One thread-block cluster per scene.  ws: pcb_furthest_point_sampling_ws_bytes
 * (0 unless N exceeds what a cluster holds on chip; ws may then be NULL). */
size_t pcb_furthest_point_sampling_ws_bytes(int64_t B, int64_t N);
int pcb_furthest_point_sampling(const float* xyz, int64_t B, int64_t N, int64_t npoint, int32_t* idx, void* ws, size_t ws_bytes, void* stream);
/* idx [B, M, nsample]: the first nsample k (ascending) with |new_xyz[m] - xyz[k]|^2 < radius^2; the remaining slots repeat the first hit;
 * a row with no hit is all zeros. */
int pcb_ball_query(const float* new_xyz, const float* xyz, int64_t B, int64_t M, int64_t N, float radius, int nsample, int32_t* idx,
                   void* stream);
/* dist2, idx [B, n, 3]: the three nearest known points of each unknown point (squared distances; ties keep the earlier k); when m < 3
 * the missing entries are dist2 = inf, idx = 0. */
int pcb_three_nn(const float* unknown, const float* known, int64_t B, int64_t n, int64_t m, float* dist2, int32_t* idx, void* stream);
/* out[b, c, p] = features[b, c, idx[b, p]], p < L: gather_points (idx [B, M], L = M) and group_points (idx [B, M, S], L = M * S,
 * out [B, C, M, S]).  An index outside [0, N) reads 0. */
int pcb_gather_points(const float* features, const int32_t* idx, int64_t B, int64_t C, int64_t N, int64_t L, float* out, void* stream);
/* out[b, c, j] = (f[i1] * w1 + f[i2] * w2) + f[i3] * w3 over features [B, C, m], idx / weight [B, n, 3]; out [B, C, n]. */
int pcb_three_interpolate(const float* features, const int32_t* idx, const float* weight, int64_t B, int64_t C, int64_t m, int64_t n,
                          float* out, void* stream);
/* Adjoints, deterministic: every source point's readers are listed in ascending output position (stable radix sort of the index
 * tensor) and summed in that order in fp64; grad_features is written in full (zeros where nothing reads).  ws: pcb_points_grad_ws_bytes(B,
 * N, L) with L = readers per scene (M, M * S; 3 * n for three_interpolate, whose source count is m). */
size_t pcb_points_grad_ws_bytes(int64_t B, int64_t N, int64_t L);
int pcb_gather_points_grad(const float* grad_out, const int32_t* idx, int64_t B, int64_t C, int64_t N, int64_t L, float* grad_features,
                           void* ws, size_t ws_bytes, void* stream);
int pcb_three_interpolate_grad(const float* grad_out, const int32_t* idx, const float* weight, int64_t B, int64_t C, int64_t n, int64_t m,
                               float* grad_features, void* ws, size_t ws_bytes, void* stream);

/* ----------------------------------------------------------------------------------------------- sparse-conv detection backbone (8f-7) */
/* Batched voxelisation of a collated VoteNet batch, xyz fp32 [B, N, 3] (`downstream/votenet_det_new/models/backbone/sparseconv/
 * voxelized_dataset.py:33-65`: per scene floor(xyz / voxel_size) in fp32, `ME.utils.sparse_quantize(coords, return_index=True)`).
 * One row per occupied (scene, voxel), scene-major, ascending first index within a scene: out_coords int32 [M, 4] = (b, x, y, z),
 * inds int32 [M] = the scene-local index of the voxel's first (smallest-index) point, offsets int64 [B + 1] (device): scene b is rows
 * [offsets[b], offsets[b+1]).  out_coords / inds hold up to B * N rows.  SYNCHRONISES once: offsets_host (host, B + 1 entries) receives
 * the offsets, M = offsets_host[B].  A cell index outside +-2^20 returns PCB_ERR_RANGE.  B < 1, N < 1, voxel_size <= 0, NULL pointers
 * and a short workspace return PCB_ERR_ARG. */
size_t pcb_voxelize_scenes_ws_bytes(int64_t B, int64_t N);
int pcb_voxelize_scenes(const float* xyz, int64_t B, int64_t N, float voxel_size, int32_t* out_coords, int32_t* inds, int64_t* offsets,
                        int64_t* offsets_host, void* ws, size_t ws_bytes, void* stream);
/* Furthest-point sampling of B scenes of different sizes in one launch: points fp32 [M, 3] grouped by scene, device offsets [B + 1]
 * (scene b is rows [offsets[b], offsets[b+1])), max_n an upper bound on every scene's size (sizes the clusters and the workspace; a
 * bound above M counts as M).  idx [B, npoint] of scene-local indices, for every scene identical to pcb_furthest_point_sampling on that
 * scene alone.  A scene that is empty, larger than max_n or outside [0, M) gets -1 in every slot.  B < 1, M < B, max_n < 1 and NULL
 * pointers return PCB_ERR_ARG.  ws: pcb_furthest_point_sampling_ragged_ws_bytes (0 unless max_n exceeds what a cluster holds on chip). */
size_t pcb_furthest_point_sampling_ragged_ws_bytes(int64_t B, int64_t M, int64_t max_n);
int pcb_furthest_point_sampling_ragged(const float* xyz, const int64_t* offsets, int64_t B, int64_t M, int64_t max_n, int64_t npoint,
                                       int32_t* idx, void* ws, size_t ws_bytes, void* stream);
/* Adjoint of the row gather out[p, :] = rows[idx[p], :], p < L, over rows fp32 [M, C] (row-major): grad_rows [M, C] written in full,
 * each row the fp64 sum of its readers' gradients in ascending p (deterministic; an index outside [0, M) is read by nobody).
 * ws: pcb_points_grad_ws_bytes(1, M, L). */
int pcb_gather_rows_grad(const float* grad_out, const int32_t* idx, int64_t L, int64_t C, int64_t M, float* grad_rows, void* ws,
                         size_t ws_bytes, void* stream);

/* ----------------------------------------------------------------------------------------------- PointNet++ shared MLPs (8f-16) */
/* The two ends of a set-abstraction module's shared MLP (`pointnet2_modules.py` PointnetSAModuleVotes, `pytorch_utils.py` SharedMLP) that
 * differ from a plain 1x1 convolution; the layers between are pcb_unit_* calls on a K = 1 identity table.  Rows are point-major: row
 * r = (b npoint + i) S + s is sample s of centre i of scene b (M = B npoint centres, R = M S rows).  All fp32 with one rounding per
 * operation, no contraction except inside the BatchNorm expression; nothing synchronises.
 *
 * pcb_sa_layer0: the first layer without the grouped [R, 3 + C] input.  rel[r] (fp32 [R, 3]) = (xyz[b, j] - new_xyz[b, i]), then / radius
 *   when radius > 0 (the original's normalize_xyz; 0: no division), j = idx[r] (int32 [B, npoint, S], ball query), and
 *   z[r, c] = P[b N + j, c] + ((rel_0 Wx[0][c] + rel_1 Wx[1][c]) + rel_2 Wx[2][c]) for c < C0 (row stride ldz), where Wx (fp32 [3][C0])
 *   holds the layer's three xyz columns and P (fp32 [B N, C0], row stride ldp, or NULL for a module without features) = the feature
 *   columns applied to every point once.  gidx[r] = b N + j (int32 [R]), -1 where j lies outside [0, N) (that row then reads zeros).
 * pcb_sa_pool: the last layer's BatchNorm -> ReLU -> max over the S samples of each centre, by selection: sel[i, c] (int32 [M, C]) = the
 *   slot of the largest z (gamma[c] >= 0) or of the smallest z (gamma[c] < 0), the smallest slot among equals, and
 *   out[i, c] (row stride ldo) = max(0, (z - mean) invstd gamma + beta) at that slot.  invstd > 0 and every rounding is monotone, so out
 *   equals the maximum of the same expression over all S slots bit for bit.  mean / invstd: pcb_bn_stats_seg (training) or the running
 *   statistics.
 * pcb_sa_pool_grad: dY (fp32 [R, C], written in full) = g[i, c] (row stride ldg) on the selected slot where out[i, c] > 0, else 0: the
 *   gradient of the pre-pool activation, for pcb_bn_backward_seg on z.
 * pcb_sa_xyz_rows: rows (fp32 [R + M, 3]) for pcb_gather_rows_grad over the index list [gidx | b N + inds]: rows[r] = grel[r] / radius
 *   (radius > 0; grel[r] itself otherwise), grel = the gradient of rel, and rows[R + i] = d_new_xyz[i] (fp32 [M, 3] or NULL: 0) minus the
 *   sum of centre i's S rows in ascending s.
 * Sizes below 1, R, M C or B N >= 2^31, a NaN radius, strides below the widths and NULL pointers return PCB_ERR_ARG before the launch. */
int pcb_sa_layer0(const float* xyz, const float* new_xyz, const int32_t* idx, int64_t B, int64_t N, int64_t npoint, int S, float radius,
                  const float* P, int ldp, const float* Wx, int C0, float* rel, int32_t* gidx, float* z, int ldz, void* stream);
int pcb_sa_pool(const float* z, int ldz, int64_t M, int S, int C, const float* mean, const float* invstd, const float* gamma,
                const float* beta, int32_t* sel, float* out, int ldo, void* stream);
int pcb_sa_pool_grad(const float* g, int ldg, const int32_t* sel, const float* out, int ldo, int64_t M, int S, int C, float* dY,
                     void* stream);
int pcb_sa_xyz_rows(const float* grel, const float* d_new_xyz, int64_t M, int S, float radius, float* rows, void* stream);

/* ----------------------------------------------------------------------------------------------- VoteNet heads (8f-18) */
/* The elementwise ends of VoteNet's voting module (`models/voting_module.py`) and proposal head (`models/proposal_module.py`
 * decode_scores) around their last 1x1 convolution, whose output z (fp32, point-major rows, row stride ldz) the caller computes with
 * pcb_conv_forward_split; the layers before it are pcb_unit_* calls on a K = 1 identity table.  Forward arithmetic is the original's
 * torch expressions on the same z, one rounding per operation: the outputs are bit-identical to them.  Every output element is written
 * by one thread (deterministic, no atomics).  Gradients are read through pcb_strided element strides (NULL, or a NULL `p`: absent, read
 * as 0); the gradient of z comes out as bf16 hi/lo planes (the gradient operand of pcb_conv_wgrad_split / pcb_conv_forward_split).
 *
 * pcb_vote_epilogue: seed rows r = b S + s, V votes per seed, C feature channels, z [B S, >= (3 + C) V] with vote v in columns
 *   [v (3 + C), (v + 1)(3 + C)): vote_xyz (fp32 [B, S V, 3], contiguous) = seed_xyz[b, s] + z[r, v (3 + C) + 0..2], and vote_features
 *   (fp32 [B S V, C], point-major: row r V + v) = seed_features[r] (row stride ldf) + z[r, v (3 + C) + 3 + c].
 * pcb_vote_epilogue_grad: d_vote_xyz (scene, vote, axis) and d_vote_features (scene, vote, channel) -> dz_hi / dz_lo [B S, ldz], columns
 *   [0, Cpad) written (0 beyond (3 + C) V); d_seed_features (fp32 [B S, C], row stride ldd, or NULL) = sum over v of d_vote_features
 *   and d_seed_xyz (fp32 [B, S, 3] or NULL) = sum over v of d_vote_xyz, in ascending v: the residual paths.
 * pcb_proposal_epilogue: z [B K, >= X] in decode_scores' column order (objectness 2, center 3, heading scores NH, heading residuals NH,
 *   size scores NS, size residuals 3 NS, semantic classes), aggregated_vote_xyz fp32 [B, K, 3]: center [B, K, 3] = aggregated_vote_xyz +
 *   z[:, 2:5]; heading_residuals [B, K, NH] = z[:, 5+NH : 5+2NH] * heading_unit (fp32(pi / NH): torch's fp32 tensor times a Python
 *   float); size_residuals [B, K, NS, 3] = the size-residual columns * mean_size (HOST fp32 [NS, 3], NS <= 64, copied into the launch).
 * pcb_proposal_epilogue_grad: grads = HOST array of 9 pcb_strided in decode_scores' end_points order -- objectness_scores, center,
 *   heading_scores, heading_residuals_normalized, heading_residuals, size_scores, size_residuals_normalized (sx: the axis stride),
 *   size_residuals (sx too), sem_cls_scores -- each with strides (scene, proposal, channel).  dz (columns [0, Xpad), 0 beyond X =
 *   5 + 2 NH + 4 NS + C) = the gradient of the view reading each column, the residual columns plus heading_unit x d heading_residuals
 *   and mean_size x d size_residuals; written as bf16 hi/lo planes (dz_hi / dz_lo) and / or fp32 (dz), each NULL to skip, row stride ldz.
 *   d_aggregated_vote_xyz (fp32 [B, K, 3] or NULL) = the center gradient.
 * Sizes below 1, B S V or B K >= 2^31, NS > 64, strides below the widths and NULL required pointers return PCB_ERR_ARG before the
 * launch. */
int pcb_vote_epilogue(const float* seed_xyz, const float* seed_features, int ldf, const float* z, int ldz, int64_t B, int64_t S, int V,
                      int C, float* vote_xyz, float* vote_features, void* stream);
int pcb_vote_epilogue_grad(const pcb_strided* d_vote_xyz, const pcb_strided* d_vote_features, int64_t B, int64_t S, int V, int C,
                           uint16_t* dz_hi, uint16_t* dz_lo, int ldz, int Cpad, float* d_seed_features, int ldd, float* d_seed_xyz,
                           void* stream);
int pcb_proposal_epilogue(const float* z, int ldz, const float* aggregated_vote_xyz, int64_t B, int64_t K, int NH, int NS,
                          float heading_unit, const float* mean_size, float* center, float* heading_residuals, float* size_residuals,
                          void* stream);
int pcb_proposal_epilogue_grad(const pcb_strided* grads, int64_t B, int64_t K, int NH, int NS, int C, float heading_unit,
                               const float* mean_size, uint16_t* dz_hi, uint16_t* dz_lo, float* dz, int ldz, int Xpad,
                               float* d_aggregated_vote_xyz, void* stream);

/* ----------------------------------------------------------------------------------------------- optimiser */
/* torch.optim.SGD semantics on a flat buffer:  d = g*grad_scale + wd*p;  buf = first ? d : momentum*buf + (1-dampening)*d;  p -= lr*buf
 * (pretraining: dampening 0, `lib/ddp_trainer.py:107-111`; semseg finetuning: 0.1, `downstream/semseg/lib/solvers.py:50-57`) */
int pcb_sgd_step(float* p, const float* g, float* buf, int64_t n, float lr, float momentum, float weight_decay,
                 float grad_scale, int first, float dampening, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PCB200_H_ */
