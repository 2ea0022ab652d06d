// VoteNet detection evaluation (`downstream/votenet_det_new/models/ap_helper.py`, `lib/utils/{nms,eval_det,box_util}.py`) on the device:
//   * pcb_det_decode_pred / pcb_det_decode_gt: one thread per proposal / label -- argmaxes, residual gathers and fp32 softmaxes
//     (predictions), then the 8 corners in upright-camera coordinates from ONE box routine shared by both sides (fp64)
//   * pcb_det_points_in_box: points of each scene inside each box (`remove_empty_box`), points tiled through shared memory
//   * pcb_det_nms: one CTA per scene -- rank the candidates, build the K x K "suppresses" bitmask in parallel, one warp walks it
//   * pcb_det_ap: oriented IoU of every detection against the ground truth of its (scan, class), one stable radix sort of (class,
//     descending score) keys (sort.cuh), VOC matching by an integer atomicMin of the sorted rank per ground-truth box, and per class the
//     cumulative counts, the precision envelope and the AP sum in a fixed order.
// Every fp64 expression below is written with __dmul_rn / __dadd_rn / __dsub_rn where the reference rounds once per operation, so the
// compiler cannot contract it into an FMA; only integer atomics are used.
#include <cub/cub.cuh>
#include "sort.cuh"

using namespace pcb;

namespace {

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
// np.maximum / np.minimum: a NaN operand gives NaN
__device__ __forceinline__ double np_max(double a, double b) { return (isnan(a) || isnan(b)) ? (double)NAN : (a > b ? a : b); }
__device__ __forceinline__ double np_min(double a, double b) { return (isnan(a) || isnan(b)) ? (double)NAN : (a < b ? a : b); }

// torch.argmax: the first index among the maximal values, a NaN counting as maximal
__device__ __forceinline__ int argmax_first(const float* x, int n) {
  int bi = 0;
  float bv = x[0];
  for (int i = 1; i < n && !isnan(bv); ++i)
    if (x[i] > bv || isnan(x[i])) { bv = x[i]; bi = i; }
  return bi;
}

// numpy's fp32 sum along a contiguous row (pairwise_sum of numpy's loops_utils.h: a plain loop below 8 items, 8 running sums up to
// 128, halves split at a multiple of 8 above), starting from 0 as np.sum does.  Unrolled to depth 3, enough for n <= 1024.
__device__ __forceinline__ float np_block_sum(const float* a, int n) {
  if (n < 8) {
    float r = 0.f;
    for (int i = 0; i < n; ++i) r = __fadd_rn(r, a[i]);
    return r;
  }
  float r[8];
  for (int j = 0; j < 8; ++j) r[j] = a[j];
  int i = 8;
  for (; i < n - (n % 8); i += 8)
    for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], a[i + j]);
  float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])), __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
  for (; i < n; ++i) res = __fadd_rn(res, a[i]);
  return res;
}
template <int DEPTH> __device__ __forceinline__ float np_pairwise_sum(const float* a, int n) {
  if constexpr (DEPTH == 0) {
    return np_block_sum(a, n);
  } else {
    if (n <= 128) return np_block_sum(a, n);
    int h = n / 2;
    h -= h % 8;
    return __fadd_rn(np_pairwise_sum<DEPTH - 1>(a, h), np_pairwise_sum<DEPTH - 1>(a + h, n - h));
  }
}

// `softmax` of ap_helper.py:33-38 over one fp32 row: e = exp(x - max) rounded to fp32 (exp in fp64), p = e / (np.sum of e)
__device__ void np_softmax(const float* x, int n, float* e) {
  float m = x[0];
  for (int i = 1; i < n; ++i) m = fmaxf(m, x[i]);
  for (int i = 0; i < n; ++i) e[i] = (float)exp((double)__fsub_rn(x[i], m));
}

// The box routine of both sides: `get_3d_box(box_size, heading_angle, center)` (box_util.py:210-225) with R = roty(angle), one rounding
// per operation: corner k = (c x_k + s z_k, y_k, -s x_k + c z_k) + center, x = +-l/2, y = +-h/2, z = +-w/2 in the reference's order.
// box: (cx, cy, cz) upright camera, (l, w, h), (cos, sin) -- what pcb_det_points_in_box reads back.
__device__ void build_box(double cx, double cy, double cz, double l, double w, double h, double angle, double* corners, double* box) {
  const double c = cos(angle), s = sin(angle);
  const double hl = l / 2, hw = w / 2, hh = h / 2;
  const double xs[8] = {hl, hl, -hl, -hl, hl, hl, -hl, -hl};
  const double ys[8] = {hh, hh, hh, hh, -hh, -hh, -hh, -hh};
  const double zs[8] = {hw, -hw, -hw, hw, hw, -hw, -hw, hw};
  for (int k = 0; k < 8; ++k) {
    // np.dot row i of R: (R[i,0] x + R[i,1] y) + R[i,2] z; the zero / unit entries of roty are exact
    corners[3 * k + 0] = add(add(mul(c, xs[k]), mul(0.0, ys[k])), mul(s, zs[k])) + cx;
    corners[3 * k + 1] = add(add(mul(0.0, xs[k]), mul(1.0, ys[k])), mul(0.0, zs[k])) + cy;
    corners[3 * k + 2] = add(add(mul(-s, xs[k]), mul(0.0, ys[k])), mul(c, zs[k])) + cz;
  }
  box[0] = cx; box[1] = cy; box[2] = cz; box[3] = l; box[4] = w; box[5] = h; box[6] = c; box[7] = s;
}

// `class2angle`: rule 0 (ScanNet) returns 0; rule 1 (SUN RGB-D) cls * 2 pi / H + residual, minus 2 pi above pi
__device__ __forceinline__ double heading(int rule, int64_t cls, double residual, int H) {
  if (rule == 0) return 0.0;
  const double per = 2 * M_PI / (double)H;
  double a = add(mul((double)cls, per), residual);
  if (a > M_PI) a = sub(a, 2 * M_PI);
  return a;
}

constexpr int MAX_CLS = 1024;

__global__ void decode_pred_kernel(const float* __restrict__ center, const float* __restrict__ hs, const float* __restrict__ hr,
                                   const float* __restrict__ ss, const float* __restrict__ sr, const float* __restrict__ cs,
                                   const float* __restrict__ os, int64_t BK, int H, int S, int C, const double* __restrict__ mean_size,
                                   int rule, double* __restrict__ corners, double* __restrict__ box, int32_t* __restrict__ sem_cls,
                                   float* __restrict__ obj_prob, float* __restrict__ sem_prob) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= BK) return;
  const int hc = argmax_first(hs + i * H, H);
  const int sc = argmax_first(ss + i * S, S);
  const float* x = cs + i * C;
  sem_cls[i] = argmax_first(x, C);
  float* p = sem_prob + i * C;
  np_softmax(x, C, p);
  const float sum = np_pairwise_sum<3>(p, C);
  for (int c = 0; c < C; ++c) p[c] = __fdiv_rn(p[c], sum);
  float e[2];
  np_softmax(os + i * 2, 2, e);
  obj_prob[i] = __fdiv_rn(e[1], __fadd_rn(__fadd_rn(0.f, e[0]), e[1]));
  const double a = heading(rule, hc, (double)hr[i * H + hc], H);
  const float* r = sr + (i * S + sc) * 3;
  const double* ms = mean_size + sc * 3;
  // center: flip_axis_to_camera (x, y, z) -> (x, -z, y)
  build_box((double)center[i * 3], -(double)center[i * 3 + 2], (double)center[i * 3 + 1], ms[0] + (double)r[0], ms[1] + (double)r[1],
            ms[2] + (double)r[2], a, corners + i * 24, box + i * 8);
}

__global__ void decode_gt_kernel(const float* __restrict__ center, const int64_t* __restrict__ hc, const float* __restrict__ hr,
                                 const int64_t* __restrict__ scl, const float* __restrict__ sr, int64_t BK, int H, int S,
                                 const double* __restrict__ mean_size, int rule, double* __restrict__ corners, double* __restrict__ box,
                                 int32_t* __restrict__ status) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= BK) return;
  const int64_t sc = scl[i];
  if (sc < 0 || sc >= S || (rule == 1 && (hc[i] < 0 || hc[i] >= H))) { atomicOr(status, PCB_ERR_RANGE); return; }
  const double a = heading(rule, hc[i], (double)hr[i], H);
  const double* ms = mean_size + sc * 3;
  build_box((double)center[i * 3], -(double)center[i * 3 + 2], (double)center[i * 3 + 1], ms[0] + (double)sr[i * 3],
            ms[1] + (double)sr[i * 3 + 1], ms[2] + (double)sr[i * 3 + 2], a, corners + i * 24, box + i * 8);
}

// ------------------------------------------------------------------------------------------------ points per box
// grid (scene, block of 32 boxes, point split); lane = box, warp = a stride of the point tile.  Point p (depth) in camera coordinates is
// (x, -z, y); in the box frame lx = c dx - s dz, ly = dy, lz = s dx + c dz; inside iff |lx| <= |l|/2, |ly| <= |h|/2, |lz| <= |w|/2.
constexpr int PIB_THREADS = 256, PIB_TILE = 1024, PIB_SPLIT = 4096;
__global__ void __launch_bounds__(PIB_THREADS) points_in_box_kernel(const float* __restrict__ pts, int64_t N, int ld,
                                                                    const double* __restrict__ box, int K, int32_t* __restrict__ counts) {
  __shared__ float3 sp[PIB_TILE];
  __shared__ int red[PIB_THREADS];
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int j = blockIdx.y * 32 + lane;
  double cx = 0, cy = 0, cz = 0, hl = -1, hw = -1, hh = -1, c = 1, s = 0;
  if (j < K) {
    const double* q = box + ((int64_t)b * K + j) * 8;
    cx = q[0]; cy = q[1]; cz = q[2]; hl = fabs(q[3]) / 2; hw = fabs(q[4]) / 2; hh = fabs(q[5]) / 2; c = q[6]; s = q[7];
  }
  const int64_t p0 = (int64_t)blockIdx.z * PIB_SPLIT, p1 = min(N, p0 + PIB_SPLIT);
  int cnt = 0;
  for (int64_t t0 = p0; t0 < p1; t0 += PIB_TILE) {
    const int n = (int)min((int64_t)PIB_TILE, p1 - t0);
    __syncthreads();
    for (int k = threadIdx.x; k < n; k += PIB_THREADS) {
      const float* p = pts + ((int64_t)b * N + t0 + k) * ld;
      sp[k] = make_float3(p[0], p[1], p[2]);
    }
    __syncthreads();
    for (int k = warp; k < n; k += PIB_THREADS / 32) {
      const float3 p = sp[k];
      const double dx = sub((double)p.x, cx), dy = sub(-(double)p.z, cy), dz = sub((double)p.y, cz);
      const double lx = sub(mul(c, dx), mul(s, dz)), lz = add(mul(s, dx), mul(c, dz));
      cnt += (fabs(lx) <= hl && fabs(dy) <= hh && fabs(lz) <= hw);
    }
  }
  red[threadIdx.x] = cnt;
  __syncthreads();
  if (warp == 0 && j < K) {
    int t = 0;
    for (int w = 0; w < PIB_THREADS / 32; ++w) t += red[w * 32 + lane];
    if (t) atomicAdd(counts + (int64_t)b * K + j, t);
  }
}

// ------------------------------------------------------------------------------------------------ NMS
// One CTA per scene.  Candidates: proposals with counts >= min_points (all when counts is NULL).  Order: descending score, ties by the
// larger proposal index first (np.argsort ascending, picked from the end); a NaN score ranks above +inf, as np.argsort sorts it last, and
// -0.0 ties +0.0.  The order key is a total order, so the ranks are a permutation of [0, n).  sup[a] has bit b set iff the candidate at order a suppresses
// the one at order b > a (o > thresh in the reference's expression, fp64); a warp then walks the order greedily.
constexpr int NMS_THREADS = 512, NMS_MAXK = 1024;
// ascending order of a score as np.sort orders it: -0.0 == +0.0, every NaN above +inf
__device__ __forceinline__ uint32_t score_order(float v) {
  if (isnan(v)) return 0xFFFFFFFFu;
  if (v == 0.f) v = 0.f;
  const uint32_t u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
struct NmsBox { double x1, y1, z1, x2, y2, z2, area; int cls, idx; };

__global__ void __launch_bounds__(NMS_THREADS) nms_kernel(const double* __restrict__ corners, const float* __restrict__ score,
                                                          const int32_t* __restrict__ sem_cls, const int32_t* __restrict__ counts,
                                                          int min_points, int K, int mode, int old_type, double thresh,
                                                          int32_t* __restrict__ mask) {
  extern __shared__ __align__(16) unsigned char smem[];
  NmsBox* bx = reinterpret_cast<NmsBox*>(smem);                          // [K], by order
  const int words = (K + 31) / 32;
  uint32_t* sup = reinterpret_cast<uint32_t*>(bx + K);                   // [K][words]
  int* cand = reinterpret_cast<int*>(sup + (size_t)K * words);           // [K]: candidate flag, then the order of proposal j
  __shared__ int s_n;
  const int b = blockIdx.x;
  const double* cb = corners + (int64_t)b * K * 24;
  for (int j = threadIdx.x; j < K; j += NMS_THREADS) {
    cand[j] = counts == nullptr || counts[(int64_t)b * K + j] >= min_points;
    mask[(int64_t)b * K + j] = 0;
  }
  __syncthreads();
  // rank of candidate j: candidates with a larger score, or the same score and a larger index
  for (int j = threadIdx.x; j < K; j += NMS_THREADS) {
    if (cand[j]) {
      const uint32_t sj = score_order(score[(int64_t)b * K + j]);
      int r = 0;
      for (int i = 0; i < K; ++i) {
        if (!cand[i] || i == j) continue;
        const uint32_t si = score_order(score[(int64_t)b * K + i]);
        r += (si > sj) || (si == sj && i > j);
      }
      NmsBox q;
      const double* c = cb + j * 24;
      double mn[3] = {c[0], c[1], c[2]}, mx[3] = {c[0], c[1], c[2]};
      for (int k = 1; k < 8; ++k)
        for (int d = 0; d < 3; ++d) { mn[d] = np_min(mn[d], c[3 * k + d]); mx[d] = np_max(mx[d], c[3 * k + d]); }
      if (mode == 0) {                                                    // 2-D: camera x / z extents
        q.x1 = mn[0]; q.y1 = mn[2]; q.x2 = mx[0]; q.y2 = mx[2]; q.z1 = q.z2 = 0;
        q.area = mul(sub(q.x2, q.x1), sub(q.y2, q.y1));
      } else {
        q.x1 = mn[0]; q.y1 = mn[1]; q.z1 = mn[2]; q.x2 = mx[0]; q.y2 = mx[1]; q.z2 = mx[2];
        q.area = mul(mul(sub(q.x2, q.x1), sub(q.y2, q.y1)), sub(q.z2, q.z1));
      }
      q.cls = sem_cls[(int64_t)b * K + j];
      q.idx = j;
      bx[r] = q;
    }
  }
  if (threadIdx.x == 0) { int n = 0; for (int j = 0; j < K; ++j) n += cand[j]; s_n = n; }
  __syncthreads();
  const int n = s_n;
  // sup[a][b / 32] bit b % 32: a < b and box a suppresses box b
  for (int64_t e = threadIdx.x; e < (int64_t)n * words; e += NMS_THREADS) {
    const int a = (int)(e / words), w = (int)(e % words);
    const NmsBox A = bx[a];
    uint32_t bits = 0;
    for (int t = 0; t < 32; ++t) {
      const int bb = w * 32 + t;
      if (bb <= a || bb >= n) continue;
      const NmsBox Bx = bx[bb];
      double o;
      if (mode == 0) {
        const double xx1 = np_max(A.x1, Bx.x1), yy1 = np_max(A.y1, Bx.y1), xx2 = np_min(A.x2, Bx.x2), yy2 = np_min(A.y2, Bx.y2);
        const double ww = np_max(0.0, sub(xx2, xx1)), hh = np_max(0.0, sub(yy2, yy1));
        const double inter = mul(ww, hh);
        o = old_type ? inter / Bx.area : inter / sub(add(A.area, Bx.area), inter);
      } else {
        const double xx1 = np_max(A.x1, Bx.x1), yy1 = np_max(A.y1, Bx.y1), zz1 = np_max(A.z1, Bx.z1);
        const double xx2 = np_min(A.x2, Bx.x2), yy2 = np_min(A.y2, Bx.y2), zz2 = np_min(A.z2, Bx.z2);
        const double l = np_max(0.0, sub(xx2, xx1)), ww = np_max(0.0, sub(yy2, yy1)), hh = np_max(0.0, sub(zz2, zz1));
        const double inter = mul(mul(l, ww), hh);
        o = old_type ? inter / Bx.area : inter / sub(add(A.area, Bx.area), inter);
        if (mode == 2) o = mul(o, A.cls == Bx.cls ? 1.0 : 0.0);
      }
      if (o > thresh) bits |= 1u << t;
    }
    sup[(size_t)a * words + w] = bits;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    uint32_t removed[NMS_MAXK / 32 / 32] = {};                            // lane owns words lane, lane + 32, ... (1 word for K <= 1024)
    for (int a = 0; a < n; ++a) {
      const int w = a / 32;
      const uint32_t word = __shfl_sync(0xffffffffu, (w % 32 == lane) ? removed[w / 32] : 0u, w % 32);
      if (word >> (a % 32) & 1u) continue;
      if (lane == 0) mask[(int64_t)b * K + bx[a].idx] = 1;
      for (int v = lane; v < words; v += 32) removed[v / 32] |= sup[(size_t)a * words + v];
    }
  }
}

size_t nms_smem(int K) { return (size_t)K * sizeof(NmsBox) + (size_t)K * ((K + 31) / 32) * 4 + (size_t)K * 4; }

// ------------------------------------------------------------------------------------------------ oriented IoU
struct P2 { double x, y; };
constexpr int CLIP_MAX = 12;

// `polygon_clip` (box_util.py:16-62): Sutherland-Hodgman with the strict `inside` predicate; returns the vertex count (0 for None)
__device__ int polygon_clip(const P2* subj, int ns, const P2* clip, int nc, P2* out) {
  P2 buf[CLIP_MAX];
  int n = ns;
  for (int i = 0; i < n; ++i) out[i] = subj[i];
  P2 cp1 = clip[nc - 1];
  for (int ci = 0; ci < nc; ++ci) {
    const P2 cp2 = clip[ci];
    for (int i = 0; i < n; ++i) buf[i] = out[i];
    const int m = n;
    n = 0;
    auto inside = [&](P2 p) { return mul(sub(cp2.x, cp1.x), sub(p.y, cp1.y)) > mul(sub(cp2.y, cp1.y), sub(p.x, cp1.x)); };
    auto isect = [&](P2 s, P2 e) {
      const double dcx = sub(cp1.x, cp2.x), dcy = sub(cp1.y, cp2.y), dpx = sub(s.x, e.x), dpy = sub(s.y, e.y);
      const double n1 = sub(mul(cp1.x, cp2.y), mul(cp1.y, cp2.x)), n2 = sub(mul(s.x, e.y), mul(s.y, e.x));
      const double n3 = 1.0 / sub(mul(dcx, dpy), mul(dcy, dpx));
      return P2{mul(sub(mul(n1, dpx), mul(n2, dcx)), n3), mul(sub(mul(n1, dpy), mul(n2, dcy)), n3)};
    };
    P2 s = buf[m - 1];
    for (int i = 0; i < m; ++i) {
      const P2 e = buf[i];
      if (inside(e)) {
        if (!inside(s) && n < CLIP_MAX) out[n++] = isect(s, e);
        if (n < CLIP_MAX) out[n++] = e;
      } else if (inside(s) && n < CLIP_MAX) {
        out[n++] = isect(s, e);
      }
      s = e;
    }
    cp1 = cp2;
    if (n == 0) return 0;
  }
  return n;
}

// Area of the convex hull of p[0, n) (ConvexHull(...).volume): Andrew's monotone chain, then the shoelace sum.  Fewer than 3
// non-collinear points: 0 (Qhull raises there).
__device__ double hull_area(P2* p, int n) {
  for (int i = 1; i < n; ++i) {                                           // sort by (x, y)
    const P2 v = p[i];
    int j = i - 1;
    while (j >= 0 && (p[j].x > v.x || (p[j].x == v.x && p[j].y > v.y))) { p[j + 1] = p[j]; --j; }
    p[j + 1] = v;
  }
  P2 h[2 * CLIP_MAX];
  int k = 0;
  auto cross = [](P2 o, P2 a, P2 b) { return sub(mul(sub(a.x, o.x), sub(b.y, o.y)), mul(sub(a.y, o.y), sub(b.x, o.x))); };
  for (int i = 0; i < n; ++i) {
    while (k >= 2 && cross(h[k - 2], h[k - 1], p[i]) <= 0) --k;
    h[k++] = p[i];
  }
  for (int i = n - 2, t = k + 1; i >= 0; --i) {
    while (k >= t && cross(h[k - 2], h[k - 1], p[i]) <= 0) --k;
    h[k++] = p[i];
  }
  --k;                                                                    // the last point repeats the first
  if (k < 3) return 0.0;
  double a = 0.0;
  for (int i = 0; i < k; ++i) {
    const P2 u = h[i], v = h[(i + 1) % k];
    a = add(a, sub(mul(u.x, v.y), mul(u.y, v.x)));
  }
  return fabs(a) / 2;
}

__device__ double box3d_vol(const double* c) {
  auto len = [&](int i, int j) {
    const double dx = sub(c[3 * i], c[3 * j]), dy = sub(c[3 * i + 1], c[3 * j + 1]), dz = sub(c[3 * i + 2], c[3 * j + 2]);
    return sqrt(add(add(mul(dx, dx), mul(dy, dy)), mul(dz, dz)));
  };
  return mul(mul(len(0, 1), len(1, 2)), len(0, 4));
}

// `box3d_iou(corners1, corners2)[0]` (box_util.py:92-117)
__device__ double box3d_iou(const double* c1, const double* c2) {
  P2 r1[4], r2[4], clip[CLIP_MAX];
  for (int i = 0; i < 4; ++i) { r1[i] = P2{c1[3 * (3 - i)], c1[3 * (3 - i) + 2]}; r2[i] = P2{c2[3 * (3 - i)], c2[3 * (3 - i) + 2]}; }
  const int n = polygon_clip(r1, 4, r2, 4, clip);
  const double inter_area = n ? hull_area(clip, n) : 0.0;
  const double ymax = c2[1] < c1[1] ? c2[1] : c1[1];                      // Python min / max: the first unless the second is better
  const double ymin = c2[13] > c1[13] ? c2[13] : c1[13];
  const double dy = sub(ymax, ymin);
  const double inter_vol = mul(inter_area, dy > 0.0 ? dy : 0.0);
  return inter_vol / sub(add(box3d_vol(c1), box3d_vol(c2)), inter_vol);
}

// iou[i] = box3d_iou(c1[i], c2[i]): the IoU of pcb_det_ap, one pair per thread
__global__ void box_iou_kernel(const double* __restrict__ c1, const double* __restrict__ c2, int64_t n, double* __restrict__ iou) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) iou[i] = box3d_iou(c1 + i * 24, c2 + i * 24);
}

// ------------------------------------------------------------------------------------------------ average precision
// ground truth keyed by (scan, class); an entry outside [0, C) sorts last and is ignored
__global__ void gt_key_kernel(const int32_t* __restrict__ scan, const int32_t* __restrict__ cls, int64_t G, int C, uint64_t* __restrict__ k,
                              int32_t* __restrict__ idx, int32_t* __restrict__ npos) {
  const int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (g >= G) return;
  const bool ok = cls[g] >= 0 && cls[g] < C && scan[g] >= 0;
  k[g] = ok ? ((uint64_t)(uint32_t)scan[g] << 32) | (uint32_t)cls[g] : KEY_EMPTY;
  idx[g] = (int32_t)g;
  if (ok) atomicAdd(npos + cls[g], 1);
}

__device__ __forceinline__ int64_t lower_bound(const uint64_t* a, int64_t n, uint64_t v) {
  int64_t lo = 0, hi = n;
  while (lo < hi) { const int64_t m = (lo + hi) >> 1; if (a[m] < v) lo = m + 1; else hi = m; }
  return lo;
}

// Per detection: ovmax / jmax over the ground truth of its (scan, class) in the reference's j order (stable sort), the first maximal j,
// a NaN IoU never winning; jmax is the sorted ground-truth position (-1: none).  Also the detection's sort key: class in bits [32, ...),
// below it the score in DESCENDING order (-0.0 as +0.0, NaN last); a detection outside [0, C) gets class C.
__global__ void det_iou_kernel(const double* __restrict__ prop, int64_t P, const int32_t* __restrict__ row, const int32_t* __restrict__ cls,
                               const float* __restrict__ score, const int32_t* __restrict__ scan, int64_t D, int C,
                               const double* __restrict__ gtc, const uint64_t* __restrict__ gk, const int32_t* __restrict__ gidx, int64_t G,
                               double* __restrict__ ovmax, int32_t* __restrict__ jmax, uint64_t* __restrict__ key, int32_t* __restrict__ idx) {
  const int64_t d = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (d >= D) return;
  const int c = cls[d];
  const bool ok = c >= 0 && c < C && scan[d] >= 0 && row[d] >= 0 && row[d] < P;
  double best = -INFINITY;
  int bj = -1;
  if (ok) {
    const uint64_t k = ((uint64_t)(uint32_t)scan[d] << 32) | (uint32_t)c;
    const double* bb = prop + (int64_t)row[d] * 24;
    for (int64_t j = lower_bound(gk, G, k); j < G && gk[j] == k; ++j) {
      const double iou = box3d_iou(bb, gtc + (int64_t)gidx[j] * 24);
      if (iou > best) { best = iou; bj = (int)j; }
    }
  }
  ovmax[d] = best;
  jmax[d] = bj;
  float v = score[d];
  if (v == 0.f) v = 0.f;
  const uint32_t u = __float_as_uint(v);
  const uint32_t asc = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  key[d] = ((uint64_t)(ok ? c : C) << 32) | (uint64_t)(isnan(v) ? 0xFFFFFFFFu : ~asc);
  idx[d] = (int32_t)d;
}

// class segments of the sorted detections: [seg[2c], seg[2c+1])
__global__ void det_seg_kernel(const uint64_t* __restrict__ sk, int64_t D, int C, int32_t* __restrict__ seg) {
  const int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (p >= D) return;
  const int c = (int)(sk[p] >> 32);
  if (c >= C) return;
  if (p == 0 || (int)(sk[p - 1] >> 32) != c) seg[2 * c] = (int32_t)p;
  if (p + 1 == D || (int)(sk[p + 1] >> 32) != c) seg[2 * c + 1] = (int32_t)(p + 1);
}

// claim[t][g] = the smallest sorted position of a detection with jmax == g and ovmax > thr[t]: that detection is the true positive
__global__ void det_claim_kernel(const int32_t* __restrict__ sidx, const uint64_t* __restrict__ sk, int64_t D, int C,
                                 const double* __restrict__ ovmax, const int32_t* __restrict__ jmax, const double* __restrict__ thr, int T,
                                 int64_t G, int32_t* __restrict__ claim) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= D * T) return;
  const int t = (int)(e / D);
  const int64_t p = e - (int64_t)t * D;
  if ((int)(sk[p] >> 32) >= C) return;
  const int d = sidx[p];
  if (ovmax[d] > thr[t]) atomicMin(claim + (int64_t)t * G + jmax[d], (int32_t)p);
}

// One CTA per (class, threshold).  Forward: tp_cum by a block scan over the class's segment in chunks.  Backward: the precision envelope
// env[p] = max over q >= p of tp_cum[q] / rank[q] (a reverse max-scan), and AP = sum over true positives p of (rec[p] - rec[p-1]) * env[p]
// with rec = tp_cum / npos (voc_ap, eval_det.py:24-55).  Each thread sums its terms in chunk order, then a fixed tree: deterministic.
constexpr int APD_THREADS = 256;
__global__ void __launch_bounds__(APD_THREADS) det_ap_class_kernel(const int32_t* __restrict__ sidx, const double* __restrict__ ovmax,
                                                                   const int32_t* __restrict__ jmax, const double* __restrict__ thr,
                                                                   const int32_t* __restrict__ claim, int64_t G, const int32_t* __restrict__ seg,
                                                                   const int32_t* __restrict__ npos_c, int64_t D, int C,
                                                                   int32_t* __restrict__ cum, double* __restrict__ out) {
  using Scan = cub::BlockScan<int, APD_THREADS>;
  using MaxScan = cub::BlockScan<double, APD_THREADS>;
  __shared__ union { typename Scan::TempStorage s; typename MaxScan::TempStorage m; } tmp;
  __shared__ double red[APD_THREADS];
  __shared__ int s_carry;
  __shared__ double s_env;
  const int c = blockIdx.x, t = blockIdx.y;
  const int s0 = seg[2 * c], s1 = seg[2 * c + 1];
  const int nd = s1 - s0, npos = npos_c[c];
  const double th = thr[t];
  int32_t* cm = cum + (int64_t)t * D;
  const int32_t* cl = claim + (int64_t)t * G;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int base = s0; base < s1; base += APD_THREADS) {
    const int p = base + threadIdx.x;
    int tp = 0;
    if (p < s1) { const int d = sidx[p]; tp = ovmax[d] > th && cl[jmax[d]] == p; }
    int inc;
    Scan(tmp.s).InclusiveSum(tp, inc);
    const int carry = s_carry;
    if (p < s1) cm[p] = carry + inc;
    __syncthreads();
    if (threadIdx.x == APD_THREADS - 1) s_carry = carry + inc;
    __syncthreads();
  }
  if (threadIdx.x == 0) s_env = 0.0;
  __syncthreads();
  double acc = 0.0;
  const double np_d = (double)npos;
  for (int top = s1; top > s0; top -= APD_THREADS) {
    const int p = top - 1 - threadIdx.x;                                   // thread 0 holds the last position of the chunk
    double prec = 0.0;
    int cu = 0, prev = 0;
    if (p >= s0) {
      cu = cm[p];
      prev = p > s0 ? cm[p - 1] : 0;
      prec = (double)cu / (double)(p - s0 + 1);
    }
    double env;
    MaxScan(tmp.m).InclusiveScan(prec, env, [](double a, double b) { return a > b ? a : b; });
    const double carry = s_env;
    env = env > carry ? env : carry;
    if (p >= s0 && cu != prev) acc += ((double)cu / np_d - (double)prev / np_d) * env;
    __syncthreads();
    if (threadIdx.x == APD_THREADS - 1) s_env = env;
    __syncthreads();
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int h = APD_THREADS / 2; h; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    double* o = out + ((int64_t)t * C + c) * 4;
    if (nd == 0) { o[0] = 0.0; o[1] = 0.0; }
    else if (npos == 0) { o[0] = (double)NAN; o[1] = (double)NAN; }
    else { o[0] = red[0]; o[1] = (double)cm[s1 - 1] / np_d; }
    o[2] = (double)npos;
    o[3] = (double)nd;
  }
}

struct DetApWs { SortWs g, d; double* ovmax; int32_t* jmax; int32_t* npos; int32_t* seg; int32_t* claim; int32_t* cum; double* thr; };
DetApWs det_ap_layout(Carve& c, int64_t D, int64_t G, int C, int T) {
  return {sort_layout(c, G), sort_layout(c, D), c.take<double>(D), c.take<int32_t>(D), c.take<int32_t>(C), c.take<int32_t>(2 * C),
          c.take<int32_t>(T * G), c.take<int32_t>(T * D), c.take<double>(T)};
}

int class_bits(int C) { int b = 0; while ((1 << b) < C) ++b; return b; }

}  // namespace

extern "C" int pcb_det_decode_pred(const float* center, const float* heading_scores, const float* heading_residuals, const float* size_scores,
                                   const float* size_residuals, const float* sem_cls_scores, const float* objectness_scores, int64_t B,
                                   int64_t K, int H, int S, int C, const double* mean_size, int heading_rule, double* corners, double* box,
                                   int32_t* sem_cls, float* obj_prob, float* sem_prob, void* stream) {
  PCB_ARG(center && heading_scores && heading_residuals && size_scores && size_residuals && sem_cls_scores && objectness_scores && mean_size &&
          corners && box && sem_cls && obj_prob && sem_prob);
  PCB_ARG(B >= 1 && K >= 1 && H >= 1 && S >= 1 && C >= 1 && C <= MAX_CLS && (heading_rule == 0 || heading_rule == 1) && B * K < ((int64_t)1 << 31));
  const int64_t BK = B * K;
  decode_pred_kernel<<<blocks_for(BK, 128), 128, 0, (cudaStream_t)stream>>>(center, heading_scores, heading_residuals, size_scores,
                                                                           size_residuals, sem_cls_scores, objectness_scores, BK, H, S, C,
                                                                           mean_size, heading_rule, corners, box, sem_cls, obj_prob, sem_prob);
  return check_launch("decode_pred_kernel");
}

extern "C" int pcb_det_decode_gt(const float* center, const int64_t* heading_class, const float* heading_residual, const int64_t* size_class,
                                 const float* size_residual, int64_t B, int64_t K, int H, int S, const double* mean_size, int heading_rule,
                                 double* corners, double* box, int32_t* status, void* stream) {
  PCB_ARG(center && heading_class && heading_residual && size_class && size_residual && mean_size && corners && box && status);
  PCB_ARG(B >= 1 && K >= 1 && H >= 1 && S >= 1 && (heading_rule == 0 || heading_rule == 1) && B * K < ((int64_t)1 << 31));
  const int64_t BK = B * K;
  decode_gt_kernel<<<blocks_for(BK, 128), 128, 0, (cudaStream_t)stream>>>(center, heading_class, heading_residual, size_class, size_residual,
                                                                         BK, H, S, mean_size, heading_rule, corners, box, status);
  return check_launch("decode_gt_kernel");
}

extern "C" int pcb_det_points_in_box(const float* points, int64_t B, int64_t N, int ld, const double* box, int64_t K, int32_t* counts,
                                     void* stream) {
  PCB_ARG(points && box && counts && B >= 1 && N >= 1 && ld >= 3 && K >= 1 && B <= 65535 && K <= 65535 * 32 && N < ((int64_t)1 << 31) &&
          (N + PIB_SPLIT - 1) / PIB_SPLIT <= 65535);
  cudaStream_t st = (cudaStream_t)stream;
  PCB_CUDA(cudaMemsetAsync(counts, 0, B * K * sizeof(int32_t), st));
  const dim3 grid((unsigned)B, (unsigned)((K + 31) / 32), (unsigned)((N + PIB_SPLIT - 1) / PIB_SPLIT));
  points_in_box_kernel<<<grid, PIB_THREADS, 0, st>>>(points, N, ld, box, (int)K, counts);
  return check_launch("points_in_box_kernel");
}

extern "C" int pcb_det_nms(const double* corners, const float* score, const int32_t* sem_cls, const int32_t* counts, int min_points, int64_t B,
                           int64_t K, int mode, int old_type, double nms_iou, int32_t* pred_mask, void* stream) {
  PCB_ARG(corners && score && sem_cls && pred_mask && B >= 1 && B <= 65535 && K >= 1 && K <= NMS_MAXK && mode >= 0 && mode <= 2);
  const size_t smem = nms_smem((int)K);
  PCB_CUDA(cudaFuncSetAttribute(nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)nms_smem(NMS_MAXK)));
  nms_kernel<<<(unsigned)B, NMS_THREADS, smem, (cudaStream_t)stream>>>(corners, score, sem_cls, counts, min_points, (int)K, mode, old_type,
                                                                        nms_iou, pred_mask);
  return check_launch("nms_kernel");
}

extern "C" int pcb_det_box_iou(const double* corners1, const double* corners2, int64_t n, double* iou, void* stream) {
  PCB_ARG(corners1 && corners2 && iou && n >= 1 && n < ((int64_t)1 << 31));
  box_iou_kernel<<<blocks_for(n, 128), 128, 0, (cudaStream_t)stream>>>(corners1, corners2, n, iou);
  return check_launch("box_iou_kernel");
}

extern "C" size_t pcb_det_ap_ws_bytes(int64_t D, int64_t G, int C, int T) {
  if (D < 1 || G < 1 || C < 1 || T < 1) return 0;
  return layout_bytes(det_ap_layout, D, G, C, T);
}

extern "C" int pcb_det_ap(const double* prop_corners, int64_t P, const int32_t* det_row, const int32_t* det_cls, const float* det_score,
                          const int32_t* det_scan, int64_t D, const double* gt_corners, const int32_t* gt_scan, const int32_t* gt_cls,
                          int64_t G, int C, const double* thresholds, int T, double* out, void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(prop_corners && det_row && det_cls && det_score && det_scan && gt_corners && gt_scan && gt_cls && thresholds && out && ws);
  PCB_ARG(P >= 1 && D >= 1 && G >= 1 && C >= 1 && C <= MAX_CLS && T >= 1 && T <= 64 && D * T < ((int64_t)1 << 31) &&
          G * T < ((int64_t)1 << 31));
  Carve c{(char*)ws};
  const DetApWs w = det_ap_layout(c, D, G, C, T);
  PCB_ARG(ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  PCB_CUDA(cudaMemcpyAsync(w.thr, thresholds, T * sizeof(double), cudaMemcpyHostToDevice, st));
  PCB_CUDA(cudaMemsetAsync(w.npos, 0, C * sizeof(int32_t), st));
  PCB_CUDA(cudaMemsetAsync(w.seg, 0, 2 * C * sizeof(int32_t), st));
  PCB_CUDA(cudaMemsetAsync(w.claim, 0x7f, T * G * sizeof(int32_t), st));
  gt_key_kernel<<<blocks_for(G, 256), 256, 0, st>>>(gt_scan, gt_cls, G, C, w.g.k, w.g.idx, w.npos);
  if (int e = check_launch("gt_key_kernel")) return e;
  if (int e = sort_keys(G, w.g, 64, st)) return e;
  det_iou_kernel<<<blocks_for(D, 128), 128, 0, st>>>(prop_corners, P, det_row, det_cls, det_score, det_scan, D, C, gt_corners, w.g.sk, w.g.sidx,
                                                     G, w.ovmax, w.jmax, w.d.k, w.d.idx);
  if (int e = check_launch("det_iou_kernel")) return e;
  if (int e = sort_keys(D, w.d, 32 + class_bits(C + 1), st)) return e;
  det_seg_kernel<<<blocks_for(D, 256), 256, 0, st>>>(w.d.sk, D, C, w.seg);
  if (int e = check_launch("det_seg_kernel")) return e;
  det_claim_kernel<<<blocks_for(D * T, 256), 256, 0, st>>>(w.d.sidx, w.d.sk, D, C, w.ovmax, w.jmax, w.thr, T, G, w.claim);
  if (int e = check_launch("det_claim_kernel")) return e;
  det_ap_class_kernel<<<dim3((unsigned)C, (unsigned)T), APD_THREADS, 0, st>>>(w.d.sidx, w.ovmax, w.jmax, w.thr, w.claim, G, w.seg, w.npos, D, C,
                                                                             w.cum, out);
  return check_launch("det_ap_class_kernel");
}
