// VoteNet detection data on the GPU (include/pcb200.h "VoteNet detection data"): floor heights, choice sets, the fused point pass with
// the ScanNet instance votes, and the box labels of a ragged batch of scenes.  Every operation the original does in numpy is one
// explicitly rounded operation here (__fadd_rn / __dmul_rn ...), so nvcc cannot contract it into an FMA.
#include "common.cuh"
#include "sort.cuh"

using namespace pcb;

namespace {

constexpr int FH_THREADS = 512;
constexpr int PT_THREADS = 256;
constexpr int64_t LIM = 1ll << 31;
constexpr double PI = 3.141592653589793;      // np.pi

// ---------------------------------------------------------------------------------------------------------------- floor height

template <class T> struct Ord;
template <> struct Ord<float> {
  using K = uint32_t;
  static constexpr int BITS = 32;
  __device__ static K key(float v) { const uint32_t u = __float_as_uint(v); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
  __device__ static float val(K k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }
  __device__ static float add(float a, float b) { return __fadd_rn(a, b); }
  __device__ static float sub(float a, float b) { return __fsub_rn(a, b); }
  __device__ static float mul(float a, float b) { return __fmul_rn(a, b); }
};
template <> struct Ord<double> {
  using K = unsigned long long;
  static constexpr int BITS = 64;
  __device__ static K key(double v) {
    const K u = (K)__double_as_longlong(v);
    return (u >> 63) ? ~u : (u | (1ull << 63));
  }
  __device__ static double val(K k) { return __longlong_as_double((long long)((k >> 63) ? (k & ~(1ull << 63)) : ~k)); }
  __device__ static double add(double a, double b) { return __dadd_rn(a, b); }
  __device__ static double sub(double a, double b) { return __dsub_rn(a, b); }
  __device__ static double mul(double a, double b) { return __dmul_rn(a, b); }
};

// the key of rank r (0-based, ascending) among the n keys of z[lo .. lo + n) by 8-bit radix selection; every thread gets it
template <class T>
__device__ typename Ord<T>::K radix_select(const T* __restrict__ z, int64_t stride, int64_t lo, int64_t n, int64_t r, int* hist) {
  using K = typename Ord<T>::K;
  __shared__ int64_t s_r;
  __shared__ int s_digit;
  K prefix = 0, mask = 0;
  for (int shift = Ord<T>::BITS - 8; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
      const K k = Ord<T>::key(z[(lo + i) * stride]);
      if ((k & mask) == prefix) atomicAdd(&hist[(int)((k >> shift) & 255)], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int64_t below = 0;
      int d = 0;
      for (; d < 255; ++d) {
        if (below + hist[d] > r) break;
        below += hist[d];
      }
      s_digit = d;
      s_r = r - below;
    }
    __syncthreads();
    prefix |= (K)s_digit << shift;
    mask |= (K)255 << shift;
    r = s_r;
    __syncthreads();
  }
  return prefix;
}

template <class T>
__global__ void __launch_bounds__(FH_THREADS) floor_height_kernel(const T* __restrict__ z, int64_t stride, const int64_t* __restrict__ offsets,
                                                                 double* __restrict__ out) {
  using K = typename Ord<T>::K;
  __shared__ int hist[256];
  __shared__ unsigned long long s_le, s_gt;
  const int b = blockIdx.x;
  const int64_t lo = offsets[b], n = offsets[b + 1] - lo;
  // np.percentile(z, 0.99): q = 0.99 / 100 and the virtual index (n - 1) q, both in the data's type
  const T q = (T)0.99 / (T)100;
  const T vi = Ord<T>::mul((T)(n - 1), q);
  int64_t prev = (int64_t)floor((double)vi), next = prev + 1;
  T gamma = Ord<T>::sub(vi, (T)prev);
  if (vi >= (T)(n - 1)) {                       // numpy takes index -1 (the maximum) for both, and t = vi - (-1)
    prev = next = n - 1;
    gamma = (T)((double)vi + 1.0);
  }
  const K ka = radix_select(z, stride, lo, n, prev, hist);
  K kb = ka;
  if (next != prev) {                           // rank prev + 1: the same key while it repeats, else the next larger key
    if (threadIdx.x == 0) { s_le = 0; s_gt = ~0ull; }
    __syncthreads();
    unsigned long long le = 0, gt = ~0ull;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
      const K k = Ord<T>::key(z[(lo + i) * stride]);
      if (k <= ka) ++le;
      else if ((unsigned long long)k < gt) gt = k;
    }
    atomicAdd(&s_le, le);
    atomicMin(&s_gt, gt);
    __syncthreads();
    kb = ((int64_t)s_le > next) ? ka : (K)s_gt;
  }
  if (threadIdx.x == 0) {
    const T a = Ord<T>::val(ka), bv = Ord<T>::val(kb);
    const T diff = Ord<T>::sub(bv, a);
    // numpy's _lerp: a + (b - a) t, replaced by b - (b - a)(1 - t) where t >= 0.5
    const T r = gamma >= (T)0.5 ? Ord<T>::sub(bv, Ord<T>::mul(diff, Ord<T>::sub((T)1, gamma))) : Ord<T>::add(a, Ord<T>::mul(diff, gamma));
    out[b] = (double)r;
  }
}

// ---------------------------------------------------------------------------------------------------------------- Philox4x32-10

__device__ __forceinline__ uint4 philox(uint64_t seed, uint64_t offset, uint64_t counter) {
  uint32_t c0 = (uint32_t)counter, c1 = (uint32_t)(counter >> 32), c2 = (uint32_t)offset, c3 = (uint32_t)(offset >> 32);
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t lo0 = 0xD2511F53u * c0, hi0 = __umulhi(0xD2511F53u, c0);
    const uint32_t lo1 = 0xCD9E8D57u * c2, hi1 = __umulhi(0xCD9E8D57u, c2);
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}
__device__ __forceinline__ uint64_t philox64(uint64_t seed, uint64_t offset, uint64_t counter) {
  const uint4 r = philox(seed, offset, counter);
  return ((uint64_t)r.x << 32) | r.y;
}

// the source row of sampled row r of scene b; a choice outside [0, n_b) reads the scene's first row and flags the output (NaN coordinates)
__device__ __forceinline__ int64_t source_row(const pcb_det_batch& a, int64_t b, int64_t r, bool& bad) {
  const int64_t lo = a.offsets[b], c = a.choices[r];
  bad = c < 0 || c >= a.offsets[b + 1] - lo;
  return bad ? lo : lo + c;
}

__device__ __forceinline__ int scene_of(const int64_t* __restrict__ offsets, int64_t B, int64_t row) {
  int64_t lo = 0, hi = B - 1;                   // the last b with offsets[b] <= row (scenes are non-empty)
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (offsets[mid] <= row) lo = mid; else hi = mid - 1;
  }
  return (int)lo;
}

__global__ void choice_keys_kernel(const int64_t* __restrict__ offsets, int64_t B, int64_t M, int scene_bits, uint64_t seed, uint64_t offset,
                                   uint64_t* __restrict__ keys, int32_t* __restrict__ idx) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const int b = scene_of(offsets, B, i);
  const uint64_t r = philox64(seed, offset, (uint64_t)i);
  keys[i] = scene_bits ? (((uint64_t)b << (64 - scene_bits)) | (r >> scene_bits)) : r;
  idx[i] = (int32_t)(i - offsets[b]);
}

__global__ void choice_out_kernel(const int64_t* __restrict__ offsets, int64_t B, int64_t M, int64_t k, uint64_t seed, uint64_t offset,
                                  const int32_t* __restrict__ sorted_idx, int64_t* __restrict__ out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * k) return;
  const int64_t b = t / k, j = t - b * k, lo = offsets[b], n = offsets[b + 1] - lo;
  if (n >= k) out[t] = sorted_idx[lo + j];                     // without replacement: the first k of the scene's random order
  else out[t] = (int64_t)__umul64hi(philox64(seed, offset, (uint64_t)(M + t)), (uint64_t)n);   // with replacement: iid
}

// ---------------------------------------------------------------------------------------------------------------- point pass

__device__ __forceinline__ double dot3(double x, double y, double z, double r0, double r1, double r2) {
  return __dadd_rn(__dadd_rn(__dmul_rn(x, r0), __dmul_rn(y, r1)), __dmul_rn(z, r2));
}
// p . rotz(angle)^T for rotz = [[c, -s, 0], [s, c, 0], [0, 0, 1]]
__device__ __forceinline__ void rotate(double& x, double& y, double& z, double c, double s) {
  const double nx = dot3(x, y, z, c, -s, 0.0), ny = dot3(x, y, z, s, c, 0.0), nz = dot3(x, y, z, 0.0, 0.0, 1.0);
  x = nx; y = ny; z = nz;
}

__global__ void scannet_points_kernel(pcb_det_batch a, uint64_t* __restrict__ keys, int32_t* __restrict__ idx) {
  const int64_t k = a.num_points, r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.B * k) return;
  bool bad;
  const int64_t b = r / k, src = source_row(a, b, r, bad);
  const int C = (a.flags & PCB_DET_HEIGHT) ? 4 : 3;
  const float* v = a.vert + src * 6;
  float x = v[0], y = v[1], z = v[2];
  float* o = a.point_clouds + r * C;
  if (a.flags & PCB_DET_HEIGHT) o[3] = __fsub_rn(z, (float)a.floor[b]);      // height from the floor of all N points, before sampling
  if (a.flags & PCB_DET_AUGMENT) {                                           // sampled first, then flips and rotation
    const double* p = a.params + b * PCB_DET_NPARAM;
    if (p[0] != 0.0) x = -x;
    if (p[1] != 0.0) y = -y;
    double X = x, Y = y, Z = z;                                              // np.dot in fp64, stored back into the fp32 cloud
    rotate(X, Y, Z, p[2], p[3]);
    x = (float)X; y = (float)Y; z = (float)Z;
  }
  if (bad) x = y = z = __int_as_float(0x7fc00000);
  o[0] = x; o[1] = y; o[2] = z;
  for (int c = 0; c < 3; ++c) a.pcl_color[r * 3 + c] = v[3 + c];
  keys[r] = ((uint64_t)b << 32) | a.ins[src];                                // instance ids are arbitrary uint32 values
  idx[r] = (int32_t)r;
}

__device__ __forceinline__ uint32_t fkey(float v) { return Ord<float>::key(v); }

// per sorted position: the run (scene, instance) of its row, the run's first row (lowest output position: the sort is stable) and the
// run's min / max by order-preserving integer atomics (order-independent, so deterministic)
__global__ void instance_bounds_kernel(const pcb_det_batch a, int64_t R, const int32_t* __restrict__ sidx, const int32_t* __restrict__ rank,
                                       int32_t* __restrict__ run_of, int32_t* __restrict__ first, uint32_t* __restrict__ mn,
                                       uint32_t* __restrict__ mx) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= R) return;
  const int run = rank[p] - 1, row = sidx[p];
  const int C = (a.flags & PCB_DET_HEIGHT) ? 4 : 3;
  run_of[row] = run;
  if (p == 0 || rank[p - 1] != rank[p]) first[run] = row;
  for (int c = 0; c < 3; ++c) {
    const uint32_t kv = fkey(a.point_clouds[(int64_t)row * C + c]);
    atomicMin(&mn[run * 3 + c], kv);
    atomicMax(&mx[run * 3 + c], kv);
  }
}

__global__ void instance_votes_kernel(const pcb_det_batch a, const int32_t* __restrict__ run_of, const int32_t* __restrict__ first,
                                      const uint32_t* __restrict__ mn, const uint32_t* __restrict__ mx) {
  const int64_t k = a.num_points, r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.B * k) return;
  const int64_t b = r / k;
  const int run = run_of[r], f = first[run];
  // votes only when the semantic label of the instance's FIRST SAMPLED row (not its lowest source index) is a detected nyu40 id
  bool bad;
  const uint32_t sem = a.sem[source_row(a, b, f, bad)];          // f is a row of scene b: runs never cross scenes
  bool obj = false;
  for (int i = 0; i < a.n_ids; ++i) obj |= (int64_t)sem == a.nyu40ids[i];
  const int C = (a.flags & PCB_DET_HEIGHT) ? 4 : 3;
  float* o = a.vote_label + r * 9;
  for (int c = 0; c < 3; ++c) {
    float vote = 0.f;
    if (obj) {       // center = 0.5 (min + max) in fp32, vote = center - x
      const float center = __fmul_rn(0.5f, __fadd_rn(Ord<float>::val(mn[run * 3 + c]), Ord<float>::val(mx[run * 3 + c])));
      vote = __fsub_rn(center, a.point_clouds[r * C + c]);
    }
    o[c] = o[3 + c] = o[6 + c] = vote;                                       // three identical votes
  }
  a.vote_label_mask[r] = obj ? 1 : 0;
}

__global__ void sunrgbd_points_kernel(pcb_det_batch a) {
  const int64_t k = a.num_points, r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.B * k) return;
  bool bad;                                                                  // sampling comes last: every transform is per row
  const int64_t b = r / k, src = source_row(a, b, r, bad);
  const bool color = a.flags & PCB_DET_COLOR, height = a.flags & PCB_DET_HEIGHT;
  const double* q = a.pc + src * 6;
  double x = q[0], y = q[1], z = q[2], rgb[3];
  for (int c = 0; c < 3; ++c) rgb[c] = __dsub_rn(q[3 + c], 0.5);            // colour minus MEAN_COLOR_RGB
  double h = height ? __dsub_rn(z, a.floor[b]) : 0.0;                        // floor height before augmentation
  double v[10];
  for (int c = 0; c < 10; ++c) v[c] = a.votes[src * 10 + c];
  if (a.flags & PCB_DET_AUGMENT) {
    const double* p = a.params + b * PCB_DET_NPARAM;
    if (p[0] != 0.0) { x = -x; v[1] = -v[1]; v[4] = -v[4]; v[7] = -v[7]; }
    // votes rotate through their end points: (p + v) R^T - p R^T, not v R^T
    double e[9];
    for (int j = 0; j < 3; ++j) {
      double ex = __dadd_rn(x, v[1 + 3 * j]), ey = __dadd_rn(y, v[2 + 3 * j]), ez = __dadd_rn(z, v[3 + 3 * j]);
      rotate(ex, ey, ez, p[2], p[3]);
      e[3 * j] = ex; e[3 * j + 1] = ey; e[3 * j + 2] = ez;
    }
    rotate(x, y, z, p[2], p[3]);
    for (int j = 0; j < 3; ++j) {
      v[1 + 3 * j] = __dsub_rn(e[3 * j], x); v[2 + 3 * j] = __dsub_rn(e[3 * j + 1], y); v[3 + 3 * j] = __dsub_rn(e[3 * j + 2], z);
    }
    if (color) {     // brightness and shift per channel, jitter per point, clip to [0, 1], drop 30 % of the colours
      const double jit = __dsub_rn(__dmul_rn(0.05, a.jitter[src]), 0.025);
      const double keep = a.dropout[src] > 0.3 ? 1.0 : 0.0;
      for (int c = 0; c < 3; ++c) {
        double t = __dadd_rn(rgb[c], 0.5);
        t = __dadd_rn(__dadd_rn(__dmul_rn(t, p[5 + c]), p[8 + c]), jit);
        t = fmin(fmax(t, 0.0), 1.0);
        rgb[c] = __dsub_rn(__dmul_rn(t, keep), 0.5);
      }
    }
    const double s = p[4];                      // scale points, votes and the height column
    x = __dmul_rn(x, s); y = __dmul_rn(y, s); z = __dmul_rn(z, s);
    for (int c = 1; c < 10; ++c) v[c] = __dmul_rn(v[c], s);
    if (height) h = __dmul_rn(h, s);
  }
  const int C = 3 + (color ? 3 : 0) + (height ? 1 : 0);
  float* o = a.point_clouds + r * C;
  if (bad) x = y = z = __longlong_as_double(0x7ff8000000000000ll);
  o[0] = (float)x; o[1] = (float)y; o[2] = (float)z;
  if (color) for (int c = 0; c < 3; ++c) o[3 + c] = (float)rgb[c];
  if (height) o[C - 1] = (float)h;
  for (int c = 0; c < 9; ++c) a.vote_label[r * 9 + c] = (float)v[1 + c];
  a.vote_label_mask[r] = (int64_t)v[0];                                      // the mask is vote column 0
}

// ---------------------------------------------------------------------------------------------------------------- box labels

__device__ __forceinline__ double np_remainder(double a, double m) {           // numpy's floor-mod (npy_divmod)
  double mod = fmod(a, m);
  if (mod != 0.0) { if ((m < 0) != (mod < 0)) mod = __dadd_rn(mod, m); }
  else mod = copysign(0.0, m);
  return mod;
}

__global__ void boxes_kernel(const pcb_det_batch a) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.B * PCB_DET_MAX_OBJ) return;
  const int64_t b = t / PCB_DET_MAX_OBJ, slot = t - b * PCB_DET_MAX_OBJ;
  const int64_t K = a.box_offsets[b + 1] - a.box_offsets[b], row = a.box_offsets[b] + slot;
  const bool aug = a.flags & PCB_DET_AUGMENT;
  const double* p = a.params + b * PCB_DET_NPARAM;
  double center[3] = {0, 0, 0}, size_res[3] = {0, 0, 0}, head_res = 0.0;
  int64_t head_cls = 0, size_cls = 0, sem = 0;
  if (a.max_gt_bboxes) for (int c = 0; c < 8; ++c) a.max_gt_bboxes[t * 8 + c] = 0.0;
  if (slot < K && a.dataset == PCB_DET_SCANNET) {
    const double* bb = a.boxes + row * 7;
    double cx = bb[0], cy = bb[1], cz = bb[2], lx = bb[3], ly = bb[4];
    const double lz = bb[5];
    if (aug) {
      if (p[0] != 0.0) cx = -cx;
      if (p[1] != 0.0) cy = -cy;
      // rotate_aligned_boxes: centres rotate; the new x / y lengths are twice the largest rotated half-length corner
      rotate(cx, cy, cz, p[2], p[3]);
      const double dx = lx / 2.0, dy = ly / 2.0;
      const double sx[4] = {-1, 1, 1, -1}, sy[4] = {-1, -1, 1, 1};
      double mx = -INFINITY, my = -INFINITY;
      for (int i = 0; i < 4; ++i) {
        double X = sx[i] * dx, Y = sy[i] * dy, Z = 0.0;
        rotate(X, Y, Z, p[2], p[3]);
        mx = fmax(mx, X); my = fmax(my, Y);
      }
      lx = __dmul_rn(2.0, mx); ly = __dmul_rn(2.0, my);
    }
    int cls = 0;              // the host rejects ids outside nyu40ids (the original's IndexError)
    for (int i = 0; i < a.n_ids; ++i) if ((double)a.nyu40ids[i] == bb[6]) { cls = i; break; }
    center[0] = cx; center[1] = cy; center[2] = cz;
    const double len[3] = {lx, ly, lz};
    for (int c = 0; c < 3; ++c) size_res[c] = __dsub_rn(len[c], a.mean_size[cls * 3 + c]);      // size class = semantic class
    size_cls = sem = cls;
  } else if (slot < K) {
    const double* bb = a.boxes + row * 8;
    double cx = bb[0], cy = bb[1], cz = bb[2], l = bb[3], w = bb[4], h = bb[5];
    const double* hd = a.headings + row * 3;    // heading after flip (pi - heading) and rotation (-= angle), and its trig
    if (aug) {
      if (p[0] != 0.0) cx = -cx;
      rotate(cx, cy, cz, p[2], p[3]);
      const double s = p[4];
      cx = __dmul_rn(cx, s); cy = __dmul_rn(cy, s); cz = __dmul_rn(cz, s);
      l = __dmul_rn(l, s); w = __dmul_rn(w, s); h = __dmul_rn(h, s);
    }
    const double aug_box[8] = {cx, cy, cz, l, w, h, hd[0], bb[7]};
    for (int c = 0; c < 8; ++c) a.max_gt_bboxes[t * 8 + c] = aug_box[c];
    // angle2class
    const double two_pi = 2 * PI, apc = two_pi / (double)a.num_heading_bin;
    const double angle = np_remainder(hd[0], two_pi);
    const double shifted = np_remainder(__dadd_rn(angle, apc / 2), two_pi);
    head_cls = (int64_t)__ddiv_rn(shifted, apc);
    head_res = __dsub_rn(shifted, __dadd_rn(__dmul_rn((double)head_cls, apc), apc / 2));
    // size2class on the doubled half-sizes
    sem = (int64_t)bb[7];
    size_cls = sem;
    const double hs[3] = {l, w, h};
    for (int c = 0; c < 3; ++c) size_res[c] = __dsub_rn(__dmul_rn(hs[c], 2.0), a.mean_size[sem * 3 + c]);
    // center_label: the centre of the axis-aligned box around my_compute_box_3d's corners (not the box centre: they differ by rounding)
    const double c0 = hd[1], s0 = hd[2];
    const double xc[8] = {-l, l, l, -l, -l, l, l, -l}, yc[8] = {w, w, -w, -w, w, w, -w, -w}, zc[8] = {h, h, h, h, -h, -h, -h, -h};
    double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = 0; i < 8; ++i) {
      const double X = __dadd_rn(dot3(xc[i], yc[i], zc[i], c0, -s0, 0.0), cx);
      const double Y = __dadd_rn(dot3(xc[i], yc[i], zc[i], s0, c0, 0.0), cy);
      const double Z = __dadd_rn(dot3(xc[i], yc[i], zc[i], 0.0, 0.0, 1.0), cz);
      lo[0] = fmin(lo[0], X); lo[1] = fmin(lo[1], Y); lo[2] = fmin(lo[2], Z);
      hi[0] = fmax(hi[0], X); hi[1] = fmax(hi[1], Y); hi[2] = fmax(hi[2], Z);
    }
    for (int c = 0; c < 3; ++c) center[c] = __dadd_rn(lo[c], hi[c]) / 2;
  }
  for (int c = 0; c < 3; ++c) { a.center_label[t * 3 + c] = (float)center[c]; a.size_residual_label[t * 3 + c] = (float)size_res[c]; }
  a.heading_class_label[t] = head_cls;
  a.heading_residual_label[t] = (float)head_res;
  a.size_class_label[t] = size_cls;
  a.sem_cls_label[t] = sem;
  a.box_label_mask[t] = slot < K ? 1.f : 0.f;
}

bool offsets_ok(const int64_t* off, int64_t B, int64_t total, int64_t max_len) {
  if (!off || off[0] != 0 || off[B] != total) return false;
  for (int64_t b = 0; b < B; ++b) {
    const int64_t n = off[b + 1] - off[b];
    if (n < 0 || (max_len > 0 && n > max_len) || (max_len == 0 && n < 1)) return false;
  }
  return true;
}

int bits_for(int64_t B) { int s = 0; while ((1ll << s) < B) ++s; return s; }

struct PointsWs { SortWs s; int32_t* run_of; int32_t* first; uint32_t* mn; uint32_t* mx; };
PointsWs points_layout(Carve& c, int64_t R) {
  PointsWs w;
  w.s = sort_layout(c, R);
  w.run_of = c.take<int32_t>(R); w.first = c.take<int32_t>(R); w.mn = c.take<uint32_t>(R * 3); w.mx = c.take<uint32_t>(R * 3);
  return w;
}

bool batch_ok(const pcb_det_batch* a) {
  if (!a || a->B < 1 || a->B >= 65536 || a->M < a->B || a->M >= LIM || a->num_points < 1 || a->B * a->num_points >= LIM) return false;
  if (a->dataset != PCB_DET_SCANNET && a->dataset != PCB_DET_SUNRGBD) return false;
  if (!offsets_ok(a->offsets_host, a->B, a->M, 0) || !a->offsets || !a->params) return false;
  return true;
}

}  // namespace

extern "C" int pcb_det_floor_height(const void* z, int64_t stride, int32_t f64, const int64_t* offsets_host, const int64_t* offsets, int64_t B,
                                    double* floor, void* stream) {
  PCB_ARG(B >= 1 && B < 65536 && stride >= 1 && (f64 == 0 || f64 == 1) && z && offsets && floor);
  PCB_ARG(offsets_host && offsets_ok(offsets_host, B, offsets_host[B], 0) && offsets_host[B] < LIM);
  cudaStream_t st = (cudaStream_t)stream;
  if (f64) floor_height_kernel<double><<<(unsigned)B, FH_THREADS, 0, st>>>((const double*)z, stride, offsets, floor);
  else floor_height_kernel<float><<<(unsigned)B, FH_THREADS, 0, st>>>((const float*)z, stride, offsets, floor);
  return check_launch("floor_height_kernel");
}

extern "C" size_t pcb_det_choices_ws_bytes(int64_t M) {
  if (M < 1 || M >= LIM) return 0;
  Carve c{nullptr};
  sort_layout(c, M);
  return c.used;
}

extern "C" int pcb_det_choices(const int64_t* offsets_host, const int64_t* offsets, int64_t B, int64_t k, uint64_t seed, uint64_t offset,
                               int64_t* out, void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(B >= 1 && B < 65536 && k >= 1 && B * k < LIM && offsets && out && ws);
  PCB_ARG(offsets_host && offsets_host[B] < LIM && offsets_ok(offsets_host, B, offsets_host[B], 0));
  const int64_t M = offsets_host[B];
  PCB_ARG(ws_bytes >= pcb_det_choices_ws_bytes(M));
  Carve c{(char*)ws};
  const SortWs w = sort_layout(c, M);
  cudaStream_t st = (cudaStream_t)stream;
  choice_keys_kernel<<<blocks_for(M, PT_THREADS), PT_THREADS, 0, st>>>(offsets, B, M, bits_for(B), seed, offset, w.k, w.idx);
  if (int e = check_launch("choice_keys_kernel")) return e;
  if (int e = sort_keys(M, w, 64, st)) return e;
  choice_out_kernel<<<blocks_for(B * k, PT_THREADS), PT_THREADS, 0, st>>>(offsets, B, M, k, seed, offset, w.sidx, out);
  return check_launch("choice_out_kernel");
}

extern "C" size_t pcb_det_points_ws_bytes(int64_t B, int64_t k) {
  if (B < 1 || k < 1 || B * k >= LIM) return 0;
  Carve c{nullptr};
  points_layout(c, B * k);
  return c.used;
}

extern "C" int pcb_det_points(const pcb_det_batch* a, void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(batch_ok(a) && a->choices && a->point_clouds && a->vote_label && a->vote_label_mask);
  PCB_ARG(!(a->flags & PCB_DET_HEIGHT) || a->floor);
  const int64_t R = a->B * a->num_points;
  cudaStream_t st = (cudaStream_t)stream;
  if (a->dataset == PCB_DET_SUNRGBD) {
    PCB_ARG(a->pc && a->votes && (!(a->flags & PCB_DET_COLOR) || !(a->flags & PCB_DET_AUGMENT) || (a->jitter && a->dropout)));
    sunrgbd_points_kernel<<<blocks_for(R, PT_THREADS), PT_THREADS, 0, st>>>(*a);
    return check_launch("sunrgbd_points_kernel");
  }
  PCB_ARG(!(a->flags & PCB_DET_COLOR) && a->vert && a->sem && a->ins && a->pcl_color && a->nyu40ids && a->n_ids >= 1);
  PCB_ARG(ws && ws_bytes >= pcb_det_points_ws_bytes(a->B, a->num_points));
  Carve c{(char*)ws};
  const PointsWs w = points_layout(c, R);
  scannet_points_kernel<<<blocks_for(R, PT_THREADS), PT_THREADS, 0, st>>>(*a, w.s.k, w.s.idx);
  if (int e = check_launch("scannet_points_kernel")) return e;
  // distinct (scene, instance id) pairs of the sampled rows: a stable sort, so each run's first row is its lowest output position
  if (int e = sort_runs(R, w.s, 32 + bits_for(a->B), st)) return e;
  PCB_CUDA(cudaMemsetAsync(w.mn, 0xFF, (size_t)R * 3 * sizeof(uint32_t), st));
  PCB_CUDA(cudaMemsetAsync(w.mx, 0x00, (size_t)R * 3 * sizeof(uint32_t), st));
  instance_bounds_kernel<<<blocks_for(R, PT_THREADS), PT_THREADS, 0, st>>>(*a, R, w.s.sidx, w.s.rank, w.run_of, w.first, w.mn, w.mx);
  if (int e = check_launch("instance_bounds_kernel")) return e;
  instance_votes_kernel<<<blocks_for(R, PT_THREADS), PT_THREADS, 0, st>>>(*a, w.run_of, w.first, w.mn, w.mx);
  return check_launch("instance_votes_kernel");
}

extern "C" int pcb_det_boxes(const pcb_det_batch* a, void* stream) {
  PCB_ARG(batch_ok(a) && a->box_offsets && a->mean_size && a->n_size >= 1);
  PCB_ARG(a->box_offsets_host && a->box_offsets_host[a->B] >= 0 &&
          offsets_ok(a->box_offsets_host, a->B, a->box_offsets_host[a->B], PCB_DET_MAX_OBJ));
  PCB_ARG(a->boxes || a->box_offsets_host[a->B] == 0);
  PCB_ARG(a->center_label && a->heading_class_label && a->heading_residual_label && a->size_class_label && a->size_residual_label &&
          a->sem_cls_label && a->box_label_mask);
  if (a->dataset == PCB_DET_SCANNET) PCB_ARG(a->nyu40ids && a->n_ids >= 1 && a->n_ids <= a->n_size);
  else PCB_ARG(a->max_gt_bboxes && a->num_heading_bin >= 1 && (a->headings || a->box_offsets_host[a->B] == 0));
  boxes_kernel<<<blocks_for(a->B * PCB_DET_MAX_OBJ, PT_THREADS), PT_THREADS, 0, (cudaStream_t)stream>>>(*a);
  return check_launch("boxes_kernel");
}
