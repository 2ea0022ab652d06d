// Semantic-segmentation training augmentation -- the per-scene CPU work of the reference's finetune loader
// (`downstream/semseg/lib/dataset.py:275-309`):
//   * point bounds (per-axis min / max) for the elastic noise grid and the S3DIS clip                  -> pcb_point_bounds
//   * `ElasticDistortion` (`lib/transforms.py:187-217`): box-blurred noise grid, trilinear interpolation   -> pcb_elastic_distort
//   * `floor(homo(xyz) @ T.T[:, :3])` minus its minimum (`lib/voxelizer.py:134-142`)                      -> pcb_affine_floor
//   * flip, auto-contrast, colour translation, colour jitter (`dataset.py:344-350`)                       -> pcb_semseg_input_transform
// Every product and sum is one IEEE operation in the reference's operand order (`__fmul_rn` / `__dadd_rn` ...), so the host oracle
// (`oracle/semseg_data_cpu.py`) reproduces the results bit for bit.  Reductions are min / max (order-independent); no float atomics.
#include <float.h>
#include "common.cuh"

using namespace pcb;

namespace {

constexpr int VB = 1 << 20;          // |voxel index| < 2^20, as pcb_voxelize
constexpr int RB = 256;              // blocks of the partial-reduction passes
constexpr int RT = 256;              // threads per block

inline unsigned reduce_blocks(int64_t n) { const unsigned b = blocks_for(n, RT); return b < RB ? (b ? b : 1) : RB; }

// in-block min / max of K lanes per thread (float), thread 0's lanes hold the result
template <int K>
__device__ void block_minmax(float (&lo)[K], float (&hi)[K]) {
  __shared__ float slo[K][RT], shi[K][RT];
  for (int k = 0; k < K; ++k) { slo[k][threadIdx.x] = lo[k]; shi[k][threadIdx.x] = hi[k]; }
  __syncthreads();
  for (int s = RT / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s)
      for (int k = 0; k < K; ++k) {
        slo[k][threadIdx.x] = fminf(slo[k][threadIdx.x], slo[k][threadIdx.x + s]);
        shi[k][threadIdx.x] = fmaxf(shi[k][threadIdx.x], shi[k][threadIdx.x + s]);
      }
    __syncthreads();
  }
  for (int k = 0; k < K; ++k) { lo[k] = slo[k][0]; hi[k] = shi[k][0]; }
}

// ---------------------------------------------------------------- bounds

// part[b] = (min x, min y, min z, max x, max y, max z) of block b's grid-stride slice
__global__ void bounds_partial_kernel(const float* __restrict__ xyz, int64_t n, float* __restrict__ part) {
  float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int64_t i = blockIdx.x * (int64_t)RT + threadIdx.x; i < n; i += (int64_t)gridDim.x * RT)
    for (int k = 0; k < 3; ++k) { const float v = xyz[3 * i + k]; lo[k] = fminf(lo[k], v); hi[k] = fmaxf(hi[k], v); }
  block_minmax<3>(lo, hi);
  if (threadIdx.x == 0)
    for (int k = 0; k < 3; ++k) { part[6 * blockIdx.x + k] = lo[k]; part[6 * blockIdx.x + 3 + k] = hi[k]; }
}

// one block: the partials -> out[6]
__global__ void bounds_final_kernel(const float* __restrict__ part, int nb, float* __restrict__ out) {
  float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int b = threadIdx.x; b < nb; b += RT)
    for (int k = 0; k < 3; ++k) { lo[k] = fminf(lo[k], part[6 * b + k]); hi[k] = fmaxf(hi[k], part[6 * b + 3 + k]); }
  block_minmax<3>(lo, hi);
  if (threadIdx.x == 0)
    for (int k = 0; k < 3; ++k) { out[k] = lo[k]; out[3 + k] = hi[k]; }
}

// ---------------------------------------------------------------- elastic distortion

// one 3-tap box filter along `axis` of the [gx, gy, gz, 3] grid, as scipy.ndimage.convolve does it on float32 input: the float32
// weight 1/3 widened to float64, the sum 0 + w x[i-1] + w x[i] + w x[i+1] in float64 (taps outside the grid read 0), rounded to float32
__global__ void blur_kernel(const float* __restrict__ in, float* __restrict__ out, int gx, int gy, int gz, int axis) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t total = (int64_t)gx * gy * gz * 3;
  if (e >= total) return;
  const int64_t cell = e / 3;
  const int iz = (int)(cell % gz), iy = (int)((cell / gz) % gy), ix = (int)(cell / ((int64_t)gz * gy));
  const int pos = axis == 0 ? ix : (axis == 1 ? iy : iz);
  const int dim = axis == 0 ? gx : (axis == 1 ? gy : gz);
  const int64_t stride = axis == 0 ? (int64_t)gy * gz * 3 : (axis == 1 ? (int64_t)gz * 3 : 3);
  const double w = (double)__fdiv_rn(1.f, 3.f);
  double acc = 0.0;
  for (int k = -1; k <= 1; ++k) {
    const int p = pos + k;
    const double v = (p >= 0 && p < dim) ? (double)in[e + k * stride] : 0.0;
    acc = __dadd_rn(acc, __dmul_rn(w, v));
  }
  out[e] = __double2float_rn(acc);
}

// RegularGridInterpolator's interval: the largest i in [0, dim - 2] with g[i] <= x (0 when x < g[0])
__device__ __forceinline__ int interval(const double* __restrict__ g, int dim, double x) {
  int lo = 0, hi = dim - 2;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (g[mid] <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// one thread per point: linear interpolation of the blurred grid (RegularGridInterpolator, fill 0 outside), xyz += value * magnitude
__global__ void elastic_kernel(float* __restrict__ xyz, int64_t n, const float* __restrict__ grid, int gx, int gy, int gz,
                               const double* __restrict__ axes, double magnitude) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int dims[3] = {gx, gy, gz};
  const double* g[3] = {axes, axes + gx, axes + gx + gy};
  double x[3], t[3], omt[3];
  int idx[3];
  bool oob = false;
  for (int d = 0; d < 3; ++d) {
    x[d] = (double)xyz[3 * i + d];
    const int j = interval(g[d], dims[d], x[d]);
    idx[d] = j;
    t[d] = __ddiv_rn(__dsub_rn(x[d], g[d][j]), __dsub_rn(g[d][j + 1], g[d][j]));
    omt[d] = __dsub_rn(1.0, t[d]);
    oob |= x[d] < g[d][0] || x[d] > g[d][dims[d] - 1];
  }
  double v[3] = {0.0, 0.0, 0.0};
  for (int c = 0; c < 8; ++c) {                      // itertools.product order: the last axis fastest
    const int c0 = c >> 2, c1 = (c >> 1) & 1, c2 = c & 1;
    double w = 1.0;
    w = __dmul_rn(w, c0 ? t[0] : omt[0]);
    w = __dmul_rn(w, c1 ? t[1] : omt[1]);
    w = __dmul_rn(w, c2 ? t[2] : omt[2]);
    const float* p = grid + ((((int64_t)(idx[0] + c0) * gy + (idx[1] + c1)) * gz + (idx[2] + c2)) * 3);
    for (int k = 0; k < 3; ++k) v[k] = __dadd_rn(v[k], __dmul_rn((double)p[k], w));
  }
  for (int k = 0; k < 3; ++k) {
    const double add = oob ? 0.0 : __dmul_rn(v[k], magnitude);
    xyz[3 * i + k] = __double2float_rn(__dadd_rn(x[k], add));
  }
}

// ---------------------------------------------------------------- affine floor

struct Rows3x4 { double m[12]; };

// floor(((x T[j,0] + y T[j,1]) + z T[j,2]) + T[j,3]) in float64 (homo_coords @ T.T[:, :3] with the homogeneous 1), its block minimum
// merged into mins[3] (int32 atomicMin: an exact, order-independent reduction)
__global__ void affine_floor_kernel(const float* __restrict__ xyz, int64_t n, Rows3x4 T, int32_t* __restrict__ out, int32_t* mins,
                                    int32_t* status) {
  __shared__ int32_t smin[3];
  if (threadIdx.x < 3) smin[threadIdx.x] = INT32_MAX;
  __syncthreads();
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) {
    const double x = (double)xyz[3 * i], y = (double)xyz[3 * i + 1], z = (double)xyz[3 * i + 2];
    for (int j = 0; j < 3; ++j) {
      const double* r = T.m + 4 * j;
      const double v = floor(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, r[0]), __dmul_rn(y, r[1])), __dmul_rn(z, r[2])), r[3]));
      int c = 0;
      if (fabs(v) < (double)VB) c = (int)v; else atomicOr(status, PCB_ERR_RANGE);
      out[3 * i + j] = c;
      atomicMin(&smin[j], c);
    }
  }
  __syncthreads();
  if (threadIdx.x < 3) atomicMin(&mins[threadIdx.x], smin[threadIdx.x]);
}

__global__ void shift_kernel(int32_t* __restrict__ c, int64_t n, const int32_t* __restrict__ mins) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < 3 * n) c[i] -= mins[i % 3];
}

// ---------------------------------------------------------------- flip + colour

// part[b] = colour (min r, g, b, max r, g, b) floats and coordinate max (x, y, z) ints of block b's slice
__global__ void tf_partial_kernel(const int32_t* __restrict__ coords, const float* __restrict__ feats, int64_t n, float* __restrict__ fpart,
                                  int32_t* __restrict__ ipart) {
  __shared__ int32_t sc[3];
  if (threadIdx.x < 3) sc[threadIdx.x] = INT32_MIN;
  __syncthreads();
  float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  int32_t cm[3] = {INT32_MIN, INT32_MIN, INT32_MIN};
  for (int64_t i = blockIdx.x * (int64_t)RT + threadIdx.x; i < n; i += (int64_t)gridDim.x * RT)
    for (int k = 0; k < 3; ++k) {
      const float v = feats[3 * i + k];
      lo[k] = fminf(lo[k], v); hi[k] = fmaxf(hi[k], v);
      if (coords) cm[k] = max(cm[k], coords[3 * i + k]);
    }
  for (int k = 0; k < 3; ++k) atomicMax(&sc[k], cm[k]);
  block_minmax<3>(lo, hi);
  if (threadIdx.x == 0)
    for (int k = 0; k < 3; ++k) { fpart[6 * blockIdx.x + k] = lo[k]; fpart[6 * blockIdx.x + 3 + k] = hi[k]; ipart[3 * blockIdx.x + k] = sc[k]; }
}

// one block: the partials -> red = (colour lo[3], hi[3]) and cmax[3]; status |= RANGE if auto-contrast is on and max(hi) <= 1
__global__ void tf_final_kernel(const float* __restrict__ fpart, const int32_t* __restrict__ ipart, int nb, int contrast, float* __restrict__ red,
                                int32_t* __restrict__ cmax, int32_t* status) {
  __shared__ int32_t sc[3];
  if (threadIdx.x < 3) sc[threadIdx.x] = INT32_MIN;
  __syncthreads();
  float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  int32_t cm[3] = {INT32_MIN, INT32_MIN, INT32_MIN};
  for (int b = threadIdx.x; b < nb; b += RT)
    for (int k = 0; k < 3; ++k) {
      lo[k] = fminf(lo[k], fpart[6 * b + k]); hi[k] = fmaxf(hi[k], fpart[6 * b + 3 + k]);
      cm[k] = max(cm[k], ipart[3 * b + k]);
    }
  for (int k = 0; k < 3; ++k) atomicMax(&sc[k], cm[k]);
  block_minmax<3>(lo, hi);
  if (threadIdx.x == 0) {
    for (int k = 0; k < 3; ++k) { red[k] = lo[k]; red[3 + k] = hi[k]; cmax[k] = sc[k]; }
    if (contrast && !(fmaxf(fmaxf(hi[0], hi[1]), hi[2]) > 1.f)) *status = PCB_ERR_RANGE;     // `transforms.py:53`
  }
}

struct TfArgs {
  int flip_mask, contrast, translate, normalize;
  double blend, jitter_scale, tr[3];
};

__device__ __forceinline__ double clip255(double v) { return v < 0.0 ? 0.0 : (v > 255.0 ? 255.0 : v); }

// one thread per voxel, in `Compose` order: flip -> auto-contrast -> translation -> jitter (-> optional colour normalisation)
__global__ void tf_apply_kernel(int32_t* __restrict__ coords, float* __restrict__ feats, int64_t n, const float* __restrict__ red,
                                const int32_t* __restrict__ cmax, const double* __restrict__ noise, TfArgs a) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int k = 0; k < 3; ++k)
    if (a.flip_mask >> k & 1) coords[3 * i + k] = cmax[k] - coords[3 * i + k];
  float f[3] = {feats[3 * i], feats[3 * i + 1], feats[3 * i + 2]};
  if (a.contrast) {          // float32 throughout; the Python-float blend factors are rounded to float32 first (`transforms.py:55-60`)
    const float keep = __double2float_rn(__dsub_rn(1.0, a.blend)), mix = __double2float_rn(a.blend);
    for (int k = 0; k < 3; ++k) {
      const float scale = __fdiv_rn(255.f, __fsub_rn(red[3 + k], red[k]));
      const float contrast = __fmul_rn(__fsub_rn(f[k], red[k]), scale);
      f[k] = __fadd_rn(__fmul_rn(keep, f[k]), __fmul_rn(mix, contrast));
    }
  }
  if (a.translate)           // float64 offset + float32 colour, clipped in float64, stored float32 (`transforms.py:34-35`)
    for (int k = 0; k < 3; ++k) f[k] = __double2float_rn(clip255(__dadd_rn(a.tr[k], (double)f[k])));
  if (noise)                 // noise *= std * 255; clip(noise + colour) (`transforms.py:71-73`)
    for (int k = 0; k < 3; ++k) f[k] = __double2float_rn(clip255(__dadd_rn(__dmul_rn(noise[3 * i + k], a.jitter_scale), (double)f[k])));
  if (a.normalize)           // `lib/train.py:114`: colour / 255 - 0.5 in float32
    for (int k = 0; k < 3; ++k) f[k] = __fsub_rn(__fdiv_rn(f[k], 255.f), 0.5f);
  for (int k = 0; k < 3; ++k) feats[3 * i + k] = f[k];
}

// ---------------------------------------------------------------- workspace layouts

// per-block partials, then the final (lo[3], hi[3])
struct BoundsWs { float* part; float* out; };
BoundsWs bounds_layout(Carve& c) { return {c.take<float>(RB * 6), c.take<float>(6)}; }

// the blur's second buffer (the noise grid is the first)
float* elastic_layout(Carve& c, int gx, int gy, int gz) { return c.take<float>((int64_t)gx * gy * gz * 3); }

// mins[0..2], mins[4] = the range status: one copy back to the host
int32_t* affine_layout(Carve& c) { return c.take<int32_t>(5); }

// per-block partials (colour floats, coordinate ints), the reduced colour range (lo[3], hi[3]), coordinate maxima, auto-contrast status
struct TfWs { float* fpart; int32_t* ipart; float* red; int32_t* cmax; int32_t* status; };
TfWs tf_layout(Carve& c) { return {c.take<float>(RB * 6), c.take<int32_t>(RB * 3), c.take<float>(6), c.take<int32_t>(3), c.take<int32_t>(1)}; }

}  // namespace

extern "C" size_t pcb_point_bounds_ws_bytes(void) {
  return layout_bytes(bounds_layout);
}

extern "C" int pcb_point_bounds(const float* xyz, int64_t n, float* lo, float* hi, void* ws, size_t ws_bytes, void* stream) {
  Carve c{(char*)ws};
  const BoundsWs w = bounds_layout(c);
  PCB_ARG(n > 0 && xyz && lo && hi && ws && ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned nb = reduce_blocks(n);
  bounds_partial_kernel<<<nb, RT, 0, st>>>(xyz, n, w.part);
  if (int e = check_launch("bounds_partial_kernel")) return e;
  bounds_final_kernel<<<1, RT, 0, st>>>(w.part, (int)nb, w.out);
  if (int e = check_launch("bounds_final_kernel")) return e;
  float h[6];
  PCB_CUDA(cudaMemcpyAsync(h, w.out, sizeof(h), cudaMemcpyDeviceToHost, st));
  PCB_CUDA(cudaStreamSynchronize(st));
  for (int k = 0; k < 3; ++k) { lo[k] = h[k]; hi[k] = h[3 + k]; }
  return PCB_OK;
}

extern "C" size_t pcb_elastic_distort_ws_bytes(int gx, int gy, int gz) {
  return layout_bytes(elastic_layout, gx > 0 ? gx : 1, gy > 0 ? gy : 1, gz > 0 ? gz : 1);
}

extern "C" int pcb_elastic_distort(float* xyz, int64_t n, float* noise, int gx, int gy, int gz, const double* axes, double magnitude, void* ws,
                                   size_t ws_bytes, void* stream) {
  PCB_ARG(n >= 0 && n < (1ll << 31) && gx >= 2 && gy >= 2 && gz >= 2 && (int64_t)gx * gy * gz < (1ll << 29));
  Carve c{(char*)ws};
  float* tmp = elastic_layout(c, gx, gy, gz);
  PCB_ARG(noise && axes && ws && ws_bytes >= c.used && (n == 0 || xyz));
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t total = (int64_t)gx * gy * gz * 3;
  float* bufs[2] = {noise, tmp};
  for (int pass = 0; pass < 6; ++pass) {             // two rounds of x, y, z; even count: the result lands back in `noise`
    blur_kernel<<<blocks_for(total, 256), 256, 0, st>>>(bufs[pass & 1], bufs[(pass & 1) ^ 1], gx, gy, gz, pass % 3);
    if (int e = check_launch("blur_kernel")) return e;
  }
  if (n == 0) return PCB_OK;
  elastic_kernel<<<blocks_for(n, 128), 128, 0, st>>>(xyz, n, noise, gx, gy, gz, axes, magnitude);
  return check_launch("elastic_kernel");
}

extern "C" size_t pcb_affine_floor_ws_bytes(void) {
  return layout_bytes(affine_layout);
}

extern "C" int pcb_affine_floor(const float* xyz, int64_t n, const double* T, int32_t* out, int32_t* min_out, void* ws, size_t ws_bytes,
                                void* stream) {
  Carve c{(char*)ws};
  int32_t* mins = affine_layout(c);
  PCB_ARG(n > 0 && n < (1ll << 31) && xyz && T && out && min_out && ws && ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  Rows3x4 R;
  for (int k = 0; k < 12; ++k) R.m[k] = T[k];
  int32_t* status = mins + 4;
  PCB_CUDA(cudaMemsetAsync(mins, 0x7F, 3 * sizeof(int32_t), st));      // 0x7F7F7F7F: above every in-range index
  PCB_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
  affine_floor_kernel<<<blocks_for(n, 256), 256, 0, st>>>(xyz, n, R, out, mins, status);
  if (int e = check_launch("affine_floor_kernel")) return e;
  shift_kernel<<<blocks_for(3 * n, 256), 256, 0, st>>>(out, n, mins);
  if (int e = check_launch("shift_kernel")) return e;
  int32_t h[5];
  PCB_CUDA(cudaMemcpyAsync(h, mins, sizeof(h), cudaMemcpyDeviceToHost, st));
  PCB_CUDA(cudaStreamSynchronize(st));
  if (h[4]) { set_error("pcb_affine_floor: a transformed point lies outside +-2^20 voxels"); return PCB_ERR_RANGE; }
  for (int k = 0; k < 3; ++k) min_out[k] = h[k];
  return PCB_OK;
}

extern "C" size_t pcb_semseg_input_transform_ws_bytes(void) {
  return layout_bytes(tf_layout);
}

extern "C" int pcb_semseg_input_transform(int32_t* coords, float* feats, int64_t n, int flip_mask, int contrast, double blend,
                                          const double* translation, const double* jitter_noise, double jitter_scale, int normalize, void* ws,
                                          size_t ws_bytes, void* stream) {
  Carve c{(char*)ws};
  const TfWs w = tf_layout(c);
  PCB_ARG(n > 0 && n < (1ll << 31) && (coords || flip_mask == 0) && feats && (flip_mask & ~7) == 0 && ws && ws_bytes >= c.used);
  cudaStream_t st = (cudaStream_t)stream;
  TfArgs a;
  a.flip_mask = flip_mask; a.contrast = contrast != 0; a.translate = translation != nullptr; a.normalize = normalize != 0;
  a.blend = blend; a.jitter_scale = jitter_scale;
  for (int k = 0; k < 3; ++k) a.tr[k] = translation ? translation[k] : 0.0;
  if (flip_mask || a.contrast) {                    // the reductions the flip and the auto-contrast read
    PCB_CUDA(cudaMemsetAsync(w.status, 0, sizeof(int32_t), st));
    const unsigned nb = reduce_blocks(n);
    tf_partial_kernel<<<nb, RT, 0, st>>>(coords, feats, n, w.fpart, w.ipart);
    if (int e = check_launch("tf_partial_kernel")) return e;
    tf_final_kernel<<<1, RT, 0, st>>>(w.fpart, w.ipart, (int)nb, a.contrast, w.red, w.cmax, w.status);
    if (int e = check_launch("tf_final_kernel")) return e;
  }
  tf_apply_kernel<<<blocks_for(n, 256), 256, 0, st>>>(coords, feats, n, w.red, w.cmax, jitter_noise, a);
  if (int e = check_launch("tf_apply_kernel")) return e;
  if (a.contrast) {
    int32_t h = 0;
    PCB_CUDA(cudaMemcpyAsync(&h, w.status, sizeof(h), cudaMemcpyDeviceToHost, st));
    PCB_CUDA(cudaStreamSynchronize(st));
    if (h) { set_error("pcb_semseg_input_transform: colour maximum <= 1 (colours must be in [0, 255])"); return PCB_ERR_RANGE; }
  }
  return PCB_OK;
}
