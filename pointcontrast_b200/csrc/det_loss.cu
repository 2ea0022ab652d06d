// VoteNet's training loss (`models/loss_helper.py::get_loss`, `lib/utils/nn_distance.py`) and its gradients on the device:
//   * det_loss_scene_kernel: grid (scene, part).  Each thread takes seeds, proposals and label slots in a fixed stride and computes the
//     per-element terms in fp32 as the original's torch ops round them (no FMA contraction), keeps the argmins the backward needs in
//     `state`, and adds its share of the 14 batch sums in fp64; the CTA reduces them in a fixed tree order into one row per (scene, part).
//   * det_loss_finish_kernel: one warp sums those rows in ascending order (fp64), rounds each term once and writes the 13 outputs.
//   * det_loss_backward_kernel: the same grid; every gradient element is written by exactly one thread, the dist2 gradients of a
//     proposal summed over the label slots in ascending order.  No atomics anywhere.
#include <math.h>
#include "common.cuh"

using namespace pcb;

namespace {

constexpr int THREADS = 256;
constexpr int MAX_PARTS = 8;
constexpr int MAX_NS = 64;
// the batch sums, in this order
enum { Q_VOTE, Q_VOTE_MASK, Q_OBJ, Q_OBJ_MASK, Q_C1, Q_LABEL, Q_C2, Q_BOX_MASK, Q_HCLS, Q_HREG, Q_SCLS, Q_SREG, Q_SEM, Q_ACC, NQ };
// the outputs, in this order
enum { O_VOTE, O_OBJ, O_CENTER, O_HCLS, O_HREG, O_SCLS, O_SREG, O_SEM, O_BOX, O_LOSS, O_POS, O_NEG, O_ACC, NOUT };
// the denominators kept in `state` for the backward
enum { D_VOTE, D_OBJ, D_LABEL, D_BOX, ND };

struct MeanSize { float v[3 * MAX_NS]; };

struct StateLayout {
  double* den;        // [ND]: the fp32 denominators sum + 1e-6
  int32_t* vote_pick;  // [B, S]: j * V + v of the (GT vote, predicted vote) pair the vote min returned
  int32_t* cidx1;      // [B, K]: nearest label slot of each predicted center
  int32_t* cidx2;      // [B, K2]: nearest predicted center of each label slot
};
StateLayout state_layout(Carve& c, int64_t B, int64_t S, int64_t K, int64_t K2) {
  StateLayout s;
  s.den = c.take<double>(ND);
  s.vote_pick = c.take<int32_t>(B * S);
  s.cidx1 = c.take<int32_t>(B * K);
  s.cidx2 = c.take<int32_t>(B * K2);
  return s;
}
int parts_for(int64_t S, int64_t K, int64_t K2) {
  const int64_t n = S > K ? (S > K2 ? S : K2) : (K > K2 ? K : K2);
  const int64_t p = (n + THREADS - 1) / THREADS;
  return (int)(p < 1 ? 1 : (p > MAX_PARTS ? MAX_PARTS : p));
}
double* ws_layout(Carve& c, int64_t B, int parts) { return c.take<double>(B * parts * NQ); }

__device__ __forceinline__ float at(const pcb_strided& t, int64_t b, int64_t k, int64_t c, int64_t x = 0) {
  return t.p[b * t.sb + k * t.sk + c * t.sc + x * t.sx];
}
// (dx dx + dy dy) + dz dz and (|dx| + |dy|) + |dz| of nn_distance, pc1 - pc2
__device__ __forceinline__ float sqdist(const float* a, const float* b) {
  const float dx = __fsub_rn(a[0], b[0]), dy = __fsub_rn(a[1], b[1]), dz = __fsub_rn(a[2], b[2]);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}
__device__ __forceinline__ float l1dist(const float* a, const float* b) {
  return __fadd_rn(__fadd_rn(fabsf(__fsub_rn(a[0], b[0])), fabsf(__fsub_rn(a[1], b[1]))), fabsf(__fsub_rn(a[2], b[2])));
}
// torch.min(dim): the first minimum, a NaN counting as the minimum
__device__ __forceinline__ bool takes_min(float d, float best) { return d < best || (isnan(d) && !isnan(best)); }
__device__ __forceinline__ float sgn(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }
// huber_loss(x, delta=1): q = clamp(|x|, max=1), 0.5 q^2 + (|x| - q); its derivative is clamp(x, -1, 1)
__device__ __forceinline__ float huber(float x) {
  const float a = fabsf(x), q = a > 1.f ? 1.f : a;
  return __fadd_rn(__fmul_rn(0.5f, __fmul_rn(q, q)), __fsub_rn(a, q));
}
__device__ __forceinline__ float huber_grad(float x) { return x > 1.f ? 1.f : (x < -1.f ? -1.f : x); }
// log_softmax row statistics of a strided row: m = the maximum (NaN propagates), s = sum of expf(x - m) in ascending order
__device__ __forceinline__ void row_stats(const pcb_strided& t, int64_t b, int64_t k, int n, float& m, float& s) {
  m = at(t, b, k, 0);
  for (int c = 1; c < n; ++c) {
    const float x = at(t, b, k, c);
    if (x > m || isnan(x)) m = x;
  }
  s = 0.f;
  for (int c = 0; c < n; ++c) s = __fadd_rn(s, expf(__fsub_rn(at(t, b, k, c), m)));
}
// nll_loss(log_softmax(x), y) = -((x[y] - m) - log s)
__device__ __forceinline__ float cross_entropy(const pcb_strided& t, int64_t b, int64_t k, int n, int64_t y) {
  float m, s;
  row_stats(t, b, k, n, m, s);
  return -__fsub_rn(__fsub_rn(at(t, b, k, y), m), logf(s));
}
// g (softmax - onehot(y)) over a strided row into a dense row
__device__ __forceinline__ void cross_entropy_grad(const pcb_strided& t, int64_t b, int64_t k, int n, int64_t y, float g, float* out) {
  float m, s;
  row_stats(t, b, k, n, m, s);
  for (int c = 0; c < n; ++c) out[c] = __fmul_rn(g, __fsub_rn(__fdiv_rn(expf(__fsub_rn(at(t, b, k, c), m)), s), c == y ? 1.f : 0.f));
}
__device__ __forceinline__ void fill(float* out, int n, float v) {
  for (int c = 0; c < n; ++c) out[c] = v;
}
__device__ __forceinline__ void gt_center(const pcb_det_loss_args& a, int64_t b, int64_t j, float* g) {
  const float* p = a.center_label + (b * a.K2 + j) * a.center_label_ld;
  g[0] = p[0]; g[1] = p[1]; g[2] = p[2];
}
__device__ __forceinline__ void center_of(const pcb_det_loss_args& a, int64_t b, int64_t k, float* c) {
  c[0] = at(a.center, b, k, 0); c[1] = at(a.center, b, k, 1); c[2] = at(a.center, b, k, 2);
}
// the nearest label slot of point p (squared distance, first minimum)
__device__ __forceinline__ int nearest_slot(const pcb_det_loss_args& a, int64_t b, const float* p, float& best) {
  int bi = 0;
  best = INFINITY;
  for (int64_t j = 0; j < a.K2; ++j) {
    float g[3];
    gt_center(a, b, j, g);
    const float d = sqdist(p, g);
    if (j == 0 || takes_min(d, best)) { best = d; bi = (int)j; }
  }
  return bi;
}
// the GT votes of seed i (vote_label gathered at seed_inds, plus seed_xyz); false when the index lies outside [0, N)
__device__ __forceinline__ bool gt_votes(const pcb_det_loss_args& a, int64_t b, int64_t i, float* gv, float& mask) {
  const int64_t idx = a.seed_inds_i64 ? ((const int64_t*)a.seed_inds)[b * a.S + i] : (int64_t)((const int32_t*)a.seed_inds)[b * a.S + i];
  if (idx < 0 || idx >= a.N) return false;
  const float* vl = a.vote_label + (b * a.N + idx) * 9;
  const float* sx = a.seed_xyz + (b * a.S + i) * 3;
  for (int j = 0; j < 9; ++j) gv[j] = __fadd_rn(vl[j], sx[j % 3]);
  mask = (float)a.vote_label_mask[b * a.N + idx];
  return true;
}

__device__ __forceinline__ void block_sums(double (*red)[THREADS], const double* acc, double* row) {
  for (int q = 0; q < NQ; ++q) red[q][threadIdx.x] = acc[q];
  __syncthreads();
  for (int h = THREADS / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h)
      for (int q = 0; q < NQ; ++q) red[q][threadIdx.x] += red[q][threadIdx.x + h];
    __syncthreads();
  }
  if ((int)threadIdx.x < NQ) row[threadIdx.x] = red[threadIdx.x][0];
}

__global__ void __launch_bounds__(THREADS) det_loss_scene_kernel(pcb_det_loss_args a, MeanSize ms, int parts, int64_t* obj_label,
                                                                  float* obj_mask, int64_t* assignment, StateLayout st, double* partial) {
  __shared__ double red[NQ][THREADS];
  const int64_t b = blockIdx.x;
  const int64_t t0 = (int64_t)blockIdx.y * THREADS + threadIdx.x, step = (int64_t)parts * THREADS;
  double acc[NQ];
  for (int q = 0; q < NQ; ++q) acc[q] = 0.0;

  // ---- vote term
  for (int64_t i = t0; i < a.S; i += step) {
    float gv[9], mask, dist = NAN;
    int pick = 0;
    if (gt_votes(a, b, i, gv, mask)) {
      const float* vx = a.vote_xyz + (b * a.S + i) * a.V * 3;
      for (int j = 0; j < 3; ++j) {
        float dj = 0.f;
        int vj = 0;
        for (int64_t v = 0; v < a.V; ++v) {
          const float d = l1dist(vx + v * 3, gv + 3 * j);
          if (v == 0 || takes_min(d, dj)) { dj = d; vj = (int)v; }
        }
        if (j == 0 || takes_min(dj, dist)) { dist = dj; pick = j * (int)a.V + vj; }
      }
    } else {
      mask = NAN;
    }
    st.vote_pick[b * a.S + i] = pick;
    acc[Q_VOTE] += (double)__fmul_rn(dist, mask);
    acc[Q_VOTE_MASK] += (double)mask;
  }

  // ---- proposals: assignment, objectness, center dist1, heading / size / semantic terms
  for (int64_t k = t0; k < a.K; k += step) {
    const int64_t r = b * a.K + k;
    float d1;
    const int j = nearest_slot(a, b, a.aggregated_vote_xyz + r * 3, d1);
    const float e = sqrtf(__fadd_rn(d1, 1e-6f));
    const int lab = e < 0.3f ? 1 : 0;
    const float m = (lab || e > 0.6f) ? 1.f : 0.f, l = (float)lab;
    obj_label[r] = lab;
    obj_mask[r] = m;
    assignment[r] = j;

    acc[Q_OBJ] += (double)__fmul_rn(__fmul_rn(lab ? 0.8f : 0.2f, cross_entropy(a.objectness_scores, b, k, 2, lab)), m);
    acc[Q_OBJ_MASK] += (double)m;
    const float x0 = at(a.objectness_scores, b, k, 0), x1 = at(a.objectness_scores, b, k, 1);
    const int pred = (isnan(x0) || !(x1 > x0 || isnan(x1))) ? 0 : 1;       // torch.argmax: first maximum, NaN maximal
    acc[Q_ACC] += (double)(pred == lab ? m : 0.f);

    float c[3], dc;
    center_of(a, b, k, c);
    st.cidx1[r] = nearest_slot(a, b, c, dc);
    acc[Q_C1] += (double)__fmul_rn(dc, l);
    acc[Q_LABEL] += (double)l;

    const int64_t g = b * a.K2 + j;
    const int64_t hc = a.heading_class_label[g], sc = a.size_class_label[g], cc = a.sem_cls_label[g];
    float hcls = NAN, hreg = NAN, scls = NAN, sreg = NAN, sem = NAN;
    if (hc >= 0 && hc < a.NH) {
      hcls = cross_entropy(a.heading_scores, b, k, a.NH, hc);
      hreg = huber(__fsub_rn(at(a.heading_residuals_normalized, b, k, hc), __fmul_rn(a.heading_residual_label[g], a.heading_scale)));
    }
    if (sc >= 0 && sc < a.NS) {
      scls = cross_entropy(a.size_scores, b, k, a.NS, sc);
      float h[3];
      for (int x = 0; x < 3; ++x)
        h[x] = huber(__fsub_rn(at(a.size_residuals_normalized, b, k, sc, x), __fdiv_rn(a.size_residual_label[g * 3 + x], ms.v[sc * 3 + x])));
      sreg = __fdiv_rn(__fadd_rn(__fadd_rn(h[0], h[1]), h[2]), 3.f);
    }
    if (cc >= 0 && cc < a.C) sem = cross_entropy(a.sem_cls_scores, b, k, a.C, cc);
    acc[Q_HCLS] += (double)__fmul_rn(hcls, l);
    acc[Q_HREG] += (double)__fmul_rn(hreg, l);
    acc[Q_SCLS] += (double)__fmul_rn(scls, l);
    acc[Q_SREG] += (double)__fmul_rn(sreg, l);
    acc[Q_SEM] += (double)__fmul_rn(sem, l);
  }

  // ---- label slots: center dist2
  for (int64_t j = t0; j < a.K2; j += step) {
    float g[3], best = INFINITY;
    gt_center(a, b, j, g);
    int bk = 0;
    for (int64_t k = 0; k < a.K; ++k) {
      float c[3];
      center_of(a, b, k, c);
      const float d = sqdist(c, g);
      if (k == 0 || takes_min(d, best)) { best = d; bk = (int)k; }
    }
    st.cidx2[b * a.K2 + j] = bk;
    const float bm = a.box_label_mask[b * a.K2 + j];
    acc[Q_C2] += (double)__fmul_rn(best, bm);
    acc[Q_BOX_MASK] += (double)bm;
  }
  block_sums(red, acc, partial + (b * parts + blockIdx.y) * NQ);
}

__global__ void det_loss_finish_kernel(const double* partial, int64_t rows, int64_t BK, float* out, double* den) {
  __shared__ double tot[NQ];
  const int q = threadIdx.x;
  if (q < NQ) {
    double s = 0.0;
    for (int64_t r = 0; r < rows; ++r) s += partial[r * NQ + q];
    tot[q] = s;
  }
  __syncwarp();
  if (q != 0) return;
  // the original's denominators sum(x) + 1e-6 are fp32 (the sums of 0/1 values are exact below 2^24)
  double den_of[NQ];
  for (int d : {Q_VOTE_MASK, Q_OBJ_MASK, Q_LABEL, Q_BOX_MASK}) den_of[d] = (double)__fadd_rn((float)tot[d], 1e-6f);
  auto mean = [&](int num, int d) { return (float)(tot[num] / den_of[d]); };
  float o[NOUT];
  o[O_VOTE] = mean(Q_VOTE, Q_VOTE_MASK);
  o[O_OBJ] = mean(Q_OBJ, Q_OBJ_MASK);
  o[O_CENTER] = (float)(tot[Q_C1] / den_of[Q_LABEL] + tot[Q_C2] / den_of[Q_BOX_MASK]);
  o[O_HCLS] = mean(Q_HCLS, Q_LABEL);
  o[O_HREG] = mean(Q_HREG, Q_LABEL);
  o[O_SCLS] = mean(Q_SCLS, Q_LABEL);
  o[O_SREG] = mean(Q_SREG, Q_LABEL);
  o[O_SEM] = mean(Q_SEM, Q_LABEL);
  // box_loss and loss as get_loss writes them, in fp32 and in its order
  o[O_BOX] = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(o[O_CENTER], __fmul_rn(0.1f, o[O_HCLS])), o[O_HREG]), __fmul_rn(0.1f, o[O_SCLS])),
                       o[O_SREG]);
  o[O_LOSS] = __fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(o[O_VOTE], __fmul_rn(0.5f, o[O_OBJ])), o[O_BOX]), __fmul_rn(0.1f, o[O_SEM])), 10.f);
  // sum / float(B K) with a Python float: torch multiplies by the fp32 reciprocal
  const float inv = 1.f / (float)BK;
  o[O_POS] = __fmul_rn((float)tot[Q_LABEL], inv);
  o[O_NEG] = __fsub_rn(__fmul_rn((float)tot[Q_OBJ_MASK], inv), o[O_POS]);
  o[O_ACC] = mean(Q_ACC, Q_OBJ_MASK);
  for (int i = 0; i < NOUT; ++i) out[i] = o[i];
  den[D_VOTE] = den_of[Q_VOTE_MASK];
  den[D_OBJ] = den_of[Q_OBJ_MASK];
  den[D_LABEL] = den_of[Q_LABEL];
  den[D_BOX] = den_of[Q_BOX_MASK];
}

struct Grads {
  float *vote_xyz, *seed_xyz, *center, *obj, *hs, *hr, *ss, *sr, *sem;
};

__global__ void __launch_bounds__(THREADS) det_loss_backward_kernel(pcb_det_loss_args a, MeanSize ms, int parts, const float* grad,
                                                                     const int64_t* obj_label, const float* obj_mask,
                                                                     const int64_t* assignment, StateLayout st, Grads gr) {
  const int64_t b = blockIdx.x;
  const int64_t t0 = (int64_t)blockIdx.y * THREADS + threadIdx.x, step = (int64_t)parts * THREADS;
  // fold d box_loss and d loss into the eight terms as autograd does on the original graph (loss = 10 (vote + 0.5 obj + box + 0.1 sem))
  const float gl = __fmul_rn(grad[O_LOSS], 10.f), gb = __fadd_rn(grad[O_BOX], gl);
  float G[O_BOX];
  G[O_VOTE] = __fadd_rn(grad[O_VOTE], gl);
  G[O_OBJ] = __fadd_rn(grad[O_OBJ], __fmul_rn(0.5f, gl));
  G[O_CENTER] = __fadd_rn(grad[O_CENTER], gb);
  G[O_HCLS] = __fadd_rn(grad[O_HCLS], __fmul_rn(0.1f, gb));
  G[O_HREG] = __fadd_rn(grad[O_HREG], gb);
  G[O_SCLS] = __fadd_rn(grad[O_SCLS], __fmul_rn(0.1f, gb));
  G[O_SREG] = __fadd_rn(grad[O_SREG], gb);
  G[O_SEM] = __fadd_rn(grad[O_SEM], __fmul_rn(0.1f, gl));
  auto scale = [&](int o, int d) { return (float)((double)G[o] / st.den[d]); };
  const float s_vote = scale(O_VOTE, D_VOTE), s_obj = scale(O_OBJ, D_OBJ), s_c1 = scale(O_CENTER, D_LABEL), s_c2 = scale(O_CENTER, D_BOX);
  const float s_hcls = scale(O_HCLS, D_LABEL), s_hreg = scale(O_HREG, D_LABEL), s_scls = scale(O_SCLS, D_LABEL);
  const float s_sreg = scale(O_SREG, D_LABEL), s_sem = scale(O_SEM, D_LABEL);

  // ---- votes: only the (GT vote, predicted vote) pair the min returned gets a gradient
  for (int64_t i = t0; i < a.S; i += step) {
    float gv[9], mask, gvote[3] = {NAN, NAN, NAN};
    const int pick = st.vote_pick[b * a.S + i], j = pick / (int)a.V, vp = pick % (int)a.V;
    const float* vx = a.vote_xyz + (b * a.S + i) * a.V * 3;
    if (gt_votes(a, b, i, gv, mask)) {
      const float w = __fmul_rn(s_vote, mask);
      for (int x = 0; x < 3; ++x) gvote[x] = __fmul_rn(w, sgn(__fsub_rn(vx[vp * 3 + x], gv[3 * j + x])));
    }
    if (gr.vote_xyz)
      for (int64_t v = 0; v < a.V; ++v)
        for (int x = 0; x < 3; ++x) gr.vote_xyz[((b * a.S + i) * a.V + v) * 3 + x] = v == vp ? gvote[x] : 0.f;
    if (gr.seed_xyz)
      for (int x = 0; x < 3; ++x) gr.seed_xyz[(b * a.S + i) * 3 + x] = -gvote[x];
  }

  // ---- proposals
  for (int64_t k = t0; k < a.K; k += step) {
    const int64_t r = b * a.K + k, g = b * a.K2 + assignment[r];
    const int lab = (int)obj_label[r];
    const float l = (float)lab, m = obj_mask[r];
    if (gr.obj)
      cross_entropy_grad(a.objectness_scores, b, k, 2, lab, __fmul_rn(__fmul_rn(s_obj, m), lab ? 0.8f : 0.2f), gr.obj + r * 2);
    if (gr.center) {
      float c[3], q[3], gc[3];
      center_of(a, b, k, c);
      gt_center(a, b, st.cidx1[r], q);
      const float w1 = __fmul_rn(s_c1, l);
      for (int x = 0; x < 3; ++x) gc[x] = __fmul_rn(w1, __fmul_rn(2.f, __fsub_rn(c[x], q[x])));
      for (int64_t j = 0; j < a.K2; ++j) {
        if (st.cidx2[b * a.K2 + j] != k) continue;
        gt_center(a, b, j, q);
        const float w2 = __fmul_rn(s_c2, a.box_label_mask[b * a.K2 + j]);
        for (int x = 0; x < 3; ++x) gc[x] = __fadd_rn(gc[x], __fmul_rn(w2, __fmul_rn(2.f, __fsub_rn(c[x], q[x]))));
      }
      for (int x = 0; x < 3; ++x) gr.center[r * 3 + x] = gc[x];
    }
    const int64_t hc = a.heading_class_label[g], sc = a.size_class_label[g], cc = a.sem_cls_label[g];
    const bool hok = hc >= 0 && hc < a.NH, sok = sc >= 0 && sc < a.NS;
    if (gr.hs) {
      if (hok) cross_entropy_grad(a.heading_scores, b, k, a.NH, hc, __fmul_rn(s_hcls, l), gr.hs + r * a.NH);
      else fill(gr.hs + r * a.NH, a.NH, NAN);
    }
    if (gr.hr) {
      float* o = gr.hr + r * a.NH;
      fill(o, a.NH, hok ? 0.f : NAN);
      if (hok) {
        const float d = __fsub_rn(at(a.heading_residuals_normalized, b, k, hc), __fmul_rn(a.heading_residual_label[g], a.heading_scale));
        o[hc] = __fmul_rn(__fmul_rn(s_hreg, l), huber_grad(d));
      }
    }
    if (gr.ss) {
      if (sok) cross_entropy_grad(a.size_scores, b, k, a.NS, sc, __fmul_rn(s_scls, l), gr.ss + r * a.NS);
      else fill(gr.ss + r * a.NS, a.NS, NAN);
    }
    if (gr.sr) {
      float* o = gr.sr + r * a.NS * 3;
      fill(o, a.NS * 3, sok ? 0.f : NAN);
      if (sok) {
        const float w = __fdiv_rn(__fmul_rn(s_sreg, l), 3.f);       // the mean over the 3 components
        for (int x = 0; x < 3; ++x) {
          const float d = __fsub_rn(at(a.size_residuals_normalized, b, k, sc, x), __fdiv_rn(a.size_residual_label[g * 3 + x], ms.v[sc * 3 + x]));
          o[sc * 3 + x] = __fmul_rn(w, huber_grad(d));
        }
      }
    }
    if (gr.sem) {
      if (cc >= 0 && cc < a.C) cross_entropy_grad(a.sem_cls_scores, b, k, a.C, cc, __fmul_rn(s_sem, l), gr.sem + r * a.C);
      else fill(gr.sem + r * a.C, a.C, NAN);
    }
  }
}

int check_args(const pcb_det_loss_args* a) {
  PCB_ARG(a);
  PCB_ARG(a->B >= 1 && a->B <= 65535 && a->S >= 1 && a->V >= 1 && a->N >= 1 && a->K >= 1 && a->K2 >= 1);
  PCB_ARG(a->NH >= 1 && a->NS >= 1 && a->NS <= MAX_NS && a->C >= 1 && a->center_label_ld >= 3);
  const int64_t lim = (int64_t)1 << 31;
  PCB_ARG(a->S * a->V < lim && a->B * a->S * a->V * 3 < lim && a->B * a->N * 9 < lim && a->B * a->K * a->NS * 3 < lim &&
          a->B * a->K * a->NH < lim && a->B * a->K * a->C < lim && a->B * a->K2 * a->center_label_ld < lim);
  PCB_ARG(a->mean_size && a->seed_xyz && a->seed_inds && a->vote_xyz && a->vote_label && a->vote_label_mask && a->aggregated_vote_xyz);
  PCB_ARG(a->center.p && a->objectness_scores.p && a->heading_scores.p && a->heading_residuals_normalized.p && a->size_scores.p &&
          a->size_residuals_normalized.p && a->sem_cls_scores.p);
  PCB_ARG(a->center_label && a->heading_class_label && a->heading_residual_label && a->size_class_label && a->size_residual_label &&
          a->sem_cls_label && a->box_label_mask);
  return PCB_OK;
}

MeanSize mean_size_of(const pcb_det_loss_args* a) {
  MeanSize m = {};
  for (int i = 0; i < 3 * a->NS; ++i) m.v[i] = a->mean_size[i];
  return m;
}

}  // namespace

extern "C" size_t pcb_det_loss_ws_bytes(int64_t B, int64_t S, int64_t K, int64_t K2) {
  if (B < 1 || S < 1 || K < 1 || K2 < 1) return 0;
  return layout_bytes(ws_layout, B, parts_for(S, K, K2));
}

extern "C" size_t pcb_det_loss_state_bytes(int64_t B, int64_t S, int64_t K, int64_t K2) {
  if (B < 1 || S < 1 || K < 1 || K2 < 1) return 0;
  return layout_bytes(state_layout, B, S, K, K2);
}

extern "C" int pcb_det_loss_forward(const pcb_det_loss_args* args, float* out, int64_t* objectness_label, float* objectness_mask,
                                    int64_t* object_assignment, void* state, size_t state_bytes, void* ws, size_t ws_bytes, void* stream) {
  if (int e = check_args(args)) return e;
  const pcb_det_loss_args& a = *args;
  PCB_ARG(out && objectness_label && objectness_mask && object_assignment && state && ws);
  PCB_ARG(state_bytes >= pcb_det_loss_state_bytes(a.B, a.S, a.K, a.K2) && ws_bytes >= pcb_det_loss_ws_bytes(a.B, a.S, a.K, a.K2));
  const int parts = parts_for(a.S, a.K, a.K2);
  Carve cs{(char*)state}, cw{(char*)ws};
  const StateLayout st = state_layout(cs, a.B, a.S, a.K, a.K2);
  double* partial = ws_layout(cw, a.B, parts);
  cudaStream_t s = (cudaStream_t)stream;
  det_loss_scene_kernel<<<dim3((unsigned)a.B, (unsigned)parts), THREADS, 0, s>>>(a, mean_size_of(args), parts, objectness_label,
                                                                                 objectness_mask, object_assignment, st, partial);
  if (int e = check_launch("det_loss_scene_kernel")) return e;
  det_loss_finish_kernel<<<1, 32, 0, s>>>(partial, a.B * parts, a.B * a.K, out, st.den);
  return check_launch("det_loss_finish_kernel");
}

extern "C" int pcb_det_loss_backward(const pcb_det_loss_args* args, const float* grad, const int64_t* objectness_label,
                                     const float* objectness_mask, const int64_t* object_assignment, const void* state, size_t state_bytes,
                                     float* d_vote_xyz, float* d_seed_xyz, float* d_center, float* d_objectness_scores, float* d_heading_scores,
                                     float* d_heading_residuals_normalized, float* d_size_scores, float* d_size_residuals_normalized,
                                     float* d_sem_cls_scores, void* stream) {
  if (int e = check_args(args)) return e;
  const pcb_det_loss_args& a = *args;
  PCB_ARG(grad && objectness_label && objectness_mask && object_assignment && state);
  PCB_ARG(state_bytes >= pcb_det_loss_state_bytes(a.B, a.S, a.K, a.K2));
  const int parts = parts_for(a.S, a.K, a.K2);
  Carve cs{(char*)state};
  const StateLayout st = state_layout(cs, a.B, a.S, a.K, a.K2);
  const Grads g{d_vote_xyz, d_seed_xyz, d_center, d_objectness_scores, d_heading_scores, d_heading_residuals_normalized, d_size_scores,
                d_size_residuals_normalized, d_sem_cls_scores};
  det_loss_backward_kernel<<<dim3((unsigned)a.B, (unsigned)parts), THREADS, 0, (cudaStream_t)stream>>>(
      a, mean_size_of(args), parts, grad, objectness_label, objectness_mask, object_assignment, st, g);
  return check_launch("det_loss_backward_kernel");
}
