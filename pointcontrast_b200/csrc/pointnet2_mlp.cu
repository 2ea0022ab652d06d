// The grouping and pooling ends of VoteNet's PointNet++ shared MLPs (include/pcb200.h "PointNet++ shared MLPs", DESIGN.md 8f-16):
// the first layer of a set-abstraction module evaluated on the ball-query neighbourhoods without materialising the grouped input, the
// max pool over each neighbourhood by selection, and the backward passes that are specific to the two.  The layers between them are
// the fused units (unit.cu) on a K = 1 identity table; the pooled layer's BatchNorm statistics and backward are bn.cu's.
#include "common.cuh"

using namespace pcb;

namespace {
constexpr int64_t LIM = 1ll << 31;

// z[r, c] = P[b N + j, c] + ((rel_0 Wx[0][c] + rel_1 Wx[1][c]) + rel_2 Wx[2][c]), rel = (xyz[b, j] - new_xyz[b, i]) [/ radius], for row
// r = (b npoint + i) S + s and j = idx[r].  One thread per (row, channel); the channel-0 thread also writes rel and the global index.
__global__ void sa_layer0_kernel(const float* __restrict__ xyz, const float* __restrict__ new_xyz, const int32_t* __restrict__ idx,
                                 int64_t N, int64_t M, int S, float radius, const float* __restrict__ P, int ldp,
                                 const float* __restrict__ Wx, int C0, float* __restrict__ rel, int32_t* __restrict__ gidx,
                                 float* __restrict__ z, int ldz, int64_t total) {
  pdl_wait(); pdl_trigger();
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int c = (int)(t % C0);
  const int64_t r = t / C0;
  const int64_t ci = r / S;                       // centre, batch-major: b * M + i
  const int64_t b = ci / M;
  const int j = idx[r];
  const bool ok = j >= 0 && j < N;
  const float* p = xyz + (b * N + (ok ? j : 0)) * 3;
  const float* q = new_xyz + ci * 3;
  float d0 = __fsub_rn(ok ? p[0] : 0.f, q[0]), d1 = __fsub_rn(ok ? p[1] : 0.f, q[1]), d2 = __fsub_rn(ok ? p[2] : 0.f, q[2]);
  if (radius > 0.f) { d0 = __fdiv_rn(d0, radius); d1 = __fdiv_rn(d1, radius); d2 = __fdiv_rn(d2, radius); }
  float v = __fadd_rn(__fadd_rn(__fmul_rn(d0, Wx[c]), __fmul_rn(d1, Wx[C0 + c])), __fmul_rn(d2, Wx[2 * C0 + c]));
  if (P) v = __fadd_rn(ok ? P[(b * N + j) * (int64_t)ldp + c] : 0.f, v);
  z[r * (int64_t)ldz + c] = v;
  if (c == 0) {
    rel[r * 3] = d0; rel[r * 3 + 1] = d1; rel[r * 3 + 2] = d2;
    gidx[r] = ok ? (int32_t)(b * N + j) : -1;
  }
}

// Per (centre, channel): the slot s < S of the extreme z on gamma's side (maximum for gamma >= 0, minimum for gamma < 0; the smallest
// slot among equals), and out = relu(BN(z at that slot)) in bn_apply_kernel's expression.
__global__ void sa_pool_kernel(const float* __restrict__ z, int ldz, int64_t M, int S, int C, const float* __restrict__ mean,
                               const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                               int32_t* __restrict__ sel, float* __restrict__ out, int ldo) {
  pdl_wait(); pdl_trigger();
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= M * C) return;
  const int c = (int)(t % C);
  const int64_t i = t / C;
  const float* zc = z + i * S * (int64_t)ldz + c;
  const float g = gamma[c];
  const bool lo = g < 0.f;
  float best = zc[0];
  int bs = 0;
  for (int s = 1; s < S; ++s) {
    const float v = zc[(int64_t)s * ldz];
    if (lo ? v < best : v > best) { best = v; bs = s; }
  }
  const float y = (best - mean[c]) * invstd[c] * g + beta[c];
  sel[t] = bs;
  out[i * (int64_t)ldo + c] = fmaxf(y, 0.f);
}

// dY [M S, C] (dense, written in full) = the gradient of relu(BN(z)) that the max pool passes back: g where the pooled output is
// positive, on the selected slot only.
__global__ void sa_pool_grad_kernel(const float* __restrict__ g, int ldg, const int32_t* __restrict__ sel, const float* __restrict__ out,
                                    int ldo, int64_t M, int S, int C, float* __restrict__ dY) {
  pdl_wait(); pdl_trigger();
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= M * C) return;
  const int c = (int)(t % C);
  const int64_t i = t / C;
  const float gv = out[i * (int64_t)ldo + c] > 0.f ? g[i * (int64_t)ldg + c] : 0.f;
  const int bs = sel[t];
  float* d = dY + i * S * (int64_t)C + c;
  for (int s = 0; s < S; ++s) d[(int64_t)s * C] = s == bs ? gv : 0.f;
}

// rows [R + M, 3]: rows[r] = grel[r] / radius (the gradient reaching point idx[r]), rows[R + i] = d_new_xyz[i] - sum_s rows[i S + s]
// in ascending s (the gradient reaching centre i).  One thread per (centre, axis).
__global__ void sa_xyz_rows_kernel(const float* __restrict__ grel, const float* __restrict__ d_new_xyz, int64_t M, int S, float radius,
                                   float* __restrict__ rows) {
  pdl_wait(); pdl_trigger();
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= M * 3) return;
  const int k = (int)(t % 3);
  const int64_t i = t / 3;
  float acc = 0.f;
  for (int s = 0; s < S; ++s) {
    const int64_t e = (i * S + s) * 3 + k;
    const float v = radius > 0.f ? __fdiv_rn(grel[e], radius) : grel[e];
    rows[e] = v;
    acc = __fadd_rn(acc, v);
  }
  rows[(M * S + i) * 3 + k] = __fsub_rn(d_new_xyz ? d_new_xyz[t] : 0.f, acc);
}
}  // namespace

extern "C" int pcb_sa_layer0(const float* xyz, const float* new_xyz, const int32_t* idx, int64_t B, int64_t N, int64_t M, int S,
                             float radius, const float* P, int ldp, const float* Wx, int C0, float* rel, int32_t* gidx, float* z, int ldz,
                             void* stream) {
  PCB_ARG(B >= 1 && N >= 1 && M >= 1 && S >= 1 && C0 >= 1 && N < LIM && B * N < LIM && B * M * S < LIM && ldz >= C0 && radius == radius);
  PCB_ARG(!P || ldp >= C0);
  PCB_ARG(xyz && new_xyz && idx && Wx && rel && gidx && z);
  const int64_t total = B * M * S * C0;
  launch_kernel(sa_layer0_kernel, blocks_for(total, 256), 256, 0, (cudaStream_t)stream, xyz, new_xyz, idx, N, M, S, radius, P, ldp, Wx, C0,
                rel, gidx, z, ldz, total);
  return check_launch("sa_layer0_kernel");
}

extern "C" int pcb_sa_pool(const float* z, int ldz, int64_t M, int S, int C, const float* mean, const float* invstd, const float* gamma,
                           const float* beta, int32_t* sel, float* out, int ldo, void* stream) {
  PCB_ARG(M >= 1 && S >= 1 && C >= 1 && M * S < LIM && M * C < LIM && ldz >= C && ldo >= C);
  PCB_ARG(z && mean && invstd && gamma && beta && sel && out);
  launch_kernel(sa_pool_kernel, blocks_for(M * C, 256), 256, 0, (cudaStream_t)stream, z, ldz, M, S, C, mean, invstd, gamma, beta, sel, out,
                ldo);
  return check_launch("sa_pool_kernel");
}

extern "C" int pcb_sa_pool_grad(const float* g, int ldg, const int32_t* sel, const float* out, int ldo, int64_t M, int S, int C, float* dY,
                                void* stream) {
  PCB_ARG(M >= 1 && S >= 1 && C >= 1 && M * S < LIM && M * C < LIM && ldg >= C && ldo >= C);
  PCB_ARG(g && sel && out && dY);
  launch_kernel(sa_pool_grad_kernel, blocks_for(M * C, 256), 256, 0, (cudaStream_t)stream, g, ldg, sel, out, ldo, M, S, C, dY);
  return check_launch("sa_pool_grad_kernel");
}

extern "C" int pcb_sa_xyz_rows(const float* grel, const float* d_new_xyz, int64_t M, int S, float radius, float* rows, void* stream) {
  PCB_ARG(M >= 1 && S >= 1 && M * S < LIM && radius == radius);
  PCB_ARG(grel && rows);
  launch_kernel(sa_xyz_rows_kernel, blocks_for(M * 3, 256), 256, 0, (cudaStream_t)stream, grel, d_new_xyz, M, S, radius, rows);
  return check_launch("sa_xyz_rows_kernel");
}
