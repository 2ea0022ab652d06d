// The elementwise ends of VoteNet's voting and proposal heads (include/pcb200.h "VoteNet heads", DESIGN.md 8f-18): what
// `voting_module.py` and `decode_scores` compute from the last 1x1 convolution's output z, and the adjoints that turn the gradients of
// those outputs back into the gradient of z as bf16 hi/lo planes for the weight-gradient and data-gradient kernels.  The convolutions
// and the BatchNorm units around them are conv.cu's and unit.cu's.  Every output element is written by one thread (no atomics).
#include "common.cuh"

using namespace pcb;

namespace {
constexpr int64_t LIM = 1ll << 31;
constexpr int MAX_NS = 64;
constexpr int NGRAD = 9;

struct MeanSize { float v[3 * MAX_NS]; };
struct Grads { pcb_strided g[NGRAD]; };

// fp32 -> bf16 hi + bf16 lo (x ~= hi + lo to 2^-17), the gradient operand format of the tensor-core conv kernels (bn.cu store_split4)
__device__ __forceinline__ void store_split_bf16(float v, uint16_t* hi, uint16_t* lo) {
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  const __nv_bfloat16 l = __float2bfloat16_rn(v - __bfloat162float(h));
  *hi = __bfloat16_as_ushort(h);
  *lo = __bfloat16_as_ushort(l);
}

__device__ __forceinline__ float rd(const pcb_strided& g, int64_t b, int64_t k, int64_t c) {
  return g.p ? g.p[b * g.sb + k * g.sk + c * g.sc] : 0.f;
}

// vote_xyz[b, s V + v, i] = seed_xyz[b, s, i] + z[r, v (3 + C) + i];  vote_features[r V + v, c] = X[r, c] + z[r, v (3 + C) + 3 + c]
// (r = b S + s).  One thread per (r, v, column of 3 + C).
__global__ void vote_epilogue_kernel(const float* __restrict__ seed_xyz, const float* __restrict__ X, int ldf, const float* __restrict__ z,
                                     int ldz, int V, int C, float* __restrict__ vote_xyz, float* __restrict__ vote_features, int64_t total) {
  pdl_wait(); pdl_trigger();
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int W = 3 + C;
  const int j = (int)(t % W);
  const int64_t rv = t / W;                       // r V + v
  const int v = (int)(rv % V);
  const int64_t r = rv / V;
  const float off = z[r * ldz + (int64_t)v * W + j];
  if (j < 3) vote_xyz[rv * 3 + j] = __fadd_rn(seed_xyz[r * 3 + j], off);
  else vote_features[rv * C + (j - 3)] = __fadd_rn(X[r * ldf + (j - 3)], off);
}

// dz[r, j] (bf16 hi/lo, columns [0, Cpad)) = d_vote_xyz / d_vote_features at the element z[r, j] produced, 0 in the padding;
// d_seed_features[r, c] = sum_v d_vote_features[b, c, s V + v] and d_seed_xyz[r, i] = sum_v d_vote_xyz[b, s V + v, i], ascending v.
__global__ void vote_epilogue_grad_kernel(pcb_strided gx, pcb_strided gf, int64_t S, int V, int C, uint16_t* __restrict__ dz_hi,
                                          uint16_t* __restrict__ dz_lo, int ldz, int Cpad, float* __restrict__ d_seed_features, int ldd,
                                          float* __restrict__ d_seed_xyz, int64_t total) {
  pdl_wait(); pdl_trigger();
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int j = (int)(t % Cpad);
  const int64_t r = t / Cpad;
  const int64_t b = r / S, s = r % S;
  const int W = 3 + C;
  float d = 0.f;
  if (j < W * V) {
    const int v = j / W, k = j % W;
    d = k < 3 ? rd(gx, b, s * V + v, k) : rd(gf, b, s * V + v, k - 3);
  }
  store_split_bf16(d, dz_hi + r * ldz + j, dz_lo + r * ldz + j);
  if (d_seed_features && j < C) {
    float acc = 0.f;
    for (int v = 0; v < V; ++v) acc = __fadd_rn(acc, rd(gf, b, s * V + v, j));
    d_seed_features[r * ldd + j] = acc;
  }
  if (d_seed_xyz && j < 3) {
    float acc = 0.f;
    for (int v = 0; v < V; ++v) acc = __fadd_rn(acc, rd(gx, b, s * V + v, j));
    d_seed_xyz[r * 3 + j] = acc;
  }
}

// center[r, i] = aggregated_vote_xyz[r, i] + z[r, 2 + i]; heading_residuals[r, h] = z[r, 5 + NH + h] * unit;
// size_residuals[r, q] = z[r, 5 + 2 NH + NS + q] * mean_size[q] (q = cluster * 3 + axis).  One thread per (r, column of 3 + NH + 3 NS).
__global__ void proposal_epilogue_kernel(const float* __restrict__ z, int ldz, const float* __restrict__ agg, int NH, int NS, float unit,
                                         MeanSize ms, float* __restrict__ center, float* __restrict__ hr, float* __restrict__ sr,
                                         int64_t total) {
  pdl_wait(); pdl_trigger();
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int W = 3 + NH + 3 * NS;
  const int j = (int)(t % W);
  const int64_t r = t / W;
  const float* zr = z + r * ldz;
  if (j < 3) center[r * 3 + j] = __fadd_rn(agg[r * 3 + j], zr[2 + j]);
  else if (j < 3 + NH) hr[r * NH + (j - 3)] = __fmul_rn(zr[5 + NH + (j - 3)], unit);
  else {
    const int q = j - 3 - NH;
    sr[r * 3 * NS + q] = __fmul_rn(zr[5 + 2 * NH + NS + q], ms.v[q]);
  }
}

// dz[r, j] for the columns of decode_scores (objectness 2, center 3, heading scores NH, heading residuals NH, size scores NS, size
// residuals 3 NS, semantic classes C, then 0 up to Xpad): the gradient of the view that reads column j, plus unit x the gradient of
// heading_residuals / mean_size x the gradient of size_residuals on the residual columns.  d_aggregated_vote_xyz = the center gradient.
__global__ void proposal_epilogue_grad_kernel(Grads G, int64_t K, int NH, int NS, int C, float unit, MeanSize ms,
                                              uint16_t* __restrict__ dz_hi, uint16_t* __restrict__ dz_lo, float* __restrict__ dz, int ldz,
                                              int Xpad, float* __restrict__ d_agg, int64_t total) {
  pdl_wait(); pdl_trigger();
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int j = (int)(t % Xpad);
  const int64_t r = t / Xpad;
  const int64_t b = r / K, k = r % K;
  const int h0 = 5, h1 = 5 + NH, s0 = 5 + 2 * NH, s1 = s0 + NS, c0 = s1 + 3 * NS, X = c0 + C;
  float d = 0.f;
  if (j < 2) d = rd(G.g[0], b, k, j);
  else if (j < h0) {
    d = rd(G.g[1], b, k, j - 2);
    if (d_agg) d_agg[r * 3 + (j - 2)] = d;
  } else if (j < h1) d = rd(G.g[2], b, k, j - h0);
  else if (j < s0) d = __fadd_rn(rd(G.g[3], b, k, j - h1), __fmul_rn(rd(G.g[4], b, k, j - h1), unit));
  else if (j < s1) d = rd(G.g[5], b, k, j - s0);
  else if (j < c0) {
    const int q = j - s1, cl = q / 3, ax = q % 3;
    const pcb_strided& n = G.g[6];
    const pcb_strided& m = G.g[7];
    const float gn = n.p ? n.p[b * n.sb + k * n.sk + cl * n.sc + ax * n.sx] : 0.f;
    const float gm = m.p ? m.p[b * m.sb + k * m.sk + cl * m.sc + ax * m.sx] : 0.f;
    d = __fadd_rn(gn, __fmul_rn(gm, ms.v[q]));
  } else if (j < X) d = rd(G.g[8], b, k, j - c0);
  if (dz_hi) store_split_bf16(d, dz_hi + r * ldz + j, dz_lo + r * ldz + j);
  if (dz) dz[r * ldz + j] = d;
}

bool mean_size_ok(const float* mean_size, int NS, MeanSize& ms) {
  if (!mean_size || NS < 1 || NS > MAX_NS) return false;
  for (int q = 0; q < 3 * MAX_NS; ++q) ms.v[q] = q < 3 * NS ? mean_size[q] : 0.f;
  return true;
}
}  // namespace

extern "C" int pcb_vote_epilogue(const float* seed_xyz, const float* seed_features, int ldf, const float* z, int ldz, int64_t B, int64_t S,
                                 int V, int C, float* vote_xyz, float* vote_features, void* stream) {
  PCB_ARG(B >= 1 && S >= 1 && V >= 1 && C >= 1 && B * S * V < LIM && ldf >= C && ldz >= (3 + C) * V);
  PCB_ARG(seed_xyz && seed_features && z && vote_xyz && vote_features);
  const int64_t total = B * S * V * (3 + C);
  launch_kernel(vote_epilogue_kernel, blocks_for(total, 256), 256, 0, (cudaStream_t)stream, seed_xyz, seed_features, ldf, z, ldz, V, C,
                vote_xyz, vote_features, total);
  return check_launch("vote_epilogue_kernel");
}

extern "C" int pcb_vote_epilogue_grad(const pcb_strided* d_vote_xyz, const pcb_strided* d_vote_features, int64_t B, int64_t S, int V, int C,
                                      uint16_t* dz_hi, uint16_t* dz_lo, int ldz, int Cpad, float* d_seed_features, int ldd, float* d_seed_xyz,
                                      void* stream) {
  PCB_ARG(B >= 1 && S >= 1 && V >= 1 && C >= 1 && B * S * V < LIM && Cpad >= (3 + C) * V && ldz >= Cpad);
  PCB_ARG(!d_seed_features || ldd >= C);
  PCB_ARG(dz_hi && dz_lo);
  const pcb_strided none = {};
  const pcb_strided gx = d_vote_xyz ? *d_vote_xyz : none, gf = d_vote_features ? *d_vote_features : none;
  const int64_t total = B * S * Cpad;
  launch_kernel(vote_epilogue_grad_kernel, blocks_for(total, 256), 256, 0, (cudaStream_t)stream, gx, gf, S, V, C, dz_hi, dz_lo, ldz, Cpad,
                d_seed_features, ldd, d_seed_xyz, total);
  return check_launch("vote_epilogue_grad_kernel");
}

extern "C" int pcb_proposal_epilogue(const float* z, int ldz, const float* aggregated_vote_xyz, int64_t B, int64_t K, int NH, int NS,
                                     float heading_unit, const float* mean_size, float* center, float* heading_residuals,
                                     float* size_residuals, void* stream) {
  MeanSize ms;
  PCB_ARG(B >= 1 && K >= 1 && NH >= 1 && B * K < LIM && mean_size_ok(mean_size, NS, ms) && ldz >= 5 + 2 * NH + 4 * NS);
  PCB_ARG(z && aggregated_vote_xyz && center && heading_residuals && size_residuals);
  const int64_t total = B * K * (3 + NH + 3 * NS);
  launch_kernel(proposal_epilogue_kernel, blocks_for(total, 256), 256, 0, (cudaStream_t)stream, z, ldz, aggregated_vote_xyz, NH, NS,
                heading_unit, ms, center, heading_residuals, size_residuals, total);
  return check_launch("proposal_epilogue_kernel");
}

extern "C" int pcb_proposal_epilogue_grad(const pcb_strided* grads, int64_t B, int64_t K, int NH, int NS, int C, float heading_unit,
                                          const float* mean_size, uint16_t* dz_hi, uint16_t* dz_lo, float* dz, int ldz, int Xpad,
                                          float* d_aggregated_vote_xyz, void* stream) {
  MeanSize ms;
  PCB_ARG(B >= 1 && K >= 1 && NH >= 1 && C >= 1 && B * K < LIM && mean_size_ok(mean_size, NS, ms));
  PCB_ARG(Xpad >= 5 + 2 * NH + 4 * NS + C && ldz >= Xpad);
  PCB_ARG(grads && (dz_hi || dz) && (!dz_hi || dz_lo));
  Grads G;
  for (int i = 0; i < NGRAD; ++i) G.g[i] = grads[i];
  const int64_t total = B * K * Xpad;
  launch_kernel(proposal_epilogue_grad_kernel, blocks_for(total, 256), 256, 0, (cudaStream_t)stream, G, K, NH, NS, C, heading_unit, ms,
                dz_hi, dz_lo, dz, ldz, Xpad, d_aggregated_vote_xyz, total);
  return check_launch("proposal_epilogue_grad_kernel");
}
