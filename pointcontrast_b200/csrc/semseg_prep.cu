// S3DIS to training PLY on the GPU (DESIGN.md 8f-14): the compute of the reference's
// `downstream/semseg/lib/datasets/preprocessing/stanford.py` `Stanford3DDatasetConverter.convert_to_ply` for one room, whose
// annotation files' bytes are concatenated into one buffer:
//   * the line structure of Python's text-mode iteration (`for l in f`, `:50`): universal newlines, a last line without one  -> pcb_text_lines
//   * `[float(li) for li in l.split()]` per line with the `try/except` that skips a line (`:51-55`), the float32 / uint8 casts
//     (`:59-62`), the file's label (`:91`) and the 1 cm cell `floor(float64(x) / 0.01)` of `sparse_quantize` (`:98-105`)  -> pcb_s3dis_parse
//   * the rows `np.concatenate((coords[inds], feats[inds], collabels[:, None]), 1)` as the PLY body `lib/pc_utils.py:41-70` writes
//     (x, y, z <f4, red, green, blue, label u1)                                                                            -> pcb_ply_rows
// The quantisation between the last two is pcb_voxelize_labels.  The parser decides on the device only what it can decide exactly
// (Clinger's fast path on the `float()` grammar of [0-9+-.eE]); every other line is marked for the host, which parses it with Python's
// own expression, so the result is the original's for any input.
#include <cub/cub.cuh>
#include "common.cuh"

using namespace pcb;

namespace {

constexpr int CHUNK = 16;                   // bytes per thread of the line pass: one 16-byte vector load
constexpr int MAX_LINE = 512;               // longer lines go to the host
constexpr int MAX_DIGITS = 19;              // Clinger: at most 19 significant digits ...
constexpr uint64_t MAX_MANTISSA = 1ull << 53;   // ... whose value is exact in fp64 ...
constexpr int MAX_POW10 = 22;               // ... scaled by an exact power of ten

__constant__ double kPow10[MAX_POW10 + 1] = {1e0,  1e1,  1e2,  1e3,  1e4,  1e5,  1e6,  1e7,  1e8,  1e9,  1e10, 1e11,
                                             1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};

// the file of byte / line position p: the last f with off[f] <= p (off non-decreasing, off[0] == 0)
__device__ __forceinline__ int file_of(const int64_t* __restrict__ off, int F, int64_t p) {
  int lo = 0, hi = F - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= p) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// The line starts of bytes [c * CHUNK, c * CHUNK + CHUNK) ∩ [0, n), as a bit mask: byte p starts a line when it is the first byte of
// its file, or follows '\n', or follows a '\r' that is not followed by '\n' (Python's universal newlines).  An empty file holds no
// byte, hence no line.  flags != NULL: also ORs PCB_TEXT_NONASCII into flags[f] of every file with a byte >= 0x80 in the chunk.
__device__ __forceinline__ uint32_t chunk_starts(const uint8_t* __restrict__ text, int64_t n, const int64_t* __restrict__ off, int F,
                                                 int64_t c, int32_t* __restrict__ flags) {
  const int64_t p0 = c * CHUNK;
  uint8_t b[CHUNK];
  *reinterpret_cast<uint4*>(b) = *reinterpret_cast<const uint4*>(text + p0);
  int f = file_of(off, F, p0);
  int64_t next = f + 1 < F ? off[f + 1] : INT64_MAX;
  uint8_t prev = p0 > 0 ? text[p0 - 1] : '\n';
  uint32_t mask = 0;
  bool high = false;
  const int m = (int)min((int64_t)CHUNK, n - p0);
  for (int k = 0; k < m; ++k) {
    const int64_t p = p0 + k;
    if (p >= next) {                                      // a file starts here (skip the empty ones before it)
      if (high && flags) atomicOr(&flags[f], PCB_TEXT_NONASCII);
      high = false;
      while (f + 1 < F && off[f + 1] <= p) ++f;
      next = f + 1 < F ? off[f + 1] : INT64_MAX;
    }
    const uint8_t ch = b[k];
    if (p == off[f] || prev == '\n' || (prev == '\r' && ch != '\n')) mask |= 1u << k;
    high |= ch >= 0x80;
    prev = ch;
  }
  if (high && flags) atomicOr(&flags[f], PCB_TEXT_NONASCII);
  return mask;
}

__global__ void line_count_kernel(const uint8_t* __restrict__ text, int64_t n, const int64_t* __restrict__ off, int F, int64_t nchunks,
                                  int64_t* __restrict__ counts, int32_t* __restrict__ flags) {
  pdl_wait();
  pdl_trigger();
  const int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (c < nchunks) counts[c] = __popc(chunk_starts(text, n, off, F, c, flags));
  else if (c == nchunks) counts[c] = 0;
}

__global__ void line_scatter_kernel(const uint8_t* __restrict__ text, int64_t n, const int64_t* __restrict__ off, int F, int64_t nchunks,
                                    const int64_t* __restrict__ chunk_off, int64_t* __restrict__ line_start) {
  pdl_wait();
  pdl_trigger();
  const int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (c > nchunks) return;
  if (c == nchunks) { line_start[chunk_off[nchunks]] = n; return; }
  uint32_t mask = chunk_starts(text, n, off, F, c, nullptr);
  int64_t j = chunk_off[c];
  while (mask) {
    const int k = __ffs(mask) - 1;
    mask &= mask - 1;
    line_start[j++] = c * CHUNK + k;
  }
}

// str.split()'s ASCII whitespace
__device__ __forceinline__ bool is_space(uint8_t ch) { return ch == ' ' || (ch >= '\t' && ch <= '\r') || (ch >= 0x1c && ch <= 0x1f); }

enum Token { TOK_EXACT, TOK_HOST, TOK_INVALID };

// float() of token [a, b) (ASCII, no whitespace).  TOK_INVALID: float() raises; TOK_HOST: float() may accept it (inf, nan, digit
// underscores) or the value is not on Clinger's fast path; TOK_EXACT: *v is float()'s correctly rounded value.
__device__ Token parse_token(const uint8_t* __restrict__ s, int a, int b, double* v) {
  bool host = false;
  for (int k = a; k < b; ++k) {
    const uint8_t ch = s[k];
    if ((ch >= '0' && ch <= '9') || ch == '+' || ch == '-' || ch == '.' || ch == 'e' || ch == 'E') continue;
    const uint8_t lower = ch | 0x20;                      // the letters of inf / infinity / nan, and digit underscores
    if (ch == '_' || lower == 'i' || lower == 'n' || lower == 'f' || lower == 'a' || lower == 't' || lower == 'y') host = true;
    else return TOK_INVALID;
  }
  if (host) return TOK_HOST;
  // [+-]? (digits [. digits?] | . digits) ([eE] [+-]? digits)?
  int k = a;
  const bool neg = s[k] == '-';
  if (s[k] == '+' || s[k] == '-') ++k;
  uint64_t mant = 0;
  int sig = 0, frac = 0, intd = 0, fracd = 0;
  for (; k < b && s[k] >= '0' && s[k] <= '9'; ++k, ++intd) {
    if (mant || s[k] != '0') { if (++sig <= MAX_DIGITS) mant = mant * 10 + (s[k] - '0'); }
  }
  if (k < b && s[k] == '.') {
    for (++k; k < b && s[k] >= '0' && s[k] <= '9'; ++k, ++fracd) {
      if (mant || s[k] != '0') { if (++sig <= MAX_DIGITS) mant = mant * 10 + (s[k] - '0'); }
      ++frac;
    }
  }
  if (intd + fracd == 0) return TOK_INVALID;
  int e = 0, ed = 0;
  if (k < b && (s[k] == 'e' || s[k] == 'E')) {
    ++k;
    const bool eneg = k < b && s[k] == '-';
    if (k < b && (s[k] == '+' || s[k] == '-')) ++k;
    for (; k < b && s[k] >= '0' && s[k] <= '9'; ++k, ++ed)
      if (ed < 6) e = e * 10 + (s[k] - '0');
    if (ed == 0) return TOK_INVALID;
    if (ed >= 6) host = true;
    e = eneg ? -e : e;
  }
  if (k != b) return TOK_INVALID;
  if (mant == 0 && sig == 0) { *v = neg ? -0.0 : 0.0; return TOK_EXACT; }
  const int e10 = e - frac;
  if (host || sig > MAX_DIGITS || mant > MAX_MANTISSA || e10 > MAX_POW10 || e10 < -MAX_POW10) return TOK_HOST;
  const double m = (double)mant;                          // exact: mant <= 2^53
  const double r = e10 >= 0 ? __dmul_rn(m, kPow10[e10]) : __ddiv_rn(m, kPow10[-e10]);
  *v = neg ? -r : r;
  return TOK_EXACT;
}

// the 1 cm cell of a coordinate: floor(float64(x) / 0.01) in true fp64 division; outside +-2^30 it is clamped there, which
// pcb_voxelize_labels reports as out of range
__device__ __forceinline__ int32_t cell_of(float x) {
  const double q = floor(__ddiv_rn((double)x, 0.01));
  return q >= 1073741824.0 ? 1073741824 : (q <= -1073741824.0 ? -1073741824 : (int32_t)q);   // NaN -> 0 never occurs: x is finite
}

__global__ void parse_kernel(const uint8_t* __restrict__ text, const int64_t* __restrict__ off, int F, const int32_t* __restrict__ file_label,
                             const int32_t* __restrict__ flags, const int64_t* __restrict__ line_start, int64_t L, float* __restrict__ xyz,
                             uint8_t* __restrict__ rgb, int32_t* __restrict__ label, int32_t* __restrict__ cell, uint8_t* __restrict__ status) {
  pdl_wait();
  pdl_trigger();
  const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (j >= L) return;
  const int64_t a = line_start[j];
  const int f = file_of(off, F, a);
  const int64_t b = min(line_start[j + 1], off[f + 1]);
  label[j] = file_label[f];
  uint8_t st = PCB_LINE_KEPT;
  double v[6] = {0, 0, 0, 0, 0, 0};
  if ((flags[f] & PCB_TEXT_NONASCII) || b - a > MAX_LINE) {
    st = PCB_LINE_HOST;
  } else {
    const uint8_t* s = text + a;
    const int len = (int)(b - a);
    int ntok = 0;
    bool host = false, invalid = false;
    for (int k = 0; k < len;) {
      while (k < len && is_space(s[k])) ++k;
      if (k == len) break;
      const int t0 = k;
      while (k < len && !is_space(s[k])) ++k;
      double x = 0;
      const Token t = parse_token(s, t0, k, &x);
      invalid |= t == TOK_INVALID;
      host |= t == TOK_HOST;
      if (ntok < 6) v[ntok] = x;
      ++ntok;
    }
    st = invalid ? PCB_LINE_SKIPPED : host ? PCB_LINE_HOST : ntok != 6 ? PCB_LINE_ERROR : PCB_LINE_KEPT;
  }
  if (st == PCB_LINE_KEPT) {
    for (int k = 0; k < 3; ++k) {
      const float c = __double2float_rn(v[3 + k]);         // `np.array(...).astype(np.float32)`, then `.astype(np.uint8)`
      if (!(c >= 0.f && c < 256.f)) st = PCB_LINE_HOST;    // outside the cast's defined range: numpy's platform result, on the host
      rgb[3 * j + k] = st == PCB_LINE_KEPT ? (uint8_t)c : 0;
    }
  }
  for (int k = 0; k < 3; ++k) {
    const float x = __double2float_rn(v[k]);
    xyz[3 * j + k] = x;
    cell[3 * j + k] = st == PCB_LINE_KEPT ? cell_of(x) : 0;
  }
  status[j] = st;
}

__global__ void ply_rows_kernel(const float* __restrict__ xyz, const uint8_t* __restrict__ rgb, const int32_t* __restrict__ sel,
                                const int32_t* __restrict__ vlabel, int64_t m, uint4* __restrict__ rows) {
  pdl_wait();
  pdl_trigger();
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= m) return;
  const int64_t p = sel[i];
  rows[i] = make_uint4(__float_as_uint(xyz[3 * p]), __float_as_uint(xyz[3 * p + 1]), __float_as_uint(xyz[3 * p + 2]),
                       (uint32_t)rgb[3 * p] | ((uint32_t)rgb[3 * p + 1] << 8) | ((uint32_t)rgb[3 * p + 2] << 16) |
                           ((uint32_t)(vlabel[i] & 0xff) << 24));
}

void text_lines_layout(Carve& c, int64_t nchunks, void** cub, size_t* cub_bytes) {
  size_t cb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, cb, (int64_t*)nullptr, (int64_t*)nullptr, (int)(nchunks + 1));
  *cub = c.take<char>((int64_t)cb);
  *cub_bytes = cb;
}

}  // namespace

extern "C" size_t pcb_text_lines_ws_bytes(int64_t nbytes) {
  void* cub; size_t cb;
  return layout_bytes(text_lines_layout, (nbytes + CHUNK - 1) / CHUNK, &cub, &cb);
}

extern "C" int pcb_text_lines(const uint8_t* text, int64_t nbytes, const int64_t* file_off, int32_t nfiles, int64_t* chunk_off,
                              int32_t* flags, int64_t* n_lines, void* ws, size_t ws_bytes, void* stream) {
  PCB_ARG(text && file_off && chunk_off && flags && n_lines && nbytes >= 0 && nfiles >= 1);
  const int64_t nchunks = (nbytes + CHUNK - 1) / CHUNK;
  PCB_ARG(nchunks + 1 < INT32_MAX && reinterpret_cast<uintptr_t>(text) % 16 == 0);
  PCB_ARG(ws_bytes >= pcb_text_lines_ws_bytes(nbytes) && (ws || ws_bytes == 0));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Carve c{static_cast<char*>(ws)};
  void* cub; size_t cb;
  text_lines_layout(c, nchunks, &cub, &cb);
  PCB_CUDA(cudaMemsetAsync(flags, 0, sizeof(int32_t) * nfiles, st));
  launch_kernel(line_count_kernel, blocks_for(nchunks + 1, 256), 256, 0, st, text, nbytes, file_off, (int)nfiles, nchunks, chunk_off, flags);
  if (int rc = check_launch("line_count_kernel")) return rc;
  PCB_CUDA(cub::DeviceScan::ExclusiveSum(cub, cb, chunk_off, chunk_off, (int)(nchunks + 1), st));
  PCB_CUDA(cudaMemcpyAsync(n_lines, chunk_off + nchunks, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  PCB_CUDA(cudaStreamSynchronize(st));
  return PCB_OK;
}

extern "C" int pcb_s3dis_parse(const uint8_t* text, int64_t nbytes, const int64_t* file_off, const int32_t* file_label, int32_t nfiles,
                               const int64_t* chunk_off, int32_t* flags, int64_t n_lines, int64_t* line_start, float* xyz, uint8_t* rgb,
                               int32_t* label, int32_t* cell, uint8_t* status, void* stream) {
  PCB_ARG(text && file_off && file_label && chunk_off && flags && line_start && nbytes >= 0 && nfiles >= 1 && n_lines >= 0);
  PCB_ARG(reinterpret_cast<uintptr_t>(text) % 16 == 0);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t nchunks = (nbytes + CHUNK - 1) / CHUNK;
  launch_kernel(line_scatter_kernel, blocks_for(nchunks + 1, 256), 256, 0, st, text, nbytes, file_off, (int)nfiles, nchunks, chunk_off, line_start);
  if (int rc = check_launch("line_scatter_kernel")) return rc;
  if (n_lines == 0) return PCB_OK;
  PCB_ARG(xyz && rgb && label && cell && status);
  launch_kernel(parse_kernel, blocks_for(n_lines, 128), 128, 0, st, text, file_off, (int)nfiles, file_label, (const int32_t*)flags,
                (const int64_t*)line_start, n_lines, xyz, rgb, label, cell, status);
  return check_launch("parse_kernel");
}

extern "C" int pcb_ply_rows(const float* xyz, const uint8_t* rgb, const int32_t* sel, const int32_t* labels, int64_t m, uint8_t* rows,
                            void* stream) {
  if (m == 0) return PCB_OK;
  PCB_ARG(xyz && rgb && sel && labels && rows && m > 0 && reinterpret_cast<uintptr_t>(rows) % 16 == 0);
  launch_kernel(ply_rows_kernel, blocks_for(m, 256), 256, 0, static_cast<cudaStream_t>(stream), xyz, rgb, sel, labels, m,
                reinterpret_cast<uint4*>(rows));
  return check_launch("ply_rows_kernel");
}
