// GNN message passing: batched CSR build from the reference's dense adjacency, and the
// gather -> scale -> segmented-reduce ("scatter") kernel that replaces torch.bmm(edge, x)
// (gnn_transformer.py:80).
//
// Adjacency format ("packed edges"): graphs are concatenated in batch order; rows are the
// destination nodes in (graph b, node i) order, `rowptr` is cumulative over the whole batch,
// `col` holds LOCAL source-node ids j in [0, N), `val` = A[b, i, j] as fp32 (the reference casts
// its float64 adjacency with edge.float(), gnn_transformer.py:80).
//
// Feature rows live in the encoder's segment-major node buffer (DESIGN.md): all code rows of all
// graphs, then all sub-token rows, then all AST/edit rows.  seg_row() maps (b, node) to that row.
// With n_sub = n_ast = 0 the map is the identity (synthetic single-segment graphs).
#include "common.cuh"
#include "fira_b200.h"

namespace {

constexpr int D = 256;

struct Segs { int B, n0, n1, n2; };   // n0 code, n1 sub-token, n2 AST/edit rows per graph

__device__ __forceinline__ long seg_row(const Segs& s, int b, int j) {
  if (j < s.n0) return (long)b * s.n0 + j;
  if (j < s.n0 + s.n1) return (long)s.B * s.n0 + (long)b * s.n1 + (j - s.n0);
  return (long)s.B * (s.n0 + s.n1) + (long)b * s.n2 + (j - s.n0 - s.n1);
}
// inverse: segment-major row -> (b, node)
__device__ __forceinline__ void seg_unrow(const Segs& s, long r, int& b, int& i) {
  const long e0 = (long)s.B * s.n0, e1 = e0 + (long)s.B * s.n1;
  if (r < e0) { b = (int)(r / s.n0); i = (int)(r % s.n0); }
  else if (r < e1) { long q = r - e0; b = (int)(q / s.n1); i = s.n0 + (int)(q % s.n1); }
  else { long q = r - e1; b = (int)(q / s.n2); i = s.n0 + s.n1 + (int)(q % s.n2); }
}

// ---------------------------------------------------------------- dense -> CSR
template <typename E> __device__ __forceinline__ float edge_to_float(E v) { return (float)v; }
template <> __device__ __forceinline__ float edge_to_float<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename E> __device__ __forceinline__ bool edge_nonzero(E v) { return v != (E)0; }
template <> __device__ __forceinline__ bool edge_nonzero<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v) != 0.f; }

// pass 1: one warp per (b, i): count the non-zeros of A[b, i, :]
template <typename E>
__global__ void dense_count_kernel(const E* __restrict__ a, long sb, long si, long sj, int B, int N,
                                   int* __restrict__ counts) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const long rows = (long)B * N;
  const int lane = threadIdx.x & 31;
  for (long r = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < rows;
       r += (long)gridDim.x * (blockDim.x >> 5)) {
    const E* row = a + (r / N) * sb + (r % N) * si;
    int c = 0;
    for (int j = lane; j < N; j += 32) c += edge_nonzero(row[(long)j * sj]) ? 1 : 0;
    c = __reduce_add_sync(0xffffffffu, c);
    if (lane == 0) counts[r] = c;
  }
}

// exclusive scan of n counts into rowptr[0..n] by ONE 1024-thread CTA (n = B*650 <= a few 100k)
__global__ void scan_kernel(const int* __restrict__ counts, int* __restrict__ rowptr, long n) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ int warp_tot[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long base = 0; base < n; base += 1024) {
    long i = base + threadIdx.x;
    int v = i < n ? counts[i] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) warp_tot[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int w = warp_tot[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
      warp_tot[lane] = w;
    }
    __syncthreads();
    int excl = carry + (warp ? warp_tot[warp - 1] : 0) + x - v;
    if (i < n) rowptr[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) rowptr[n] = carry;
}

// pass 2: same traversal, ballot-compacted writes (columns stay sorted)
template <typename E>
__global__ void dense_fill_kernel(const E* __restrict__ a, long sb, long si, long sj, int B, int N,
                                  const int* __restrict__ rowptr, int* __restrict__ col, float* __restrict__ val) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const long rows = (long)B * N;
  const int lane = threadIdx.x & 31;
  for (long r = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < rows;
       r += (long)gridDim.x * (blockDim.x >> 5)) {
    const E* row = a + (r / N) * sb + (r % N) * si;
    int pos = rowptr[r];
    for (int j0 = 0; j0 < N; j0 += 32) {
      const int j = j0 + lane;
      E v = j < N ? row[(long)j * sj] : (E)0;
      const bool nz = j < N && edge_nonzero(v);
      const unsigned bal = __ballot_sync(0xffffffffu, nz);
      if (nz) {
        int o = pos + __popc(bal & ((1u << lane) - 1u));
        col[o] = j; val[o] = edge_to_float(v);
      }
      pos += __popc(bal);
    }
  }
}

__global__ void csr_rowsum_kernel(const int* __restrict__ rowptr, const float* __restrict__ val, Segs s, int N,
                                  float* __restrict__ out) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const long R = (long)s.B * N;
  for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < R; r += (long)gridDim.x * blockDim.x) {
    int b, i; seg_unrow(s, r, b, i);
    const long g = (long)b * N + i;
    float t = 0.f;
    for (int e = rowptr[g]; e < rowptr[g + 1]; ++e) t += val[e];
    out[r] = t;
  }
}

// ---------------------------------------------------------------- the GNN "scatter": Y = A X (+ addend)
// A QUARTER warp (LPR = 8 lanes) owns one destination row, 32 features per lane, so a warp carries four independent
// rowptr -> (col,val) -> neighbour-row chains; with a whole warp per row the bf16 rows (512 B) are too short to keep
// enough bytes in flight.  The (col, val) segment of a row is fetched by the row's lanes in parallel and broadcast by
// shuffle (segmented reduction with no atomics: CSR is destination-sorted); fp32 accumulation in source order
// (deterministic).
// A lane's features are INTERLEAVED in 8-feature chunks (chunk j of lane l = features j*LPR*8 + l*8 .. +7), so
// one load/store instruction of a row group covers a contiguous LPR*16 B (bf16) span; with the blocked layout
// (lane l = features l*F ..) every instruction touched half of each 32-B sector (ncu: 49 % excessive sectors).
// Algorithmic bytes per pass: 2 * R * D * sizeof(T) + (R + 1) * 4 + nnz * 8   (SURVEY.md section 8d).
template <typename T>
__global__ void __launch_bounds__(256) csr_spmm_part_kernel(const int* __restrict__ rowptr, const int* __restrict__ col,
                                                            const float* __restrict__ val, const T* __restrict__ x,
                                                            const T* __restrict__ addend, T* __restrict__ y, Segs s,
                                                            int N) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  constexpr int LPR = 8;                          // lanes per destination row
  constexpr int F = D / LPR;                      // features per lane
  constexpr int RPW = 32 / LPR;                   // rows per warp
  const long R = (long)s.B * N;
  const int lane = threadIdx.x & 31;
  const int hl = lane % LPR;                      // lane within its row group
  const int hbase = lane - hl;                    // shuffle source offset of this group
  const unsigned hmask = ((1u << LPR) - 1u) << hbase;
  const long part0 = ((long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW + lane / LPR;
  const long nparts = (long)gridDim.x * (blockDim.x >> 5) * RPW;
  for (long r = part0; r < R; r += nparts) {
    int b, i; seg_unrow(s, r, b, i);
    const long g = (long)b * N + i;
    const int e0 = rowptr[g], e1 = rowptr[g + 1];
    float acc[F];
    if (addend) {
#pragma unroll
      for (int q = 0; q < F; q += 8) Act<T>::load8(addend + r * D + q * LPR + hl * 8, acc + q);
    } else {
#pragma unroll
      for (int k = 0; k < F; ++k) acc[k] = 0.f;
    }
    for (int eb = e0; eb < e1; eb += LPR) {
      const int n = min(LPR, e1 - eb);
      int c = 0; float w = 0.f;
      if (hl < n) { c = col[eb + hl]; w = val[eb + hl]; }
      for (int t = 0; t < n; ++t) {
        const int c0 = __shfl_sync(hmask, c, hbase + t);
        const float w0 = __shfl_sync(hmask, w, hbase + t);
        float v0[F];
        const T* p0 = x + seg_row(s, b, c0) * D + hl * 8;
#pragma unroll
        for (int q = 0; q < F; q += 8) Act<T>::load8(p0 + q * LPR, v0 + q);
#pragma unroll
        for (int k = 0; k < F; ++k) acc[k] = fmaf(w0, v0[k], acc[k]);
      }
    }
#pragma unroll
    for (int q = 0; q < F; q += 8) Act<T>::store8(y + r * D + q * LPR + hl * 8, acc + q);
  }
}

}  // namespace

#define DISPATCH_T(dtype, ...)                                                            \
  if ((dtype) == FIRA_F32) { using T = float; __VA_ARGS__ }                               \
  else if ((dtype) == FIRA_BF16) { using T = __nv_bfloat16; __VA_ARGS__ }                 \
  else { fira_set_error(FIRA_ERR_DTYPE, "unknown dtype %d", (int)(dtype)); return FIRA_ERR_DTYPE; }

extern "C" {

// edge_dtype: 0 f32, 1 bf16, 2 f64, 3 f16 is not supported (the reference only produces f64/f32)
int fira_csr_count_dense(const void* edge, int edge_dtype, long stride_b, long stride_i, long stride_j, int B, int N,
                         int* counts, int* rowptr, void* stream) {
  FIRA_CHECK_ARG(B > 0 && N > 0, FIRA_ERR_SHAPE, "csr_count_dense: B=%d N=%d", B, N);
  cudaStream_t st = (cudaStream_t)stream;
  const long rows = (long)B * N;
  int grid = (int)((rows + 7) / 8 < fira_num_sms() * 8 ? (rows + 7) / 8 : fira_num_sms() * 8);
  if (edge_dtype == 0) launch_k(dense_count_kernel<float>, dim3(grid), dim3(256), 0, st, (const float*)edge, stride_b, stride_i, stride_j, B, N, counts);
  else if (edge_dtype == 2) launch_k(dense_count_kernel<double>, dim3(grid), dim3(256), 0, st, (const double*)edge, stride_b, stride_i, stride_j, B, N, counts);
  else if (edge_dtype == 1) launch_k(dense_count_kernel<__nv_bfloat16>, dim3(grid), dim3(256), 0, st, (const __nv_bfloat16*)edge, stride_b, stride_i, stride_j, B, N, counts);
  else { fira_set_error(FIRA_ERR_DTYPE, "csr_count_dense: edge dtype %d", edge_dtype); return FIRA_ERR_DTYPE; }
  FIRA_CHECK_LAUNCH("fira_csr_count_dense");
  launch_k(scan_kernel, dim3(1), dim3(1024), 0, st, counts, rowptr, rows);
  FIRA_CHECK_LAUNCH("fira_csr_count_dense/scan");
  return FIRA_OK;
}

int fira_csr_fill_dense(const void* edge, int edge_dtype, long stride_b, long stride_i, long stride_j, int B, int N,
                        const int* rowptr, int* col, float* val, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const long rows = (long)B * N;
  int grid = (int)((rows + 7) / 8 < fira_num_sms() * 8 ? (rows + 7) / 8 : fira_num_sms() * 8);
  if (edge_dtype == 0) launch_k(dense_fill_kernel<float>, dim3(grid), dim3(256), 0, st, (const float*)edge, stride_b, stride_i, stride_j, B, N, rowptr, col, val);
  else if (edge_dtype == 2) launch_k(dense_fill_kernel<double>, dim3(grid), dim3(256), 0, st, (const double*)edge, stride_b, stride_i, stride_j, B, N, rowptr, col, val);
  else if (edge_dtype == 1) launch_k(dense_fill_kernel<__nv_bfloat16>, dim3(grid), dim3(256), 0, st, (const __nv_bfloat16*)edge, stride_b, stride_i, stride_j, B, N, rowptr, col, val);
  else { fira_set_error(FIRA_ERR_DTYPE, "csr_fill_dense: edge dtype %d", edge_dtype); return FIRA_ERR_DTYPE; }
  FIRA_CHECK_LAUNCH("fira_csr_fill_dense");
  return FIRA_OK;
}

int fira_csr_rowsum(const int* rowptr, const float* val, int B, int n_code, int n_sub, int n_ast, float* out,
                    void* stream) {
  Segs s{B, n_code, n_sub, n_ast};
  const int N = n_code + n_sub + n_ast;
  FIRA_CHECK_ARG(n_code > 0 && n_sub >= 0 && n_ast >= 0, FIRA_ERR_SHAPE, "csr_rowsum: segments");
  const long R = (long)B * N;
  launch_k(csr_rowsum_kernel, dim3((int)((R + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, rowptr, val, s, N, out);
  FIRA_CHECK_LAUNCH("fira_csr_rowsum");
  return FIRA_OK;
}

int fira_gcn_aggregate(const int* rowptr, const int* col, const float* val, const void* x, const void* addend,
                       void* y, int B, int n_code, int n_sub, int n_ast, int dim, int dtype, void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "gcn_aggregate: dim %d != 256", dim);
  FIRA_CHECK_ARG(n_code > 0 && n_sub >= 0 && n_ast >= 0 && B > 0, FIRA_ERR_SHAPE, "gcn_aggregate: segments");
  FIRA_CHECK_ARG(fira_aligned16(x) && fira_aligned16(y) && fira_aligned16(addend), FIRA_ERR_ALIGN,
                 "gcn_aggregate: 16-B alignment");
  FIRA_CHECK_ARG(x != y, FIRA_ERR_ARG, "gcn_aggregate: in-place not supported");
  Segs s{B, n_code, n_sub, n_ast};
  const int N = n_code + n_sub + n_ast;
  const long R = (long)B * N;
  const long ctas = (R + 31) / 32;                // 8 warps x 4 rows per CTA
  const long cap = (long)fira_num_sms() * 8 * 4;
  const int grid = (int)(ctas < cap ? ctas : cap);
  DISPATCH_T(dtype, launch_k(csr_spmm_part_kernel<T>, dim3(grid), dim3(256), 0, (cudaStream_t)stream,
      rowptr, col, val, (const T*)x, (const T*)addend, (T*)y, s, N);)
  FIRA_CHECK_LAUNCH("fira_gcn_aggregate");
  return FIRA_OK;
}

}  // extern "C"
