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
#include <stdlib.h>
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
// One warp owns one destination row: 32 lanes x 8 features = the whole 256-wide row, so each
// neighbour row is ONE fully coalesced 1 KB (fp32) / 512 B (bf16) read; the (col, val) segment of
// the row is fetched by the lanes in parallel and broadcast by shuffle (segmented reduction with no
// atomics: CSR is destination-sorted).  fp32 accumulation in source order (deterministic).
// Algorithmic bytes per pass: 2 * R * D * sizeof(T) + (R + 1) * 4 + nnz * 8   (SURVEY.md section 8d).
template <typename T>
__global__ void __launch_bounds__(256) csr_spmm_kernel(const int* __restrict__ rowptr, const int* __restrict__ col,
                                                       const float* __restrict__ val, const T* __restrict__ x,
                                                       const T* __restrict__ addend, T* __restrict__ y, Segs s, int N) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const long R = (long)s.B * N;
  const int lane = threadIdx.x & 31;
  const long warp0 = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long nwarps = (long)gridDim.x * (blockDim.x >> 5);
  for (long r = warp0; r < R; r += nwarps) {
    int b, i; seg_unrow(s, r, b, i);
    const long g = (long)b * N + i;
    const int e0 = rowptr[g], e1 = rowptr[g + 1];
    float acc[8];
    if (addend) Act<T>::load8(addend + r * D + lane * 8, acc);
    else {
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    }
    for (int eb = e0; eb < e1; eb += 32) {
      const int n = min(32, e1 - eb);
      int c = 0; float w = 0.f;
      if (lane < n) { c = col[eb + lane]; w = val[eb + lane]; }
      int t = 0;
      for (; t + 1 < n; t += 2) {      // two neighbour rows in flight per lane
        const int c0 = __shfl_sync(0xffffffffu, c, t), c1 = __shfl_sync(0xffffffffu, c, t + 1);
        const float w0 = __shfl_sync(0xffffffffu, w, t), w1 = __shfl_sync(0xffffffffu, w, t + 1);
        float v0[8], v1[8];
        Act<T>::load8(x + seg_row(s, b, c0) * D + lane * 8, v0);
        Act<T>::load8(x + seg_row(s, b, c1) * D + lane * 8, v1);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = fmaf(w0, v0[k], acc[k]);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = fmaf(w1, v1[k], acc[k]);
      }
      if (t < n) {
        const int c0 = __shfl_sync(0xffffffffu, c, t);
        const float w0 = __shfl_sync(0xffffffffu, w, t);
        float v0[8];
        Act<T>::load8(x + seg_row(s, b, c0) * D + lane * 8, v0);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = fmaf(w0, v0[k], acc[k]);
      }
    }
    Act<T>::store8(y + r * D + lane * 8, acc);
  }
}

// Version 4: HALF a warp per destination row, 16 features per lane (two 16-byte loads for bf16, four for
// fp32).  A warp then carries two independent rows, i.e. twice the rows -- and twice the dependent
// rowptr -> (col,val) -> feature-row chains -- in flight for the same number of resident warps; the bf16
// rows (512 B) are too short for a full warp to keep enough bytes in flight (v1: 0.29 of peak in bf16).
// A lane's features are INTERLEAVED in 8-feature chunks (chunk j of lane l = features j*LPR*8 + l*8 .. +7), so
// one load/store instruction of a row group covers a contiguous LPR*16 B (bf16) span; with the blocked layout
// (lane l = features l*F ..) every instruction touched half of each 32-B sector (ncu: 49 % excessive sectors).
template <typename T, int LPR, int UNROLL = 1>     // LPR lanes per destination row (16 or 8): 32/LPR rows in flight per warp
__global__ void __launch_bounds__(256) csr_spmm_part_kernel(const int* __restrict__ rowptr, const int* __restrict__ col,
                                                            const float* __restrict__ val, const T* __restrict__ x,
                                                            const T* __restrict__ addend, T* __restrict__ y, Segs s,
                                                            int N) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  constexpr int F = D / LPR;                      // features per lane (16 or 32)
  constexpr int RPW = 32 / LPR;                   // rows per warp
  const long R = (long)s.B * N;
  const int lane = threadIdx.x & 31;
  const int hl = lane % LPR;                      // lane within its row group
  const int hbase = lane - hl;                    // shuffle source offset of this group
  const unsigned hmask = (LPR == 32 ? 0xffffffffu : ((1u << LPR) - 1u)) << hbase;
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
      int t = 0;
      if constexpr (UNROLL == 2) {       // variant 7 (A/B): two neighbour rows in flight per lane group, CSR order kept
        for (; t + 1 < n; t += 2) {
          const int c0 = __shfl_sync(hmask, c, hbase + t), c1 = __shfl_sync(hmask, c, hbase + t + 1);
          const float w0 = __shfl_sync(hmask, w, hbase + t), w1 = __shfl_sync(hmask, w, hbase + t + 1);
          float v0[F], v1[F];
          const T* p0 = x + seg_row(s, b, c0) * D + hl * 8;
          const T* p1 = x + seg_row(s, b, c1) * D + hl * 8;
#pragma unroll
          for (int q = 0; q < F; q += 8) Act<T>::load8(p0 + q * LPR, v0 + q);
#pragma unroll
          for (int q = 0; q < F; q += 8) Act<T>::load8(p1 + q * LPR, v1 + q);
#pragma unroll
          for (int k = 0; k < F; ++k) acc[k] = fmaf(w0, v0[k], acc[k]);
#pragma unroll
          for (int k = 0; k < F; ++k) acc[k] = fmaf(w1, v1[k], acc[k]);
        }
      }
      for (; t < n; ++t) {
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

// Version 6 (opt-in, FIRA_SPMM_VARIANT=6, not measured): the v4 row mapping on a persistent one-wave grid with the
// metadata software-pipelined two rows ahead.  In v4 every CTA lives exactly one dependent chain
// rowptr -> (col,val) -> neighbour rows (three DRAM latencies).  Here a row group
// walks ~R / (SMs * 4 * 16) rows; while the neighbour rows of row k are gathered, the first (col,val) chunk of row
// k+1 and the rowptr pair of row k+2 are already in flight, so a row costs ~one latency instead of three.
template <typename T, int LPR>
__global__ void __launch_bounds__(256) csr_spmm_pipe_kernel(const int* __restrict__ rowptr, const int* __restrict__ col,
                                                            const float* __restrict__ val, const T* __restrict__ x,
                                                            const T* __restrict__ addend, T* __restrict__ y, Segs s,
                                                            int N) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  constexpr int F = D / LPR;
  constexpr int RPW = 32 / LPR;
  const long R = (long)s.B * N;
  const int lane = threadIdx.x & 31;
  const int hl = lane % LPR;
  const int hbase = lane - hl;
  const unsigned hmask = (LPR == 32 ? 0xffffffffu : ((1u << LPR) - 1u)) << hbase;
  const long part0 = ((long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW + lane / LPR;
  const long nparts = (long)gridDim.x * (blockDim.x >> 5) * RPW;
  auto row_meta = [&](long r, int& b, int& lo, int& hi) {
    int i; seg_unrow(s, r, b, i);
    const long g = (long)b * N + i;
    lo = rowptr[g]; hi = rowptr[g + 1];
  };
  long r = part0;
  int b0 = 0, e0 = 0, e1 = 0, c = 0;             // row k: graph, edge range, first (col, val) chunk
  float w = 0.f;
  int b1 = 0, f0 = 0, f1 = 0;                    // row k+1: graph, edge range
  if (r < R) {
    row_meta(r, b0, e0, e1);
    if (hl < e1 - e0) { c = col[e0 + hl]; w = val[e0 + hl]; }
  }
  if (r + nparts < R) row_meta(r + nparts, b1, f0, f1);
  while (r < R) {
    int cn = 0; float wn = 0.f;                  // in flight during this row: (col,val) of row k+1 ...
    if (r + nparts < R && hl < f1 - f0) { cn = col[f0 + hl]; wn = val[f0 + hl]; }
    int b2 = 0, g0 = 0, g1 = 0;                  // ... and the rowptr pair of row k+2
    if (r + 2 * nparts < R) row_meta(r + 2 * nparts, b2, g0, g1);
    float acc[F];
    if (addend) {
#pragma unroll
      for (int q = 0; q < F; q += 8) Act<T>::load8(addend + r * D + q * LPR + hl * 8, acc + q);
    } else {
#pragma unroll
      for (int k = 0; k < F; ++k) acc[k] = 0.f;
    }
    for (int eb = e0; eb < e1; eb += LPR) {
      if (eb != e0) {                            // rows with more than LPR neighbours: later chunks are not prefetched
        c = 0; w = 0.f;
        if (hl < e1 - eb) { c = col[eb + hl]; w = val[eb + hl]; }
      }
      const int n = min(LPR, e1 - eb);
      int t = 0;
      for (; t + 1 < n; t += 2) {                // two neighbour rows in flight per lane
        const int c0 = __shfl_sync(hmask, c, hbase + t), c1 = __shfl_sync(hmask, c, hbase + t + 1);
        const float w0 = __shfl_sync(hmask, w, hbase + t), w1 = __shfl_sync(hmask, w, hbase + t + 1);
        float v0[F], v1[F];
        const T* p0 = x + seg_row(s, b0, c0) * D + hl * 8;
        const T* p1 = x + seg_row(s, b0, c1) * D + hl * 8;
#pragma unroll
        for (int q = 0; q < F; q += 8) { Act<T>::load8(p0 + q * LPR, v0 + q); Act<T>::load8(p1 + q * LPR, v1 + q); }
#pragma unroll
        for (int k = 0; k < F; ++k) acc[k] = fmaf(w1, v1[k], fmaf(w0, v0[k], acc[k]));
      }
      if (t < n) {
        const int c0 = __shfl_sync(hmask, c, hbase + t);
        const float w0 = __shfl_sync(hmask, w, hbase + t);
        float v0[F];
        const T* p0 = x + seg_row(s, b0, c0) * D + hl * 8;
#pragma unroll
        for (int q = 0; q < F; q += 8) Act<T>::load8(p0 + q * LPR, v0 + q);
#pragma unroll
        for (int k = 0; k < F; ++k) acc[k] = fmaf(w0, v0[k], acc[k]);
      }
    }
#pragma unroll
    for (int q = 0; q < F; q += 8) Act<T>::store8(y + r * D + q * LPR + hl * 8, acc + q);
    r += nparts;
    b0 = b1; e0 = f0; e1 = f1; c = cn; w = wn;
    b1 = b2; f0 = g0; f1 = g1;
  }
}

// Version 3: bulk-async (TMA engine, SASS UBLKCP) staging of the neighbour rows in shared memory.
// Little's law asks for tens of KB of reads in flight per SM; v1/v2 hold the gathered rows in
// registers and spend most of a row's life on the two dependent metadata round trips, so they sit at
// ~13 KB/SM.  Here a warp takes a group of GR consecutive destination rows, builds their edge list
// once (one rowptr round trip, one col/val round trip), then every lane fires ONE
// cp.async.bulk of a whole 1 KB / 512 B neighbour row into the warp's shared-memory stage -- up to EB
// rows in flight per warp at zero register cost -- and after a single mbarrier wait the warp reduces
// the staged rows in CSR order (segmented reduction, no atomics).  `addend` rides along as a
// pseudo-edge of weight 1.
constexpr int GR = 8;    // destination rows per warp group
constexpr int EB = 16;   // staged neighbour rows per batch

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}

template <typename T, int WARPS>
__global__ void __launch_bounds__(WARPS * 32) csr_spmm_bulk_kernel(const int* __restrict__ rowptr,
                                                                   const int* __restrict__ col,
                                                                   const float* __restrict__ val,
                                                                   const T* __restrict__ x,
                                                                   const T* __restrict__ addend, T* __restrict__ y,
                                                                   Segs s, int N) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ __align__(8) unsigned long long bars[WARPS];
  constexpr uint32_t ROW_BYTES = D * sizeof(T);
  const long R = (long)s.B * N;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T* stage = reinterpret_cast<T*>(smem_raw) + (size_t)warp * EB * D;
  const uint32_t bar = smem_u32(&bars[warp]);
  if (lane == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  uint32_t parity = 0;
  const long group0 = (long)blockIdx.x * WARPS + warp;
  const long ngroups = (long)gridDim.x * WARPS;
  const int extra = addend ? 1 : 0;
  for (long r0 = group0 * GR; r0 < R; r0 += ngroups * GR) {
    // ---- metadata: one round trip for rowptr, prefix over the group's rows
    int my_e0 = 0, my_n = 0, my_b = 0;
    if (lane < GR && r0 + lane < R) {
      int b, i; seg_unrow(s, r0 + lane, b, i);
      const long g = (long)b * N + i;
      my_e0 = rowptr[g]; my_n = rowptr[g + 1] - my_e0 + extra; my_b = b;
    }
    int incl = my_n;                                        // inclusive prefix over lanes 0..GR-1
#pragma unroll
    for (int o = 1; o < GR; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    const int total = __shfl_sync(0xffffffffu, incl, GR - 1);
    const int my_start = incl - my_n;
    int cur = -1;                                           // destination slot being accumulated
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int kb = 0; kb < total; kb += EB) {
      const int cnt = min(EB, total - kb);
      // ---- this lane's edge of the batch: slot, source row pointer, weight (one col/val round trip)
      int slot = 0; float w = 0.f; const T* src = nullptr;
      const int id = kb + lane;
#pragma unroll
      for (int q = 0; q < GR; ++q) {
        const int st = __shfl_sync(0xffffffffu, my_start, q), nn = __shfl_sync(0xffffffffu, my_n, q);
        const int ee = __shfl_sync(0xffffffffu, my_e0, q), bq = __shfl_sync(0xffffffffu, my_b, q);
        if (lane < cnt && id >= st && id < st + nn) {
          slot = q;
          const int j = id - st;
          if (extra && j == nn - 1) { src = addend + (r0 + q) * D; w = 1.f; }
          else { src = x + seg_row(s, bq, col[ee + j]) * D; w = val[ee + j]; }
        }
      }
      // ---- fire the bulk copies: lane 0 arms the barrier with the byte count, every lane copies its row
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // stage reads (generic) before async refill
      if (lane == 0) mbar_expect_tx(bar, (uint32_t)cnt * ROW_BYTES);
      __syncwarp();
      if (lane < cnt) bulk_g2s(smem_u32(stage + (size_t)lane * D), src, ROW_BYTES, bar);
      uint32_t spins = 0;
      while (!mbar_try_wait(bar, parity)) { if (++spins > (1u << 24)) __trap(); }
      parity ^= 1;
      // ---- segmented reduction of the staged rows, CSR order
      for (int k = 0; k < cnt; ++k) {
        const int sk = __shfl_sync(0xffffffffu, slot, k);
        const float wk = __shfl_sync(0xffffffffu, w, k);
        if (sk != cur) {
          if (cur >= 0) Act<T>::store8(y + (r0 + cur) * D + lane * 8, acc);
#pragma unroll
          for (int q = 0; q < 8; ++q) acc[q] = 0.f;
          for (int z = cur + 1; z < sk; ++z) Act<T>::store8(y + (r0 + z) * D + lane * 8, acc);   // edge-less rows
          cur = sk;
        }
        float v[8];
        Act<T>::load8(stage + (size_t)k * D + lane * 8, v);
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = fmaf(wk, v[q], acc[q]);
      }
      __syncwarp();                                         // all lanes done reading before the stage is refilled
    }
    if (cur >= 0) Act<T>::store8(y + (r0 + cur) * D + lane * 8, acc);
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q] = 0.f;
    for (int z = cur + 1; z < GR && r0 + z < R; ++z) Act<T>::store8(y + (r0 + z) * D + lane * 8, acc);
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
  // default: a QUARTER warp per destination row (variant 8: four independent rowptr -> (col,val) -> neighbour-row chains
  // per warp, 32 features = 64-128 B per lane and neighbour row), more independent chains in flight than half a warp
  // (variant 4) or a whole warp (variant 1) per row.  FIRA_SPMM_VARIANT overrides (A/B runs).
  static const int forced = [] { const char* e = getenv("FIRA_SPMM_VARIANT"); return e ? atoi(e) : 0; }();
  const int variant = forced ? forced : 8;
  if (variant == 1) {                      // round-1 baseline kernel, kept for A/B profiling
    long ctas = (R + 7) / 8;
    const long cap = (long)fira_num_sms() * 8 * 4;
    int grid = (int)(ctas < cap ? ctas : cap);
    DISPATCH_T(dtype, launch_k(csr_spmm_kernel<T>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, rowptr, col, val, (const T*)x,
                                                                                   (const T*)addend, (T*)y, s, N);)
  } else if (variant == 4) {
    long ctas = (R + 15) / 16;               // 8 warps x 2 rows
    const long cap = (long)fira_num_sms() * 8 * 4;
    int grid = (int)(ctas < cap ? ctas : cap);
    DISPATCH_T(dtype, launch_k(csr_spmm_part_kernel<T, 16>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, 
        rowptr, col, val, (const T*)x, (const T*)addend, (T*)y, s, N);)
  } else if (variant >= 7 && variant <= 10) {
    // 7: half a warp per row, two neighbour rows in flight; 8 (default): a quarter warp per row; 9: an eighth of a warp per
    // row (bf16); 10: a quarter warp per row, two neighbour rows in flight
    const int rows_per_cta = variant == 7 ? 16 : (variant == 9 ? 64 : 32);
    long ctas = (R + rows_per_cta - 1) / rows_per_cta;
    const long cap = (long)fira_num_sms() * 8 * 4;
    int grid = (int)(ctas < cap ? ctas : cap);
    if (variant == 7) {
      DISPATCH_T(dtype, launch_k(csr_spmm_part_kernel<T, 16, 2>, dim3(grid), dim3(256), 0, (cudaStream_t)stream,
          rowptr, col, val, (const T*)x, (const T*)addend, (T*)y, s, N);)
    } else if (variant == 8) {
      DISPATCH_T(dtype, launch_k(csr_spmm_part_kernel<T, 8, 1>, dim3(grid), dim3(256), 0, (cudaStream_t)stream,
          rowptr, col, val, (const T*)x, (const T*)addend, (T*)y, s, N);)
    } else if (variant == 9) {
      DISPATCH_T(dtype, launch_k(csr_spmm_part_kernel<T, 4, 1>, dim3(grid), dim3(256), 0, (cudaStream_t)stream,
          rowptr, col, val, (const T*)x, (const T*)addend, (T*)y, s, N);)
    } else {
      DISPATCH_T(dtype, launch_k(csr_spmm_part_kernel<T, 8, 2>, dim3(grid), dim3(256), 0, (cudaStream_t)stream,
          rowptr, col, val, (const T*)x, (const T*)addend, (T*)y, s, N);)
    }
  } else if (variant == 6) {                 // persistent one-wave grid, metadata pipelined two rows ahead (unmeasured)
    const int rows_per_cta = dtype == FIRA_BF16 ? 16 : 8;
    long ctas = (R + rows_per_cta - 1) / rows_per_cta;
    const long cap = (long)fira_num_sms() * 4;               // 64 registers/thread -> 4 CTAs of 256 threads per SM
    int grid = (int)(ctas < cap ? ctas : cap);
    if (dtype == FIRA_BF16) {
      launch_k(csr_spmm_pipe_kernel<__nv_bfloat16, 16>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, 
          rowptr, col, val, (const __nv_bfloat16*)x, (const __nv_bfloat16*)addend, (__nv_bfloat16*)y, s, N);
    } else {
      launch_k(csr_spmm_pipe_kernel<float, 32>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, 
          rowptr, col, val, (const float*)x, (const float*)addend, (float*)y, s, N);
    }
  } else if (variant == 3) {
    constexpr int WARPS = 6;
    const size_t smem = (size_t)WARPS * EB * D * (dtype == FIRA_F32 ? 4 : 2);
    static bool attr_done = false;
    if (!attr_done) {
      cudaFuncSetAttribute(csr_spmm_bulk_kernel<float, WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           WARPS * EB * D * 4);
      cudaFuncSetAttribute(csr_spmm_bulk_kernel<__nv_bfloat16, WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           WARPS * EB * D * 2);
      attr_done = true;
    }
    long ctas = (R + (long)GR * WARPS - 1) / ((long)GR * WARPS);
    const long cap = (long)fira_num_sms() * 8;
    int grid = (int)(ctas < cap ? ctas : cap);
    DISPATCH_T(dtype, launch_k(csr_spmm_bulk_kernel<T, WARPS>, dim3(grid), dim3(WARPS * 32), smem, (cudaStream_t)stream, 
        rowptr, col, val, (const T*)x, (const T*)addend, (T*)y, s, N);)
  } else {
    fira_set_error(FIRA_ERR_ARG, "gcn_aggregate: unknown FIRA_SPMM_VARIANT %d (1, 3, 4, 6)", variant);
    return FIRA_ERR_ARG;
  }
  FIRA_CHECK_LAUNCH("fira_gcn_aggregate");
  return FIRA_OK;
}

}  // extern "C"
