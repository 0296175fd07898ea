// Fused GCN layer for the bf16 throughput path (gnn_transformer.py:74-86), ONE kernel per layer and direction:
//
//   forward  (MODE 0):  Z = (A H) Wc^T + rowsum(A) (x) c1 + b2 ;  out = LN(dropout(Z) + H)          Wc = W2 W1, c1 = W2 b1
//   backward (MODE 1):  AdZ = A^T dZ (side output for dWc = AdZ^T H) ;  dH = AdZ Wc + d_resid
//
// gather -> transform -> epilogue without a round trip through HBM between them:
//   * 4 gather warps build the aggregated 128-row tile (A H)[rows, 0:256] straight in shared memory, in the
//     K-major SWIZZLE_128B layout wgmma reads (the tile IS the A operand): a quarter warp per destination row,
//     16-byte loads, 8 x 128 B of neighbour rows in flight per lane group, fp32 accumulation in CSR order, the tile's
//     rowptr / (col, val) metadata prefetched into shared memory first (one dependent latency per row, not three);
//   * the 256 x 256 weight (128 KB bf16) is loaded ONCE per CTA by TMA and stays resident (persistent CTAs, one per SM);
//   * two consumer warpgroups (rows 0-63 / 64-127 of the tile) issue 16 wgmma m64 n256 k16 each per tile, fp32
//     accumulator in registers; the A tile is handed back as soon as they complete, so the gather of tile t+1
//     overlaps the epilogue of tile t;
//   * the epilogue works on the register fragments: add bias + rowsum*c1, write Z, apply dropout + residual +
//     LayerNorm (a row's 256 columns live in the 4 threads of a lane quad: two shuffles for the row statistics) and
//     write the normalised rows.
// Rows are addressed through a CSR in BUFFER order (rowptr[r], col = buffer row; fira_csr_to_rows builds it from the
// (graph, node)-ordered CSR), so the kernel does not care whether the node buffer is padded segment-major or packed.
#include "tc_common.cuh"
#include "fira_b200.h"

namespace {

using namespace tc;

constexpr int D = 256;
constexpr int TM = 128;                    // rows per tile: two m64 warpgroups
constexpr int N_CONSUMER = 256;            // warps 0-7
constexpr int N_GATHER = 4;                // warps 8-11
constexpr int THREADS = N_CONSUMER + N_GATHER * 32;
constexpr int EC = 1024;                   // edges of a tile staged in shared memory (larger tiles read col/val from global)
constexpr uint32_t B_BYTES = D * D * 2;    // 131072: 4 k-blocks x [256 n-rows x 128 B]
constexpr uint32_t A_BYTES = TM * D * 2;   // 65536:  4 k-blocks x [128 rows x 128 B]
constexpr uint32_t OFF_A = B_BYTES, OFF_ROWPTR = OFF_A + A_BYTES, OFF_COL = OFF_ROWPTR + 544, OFF_VAL = OFF_COL + EC * 4,
                   OFF_RS = OFF_VAL + EC * 4, SMEM_BYTES = OFF_RS + 4 * TM * 4;
constexpr int GATHER_BAR = 1;              // named barrier of the gather warps

struct Params {
  const int* rowptr; const int* col; const float* val;      // buffer-order CSR
  const __nv_bfloat16* x;                                    // H (fwd) or dZ (bwd), [R, 256]
  long R;
  // MODE 0
  const float* bias; const float* c1; const float* gamma; const float* beta;
  __nv_bfloat16* z; __nv_bfloat16* outA; __nv_bfloat16* outB; long split;
  float* mean; float* rstd;
  float p_drop; uint64_t seed; const uint64_t* seed_ctr; uint32_t stream_id;
  // MODE 1
  const __nv_bfloat16* addend; __nv_bfloat16* agg_out; __nv_bfloat16* y;
};

__device__ __forceinline__ void tile_range(long R, int cta, int ncta, int t, long& r0, int& rows, int& ntiles) {
  const long rpc = (R + ncta - 1) / ncta;
  const long lo = (long)cta * rpc;
  const long hi = lo + rpc < R ? lo + rpc : R;
  const long n = hi > lo ? hi - lo : 0;
  ntiles = (int)((n + TM - 1) / TM);
  if (ntiles == 0) { r0 = 0; rows = 0; return; }
  long chunk = (n + ntiles - 1) / ntiles;
  chunk = (chunk + 7) & ~7L;
  if (chunk > TM) chunk = TM;
  r0 = lo + (long)t * chunk;
  const long e = r0 + chunk < hi ? r0 + chunk : hi;
  rows = (int)(e > r0 ? e - r0 : 0);
}

__device__ __forceinline__ uint4 pack8(const float* v) {
  uint4 r;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
  return r;
}
__device__ __forceinline__ void unpack8(const uint4& raw, float* v) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float2 f = __bfloat1622float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
}

// 12 warps cap the kernel at 168 registers: the LayerNorm epilogue over the 128-register accumulator spills (ptxas -v: up
// to 1.2 KB); the kernel is opt-in (FIRA_GCN_FUSED) and has not been timed on the H100
template <int MODE>
__global__ void __launch_bounds__(THREADS, 1) gcn_fused_kernel(const __grid_constant__ CUtensorMap tmW, Params p) {
  extern __shared__ unsigned char smem_raw[];
  __shared__ __align__(8) unsigned long long b_full, a_full, a_empty;
  const uint32_t base = (smem_addr(smem_raw) + 1023u) & ~1023u;
  unsigned char* sm = smem_raw + (base - smem_addr(smem_raw));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cta = blockIdx.x, ncta = gridDim.x;
  long r0_; int rows_, ntiles;
  tile_range(p.R, cta, ncta, 0, r0_, rows_, ntiles);

  if (threadIdx.x == 0) {
    mbar_init(smem_addr(&b_full), 1);
    mbar_init(smem_addr(&a_full), N_GATHER * 32);
    mbar_init(smem_addr(&a_empty), N_CONSUMER);
    mbar_init_fence();
    tma_prefetch_desc(&tmW);
  }
  __syncthreads();
  pdl_wait(); pdl_trigger();       // PDL: the prologue above overlapped the previous kernel's tail (common.cuh)

  if (warp >= N_CONSUMER / 32) {
    // ======================================================= gather warps: A tile = (A_hat X)[tile rows, :]
    const int gw = warp - N_CONSUMER / 32;           // 0..3
    const int gtid = gw * 32 + lane;                 // 0..127
    const int q = lane >> 3, ql = lane & 7;          // quarter-warp (row slot) / lane within it
    int* s_rowptr = reinterpret_cast<int*>(sm + OFF_ROWPTR);
    int* s_col = reinterpret_cast<int*>(sm + OFF_COL);
    float* s_val = reinterpret_cast<float*>(sm + OFF_VAL);
    float* s_rs = reinterpret_cast<float*>(sm + OFF_RS);
    for (int t = 0; t < ntiles; ++t) {
      long r0; int rows, nt_;
      tile_range(p.R, cta, ncta, t, r0, rows, nt_);
      // ---- tile metadata -> shared memory (every gather warp is done with the previous tile's metadata first)
      if (t >= 1) named_bar(GATHER_BAR, N_GATHER * 32);
      for (int i = gtid; i <= rows; i += N_GATHER * 32) s_rowptr[i] = p.rowptr[r0 + i];
      named_bar(GATHER_BAR, N_GATHER * 32);
      const int e_lo = s_rowptr[0], e_hi = s_rowptr[rows];
      const int nE = e_hi - e_lo;
      const bool staged = nE <= EC;
      if (staged)
        for (int i = gtid; i < nE; i += N_GATHER * 32) { s_col[i] = p.col[e_lo + i]; s_val[i] = p.val[e_lo + i]; }
      if (t >= 1 && gtid == 0) mbar_wait(smem_addr(&a_empty), (t - 1) & 1);   // wgmma of tile t-1 have read the A tile
      named_bar(GATHER_BAR, N_GATHER * 32);
      const int* cp = staged ? s_col : p.col + e_lo;
      const float* vp = staged ? s_val : p.val + e_lo;
      // each warp: rows gw*32 + it*4 + q
#pragma unroll 1
      for (int it = 0; it < 8; ++it) {
        const int r = gw * 32 + it * 4 + q;
        if (r < rows) {
          const int e0 = s_rowptr[r] - e_lo, e1 = s_rowptr[r + 1] - e_lo;
          float acc[4][8];
#pragma unroll
          for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[j][i] = 0.f;
          float rsum = 0.f;
          int e = e0;
          for (; e + 1 < e1; e += 2) {
            const int c0 = cp[e], c1 = cp[e + 1];
            const float w0 = vp[e], w1 = vp[e + 1];
            const uint4* s0 = reinterpret_cast<const uint4*>(p.x + (long)c0 * D + ql * 8);
            const uint4* s1 = reinterpret_cast<const uint4*>(p.x + (long)c1 * D + ql * 8);
            uint4 a[4], b[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) a[j] = __ldg(s0 + j * 8);       // features j*64 + ql*8 .. +7
#pragma unroll
            for (int j = 0; j < 4; ++j) b[j] = __ldg(s1 + j * 8);
            rsum += w0 + w1;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              float f[8];
              unpack8(a[j], f);
#pragma unroll
              for (int i = 0; i < 8; ++i) acc[j][i] = fmaf(w0, f[i], acc[j][i]);
              unpack8(b[j], f);
#pragma unroll
              for (int i = 0; i < 8; ++i) acc[j][i] = fmaf(w1, f[i], acc[j][i]);
            }
          }
          if (e < e1) {
            const int c0 = cp[e];
            const float w0 = vp[e];
            const uint4* s0 = reinterpret_cast<const uint4*>(p.x + (long)c0 * D + ql * 8);
            uint4 a[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) a[j] = __ldg(s0 + j * 8);
            rsum += w0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              float f[8];
              unpack8(a[j], f);
#pragma unroll
              for (int i = 0; i < 8; ++i) acc[j][i] = fmaf(w0, f[i], acc[j][i]);
            }
          }
          // bf16 row -> swizzled K-major A tile: k-block j, 16-byte chunk ql of row r
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const uint4 v = pack8(acc[j]);
            *reinterpret_cast<uint4*>(sm + OFF_A + j * 16384 + sw128_offset(r, ql)) = v;
            if (MODE == 1) *reinterpret_cast<uint4*>(p.agg_out + (r0 + r) * D + j * 64 + ql * 8) = v;
          }
          if (MODE == 0 && ql == 0) s_rs[(t & 3) * TM + r] = rsum;
        }
      }
      fence_proxy_async();                           // my generic-proxy writes -> visible to the wgmma (async proxy) reads
      mbar_arrive(smem_addr(&a_full));
    }
    return;
  }

  // ======================================================= consumers: warpgroup wg = tile rows [64 wg, +64)
  const int wg = warp >> 2, q4 = lane & 3;
  if (threadIdx.x == 0 && ntiles > 0) {
    // ---- weight: resident B operand, 4 k-blocks of [256 n x 64 k]
    mbar_expect_tx(smem_addr(&b_full), B_BYTES);
#pragma unroll
    for (int kb = 0; kb < 4; ++kb) tma_load_2d(base + kb * 32768, &tmW, kb * 64, 0, smem_addr(&b_full));
  }
  if (ntiles > 0) mbar_wait(smem_addr(&b_full), 0);
  const float* s_rs = reinterpret_cast<const float*>(sm + OFF_RS);
  uint64_t seed = p.seed;
  if (MODE == 0 && p.seed_ctr) seed += *p.seed_ctr;
  const float keep_scale = (MODE == 0 && p.p_drop > 0.f) ? 1.f / (1.f - p.p_drop) : 1.f;
  const __nv_bfloat16* resid = MODE == 0 ? p.x : p.addend;
  for (int t = 0; t < ntiles; ++t) {
    long r0; int rows, nt_;
    tile_range(p.R, cta, ncta, t, r0, rows, nt_);
    float acc[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) acc[i] = 0.f;
    mbar_wait(smem_addr(&a_full), t & 1);
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < 4; ++kb)
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma<D, 0, 0>(acc, make_desc(base + OFF_A + kb * 16384 + wg * 8192 + k * 32, 16, 1024),
                       make_desc(base + kb * 32768 + k * 32, 16, 1024));
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<D / 2>(acc);
    mbar_arrive(smem_addr(&a_empty));                // the A tile may be overwritten
    // fragment rows tr[h] (tile), h = 0/1: acc[4j + 2h], acc[4j + 2h + 1] are columns 8j + 2 (lane & 3) + {0, 1}
    int tr[2];
    bool live[2];
    long grow[2];
    float rs[2], sum[2] = {0.f, 0.f}, sq[2] = {0.f, 0.f};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      tr[h] = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
      live[h] = tr[h] < rows;
      grow[h] = r0 + tr[h];
      rs[h] = (MODE == 0 && live[h]) ? s_rs[(t & 3) * TM + tr[h]] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < D / 8; ++j) {
      const int c = 8 * j + 2 * q4;
      float2 bv = make_float2(0.f, 0.f), cv = make_float2(0.f, 0.f);
      if (MODE == 0) {
        bv = __ldg(reinterpret_cast<const float2*>(p.bias + c));
        cv = __ldg(reinterpret_cast<const float2*>(p.c1 + c));
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float2 hv = make_float2(0.f, 0.f);
        if (live[h] && resid != nullptr) hv = __bfloat1622float2(__ldg(reinterpret_cast<const __nv_bfloat162*>(resid + grow[h] * D + c)));
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (MODE == 0) {
          v0 = fmaf(rs[h], cv.x, v0 + bv.x);
          v1 = fmaf(rs[h], cv.y, v1 + bv.y);
          // Z is stored as bf16 and the LayerNorm backward recomputes from the stored value: normalise the same value
          const __nv_bfloat162 zb = __floats2bfloat162_rn(v0, v1);
          if (live[h]) *reinterpret_cast<__nv_bfloat162*>(p.z + grow[h] * D + c) = zb;
          const float2 zf = __bfloat1622float2(zb);
          v0 = zf.x; v1 = zf.y;
          if (p.p_drop > 0.f) {
            const uint32_t m = dropout_keep8(seed, p.stream_id, (uint64_t)grow[h] * 32 + j, p.p_drop) >> (2 * q4);
            v0 = (m & 1) ? v0 * keep_scale : 0.f;
            v1 = (m & 2) ? v1 * keep_scale : 0.f;
          }
          v0 += hv.x; v1 += hv.y;
          acc[4 * j + 2 * h] = v0; acc[4 * j + 2 * h + 1] = v1;   // y stays in registers for the normalisation pass
          sum[h] += v0 + v1;
          sq[h] = fmaf(v0, v0, fmaf(v1, v1, sq[h]));
        } else if (live[h]) {
          *reinterpret_cast<__nv_bfloat162*>(p.y + grow[h] * D + c) = __floats2bfloat162_rn(v0 + hv.x, v1 + hv.y);
        }
      }
    }
    if (MODE == 0) {
      float mean[2], rstd[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 1);
        sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 2);
        sq[h] += __shfl_xor_sync(0xffffffffu, sq[h], 1);
        sq[h] += __shfl_xor_sync(0xffffffffu, sq[h], 2);
        mean[h] = sum[h] * (1.f / D);
        const float var = fmaxf(sq[h] * (1.f / D) - mean[h] * mean[h], 0.f);
        rstd[h] = rsqrtf(var + kLnEps);
        if (live[h] && q4 == 0 && p.mean) { p.mean[grow[h]] = mean[h]; p.rstd[grow[h]] = rstd[h]; }
      }
#pragma unroll
      for (int j = 0; j < D / 8; ++j) {
        const int c = 8 * j + 2 * q4;
        const float2 gv = __ldg(reinterpret_cast<const float2*>(p.gamma + c));
        const float2 bt = __ldg(reinterpret_cast<const float2*>(p.beta + c));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!live[h]) continue;
          const float o0 = fmaf((acc[4 * j + 2 * h] - mean[h]) * rstd[h], gv.x, bt.x);
          const float o1 = fmaf((acc[4 * j + 2 * h + 1] - mean[h]) * rstd[h], gv.y, bt.y);
          __nv_bfloat16* dst = grow[h] < p.split ? p.outA : p.outB;
          *reinterpret_cast<__nv_bfloat162*>(dst + grow[h] * D + c) = __floats2bfloat162_rn(o0, o1);
        }
      }
    }
  }
}

// ---------------------------------------------------------------- (graph, node)-ordered CSR -> buffer-order CSR
struct Segs { int B, n0, n1, n2; };
__device__ __forceinline__ long seg_row(const Segs& s, int b, int j) {
  if (j < s.n0) return (long)b * s.n0 + j;
  if (j < s.n0 + s.n1) return (long)s.B * s.n0 + (long)b * s.n1 + (j - s.n0);
  return (long)s.B * (s.n0 + s.n1) + (long)b * s.n2 + (j - s.n0 - s.n1);
}
__device__ __forceinline__ void seg_unrow(const Segs& s, long r, int& b, int& i) {
  const long e0 = (long)s.B * s.n0, e1 = e0 + (long)s.B * s.n1;
  if (r < e0) { b = (int)(r / s.n0); i = (int)(r % s.n0); }
  else if (r < e1) { long q = r - e0; b = (int)(q / s.n1); i = s.n0 + (int)(q % s.n1); }
  else { long q = r - e1; b = (int)(q / s.n2); i = s.n0 + s.n1 + (int)(q % s.n2); }
}

__global__ void rows_count_kernel(const int* __restrict__ rowptr, Segs s, int N, int* __restrict__ counts) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const long R = (long)s.B * N;
  for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < R; r += (long)gridDim.x * blockDim.x) {
    int b, i; seg_unrow(s, r, b, i);
    const long g = (long)b * N + i;
    counts[r] = rowptr[g + 1] - rowptr[g];
  }
}

// one 1024-thread CTA: exclusive scan of counts[0..n) -> out[0..n]
__global__ void rows_scan_kernel(const int* __restrict__ counts, int* __restrict__ out, long n) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ int warp_tot[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long b0 = 0; b0 < n; b0 += 1024) {
    const long i = b0 + threadIdx.x;
    const int v = i < n ? counts[i] : 0;
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
    const int excl = carry + (warp ? warp_tot[warp - 1] : 0) + x - v;
    if (i < n) out[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) out[n] = carry;
}

__global__ void rows_fill_kernel(const int* __restrict__ rowptr, const int* __restrict__ col, const float* __restrict__ val,
                                 Segs s, int N, const int* __restrict__ rowptr_g, int* __restrict__ col_g,
                                 float* __restrict__ val_g) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const long R = (long)s.B * N;
  const int lane = threadIdx.x & 31;
  for (long r = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < R; r += (long)gridDim.x * (blockDim.x >> 5)) {
    int b, i; seg_unrow(s, r, b, i);
    const long g = (long)b * N + i;
    const int e0 = rowptr[g], n = rowptr[g + 1] - e0, o0 = rowptr_g[r];
    for (int k = lane; k < n; k += 32) { col_g[o0 + k] = (int)seg_row(s, b, col[e0 + k]); val_g[o0 + k] = val[e0 + k]; }
  }
}

int launch_fused(int mode, const CUtensorMap& tm, const Params& p, cudaStream_t st) {
  static_assert(SMEM_BYTES + 1024 <= 227 * 1024, "fused GCN kernel: shared-memory budget");
  const size_t smem = SMEM_BYTES + 1024;
  cudaError_t e = mode == 0
      ? cudaFuncSetAttribute(gcn_fused_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
      : cudaFuncSetAttribute(gcn_fused_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { fira_set_error(FIRA_ERR_CUDA, "gcn_layer attr: %s", cudaGetErrorString(e)); return FIRA_ERR_CUDA; }
  long want = (p.R + 31) / 32;
  const int grid = (int)(want < fira_num_sms() ? (want < 1 ? 1 : want) : fira_num_sms());
  if (mode == 0) launch_k(gcn_fused_kernel<0>, dim3(grid), dim3(THREADS), smem, st, tm, p);
  else launch_k(gcn_fused_kernel<1>, dim3(grid), dim3(THREADS), smem, st, tm, p);
  return FIRA_OK;
}

}  // namespace

extern "C" {

int fira_csr_to_rows(const int* rowptr, const int* col, const float* val, int B, int n_code, int n_sub, int n_ast,
                     int* counts, int* rowptr_rows, int* col_rows, float* val_rows, void* stream) {
  FIRA_CHECK_ARG(rowptr && col && val && counts && rowptr_rows && col_rows && val_rows, FIRA_ERR_ARG, "csr_to_rows: null");
  FIRA_CHECK_ARG(B > 0 && n_code > 0 && n_sub >= 0 && n_ast >= 0, FIRA_ERR_SHAPE, "csr_to_rows: segments");
  Segs s{B, n_code, n_sub, n_ast};
  const int N = n_code + n_sub + n_ast;
  const long R = (long)B * N;
  cudaStream_t st = (cudaStream_t)stream;
  int grid = (int)((R + 255) / 256 < fira_num_sms() * 4 ? (R + 255) / 256 : fira_num_sms() * 4);
  launch_k(rows_count_kernel, dim3(grid), dim3(256), 0, st, rowptr, s, N, counts);
  launch_k(rows_scan_kernel, dim3(1), dim3(1024), 0, st, counts, rowptr_rows, R);
  grid = (int)((R + 7) / 8 < fira_num_sms() * 8 ? (R + 7) / 8 : fira_num_sms() * 8);
  launch_k(rows_fill_kernel, dim3(grid), dim3(256), 0, st, rowptr, col, val, s, N, rowptr_rows, col_rows, val_rows);
  FIRA_CHECK_LAUNCH("fira_csr_to_rows");
  return FIRA_OK;
}

int fira_gcn_layer_fwd(const int* rowptr_rows, const int* col_rows, const float* val_rows, const void* h,
                       const void* w_merged, const float* bias, const float* c1, const float* gamma, const float* beta,
                       void* z, void* outA, void* outB, long split, float* mean, float* rstd, long rows, int dim,
                       float p_drop, uint64_t seed, const uint64_t* seed_ctr, uint32_t stream_id, void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "gcn_layer_fwd: dim %d != 256", dim);
  FIRA_CHECK_ARG(rows > 0, FIRA_ERR_SHAPE, "gcn_layer_fwd: rows %ld", rows);
  FIRA_CHECK_ARG(rowptr_rows && col_rows && val_rows && h && w_merged && bias && c1 && gamma && beta && z && outA && outB,
                 FIRA_ERR_ARG, "gcn_layer_fwd: null argument");
  FIRA_CHECK_ARG(fira_aligned16(h) && fira_aligned16(w_merged) && fira_aligned16(z) && fira_aligned16(outA) &&
                     fira_aligned16(outB) && fira_aligned16(bias) && fira_aligned16(c1) && fira_aligned16(gamma) &&
                     fira_aligned16(beta), FIRA_ERR_ALIGN, "gcn_layer_fwd: 16-B alignment");
  FIRA_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f, FIRA_ERR_ARG, "gcn_layer_fwd: p_drop %f", p_drop);
  CUtensorMap tm;
  int rc = make_map_bf16(&tm, w_merged, D, D, D, 64, D, "gcn_layer_fwd");
  if (rc) return rc;
  Params p{};
  p.rowptr = rowptr_rows; p.col = col_rows; p.val = val_rows; p.x = (const __nv_bfloat16*)h; p.R = rows;
  p.bias = bias; p.c1 = c1; p.gamma = gamma; p.beta = beta;
  p.z = (__nv_bfloat16*)z; p.outA = (__nv_bfloat16*)outA; p.outB = (__nv_bfloat16*)outB; p.split = split;
  p.mean = mean; p.rstd = rstd; p.p_drop = p_drop; p.seed = seed; p.seed_ctr = seed_ctr; p.stream_id = stream_id;
  if ((rc = launch_fused(0, tm, p, (cudaStream_t)stream))) return rc;
  FIRA_CHECK_LAUNCH("fira_gcn_layer_fwd");
  return FIRA_OK;
}

int fira_gcn_layer_bwd(const int* rowptr_rows_t, const int* col_rows_t, const float* val_rows_t, const void* d_z,
                       const void* w_merged_t, const void* d_resid, void* agg_dz, void* d_h, long rows, int dim,
                       void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "gcn_layer_bwd: dim %d != 256", dim);
  FIRA_CHECK_ARG(rows > 0, FIRA_ERR_SHAPE, "gcn_layer_bwd: rows %ld", rows);
  FIRA_CHECK_ARG(rowptr_rows_t && col_rows_t && val_rows_t && d_z && w_merged_t && agg_dz && d_h, FIRA_ERR_ARG,
                 "gcn_layer_bwd: null argument");
  FIRA_CHECK_ARG(fira_aligned16(d_z) && fira_aligned16(w_merged_t) && fira_aligned16(d_resid) && fira_aligned16(agg_dz) &&
                     fira_aligned16(d_h), FIRA_ERR_ALIGN, "gcn_layer_bwd: 16-B alignment");
  CUtensorMap tm;
  int rc = make_map_bf16(&tm, w_merged_t, D, D, D, 64, D, "gcn_layer_bwd");
  if (rc) return rc;
  Params p{};
  p.rowptr = rowptr_rows_t; p.col = col_rows_t; p.val = val_rows_t; p.x = (const __nv_bfloat16*)d_z; p.R = rows;
  p.addend = (const __nv_bfloat16*)d_resid; p.agg_out = (__nv_bfloat16*)agg_dz; p.y = (__nv_bfloat16*)d_h;
  if ((rc = launch_fused(1, tm, p, (cudaStream_t)stream))) return rc;
  FIRA_CHECK_LAUNCH("fira_gcn_layer_bwd");
  return FIRA_OK;
}

}  // extern "C"
