// Linear + dropout + residual + LayerNorm in ONE launch (bf16 throughput mode), the block that closes every sub-layer of
// the model (gnn_transformer.py:83 GCN, :158-161 Attention, :173-174 FeedForward, :204-205 Combination):
//
//     z   = x W^T + bias (+ rs[m] * rc[n])                   [M, 256]   (stored: the backward recomputes from it)
//     out = LayerNorm(dropout_p(z) + resid) * gamma + beta               (rows < split -> outA[r], else outB[r])
//
// A 128-row tile owns whole 256-wide rows.  Pipeline: warps 0-7 = two consumer warpgroups (wgmma m64 x n256 x k16, fp32
// accumulator in registers, rows 0-63 / 64-127 of the tile), warp 8 = TMA producer (x and W k-blocks through a 3-stage
// ring, the residual tile in one go).  The epilogue works on the accumulator fragments in registers: a row's 256 columns
// are spread over the 4 threads of a lane quad, so the row statistics take two shuffles.  Two passes: (1) z -> bf16 ->
// staging boxes -> TMA store; y = dropout(z) + resid kept in the accumulator registers, row sum / sum of squares;
// (2) normalise, scale, -> staging boxes -> TMA store.  All global traffic of the epilogue is TMA (swizzled [64 x 64]
// boxes): no per-lane row stores.  Replaces fira_gemm_bf16_tc + fira_ln_residual_fwd (two launches, one round trip of
// z through L2) on the forward critical path.
#include <cuda.h>
#include <cudaTypedefs.h>
#include "tc_common.cuh"
#include "fira_b200.h"

namespace {

using namespace tc;

constexpr int BM = 128, BN = 256, BK = 64, STAGES = 3;
constexpr int N_CONSUMER = 256;                      // warps 0-7
constexpr int THREADS = N_CONSUMER + 32;             // + warp 8: TMA producer
constexpr uint32_t A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2, STAGE_BYTES = A_BYTES + B_BYTES;   // 16 KB + 32 KB
constexpr uint32_t RING_BYTES = STAGES * STAGE_BYTES;                                                // 144 KB
constexpr uint32_t RES_BYTES = BM * BN * 2;                                                          // 64 KB: 4 boxes [128 x 64]
constexpr uint32_t SMEM_BYTES = RING_BYTES + RES_BYTES + 1024;
constexpr uint32_t BOX = 64 * 64 * 2;                // one [64 rows x 64 cols] bf16 staging box
constexpr uint32_t OFF_OUT = 8 * BOX;                // z staging: ring [0, 64 KB), output staging: ring [64 KB, 128 KB)

struct LnParams {
  int M, K;
  long split;
  const float* bias; const float* rs; const float* rc; const float* gamma; const float* beta;
  float* mean; float* rstd;
  float p_drop; uint64_t seed; const uint64_t* seed_ctr; uint32_t stream_id;
  int has_b;
};

// 9 warps: 3 share an SM sub-partition's 16K registers -> <= 168 each, so the 128-register accumulator epilogue spills a
// little (ptxas -v: 584 B); the kernel is opt-in (FIRA_GEMM_LN) and has not been timed on the H100
__global__ void __launch_bounds__(THREADS, 1)
gemm_ln_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW,
               const __grid_constant__ CUtensorMap tmR, const __grid_constant__ CUtensorMap tmZ,
               const __grid_constant__ CUtensorMap tmOA, const __grid_constant__ CUtensorMap tmOB, LnParams p) {
  extern __shared__ unsigned char smem_dyn[];
  __shared__ __align__(8) unsigned long long full_bar[STAGES], empty_bar[STAGES], res_bar;
  __shared__ __align__(16) float s_bias[BN], s_rc[BN], s_gamma[BN], s_beta[BN];
  const uint32_t base = (smem_addr(smem_dyn) + 1023u) & ~1023u;
  unsigned char* sm = smem_dyn + (base - smem_addr(smem_dyn));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * BM;
  const int nkb = (p.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(smem_addr(&full_bar[s]), 1); mbar_init(smem_addr(&empty_bar[s]), N_CONSUMER); }
    mbar_init(smem_addr(&res_bar), 1);
    mbar_init_fence();
    tma_prefetch_desc(&tmX); tma_prefetch_desc(&tmW); tma_prefetch_desc(&tmR); tma_prefetch_desc(&tmZ);
    tma_prefetch_desc(&tmOA);
    if (p.has_b) tma_prefetch_desc(&tmOB);
  }
  __syncthreads();
  pdl_wait(); pdl_trigger();       // PDL: the prologue above overlapped the previous kernel's tail (common.cuh)

  if (warp == N_CONSUMER / 32) {
    // ===================== TMA producer: k-blocks of x and W, then the residual tile =====================
    if (lane == 0) {
      for (int i = 0; i < nkb; ++i) {
        const int s = i % STAGES;
        mbar_wait(smem_addr(&empty_bar[s]), ((i / STAGES) & 1) ^ 1);
        const uint32_t sa = base + s * STAGE_BYTES, sb = sa + A_BYTES, fb = smem_addr(&full_bar[s]);
        mbar_expect_tx(fb, STAGE_BYTES);
        const int kb = (i + (int)blockIdx.x) % nkb;                      // rotated k order: see gemm_tc.cu
        tma_load_2d(sa, &tmX, kb * BK, m0, fb);                          // box {64 k, 128 m}
        tma_load_2d(sb, &tmW, kb * BK, 0, fb);                           // box {64 k, 256 n}
        if (i == 0) {                                                    // residual rows: 4 boxes {64 cols, 128 rows}
          const uint32_t rb = smem_addr(&res_bar);
          mbar_expect_tx(rb, RES_BYTES);
#pragma unroll
          for (int g = 0; g < 4; ++g) tma_load_2d(base + RING_BYTES + g * 16384, &tmR, g * 64, m0, rb);
        }
      }
    }
    return;
  }

  // ===================== consumers: warpgroup wg = tile rows [64 wg, +64) =====================
  const int wg = warp >> 2;
  for (int c = threadIdx.x; c < BN; c += N_CONSUMER) {
    s_bias[c] = p.bias ? p.bias[c] : 0.f;
    s_rc[c] = p.rs ? p.rc[c] : 0.f;
    s_gamma[c] = p.gamma[c];
    s_beta[c] = p.beta[c];
  }
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  for (int i = 0; i < nkb; ++i) {
    const int s = i % STAGES;
    mbar_wait(smem_addr(&full_bar[s]), (i / STAGES) & 1);
    const uint32_t sa = base + s * STAGE_BYTES + wg * 8192, sb = base + s * STAGE_BYTES + A_BYTES;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) wgmma<BN, 0, 0>(acc, make_desc(sa + k * 32, 16, 1024), make_desc(sb + k * 32, 16, 1024));
    wgmma_commit();
    wgmma_wait<1>();
    if (i > 0) mbar_arrive(smem_addr(&empty_bar[(i - 1) % STAGES]));
  }
  wgmma_wait<0>();
  reg_fence<BN / 2>(acc);
  named_bar(1, N_CONSUMER);                          // both warpgroups are done with the ring: staging boxes live there now
  mbar_wait(smem_addr(&res_bar), 0);

  // fragment rows (tile) tr[h], h = 0/1: acc[4j + 2h], acc[4j + 2h + 1] are columns 8j + 2 (lane & 3) + {0, 1}
  const int q4 = lane & 3;
  int tr[2], br[2], m[2];
  float rsm[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    tr[h] = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    br[h] = tr[h] - wg * 64;                         // row inside this warpgroup's [64 x 64] staging boxes
    m[h] = m0 + tr[h];
    rsm[h] = (p.rs && m[h] < p.M) ? p.rs[m[h]] : 0.f;
  }
  uint64_t seed = p.seed;
  if (p.seed_ctr) seed += *p.seed_ctr;
  const float keep_scale = p.p_drop > 0.f ? 1.f / (1.f - p.p_drop) : 1.f;
  const unsigned char* res = sm + RING_BYTES;
  unsigned char* zst = sm + wg * 4 * BOX;
  unsigned char* ost = sm + OFF_OUT + wg * 4 * BOX;
  const int row0 = m0 + wg * 64;                     // first global row of this warpgroup
  float sum[2] = {0.f, 0.f}, sq[2] = {0.f, 0.f};
  // ---- pass 1: z (stored), y = dropout(z) + resid (kept in registers), row statistics
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int c = 8 * j + 2 * q4, g = j >> 3, chunk = j & 7;
    const float2 bb = *reinterpret_cast<const float2*>(s_bias + c), kk = *reinterpret_cast<const float2*>(s_rc + c);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float v0 = fmaf(rsm[h], kk.x, acc[4 * j + 2 * h] + bb.x), v1 = fmaf(rsm[h], kk.y, acc[4 * j + 2 * h + 1] + bb.y);
      // z is stored as bf16 and the LayerNorm backward recomputes from the stored value: normalise that value
      const __nv_bfloat162 zb = __floats2bfloat162_rn(v0, v1);
      *reinterpret_cast<__nv_bfloat162*>(zst + g * BOX + br[h] * 128 + ((chunk ^ (br[h] & 7)) << 4) + q4 * 4) = zb;
      const float2 zf = __bfloat1622float2(zb);
      v0 = zf.x; v1 = zf.y;
      if (p.p_drop > 0.f) {
        const uint32_t mk = dropout_keep8(seed, p.stream_id, (uint64_t)m[h] * 32 + j, p.p_drop) >> (2 * q4);
        v0 = (mk & 1) ? v0 * keep_scale : 0.f;
        v1 = (mk & 2) ? v1 * keep_scale : 0.f;
      }
      const float2 rf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(
          res + g * 16384 + tr[h] * 128 + ((chunk ^ (tr[h] & 7)) << 4) + q4 * 4));
      v0 += rf.x; v1 += rf.y;
      acc[4 * j + 2 * h] = v0; acc[4 * j + 2 * h + 1] = v1;
      sum[h] += v0 + v1;
      sq[h] = fmaf(v0, v0, fmaf(v1, v1, sq[h]));
    }
  }
  fence_proxy_async();
  named_bar(2 + wg, 128);
  if ((threadIdx.x & 127) == 0 && row0 < p.M) {
#pragma unroll
    for (int g = 0; g < 4; ++g) tma_store_2d(&tmZ, smem_addr(zst + g * BOX), g * 64, row0);
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  }
  float mean[2], rstd[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 1);
    sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 2);
    sq[h] += __shfl_xor_sync(0xffffffffu, sq[h], 1);
    sq[h] += __shfl_xor_sync(0xffffffffu, sq[h], 2);
    mean[h] = sum[h] * (1.f / BN);
    const float var = fmaxf(sq[h] * (1.f / BN) - mean[h] * mean[h], 0.f);
    rstd[h] = rsqrtf(var + kLnEps);
    if (q4 == 0 && m[h] < p.M) { p.mean[m[h]] = mean[h]; p.rstd[m[h]] = rstd[h]; }
  }
  // ---- pass 2: normalise, scale, store.  Rows below `split` go to outA[r], the others to outB[r].  Map A ends at
  // `split` (TMA clips the rest of a box that straddles it); map B covers all rows of outB and is written in 32-row
  // slabs, so the one straddling slab also writes its rows below `split` into outB -- storage the callers leave unused
  // (see fira_b200.h).
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int c = 8 * j + 2 * q4, g = j >> 3, chunk = j & 7;
    const float2 gg = *reinterpret_cast<const float2*>(s_gamma + c), ee = *reinterpret_cast<const float2*>(s_beta + c);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float o0 = fmaf((acc[4 * j + 2 * h] - mean[h]) * rstd[h], gg.x, ee.x);
      const float o1 = fmaf((acc[4 * j + 2 * h + 1] - mean[h]) * rstd[h], gg.y, ee.y);
      *reinterpret_cast<__nv_bfloat162*>(ost + g * BOX + br[h] * 128 + ((chunk ^ (br[h] & 7)) << 4) + q4 * 4) =
          __floats2bfloat162_rn(o0, o1);
    }
  }
  fence_proxy_async();
  named_bar(2 + wg, 128);
  if ((threadIdx.x & 127) == 0) {
    if (row0 < p.M) {
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        if (row0 < p.split) tma_store_2d(&tmOA, smem_addr(ost + g * BOX), g * 64, row0);
        // outB in [32 x 64] halves of the box: only the 32-row slab that straddles `split` writes rows below it
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
          if (p.has_b && row0 + 32 * hh < p.M && row0 + 32 * hh + 32 > p.split)
            tma_store_2d(&tmOB, smem_addr(ost + g * BOX + hh * 4096), g * 64, row0 + 32 * hh);
      }
    }
    tma_store_commit_wait_read();                    // the staging boxes must stay valid until TMA has read them
  }
}

}  // namespace

extern "C" int fira_gemm_ln_fwd(const void* x, long ldx, const void* w, const float* bias, const float* rs, const float* rc,
                                const void* resid, const float* gamma, const float* beta, void* z, void* outA, void* outB,
                                long split, float* mean, float* rstd, long rows, int K, float p_drop, uint64_t seed,
                                const uint64_t* seed_ctr, uint32_t stream_id, void* stream) {
  FIRA_CHECK_ARG(x && w && resid && gamma && beta && z && outA && mean && rstd, FIRA_ERR_ARG, "gemm_ln_fwd: null argument");
  FIRA_CHECK_ARG(rows > 0 && rows < (1L << 31) && K > 0 && K % 8 == 0, FIRA_ERR_SHAPE, "gemm_ln_fwd: rows %ld K %d", rows, K);
  FIRA_CHECK_ARG(ldx % 8 == 0, FIRA_ERR_ALIGN, "gemm_ln_fwd: ldx must be a multiple of 8");
  FIRA_CHECK_ARG(fira_aligned16(x) && fira_aligned16(w) && fira_aligned16(resid) && fira_aligned16(z) && fira_aligned16(outA) &&
                     fira_aligned16(outB), FIRA_ERR_ALIGN, "gemm_ln_fwd: 16-B alignment");
  FIRA_CHECK_ARG((rs == nullptr) == (rc == nullptr), FIRA_ERR_ARG, "gemm_ln_fwd: rs/rc must come together");
  FIRA_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f, FIRA_ERR_ARG, "gemm_ln_fwd: p_drop %f", p_drop);
  if (split > rows || outB == nullptr) split = rows;
  FIRA_CHECK_ARG(split >= 0, FIRA_ERR_ARG, "gemm_ln_fwd: split %ld", split);
  const int M = (int)rows;
  CUtensorMap tx, tw, tr, tz, toa, tob;
  int rc_;
  if ((rc_ = make_map_bf16(&tx, x, M, K, ldx, BK, BM, "gemm_ln_fwd"))) return rc_;
  if ((rc_ = make_map_bf16(&tw, w, BN, K, K, BK, BN, "gemm_ln_fwd"))) return rc_;
  if ((rc_ = make_map_bf16(&tr, resid, M, BN, BN, 64, BM, "gemm_ln_fwd"))) return rc_;
  if ((rc_ = make_map_bf16(&tz, z, M, BN, BN, 64, 64, "gemm_ln_fwd"))) return rc_;
  const bool has_a = split > 0, has_b = split < rows;
  // map A: rows [0, split) of outA; map B: all rows of outB (indexed by the global row; only slabs reaching `split` or
  // beyond are stored through it)
  if ((rc_ = make_map_bf16(&toa, outA, has_a ? split : 1, BN, BN, 64, 64, "gemm_ln_fwd"))) return rc_;
  tob = toa;
  if (has_b && (rc_ = make_map_bf16(&tob, outB, rows, BN, BN, 64, 32, "gemm_ln_fwd"))) return rc_;
  LnParams p{M, K, has_a ? split : 0, bias, rs, rc, gamma, beta, mean, rstd, p_drop, seed, seed_ctr, stream_id, has_b ? 1 : 0};
  cudaError_t e = cudaFuncSetAttribute(gemm_ln_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES);
  if (e != cudaSuccess) { fira_set_error(FIRA_ERR_CUDA, "gemm_ln attr: %s", cudaGetErrorString(e)); return FIRA_ERR_CUDA; }
  launch_k(gemm_ln_kernel, dim3((M + BM - 1) / BM), dim3(THREADS), SMEM_BYTES, (cudaStream_t)stream, tx, tw, tr, tz, toa, tob, p);
  FIRA_CHECK_LAUNCH("fira_gemm_ln_fwd");
  return FIRA_OK;
}
