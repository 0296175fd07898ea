// bf16 tensor-core GEMM for the throughput path: wgmma.mma_async (SASS HGMMA) with the fp32 accumulator in
// registers, operands staged in shared memory by TMA (cp.async.bulk.tensor, SASS UTMALDG) through a 2-4 stage mbarrier
// ring, warp-specialised: warps 0-7 = two consumer warpgroups (rows 0-63 / 64-127 of the tile: wgmma issue, then the
// epilogue), warp 8 = TMA producer.  One 128 x BN output tile per CTA.
//
//   C[M,N] = A (M x K) * B (K x N) + bias[n] + rs[m]*rc[n]      (optional relu; fp32 or bf16 output)
//
// Operand storage (bf16, row-major, leading dimension a multiple of 8 elements):
//   a_kmajor = 1 : A[m*lda + k]   (activations as they are)        a_kmajor = 0 : A[k*lda + m]  (dY^T, X^T)
//   b_kmajor = 1 : B[n*ldb + k]   (nn.Linear weight [out,in])      b_kmajor = 0 : B[k*ldb + n]
// The MN-major forms let the weight-gradient GEMM dW = dY^T X read dY and X in place (no transpose
// pass): TMA fetches [64 k-rows x 64 mn] boxes and the wgmma descriptor carries the MN-major
// canonical SWIZZLE_128B layout (transpose bits of the instruction).
// splits > 1: split-K across blockIdx.z, fp32 partials atomically added into a zero-filled C.
#include <cuda.h>
#include <cudaTypedefs.h>
#include <atomic>
#include <stdlib.h>
#include "tc_common.cuh"
#include "fira_b200.h"

namespace {

using namespace tc;

constexpr int BM = 128;          // two m64 warpgroups
constexpr int BK = 64;           // 64 bf16 = 128 B = one SWIZZLE_128B atom row
constexpr int N_CONSUMER = 256;  // warps 0-7
constexpr int NUM_THREADS = N_CONSUMER + 32;   // + warp 8: TMA producer
constexpr int CONSUMER_BAR = 1;  // named barrier of the consumer warps

struct TcParams {
  void* C; long ldc; int c_is_bf16;
  int M, N, K;
  const float* bias; const float* rs; const float* rc;
  int relu; int accumulate;
  int splits; int kblocks_per_split;
  int a_kmajor, b_kmajor;
  int rotate;                  // CTAs start their k loop at different k-blocks (see the producer)
  int tma_store;               // bf16 output written by TMA (cp.async.bulk.tensor store) from a swizzled staging tile
  const __nv_bfloat16* relu_mask;  // optional (TMA-store path): C[m,n] = relu_mask[m*ldc+n] > 0 ? value : 0 (relu backward)
  float* colsum;               // optional (MN-major A only): colsum[m] += sum_k A(m, k) -- the bias gradient of a wgrad product
  unsigned long long* probe;   // debugging aid (fira_debug_set_probe): CTA (0,0,0) stamps %globaltimer at its phase boundaries
};

std::atomic<unsigned long long*> g_probe{nullptr};

__device__ __forceinline__ void stamp(const TcParams& p, int slot) {
  if (p.probe && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    p.probe[slot] = t;
  }
}

// Mainloop of one consumer warpgroup: wait for a stage, 4 x wgmma m64 x BN x k16 on it, fold the A column sums in while
// they run, hand the previous stage back.  TA / TB = 1: A / B MN-major (the transpose bits are immediates of the
// instruction, so each operand-major combination is its own instantiation).
template <int BN, int STAGES, int TA, int TB>
__device__ __forceinline__ void mainloop(float* acc, float& cs, bool do_cs, int nkb, uint32_t base, const unsigned char* sm,
                                         unsigned long long* full_bar, unsigned long long* empty_bar, int wg, const TcParams& p) {
  constexpr uint32_t A_BYTES = BM * BK * 2, STAGE_BYTES = A_BYTES + BN * BK * 2;
  // column sums (MN-major A, [m/64][64 k][64 m] panels): thread <-> m column (t & 63) of its warpgroup's panel, half of k
  const int cs_m = threadIdx.x & 63, cs_k0 = ((threadIdx.x >> 6) & 1) * 32;
  for (int i = 0; i < nkb; ++i) {
    const int s = i % STAGES;
    mbar_wait(smem_addr(&full_bar[s]), (i / STAGES) & 1);
    if (i == 0 && threadIdx.x == 0) stamp(p, 4);     // first operand stage landed
    const uint32_t sa = base + s * STAGE_BYTES + wg * 8192, sb = base + s * STAGE_BYTES + A_BYTES;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
      // K-major: step 16 k = 32 B inside the 128-B swizzle row; MN-major: step 16 k-rows = 2048 B
      const uint64_t da = TA ? make_desc(sa + k * 2048, 8192, 1024) : make_desc(sa + k * 32, 16, 1024);
      const uint64_t db = TB ? make_desc(sb + k * 2048, 8192, 1024) : make_desc(sb + k * 32, 16, 1024);
      wgmma<BN, TA, TB>(acc, da, db);
    }
    wgmma_commit();
    if (do_cs) {
      const unsigned char* a = sm + (size_t)s * STAGE_BYTES + wg * 8192 + (cs_m & 7) * 2;
#pragma unroll 8
      for (int k = cs_k0; k < cs_k0 + 32; ++k)
        cs += __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(a + (k >> 3) * 1024 + (k & 7) * 128 + (((cs_m >> 3) ^ (k & 7)) << 4)));
    }
    wgmma_wait<1>();                                 // the previous stage's wgmma are complete: hand it back
    if (i > 0) mbar_arrive(smem_addr(&empty_bar[(i - 1) % STAGES]));
  }
  wgmma_wait<0>();
  reg_fence<BN / 2>(acc);
}

template <int BN, int STAGES>
__host__ __device__ constexpr uint32_t acc_region_bytes() {
  constexpr uint32_t ring = STAGES * (BM * BK * 2 + BN * BK * 2), acc = BM * (BN + 4) * 4;
  return ring > acc ? ring : acc;
}

// Stage layout in shared memory (1024-B aligned, SWIZZLE_128B):
//   K-major operand  : [rows][64 k]          rows x 128 B, 8-row groups 1024 B apart (SBO = 1024)
//   MN-major operand : [mn/64][64 k][64 mn]  each 64-mn panel is 64 k-rows x 128 B = 8 KB (LBO = 8192 between
//                      panels, SBO = 1024 between 8-k groups); one TMA box per panel.
// Once the last k-block has been consumed, the ring holds the fp32 accumulator tile [128][BN + 4] (row pitch + 16 B:
// conflict-free 16-byte reads with lane = row); the TMA-store staging boxes follow the ring.
template <int BN, int STAGES>
__global__ void __launch_bounds__(NUM_THREADS, BN == 256 ? 1 : 2)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmC, TcParams p) {
  extern __shared__ unsigned char smem_dyn[];
  __shared__ __align__(16) float s_bias[BN], s_rc[BN];   // per-column epilogue constants of this tile (TMA-store path)
  constexpr uint32_t A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2, STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int PITCH = BN + 4;                                        // floats per row of the accumulator tile
  __shared__ __align__(8) unsigned long long full_bar[STAGES], empty_bar[STAGES];

  const uint32_t base = (smem_addr(smem_dyn) + 1023u) & ~1023u;
  unsigned char* sm = smem_dyn + (base - smem_addr(smem_dyn));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kb_total = (p.K + BK - 1) / BK;
  const int kb_begin = blockIdx.z * p.kblocks_per_split;
  const int kb_end = min(kb_total, kb_begin + p.kblocks_per_split);
  const int nkb = kb_end - kb_begin;
  if (threadIdx.x == 0) stamp(p, 0);                 // kernel entry

  // bias gradient folded into the weight-gradient product: the CTAs of the first column tile also sum the A tile
  // (= dY^T) over k as it passes through shared memory, while the wgmma of the stage runs
  const bool do_cs = p.colsum != nullptr && blockIdx.x == 0;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(smem_addr(&full_bar[s]), 1); mbar_init(smem_addr(&empty_bar[s]), N_CONSUMER); }
    mbar_init_fence();
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (p.tma_store) tma_prefetch_desc(&tmC);
  }
  __syncthreads();
  if (threadIdx.x == 0) stamp(p, 1);                 // prologue done (barriers)
  pdl_wait(); pdl_trigger();       // PDL: the prologue above overlapped the previous kernel's tail (common.cuh)
  if (threadIdx.x == 0) stamp(p, 2);                 // previous kernel complete

  if (warp == N_CONSUMER / 32) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      for (int i = 0; i < nkb; ++i) {
        const int s = i % STAGES;
        const uint32_t ph = (i / STAGES) & 1;
        mbar_wait(smem_addr(&empty_bar[s]), ph ^ 1);
        const uint32_t sa = base + s * STAGE_BYTES, sb = sa + A_BYTES;
        const uint32_t fb = smem_addr(&full_bar[s]);
        mbar_expect_tx(fb, STAGE_BYTES);
        // The CTAs of one tile row all read the same A tile and those of one tile column the same B tile, at the same
        // moment.  Rotating the k-block order by the tile coordinates makes the sharers ask for different L2 lines at
        // any one time; the fp32 sum over k-blocks is order-independent up to rounding.
        const int kb = p.rotate ? kb_begin + (i + (int)(blockIdx.x + blockIdx.y)) % nkb : kb_begin + i;
        const int k0 = kb * BK;
        if (p.a_kmajor) {
          tma_load_2d(sa, &tmA, k0, m0, fb);                        // box {64 k, 128 m}
        } else {
          tma_load_2d(sa, &tmA, m0, k0, fb);                        // two boxes {64 m, 64 k}
          tma_load_2d(sa + 8192, &tmA, m0 + 64, k0, fb);
        }
        if (p.b_kmajor) {
          tma_load_2d(sb, &tmB, k0, n0, fb);                        // box {64 k, BN n}
        } else {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, &tmB, n0 + j * 64, k0, fb);
        }
      }
      stamp(p, 3);                                   // every TMA load issued
    }
    return;
  }

  // ===================== consumers: warpgroup wg owns rows [64 wg, +64) of the tile =====================
  const int wg = warp >> 2;
  if (p.tma_store) {                                 // per-column constants -> shared memory
    for (int c = threadIdx.x; c < BN; c += N_CONSUMER) {
      const int n = n0 + c;
      s_bias[c] = (p.bias && n < p.N) ? p.bias[n] : 0.f;
      s_rc[c] = (p.rs && n < p.N) ? p.rc[n] : 0.f;
    }
  }
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  float cs = 0.f;
  if (p.a_kmajor) {
    if (p.b_kmajor) mainloop<BN, STAGES, 0, 0>(acc, cs, do_cs, nkb, base, sm, full_bar, empty_bar, wg, p);
    else mainloop<BN, STAGES, 0, 1>(acc, cs, do_cs, nkb, base, sm, full_bar, empty_bar, wg, p);
  } else {
    if (p.b_kmajor) mainloop<BN, STAGES, 1, 0>(acc, cs, do_cs, nkb, base, sm, full_bar, empty_bar, wg, p);
    else mainloop<BN, STAGES, 1, 1>(acc, cs, do_cs, nkb, base, sm, full_bar, empty_bar, wg, p);
  }
  if (threadIdx.x == 0) stamp(p, 5);                 // every wgmma complete
  if (do_cs && m0 + wg * 64 + (threadIdx.x & 63) < p.M) atomicAdd(p.colsum + m0 + wg * 64 + (threadIdx.x & 63), cs);
  named_bar(CONSUMER_BAR, N_CONSUMER);               // both warpgroups are done with the ring: it becomes the accumulator tile
  float* accs = reinterpret_cast<float*>(sm);
  {
    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      *reinterpret_cast<float2*>(accs + (size_t)r * PITCH + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(accs + (size_t)(r + 8) * PITCH + 8 * j + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  named_bar(CONSUMER_BAR, N_CONSUMER);

  // ===================== epilogue: smem tile (lane = row) -> global (lane = column) =====================
  // warp -> 32 rows (quarter) and every other 64 / HB column group (colhalf).  Stores go out with lanes across the
  // columns of a row: contiguous 256-512 B (bf16) / 512 B-1 KB (fp32) per store; bias / rank-1 / relu / accumulate /
  // split-K atomics are applied on the way out with per-lane column constants.
  const int quarter = warp & 3, colhalf = warp >> 2;
  constexpr int HB = BN < 128 ? BN : 128;           // columns per pass
  constexpr int LPR = HB / 8;                       // lanes per row on the way out (8 columns per lane)
  constexpr int RPI = 32 / LPR;                     // rows per store iteration
  const int mrow0 = m0 + quarter * 32;
  auto ld32 = [&](int c0, uint32_t* r) {            // this lane's row, 32 consecutive accumulator columns
    const float* src = accs + (size_t)(quarter * 32 + lane) * PITCH + c0;
#pragma unroll
    for (int j = 0; j < 32; j += 4) *reinterpret_cast<uint4*>(r + j) = *reinterpret_cast<const uint4*>(src + j);
  };
  if (p.tma_store) {
    // ---- bf16 output through TMA: each warp converts its 32 rows, 64 columns at a time, into a [32 x 64] bf16 box in
    // the SWIZZLE_128B layout (conflict-free 16-byte st.shared: lane = row, chunk slot = chunk ^ (row & 7)) and one
    // elected lane hands the box to the TMA engine; rows past M and columns past N8 = N rounded down to 8 are clipped by
    // the tensor map (it ends on a 16-byte boundary: a map ending inside a 16-byte chunk lets the store write the rest
    // of that chunk, i.e. columns of C past N).  Columns [N8, N) go out as plain stores from the staging box.
    unsigned char* cst = sm + acc_region_bytes<BN, STAGES>() + (size_t)quarter * (BN / 64) * 4096;
    const int m = mrow0 + lane;
    const int n8 = p.N & ~7;
    const float rsm = (p.rs && m < p.M) ? p.rs[m] : 0.f;
    if (warp == 0 && lane == 0) stamp(p, 6);
    const __nv_bfloat16* mrow = nullptr;            // relu-backward mask: this lane's row of the forward activations
    if (p.relu_mask && m < p.M) {
      mrow = p.relu_mask + (long)m * p.ldc + n0;
      for (int g = colhalf; g < BN / 64; g += 2)
        if (n0 + g * 64 < p.N) asm volatile("prefetch.global.L2 [%0];" ::"l"(mrow + g * 64));
    }
#pragma unroll 1
    for (int g = colhalf; g < BN / 64; g += 2) {
      const int gc = n0 + g * 64;                   // first column of the box
      uint4 mk[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) mk[j] = make_uint4(0x3f803f80u, 0x3f803f80u, 0x3f803f80u, 0x3f803f80u);   // 1.0: keep
      if (mrow != nullptr && n0 + g * 64 + 63 < p.N) {
#pragma unroll
        for (int j = 0; j < 8; ++j) mk[j] = *reinterpret_cast<const uint4*>(mrow + g * 64 + j * 8);
      } else if (mrow != nullptr) {
        __nv_bfloat16* me = reinterpret_cast<__nv_bfloat16*>(mk);
        for (int j = 0; j < 64; ++j) if (n0 + g * 64 + j < p.N) me[j] = mrow[g * 64 + j];
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        uint32_t r[32];
        const int c0 = g * 64 + h * 32;
        ld32(c0, r);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          float v[8];
          const float4 b0 = *reinterpret_cast<const float4*>(s_bias + c0 + q * 8), b1 = *reinterpret_cast<const float4*>(s_bias + c0 + q * 8 + 4);
          const float4 k0 = *reinterpret_cast<const float4*>(s_rc + c0 + q * 8), k1 = *reinterpret_cast<const float4*>(s_rc + c0 + q * 8 + 4);
          const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
          const float kk[8] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y, k1.z, k1.w};
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            v[j] = fmaf(rsm, kk[j], __uint_as_float(r[q * 8 + j]) + bb[j]);
            if (p.relu) v[j] = fmaxf(v[j], 0.f);
          }
          {
            const __nv_bfloat162* mp = reinterpret_cast<const __nv_bfloat162*>(&mk[h * 4 + q]);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float2 f = __bfloat1622float2(mp[j]);
              if (!(f.x > 0.f)) v[2 * j] = 0.f;
              if (!(f.y > 0.f)) v[2 * j + 1] = 0.f;
            }
          }
          uint4 o;
          __nv_bfloat162* hp = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
          for (int j = 0; j < 4; ++j) hp[j] = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
          const int chunk = h * 4 + q;
          *reinterpret_cast<uint4*>(cst + g * 4096 + lane * 128 + ((chunk ^ (lane & 7)) << 4)) = o;
        }
      }
      if (n8 < p.N && gc <= n8 && n8 < gc + 64 && m < p.M) {
        // columns [N8, N) lie in one 16-byte chunk of this lane's staged row: copy them out of the staging box
        const int ch = (n8 - gc) >> 3;
        const __nv_bfloat16* src = reinterpret_cast<const __nv_bfloat16*>(cst + g * 4096 + lane * 128 + ((ch ^ (lane & 7)) << 4));
        __nv_bfloat16* dst = (__nv_bfloat16*)p.C + (long)m * p.ldc + n8;
        for (int e = 0; e < p.N - n8; ++e) dst[e] = src[e];
      }
      fence_proxy_async();
      __syncwarp();
      if (lane == 0 && gc < n8 && mrow0 < p.M) tma_store_2d(&tmC, smem_addr(cst + g * 4096), n0 + g * 64, mrow0);
    }
    if (lane == 0) tma_store_commit_wait_read();
    __syncwarp();
  } else {
    if (warp == 0 && lane == 0) stamp(p, 6);         // accumulator visible to the epilogue
    const bool first = blockIdx.z == 0;
#pragma unroll 1
    for (int hb = colhalf * HB; hb < BN; hb += 2 * HB) {
      const float* stg = accs + (size_t)(quarter * 32) * PITCH + hb;
      if (p.splits > 1) {
        // split-K partials: 16-byte vector reductions (red.global.add.v4.f32, sm_90+): a lane owns 4 consecutive
        // columns, so a row of the 128-column pass is ONE warp instruction instead of four
        const bool vec = (p.ldc & 3) == 0;
        for (int rr = 0; rr < 32; ++rr) {
          const int m = mrow0 + rr;
          if (m >= p.M) break;
          const float rsm = (p.rs && first) ? p.rs[m] : 0.f;
          float* crow = (float*)p.C + (long)m * p.ldc;
#pragma unroll
          for (int jg = 0; jg < HB / 128 + (HB % 128 ? 1 : 0); ++jg) {
            const int c = jg * 128 + lane * 4;
            const int n = n0 + hb + c;
            if (c + 3 < HB && n < p.N) {
              float4 x = *reinterpret_cast<const float4*>(stg + (size_t)rr * PITCH + c);
              float* xv = reinterpret_cast<float*>(&x);
              if (first) {
#pragma unroll
                for (int j = 0; j < 4; ++j)
                  if (n + j < p.N) {
                    if (p.bias) xv[j] += p.bias[n + j];
                    if (p.rs) xv[j] = fmaf(rsm, p.rc[n + j], xv[j]);
                  }
              }
              if (vec && n + 3 < p.N) {
                atomicAdd(reinterpret_cast<float4*>(crow + n), x);
              } else {
#pragma unroll
                for (int j = 0; j < 4; ++j)
                  if (n + j < p.N) atomicAdd(crow + n + j, xv[j]);
              }
            }
          }
        }
      } else {
        const int col = (lane % LPR) * 8;
        const int n = n0 + hb + col;
        float bv[8], rcv[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          bv[j] = (p.bias && first && n + j < p.N) ? p.bias[n + j] : 0.f;
          rcv[j] = (p.rs && first && n + j < p.N) ? p.rc[n + j] : 0.f;
        }
        const bool full = n + 7 < p.N;
        for (int it = 0; it < 32 / RPI; ++it) {
          const int rr = it * RPI + lane / LPR;
          const int m = mrow0 + rr;
          if (m >= p.M) continue;
          const float rsm = (p.rs && first) ? p.rs[m] : 0.f;
          float v[8];
          const float4 x0 = *reinterpret_cast<const float4*>(stg + (size_t)rr * PITCH + col);
          const float4 x1 = *reinterpret_cast<const float4*>(stg + (size_t)rr * PITCH + col + 4);
          v[0] = x0.x; v[1] = x0.y; v[2] = x0.z; v[3] = x0.w; v[4] = x1.x; v[5] = x1.y; v[6] = x1.z; v[7] = x1.w;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            v[j] = fmaf(rsm, rcv[j], v[j] + bv[j]);
            if (p.relu) v[j] = fmaxf(v[j], 0.f);
          }
          if (p.c_is_bf16) {
            __nv_bfloat16* cp = (__nv_bfloat16*)p.C + (long)m * p.ldc + n;
            if (full && ((p.ldc & 7) == 0)) {
              if (p.accumulate) {
                float old[8];
                Act<__nv_bfloat16>::load8(cp, old);
#pragma unroll
                for (int j = 0; j < 8; ++j) v[j] += old[j];
              }
              Act<__nv_bfloat16>::store8(cp, v);
            } else {
#pragma unroll
              for (int j = 0; j < 8; ++j)
                if (n + j < p.N) cp[j] = __float2bfloat16_rn(p.accumulate ? v[j] + __bfloat162float(cp[j]) : v[j]);
            }
          } else {
            float* cp = (float*)p.C + (long)m * p.ldc + n;
            if (full && ((p.ldc & 3) == 0)) {
              if (p.accumulate) {
                float old[8];
                Act<float>::load8(cp, old);
#pragma unroll
                for (int j = 0; j < 8; ++j) v[j] += old[j];
              }
              Act<float>::store8(cp, v);
            } else {
#pragma unroll
              for (int j = 0; j < 8; ++j) if (n + j < p.N) cp[j] = p.accumulate ? cp[j] + v[j] : v[j];
            }
          }
        }
      }
    }
  }
  if (warp == 0 && lane == 0) stamp(p, 7);           // this warp's stores issued
  if (threadIdx.x == 0) stamp(p, 8);                 // exit
}

// ---------------------------------------------------------------- host side
bool tma_store_on() {          // FIRA_GEMM_TMA_STORE=0: A/B switch back to the register / shared-memory epilogue
  static const bool on = [] { const char* e = getenv("FIRA_GEMM_TMA_STORE"); return !(e && e[0] == '0'); }();
  return on;
}

bool rotate_on() {             // FIRA_GEMM_ROTATE=0: every CTA walks k in the same order
  static const bool on = [] { const char* e = getenv("FIRA_GEMM_ROTATE"); return !(e && e[0] == '0'); }();
  return on;
}

int make_map(CUtensorMap* map, const void* ptr, long rows, long cols, long ld, int box_cols, int box_rows) {
  return make_map_bf16(map, ptr, rows, cols, ld, box_cols, box_rows, "gemm_tc");
}

template <int BN, int STAGES>
int launch_cfg(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const TcParams& p, cudaStream_t st) {
  // ring / accumulator tile, then the TMA-store staging boxes ([4 x 32 rows] x BN bf16), + 1 KB for the alignment
  constexpr size_t smem = acc_region_bytes<BN, STAGES>() + (size_t)BN * 256 + 1024;
  static_assert(smem + 2 * BN * 4 + 2 * STAGES * 8 <= 227 * 1024, "gemm_tc: shared-memory budget");
  // per launch, not cached in a static: the attribute is per device, and a static flag would be shared state
  cudaError_t e = cudaFuncSetAttribute(gemm_tc_kernel<BN, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { fira_set_error(FIRA_ERR_CUDA, "gemm_tc attr: %s", cudaGetErrorString(e)); return FIRA_ERR_CUDA; }
  dim3 grid((p.N + BN - 1) / BN, (p.M + BM - 1) / BM, p.splits);
  launch_k(gemm_tc_kernel<BN, STAGES>, dim3(grid), dim3(NUM_THREADS), smem, st, ta, tb, tc, p);
  return FIRA_OK;
}

// Two launch shapes per tile width:
//   more CTAs than SMs -> shallow ring, TWO CTAs per SM where the tile allows it (BN <= 128): one CTA's epilogue
//                         overlaps the other's TMA / wgmma phase;
//   at most one wave   -> 4-stage ring (3 for BN = 256: the fp32 accumulator tile and the staging boxes must fit too),
//                         one CTA per SM: the k-blocks of a K = 256 product are in flight at once, which is what the
//                         latency-bound 15-105 CTA launches of the decoder need.
template <int BN>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const TcParams& p, cudaStream_t st) {
  const long ctas = (long)((p.N + BN - 1) / BN) * ((p.M + BM - 1) / BM) * p.splits;
  if constexpr (BN == 256) {
    return launch_cfg<BN, 3>(ta, tb, tc, p, st);
  } else {
    if (ctas > fira_num_sms()) return launch_cfg<BN, (BN == 128 ? 2 : 3)>(ta, tb, tc, p, st);
    return launch_cfg<BN, 4>(ta, tb, tc, p, st);
  }
}

}  // namespace

// debugging aid: `probe` = device buffer of >= 16 uint64 (or NULL to switch off); the next fira_gemm_bf16_tc launches make
// CTA (0,0,0) write %globaltimer at: 0 entry, 1 prologue done, 2 previous kernel complete (PDL wait), 3 TMA loads issued,
// 4 first stage landed, 5 MMAs issued, 6 accumulator visible to the epilogue, 7 epilogue stores issued, 8 exit
extern "C" int fira_debug_set_probe(void* probe) {
  g_probe.store((unsigned long long*)probe, std::memory_order_relaxed);
  return FIRA_OK;
}

namespace {
int gemm_tc_impl(const void* A, long lda, int a_kmajor, const void* B, long ldb, int b_kmajor, void* C, long ldc,
                 int c_is_bf16, int M, int N, int K, const float* bias, const float* rs, const float* rc, int relu,
                 int accumulate, int splits, float* colsum, void* stream, const void* relu_mask = nullptr) {
  FIRA_CHECK_ARG(A && B && C, FIRA_ERR_ARG, "gemm_bf16_tc: null operand");
  FIRA_CHECK_ARG(M > 0 && N > 0 && K > 0, FIRA_ERR_SHAPE, "gemm_bf16_tc: M=%d N=%d K=%d", M, N, K);
  FIRA_CHECK_ARG((lda % 8) == 0 && (ldb % 8) == 0, FIRA_ERR_ALIGN, "gemm_bf16_tc: lda/ldb must be multiples of 8");
  FIRA_CHECK_ARG(fira_aligned16(A) && fira_aligned16(B) && fira_aligned16(C), FIRA_ERR_ALIGN, "gemm_bf16_tc: 16-B alignment");
  FIRA_CHECK_ARG((rs == nullptr) == (rc == nullptr), FIRA_ERR_ARG, "gemm_bf16_tc: rs/rc must come together");
  FIRA_CHECK_ARG(!(splits > 1 && (c_is_bf16 || relu)), FIRA_ERR_ARG, "gemm_bf16_tc: split-K needs fp32 C and no relu");
  cudaStream_t st = (cudaStream_t)stream;
  // Tile width: 256 columns per CTA amortise the A tile best, but a product with few row tiles (the decoder's
  // M = B*30 = 15 tiles) then runs on 15-60 SMs and each CTA carries a 128 x 256 epilogue.  Narrower tiles spread such
  // products over more SMs: the smallest width whose grid still fits one wave (one CTA per SM) wins.
  int BN = N > 128 ? 256 : (N > 64 ? 128 : 64);
  {
    const long mt = (M + BM - 1) / BM;
    const int sp = splits < 1 ? 1 : splits;
    for (int cand = 64; cand < BN; cand *= 2)
      if (mt * ((N + cand - 1) / cand) * sp <= fira_num_sms()) { BN = cand; break; }
  }
  CUtensorMap ta, tb;
  int rc_;
  // A: K-major -> matrix [M rows, K cols], box {64 k, 128 m};  MN-major -> matrix [K rows, M cols], box {64 m, 64 k}
  if (a_kmajor) rc_ = make_map(&ta, A, M, K, lda, BK, BM); else rc_ = make_map(&ta, A, K, M, lda, 64, BK);
  if (rc_) return rc_;
  if (b_kmajor) rc_ = make_map(&tb, B, N, K, ldb, BK, BN); else rc_ = make_map(&tb, B, K, N, ldb, 64, BK);
  if (rc_) return rc_;
  const int kb_total = (K + BK - 1) / BK;
  if (splits < 1) splits = 1;
  if (splits > kb_total) splits = kb_total;
  int per = (kb_total + splits - 1) / splits;
  splits = (kb_total + per - 1) / per;
  // bf16 output that is neither accumulated nor split: written by TMA from a swizzled staging tile ([32 rows x 64
  // columns] boxes); everything else takes the register / shared-memory epilogue
  const int tma_store = (c_is_bf16 && !accumulate && splits == 1 && (ldc % 8) == 0 && N >= 8 && tma_store_on()) ? 1 : 0;
  CUtensorMap tc = ta;
  if (tma_store) {
    rc_ = make_map(&tc, C, M, N & ~7, ldc, 64, 32);     // columns [N & ~7, N): plain stores in the epilogue
    if (rc_) return rc_;
  }
  FIRA_CHECK_ARG(relu_mask == nullptr || tma_store, FIRA_ERR_ARG,
                 "gemm_bf16_tc: the relu mask needs the TMA-store epilogue (bf16 C, no accumulate, no split-K)");
  TcParams p{C, ldc, c_is_bf16, M, N, K, bias, rs, rc, relu, accumulate, splits, per, a_kmajor, b_kmajor, rotate_on() ? 1 : 0,
             tma_store, (const __nv_bfloat16*)relu_mask, colsum,
             g_probe.load(std::memory_order_relaxed)};
  if (splits > 1 && !accumulate) {
    cudaError_t e = cudaMemset2DAsync(C, (size_t)ldc * 4, 0, (size_t)N * 4, (size_t)M, st);
    if (e != cudaSuccess) { fira_set_error(FIRA_ERR_CUDA, "gemm_bf16_tc memset: %s", cudaGetErrorString(e)); return FIRA_ERR_CUDA; }
  }
  if (BN == 256) rc_ = launch<256>(ta, tb, tc, p, st);
  else if (BN == 128) rc_ = launch<128>(ta, tb, tc, p, st);
  else rc_ = launch<64>(ta, tb, tc, p, st);
  if (rc_) return rc_;
  FIRA_CHECK_LAUNCH("fira_gemm_bf16_tc");
  return FIRA_OK;
}
}  // namespace

extern "C" int fira_gemm_bf16_tc(const void* A, long lda, int a_kmajor, const void* B, long ldb, int b_kmajor, void* C,
                                 long ldc, int c_is_bf16, int M, int N, int K, const float* bias, const float* rs,
                                 const float* rc, int relu, int accumulate, int splits, void* stream) {
  return gemm_tc_impl(A, lda, a_kmajor, B, ldb, b_kmajor, C, ldc, c_is_bf16, M, N, K, bias, rs, rc, relu, accumulate, splits,
                      nullptr, stream);
}

// Input-gradient product through a relu: dx[m,n] = h[m,n] > 0 ? sum_k dy[m,k] W[k,n] : 0 -- dy K-major, W read MN-major
// (the nn.Linear weight [out = k, in = n] as it lies in memory), h = the forward activations (same shape / leading
// dimension as dx).  The relu backward of the FeedForward block folded into the epilogue of its input-gradient product.
extern "C" int fira_gemm_bf16_tc_dx_relu(const void* dy, long lddy, const void* W, long ldw, void* dx, long lddx,
                                         const void* h, int M, int N, int K, void* stream) {
  FIRA_CHECK_ARG(h != nullptr && fira_aligned16(h), FIRA_ERR_ARG, "gemm_bf16_tc_dx_relu: mask");
  FIRA_CHECK_ARG(tma_store_on(), FIRA_ERR_ARG, "gemm_bf16_tc_dx_relu: needs the TMA-store epilogue (FIRA_GEMM_TMA_STORE=0 is set)");
  return gemm_tc_impl(dy, lddy, 1, W, ldw, 0, dx, lddx, 1, M, N, K, nullptr, nullptr, nullptr, 0, 0, 1, nullptr, stream, h);
}

// Weight-gradient product with the bias gradient folded in: C[M,N] = A^T-stored (MN-major) A times B as above, and
// d_bias[m] += sum_k A(m, k) (atomic accumulation into a zero-filled buffer), read from the A tiles as they pass through
// shared memory -- the separate column-sum pass over dY disappears.
extern "C" int fira_gemm_bf16_tc_dbias(const void* A, long lda, const void* B, long ldb, int b_kmajor, void* C, long ldc,
                                       int c_is_bf16, int M, int N, int K, int accumulate, int splits, float* d_bias,
                                       void* stream) {
  FIRA_CHECK_ARG(d_bias != nullptr, FIRA_ERR_ARG, "gemm_bf16_tc_dbias: null d_bias");
  return gemm_tc_impl(A, lda, 0, B, ldb, b_kmajor, C, ldc, c_is_bf16, M, N, K, nullptr, nullptr, nullptr, 0, accumulate,
                      splits, d_bias, stream);
}
