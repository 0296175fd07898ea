// fp32 SIMT GEMM for the parity-precision path (fp32 operands, fp32 FFMA accumulation).
//
// The reference runs every nn.Linear in fp32 (gnn_transformer.py:78,82,141-143,158,171-173,
// 200-204; Model.py:16-19,54).  "logits within 1e-4 rel" cannot be met through 12 post-LN
// layers with TF32/bf16 operands, so the parity mode keeps true fp32 products on the CUDA
// cores; the throughput mode uses the wgmma kernels in gemm_tc.cu instead.
//
// One generic kernel covers the three shapes a Linear needs:
//   forward      Y[M,N]  = X[M,K]  * W[N,K]^T (+bias, +relu, + rs[m]*rc[n])     A k-contig, B k-contig
//   grad input   dX[M,K] = dY[M,N] * W[N,K]                                      A k-contig, B n-contig
//   grad weight  dW[N,K] = dY[M,N]^T * X[M,K]   (split over M, atomics)          A m-contig, B n-contig
#include "common.cuh"
#include "fira_b200.h"

namespace {

constexpr int BK = 16;
constexpr int NTHREADS = 256;

struct GemmParams {
  const float* A; long lda; int a_kcontig;
  const float* B; long ldb; int b_kcontig;
  float* C; long ldc;
  int M, N, K;
  const float* bias;   // [N] or null
  const float* rs;     // [M] or null   rank-1 epilogue term rs[m]*rc[n]
  const float* rc;     // [N] or null
  int relu;
  int accumulate;      // C += result instead of C = result
  int splits;          // >1: every split atomically adds its partial sum into C (C pre-zeroed)
  int k_per_split;     // multiple of BK
};

// load 4 consecutive floats (along the contiguous dim) with element-wise bounds
__device__ __forceinline__ float4 guarded_load4(const float* base, long off, int valid, bool vec_ok) {
  if (valid >= 4 && vec_ok) return *reinterpret_cast<const float4*>(base + off);
  float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
  if (valid > 0) r.x = base[off];
  if (valid > 1) r.y = base[off + 1];
  if (valid > 2) r.z = base[off + 2];
  if (valid > 3) r.w = base[off + 3];
  return r;
}

// Tile loader for an operand viewed as T(x, k) with x in [0,BX) (the M or N index) and k in [0,BK).
// smem layout: s[k][x] (x contiguous), so the compute loop reads float4 along x without conflicts.
template <int BX>
struct TileLoader {
  static constexpr int F4 = BX * BK / 4;          // float4 per tile
  static constexpr int PER_T = F4 / NTHREADS;     // float4 per thread
  static_assert(F4 % NTHREADS == 0, "tile/threads mismatch");
  float4 reg[PER_T];

  __device__ __forceinline__ void load(const float* P, long ld, bool kcontig, int x0, int X, int k0, int Kend,
                                       bool vec_ok) {
#pragma unroll
    for (int i = 0; i < PER_T; ++i) {
      int f = threadIdx.x + i * NTHREADS;
      if (kcontig) {
        int x = f / (BK / 4), kq = (f % (BK / 4)) * 4;
        int gx = x0 + x, gk = k0 + kq;
        int valid = (gx < X) ? (Kend - gk) : 0;
        reg[i] = guarded_load4(P, (long)gx * ld + gk, valid, vec_ok);
      } else {
        int k = f / (BX / 4), xq = (f % (BX / 4)) * 4;
        int gx = x0 + xq, gk = k0 + k;
        int valid = (gk < Kend) ? (X - gx) : 0;
        reg[i] = guarded_load4(P, (long)gk * ld + gx, valid, vec_ok);
      }
    }
  }
  __device__ __forceinline__ void store(float (*s)[BX + 4], bool kcontig) {
#pragma unroll
    for (int i = 0; i < PER_T; ++i) {
      int f = threadIdx.x + i * NTHREADS;
      if (kcontig) {
        int x = f / (BK / 4), kq = (f % (BK / 4)) * 4;
        s[kq + 0][x] = reg[i].x; s[kq + 1][x] = reg[i].y; s[kq + 2][x] = reg[i].z; s[kq + 3][x] = reg[i].w;
      } else {
        int k = f / (BX / 4), xq = (f % (BX / 4)) * 4;
        *reinterpret_cast<float4*>(&s[k][xq]) = reg[i];
      }
    }
  }
};

// BM x BN CTA tile, each thread owns a TM x TN register block split in 4-wide strips
// (strip s covers rows ty*4 + s*(BM/(TM/4)) .. so a warp's smem reads are contiguous float4s).
template <int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__(NTHREADS) gemm_f32_kernel(GemmParams p) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  static_assert((BM / TM) * (BN / TN) == NTHREADS, "thread grid");
  constexpr int SM_ = TM / 4, SN_ = TN / 4;           // strips per thread
  constexpr int MSTRIDE = BM / SM_, NSTRIDE = BN / SN_;
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN + 4];

  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * p.k_per_split;
  const int kend = min(p.K, kbeg + p.k_per_split);
  const int tx = threadIdx.x % (BN / TN), ty = threadIdx.x / (BN / TN);

  const bool a_vec = ((p.lda & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.A) & 15) == 0);
  const bool b_vec = ((p.ldb & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.B) & 15) == 0);

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  TileLoader<BM> la;
  TileLoader<BN> lb;
  const int ntiles = (kend - kbeg + BK - 1) / BK;
  if (ntiles > 0) {
    la.load(p.A, p.lda, p.a_kcontig, m0, p.M, kbeg, kend, a_vec);
    lb.load(p.B, p.ldb, p.b_kcontig, n0, p.N, kbeg, kend, b_vec);
    la.store(As[0], p.a_kcontig);
    lb.store(Bs[0], p.b_kcontig);
  }
  __syncthreads();
  for (int t = 0; t < ntiles; ++t) {
    const int cur = t & 1;
    if (t + 1 < ntiles) {
      la.load(p.A, p.lda, p.a_kcontig, m0, p.M, kbeg + (t + 1) * BK, kend, a_vec);
      lb.load(p.B, p.ldb, p.b_kcontig, n0, p.N, kbeg + (t + 1) * BK, kend, b_vec);
    }
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int s = 0; s < SM_; ++s) {
        float4 v = *reinterpret_cast<const float4*>(&As[cur][kk][ty * 4 + s * MSTRIDE]);
        a[s * 4 + 0] = v.x; a[s * 4 + 1] = v.y; a[s * 4 + 2] = v.z; a[s * 4 + 3] = v.w;
      }
#pragma unroll
      for (int s = 0; s < SN_; ++s) {
        float4 v = *reinterpret_cast<const float4*>(&Bs[cur][kk][tx * 4 + s * NSTRIDE]);
        b[s * 4 + 0] = v.x; b[s * 4 + 1] = v.y; b[s * 4 + 2] = v.z; b[s * 4 + 3] = v.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (t + 1 < ntiles) {
      la.store(As[cur ^ 1], p.a_kcontig);
      lb.store(Bs[cur ^ 1], p.b_kcontig);
    }
    __syncthreads();
  }

  // epilogue
  const bool first_split = (blockIdx.z == 0);
  const bool c_vec = ((p.ldc & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0);
#pragma unroll
  for (int si = 0; si < SM_; ++si) {
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) {
      const int m = m0 + ty * 4 + si * MSTRIDE + ii;
      if (m >= p.M) continue;
      const float rsm = (p.rs && first_split) ? p.rs[m] : 0.f;
#pragma unroll
      for (int sj = 0; sj < SN_; ++sj) {
        const int n = n0 + tx * 4 + sj * NSTRIDE;
        float v[4];
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          float x = acc[si * 4 + ii][sj * 4 + jj];
          if (n + jj < p.N && first_split) {
            if (p.bias) x += p.bias[n + jj];
            if (p.rs) x = fmaf(rsm, p.rc[n + jj], x);
          }
          if (p.relu) x = fmaxf(x, 0.f);
          v[jj] = x;
        }
        float* cp = p.C + (long)m * p.ldc + n;
        if (p.splits > 1) {
#pragma unroll
          for (int jj = 0; jj < 4; ++jj)
            if (n + jj < p.N) atomicAdd(cp + jj, v[jj]);
        } else if (c_vec && n + 3 < p.N) {
          float4 o = make_float4(v[0], v[1], v[2], v[3]);
          if (p.accumulate) {
            const float4 c = *reinterpret_cast<const float4*>(cp);
            o.x += c.x; o.y += c.y; o.z += c.z; o.w += c.w;
          }
          *reinterpret_cast<float4*>(cp) = o;
        } else {
#pragma unroll
          for (int jj = 0; jj < 4; ++jj)
            if (n + jj < p.N) cp[jj] = p.accumulate ? cp[jj] + v[jj] : v[jj];
        }
      }
    }
  }
}

}  // namespace

extern "C" int fira_gemm_f32(const float* A, long lda, int a_kcontig, const float* B, long ldb, int b_kcontig,
                             float* C, long ldc, int M, int N, int K, const float* bias, const float* rs,
                             const float* rc, int relu, int accumulate, int splits, void* stream) {
  FIRA_CHECK_ARG(M >= 0 && N >= 0 && K >= 0, FIRA_ERR_SHAPE, "fira_gemm_f32: negative dim");
  FIRA_CHECK_ARG(A && B && C, FIRA_ERR_ARG, "fira_gemm_f32: null operand");
  FIRA_CHECK_ARG((rs == nullptr) == (rc == nullptr), FIRA_ERR_ARG, "fira_gemm_f32: rs/rc must come together");
  FIRA_CHECK_ARG(!(relu && splits > 1), FIRA_ERR_ARG, "fira_gemm_f32: relu with split-K");
  if (M == 0 || N == 0) return FIRA_OK;
  GemmParams p{A, lda, a_kcontig, B, ldb, b_kcontig, C, ldc, M, N, K, bias, rs, rc, relu, accumulate, 1, 0};
  if (splits < 1) splits = 1;
  int ktiles = (K + BK - 1) / BK;
  if (splits > ktiles) splits = ktiles > 0 ? ktiles : 1;
  int tiles_per_split = (ktiles + splits - 1) / splits;
  if (tiles_per_split < 1) tiles_per_split = 1;
  splits = ktiles > 0 ? (ktiles + tiles_per_split - 1) / tiles_per_split : 1;
  p.splits = splits;
  p.k_per_split = tiles_per_split * BK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (splits > 1 && !accumulate) {   // split partials are atomically added: start from zero
    cudaError_t e = cudaMemset2DAsync(C, (size_t)ldc * sizeof(float), 0, (size_t)N * sizeof(float), (size_t)M, st);
    if (e != cudaSuccess) { fira_set_error(FIRA_ERR_CUDA, "fira_gemm_f32 memset: %s", cudaGetErrorString(e)); return FIRA_ERR_CUDA; }
  }
  const long big_tiles = (long)((M + 127) / 128) * ((N + 127) / 128) * splits;
  if (big_tiles >= 120) {
    dim3 grid((N + 127) / 128, (M + 127) / 128, splits);
    launch_k(gemm_f32_kernel<128, 128, 8, 8>, dim3(grid), dim3(NTHREADS), 0, st, p);
  } else {
    dim3 grid((N + 63) / 64, (M + 63) / 64, splits);
    launch_k(gemm_f32_kernel<64, 64, 4, 4>, dim3(grid), dim3(NTHREADS), 0, st, p);
  }
  FIRA_CHECK_LAUNCH("fira_gemm_f32");
  return FIRA_OK;
}
