// Exact k-nearest-neighbour search of a kNN datastore (fira_icse_b200/knn.py): for every query row the k entries with
// the smallest (d_i, i), d_i = |q|^2 + norm_i - 2 q . key_i, q rounded to bf16, the products on the bf16 tensor cores
// with fp32 accumulation.
//
// Stage 1 (knn_partial_kernel): grid (query tiles of 128 rows, P key splits).  A CTA holds its 128 query rows as
// mma.sync A fragments in registers (each warp 16 rows x 256 features) and streams the keys of its split through a
// 4-stage cp.async pipeline, 64 keys per stage.  Each warp owns its 16 rows' candidate lists (k sorted 64-bit keys
// (order bits of d, i) per row in shared memory), so the epilogue needs no CTA barrier: a distance enters only when it
// beats the row's k-th key, which a lane keeps in registers, so insertions become rare once the lists fill.  The
// query tiles of one key split are adjacent block indices and run at the same time, so a split's keys come from HBM
// once and from L2 for the other tiles.  P is at most the SMs per query tile, so one wave covers the grid.
// Stage 2 (knn_merge_kernel): one warp per row merges the P sorted lists of the workspace, k rounds of a warp minimum.
//
// Every distance is computed the same way wherever its row and key sit (fixed k-step order of the MMA, the same fma),
// and the selection is exact under the total order (d, i), so the result depends on neither R, the other rows, P nor
// the SM count, and graph replays agree bit for bit.
#include "common.cuh"
#include "attn_mma.cuh"

namespace {

using namespace mma;

constexpr int kD = 256;                            // key width
constexpr int kBM = 128;                           // query rows per CTA (8 warps x 16)
constexpr int kBN = 64;                            // keys per pipeline stage
constexpr int kStages = 4;
constexpr int kThreads = 256;
constexpr int kMaxK = 64;
constexpr int kMaxSplit = 256;                     // key splits: the merge warp holds 8 list heads per lane
constexpr int kRowB = kD * 2;                      // bytes of one bf16 row
constexpr int kKeyTileB = kBN * kRowB;
constexpr int kStageB = kKeyTileB + kBN * 4;       // keys, then their norms

// byte offset of 16-B chunk c of row r in a [rows][256] bf16 tile: the XOR puts the 8 rows of an ldmatrix 8x8 matrix
// on 8 different bank groups
__device__ __forceinline__ uint32_t kswz(int r, int c) { return r * kRowB + ((c ^ (r & 7)) << 4); }

__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void* src, int bytes) {   // bytes < 16: zeros
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}

// (d, i) as one unsigned key: smaller key = nearer entry, ties in d to the smaller index
__device__ __forceinline__ uint64_t dist_key(float d, uint32_t i) {
  const uint32_t b = __float_as_uint(d);
  return ((uint64_t)((b & 0x80000000u) ? ~b : (b | 0x80000000u)) << 32) | i;
}
__device__ __forceinline__ float key_dist(uint64_t key) {
  const uint32_t b = (uint32_t)(key >> 32);
  return __uint_as_float((b & 0x80000000u) ? (b & 0x7FFFFFFFu) : ~b);
}
constexpr uint64_t kNoKey = ~0ull;

__device__ __forceinline__ uint4 load8_bf16(const __nv_bfloat16* p) { return *reinterpret_cast<const uint4*>(p); }
__device__ __forceinline__ uint4 load8_bf16(const float* p) {
  float v[8];
  Act<float>::load8(p, v);
  return make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
}

// keys [tile * 64, +64) and their norms into one stage; rows past N are zero-filled (their distances are skipped)
__device__ __forceinline__ void load_tile(unsigned char* st, const __nv_bfloat16* keys, const float* norms, long N,
                                          long tile) {
  const long k0 = tile * kBN;
  for (int c = threadIdx.x; c < kBN * 32; c += kThreads) {
    const int j = c >> 5, ch = c & 31;
    const bool ok = k0 + j < N;
    cp_async16_zfill(su32(st + kswz(j, ch)), keys + (ok ? k0 + j : 0) * kD + ch * 8, ok ? 16 : 0);
  }
  if (threadIdx.x < kBN / 4) {
    const long i = k0 + threadIdx.x * 4, n = N - i;
    const int bytes = n >= 4 ? 16 : n > 0 ? (int)n * 4 : 0;
    cp_async16_zfill(su32(st + kKeyTileB + threadIdx.x * 16), norms + (bytes ? i : 0), bytes);
  }
}

// x into the ascending list L[0..k) if it beats L[k - 1] (one thread per list)
__device__ __forceinline__ void list_insert(uint64_t* L, int k, uint64_t x) {
  if (x >= L[k - 1]) return;
  int j = k - 1;
  while (j > 0) {
    const uint64_t y = L[j - 1];
    if (y < x) break;
    L[j] = y;
    --j;
  }
  L[j] = x;
}

template <typename TQ>
__global__ void __launch_bounds__(kThreads, 1) knn_partial_kernel(const TQ* __restrict__ q, long ldq, int R,
                                                                  const __nv_bfloat16* __restrict__ keys,
                                                                  const float* __restrict__ norms, long N, int k,
                                                                  int P, uint64_t* __restrict__ ws) {
  extern __shared__ __align__(128) unsigned char smem[];
  unsigned char* stages = smem;                                       // the query tile first, then the key stages
  float* s_qn = reinterpret_cast<float*>(smem + kStages * kStageB);
  uint64_t* s_list = reinterpret_cast<uint64_t*>(s_qn + kBM);
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int r0 = blockIdx.x * kBM, p = blockIdx.y;
  const long tiles = (N + kBN - 1) / kBN;
  const long t0 = tiles * p / P, t1 = tiles * (p + 1) / P;

  for (int c = tid; c < kBM * 32; c += kThreads) {                    // queries, rounded to bf16
    const int r = c >> 5, ch = c & 31;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r0 + r < R) v = load8_bf16(q + (long)(r0 + r) * ldq + ch * 8);
    *reinterpret_cast<uint4*>(stages + kswz(r, ch)) = v;
  }
  const int ldl = k + 1;                                              // list pitch: the 8 rows of a turn hit 8 banks
  for (int i = tid; i < kBM * ldl; i += kThreads) s_list[i] = kNoKey;
  __syncthreads();
  for (int rr = 0; rr < 16; ++rr) {                                   // |q|^2 in fp32, a fixed order per row
    const int r = warp * 16 + rr;
    const uint4 v = *reinterpret_cast<const uint4*>(stages + kswz(r, lane));
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float2 f = __bfloat1622float2(h[i]); s = fmaf(f.x, f.x, s); s = fmaf(f.y, f.y, s); }
    s = warp_sum(s);
    if (lane == 0) s_qn[r] = s;
  }
  uint32_t a[16][4];                                                  // the warp's 16 rows x 256 features
#pragma unroll
  for (int kk = 0; kk < 16; ++kk) ldsm4(su32(stages + kswz(warp * 16 + (lane & 15), 2 * kk + (lane >> 4))), a[kk]);
  __syncthreads();                                                    // the query tile is free; s_qn is written

#pragma unroll
  for (int s = 0; s < kStages - 1; ++s) {
    if (t0 + s < t1) load_tile(stages + s * kStageB, keys, norms, N, t0 + s);
    cp_async_commit();
  }
  const int ra = warp * 16 + (lane >> 2);                             // this lane's rows ra and ra + 8
  const float qn0 = s_qn[ra], qn1 = s_qn[ra + 8];
  uint64_t* L0 = s_list + ra * ldl;
  uint64_t* L1 = s_list + (ra + 8) * ldl;
  uint64_t thr0 = kNoKey, thr1 = kNoKey;                              // the rows' k-th keys
  // and their distances, a cheap first test; rows past R start at -inf, so they never take a candidate
  float thd0 = r0 + ra < R ? INFINITY : -INFINITY, thd1 = r0 + ra + 8 < R ? INFINITY : -INFINITY;
  const bool live_warp = r0 + warp * 16 < R;                          // a warp of padding rows skips the product too

  for (long t = t0; t < t1; ++t) {
    cp_async_wait<kStages - 2>();
    __syncthreads();                                                  // tile t landed; tile t - 1's stage is free
    {
      const long tn = t + kStages - 1;
      if (tn < t1) load_tile(stages + ((tn - t0) % kStages) * kStageB, keys, norms, N, tn);
      cp_async_commit();
    }
    if (!live_warp) continue;                                         // (it still joins every barrier above)
    const unsigned char* st = stages + ((t - t0) % kStages) * kStageB;
    float acc[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;
#pragma unroll
    for (int kp = 0; kp < 8; ++kp)
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        uint32_t b[4];
        ldsm4(su32(st + kswz(8 * n + (lane & 7), 4 * kp + (lane >> 3))), b);
        mma16816(acc[n], a[2 * kp], b[0], b[1]);
        mma16816(acc[n], a[2 * kp + 1], b[2], b[3]);
      }
    // epilogue: acc[n][e] is row ra (e < 2) or ra + 8, key 8 n + 2 (lane & 3) + (e & 1) of the tile
    const float* snorm = reinterpret_cast<const float*>(st + kKeyTileB);
    const long base = t * kBN;
    uint32_t m0 = 0, m1 = 0;
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * n + 2 * (lane & 3) + e;
        const uint32_t i = (uint32_t)(base + col);
        const float nr = snorm[col];
        const float d0 = fmaf(-2.f, acc[n][e], qn0 + nr), d1 = fmaf(-2.f, acc[n][2 + e], qn1 + nr);
        if (base + col < N) {
          if (d0 <= thd0 && dist_key(d0, i) < thr0) m0 |= 1u << (2 * n + e);
          if (d1 <= thd1 && dist_key(d1, i) < thr1) m1 |= 1u << (2 * n + e);
        }
      }
    if (__any_sync(0xffffffffu, (m0 | m1) != 0u)) {
      for (int turn = 0; turn < 4; ++turn) {                          // the 4 lanes of a row take turns
        if ((lane & 3) == turn && (m0 | m1)) {
#pragma unroll
          for (int n = 0; n < 8; ++n)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = 8 * n + 2 * (lane & 3) + e;
              const uint32_t i = (uint32_t)(base + col);
              const float nr = snorm[col];
              if (m0 & (1u << (2 * n + e))) list_insert(L0, k, dist_key(fmaf(-2.f, acc[n][e], qn0 + nr), i));
              if (m1 & (1u << (2 * n + e))) list_insert(L1, k, dist_key(fmaf(-2.f, acc[n][2 + e], qn1 + nr), i));
            }
        }
        __syncwarp();
      }
      thr0 = L0[k - 1]; thr1 = L1[k - 1];
      thd0 = thr0 == kNoKey ? INFINITY : key_dist(thr0);
      thd1 = thr1 == kNoKey ? INFINITY : key_dist(thr1);
    }
  }
  cp_async_wait<0>();
  __syncwarp();
  for (int rr = 0; rr < 16; ++rr) {                                   // the warp's rows -> workspace [P][R][k]
    const int r = warp * 16 + rr;
    if (r0 + r >= R) break;
    for (int j = lane; j < k; j += 32) ws[((long)p * R + r0 + r) * k + j] = s_list[r * ldl + j];
  }
}

// one warp per row: k rounds, each takes the smallest head of the P sorted lists (lane l holds lists l, l + 32, ...)
__global__ void __launch_bounds__(256) knn_merge_kernel(const uint64_t* __restrict__ ws, int R, int k, int P,
                                                        int* __restrict__ idx, float* __restrict__ dist) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const int lane = threadIdx.x & 31;
  const long row = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= R) return;
  constexpr int U = kMaxSplit / 32;
  int pos[U];
  uint64_t head[U];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int l = lane + 32 * u;
    pos[u] = 0;
    head[u] = l < P ? ws[((long)l * R + row) * k] : kNoKey;
  }
  for (int j = 0; j < k; ++j) {
    uint64_t best = head[0];
    int bu = 0;
#pragma unroll
    for (int u = 1; u < U; ++u)
      if (head[u] < best) { best = head[u]; bu = u; }
    uint64_t m = best;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const uint64_t y = __shfl_xor_sync(0xffffffffu, m, o);
      m = y < m ? y : m;
    }
    if (lane == 0) {
      idx[row * k + j] = (int)(uint32_t)m;
      dist[row * k + j] = key_dist(m);
    }
    if (best == m) {                                                  // keys are unique: one lane advances
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (u == bu) {
          ++pos[u];
          head[u] = pos[u] < k ? ws[((long)(lane + 32 * u) * R + row) * k + pos[u]] : kNoKey;
        }
    }
  }
}

}  // namespace

extern "C" {

int fira_knn_search(const void* queries, long ld_q, int dtype, const void* keys, const float* norms, long N, int R,
                    int k, void* workspace, long workspace_bytes, int* idx, float* dist, void* stream) {
  FIRA_CHECK_ARG(dtype == FIRA_F32 || dtype == FIRA_BF16, FIRA_ERR_DTYPE, "knn_search: dtype %d", dtype);
  FIRA_CHECK_ARG(k >= 1 && k <= kMaxK && N >= k && N < (1L << 31) && R >= 0 && ld_q >= kD, FIRA_ERR_SHAPE,
                 "knn_search: shape (R %d, N %ld, k %d, ld_q %ld; 1 <= k <= %d, k <= N < 2^31, ld_q >= %d)", R, N, k,
                 ld_q, kMaxK, kD);
  FIRA_CHECK_ARG(queries && keys && norms && workspace && idx && dist, FIRA_ERR_ARG, "knn_search: null pointer");
  FIRA_CHECK_ARG(fira_aligned16(queries) && fira_aligned16(keys) && fira_aligned16(norms) && fira_aligned16(workspace)
                 && ld_q % 8 == 0, FIRA_ERR_ALIGN,
                 "knn_search: queries, keys, norms and workspace must be 16-byte aligned, ld_q a multiple of 8");
  if (R == 0) return FIRA_OK;
  const long per_split = 8L * k * R;
  FIRA_CHECK_ARG(workspace_bytes >= per_split, FIRA_ERR_ARG, "knn_search: workspace %ld bytes < 8 k R = %ld",
                 workspace_bytes, per_split);
  const long qtiles = (R + kBM - 1) / kBM, tiles = (N + kBN - 1) / kBN;
  long P = fira_num_sms() / qtiles;
  if (P < 1) P = 1;
  if (P > workspace_bytes / per_split) P = workspace_bytes / per_split;
  if (P > tiles) P = tiles;
  if (P > kMaxSplit) P = kMaxSplit;
  const int smem = kStages * kStageB + kBM * 4 + kBM * (k + 1) * 8;
  cudaError_t e = dtype == FIRA_F32
      ? cudaFuncSetAttribute(knn_partial_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)
      : cudaFuncSetAttribute(knn_partial_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) { fira_set_error(FIRA_ERR_CUDA, "knn_search attr: %s", cudaGetErrorString(e)); return FIRA_ERR_CUDA; }
  const dim3 grid((unsigned)qtiles, (unsigned)P);
  if (dtype == FIRA_F32)
    launch_k(knn_partial_kernel<float>, grid, dim3(kThreads), smem, (cudaStream_t)stream, (const float*)queries, ld_q,
             R, (const __nv_bfloat16*)keys, norms, N, k, (int)P, (uint64_t*)workspace);
  else
    launch_k(knn_partial_kernel<__nv_bfloat16>, grid, dim3(kThreads), smem, (cudaStream_t)stream,
             (const __nv_bfloat16*)queries, ld_q, R, (const __nv_bfloat16*)keys, norms, N, k, (int)P,
             (uint64_t*)workspace);
  FIRA_CHECK_LAUNCH("fira_knn_search (partial)");
  launch_k(knn_merge_kernel, dim3((unsigned)((R + 7) / 8)), dim3(256), 0, (cudaStream_t)stream,
           (const uint64_t*)workspace, R, k, (int)P, idx, dist);
  FIRA_CHECK_LAUNCH("fira_knn_search (merge)");
  return FIRA_OK;
}

}  // extern "C"
