// Multi-head attention core on the Hopper tensor cores (wgmma, bf16 throughput mode), gnn_transformer.py:144-156:
//     S = Q K^T / sqrt(32);  S[mask == 0] = -1e9;  P = softmax(S);  ctx = P V          (+ the backward of exactly that)
//
// The per-head problem (30 x Lk x 32) is far below a 128-row tile, and every head has its own K/V slice, so the kernel
// works on a HEAD GROUP: one CTA per (commit, 4 heads).  The 128 rows of the tile are (head hl, query t) = hl*32 + t,
// two m64 warpgroups of 64 rows each, and the A operand is the query block REPLICATED and MASKED per head:
//     A'[(hl,t), f] = Q[t, 128 g + f]  if feature f belongs to head hl (f / 32 == hl), else 0          (128 x 128)
// With that operand one M128 x N128 x K128 product against the K rows AS THEY LIE IN MEMORY (K-major, 128 features of
// the group) yields all four heads' score rows at once; the zeros make the cross-head terms vanish, the tensor core
// does 4x redundant MACs on a pipe that is otherwise idle.  The same trick runs backwards:
//     O'  = P V          (M = (hl,t), K = keys, N = 128 features; row (hl,t) keeps its own head's 32 columns)
//     dP' = dO' V^T ,  dQ' = dS K ,  dK = dS^T A'(Q) ,  dV = P^T A'(dO)      (A' as MN-major B: cross-head terms are 0)
// K and V tiles arrive by TMA (SWIZZLE_128B); one [128 keys x 64 features] box serves as K-major B (scores) and as
// MN-major B (P V, dS K) -- the bytes are the same, only the descriptor differs.  P and dS are written by the softmax
// threads into the same swizzled layout, where they serve as K-major A (P V, dS K) and as MN-major A (P^T dO, dS^T Q).
// Accumulators live in registers (wgmma fragments: a row's columns are spread over the 4 threads of a lane quad).
// Keys are processed in chunks of 128 (Lk <= 384).  The forward makes two passes over the score chunks -- row maximum,
// then the scores are recomputed for exp / sum / P -- so no online rescaling is needed.
//
// Semantics kept from the FFMA kernels (attention.cu): scale before mask, -1e9 fill (a fully masked row is uniform
// over all Lk keys), masked keys get exactly zero dK / dV unless the whole row is masked, statistics = (row max, row
// sum) [B,H,Lq,2].
#include "tc_common.cuh"
#include "fira_b200.h"

namespace attn_tc {

using namespace tc;

constexpr int DH = 32, HG = 4, GF = HG * DH;         // head dim, heads per group, features per group (128)
constexpr int KC = 128;                              // keys per chunk
constexpr int MAX_CH = 3;                            // Lk <= 384
constexpr int TILE = 128 * 128 * 2;                  // one [128 rows x 128 cols] bf16 tile = two 16 KB panels
constexpr int PANEL = 16384;
constexpr int THREADS = 256;                         // two warpgroups: tile rows [0, 64) and [64, 128)

struct Args {
  const __nv_bfloat16* q; long ldq;
  const unsigned char* key_mask;                     // [B, Lk] (NULL with ranges: every key of the ranges is valid)
  const int* ranges;                                 // NULL, or [B][4] = {first row, rows, first row, rows}: the keys of
                                                     // commit b are two row ranges of k / v (packed batches); Lk = mask pitch
  int causal, B, H, Lq, Lk;
  float scale;
  __nv_bfloat16* ctx; long ldo;                      // fwd out / bwd: forward output
  float* stats;
  // backward
  const __nv_bfloat16* d_ctx;
  __nv_bfloat16* dq; long lddq;
  __nv_bfloat16* dk; long lddk;
  __nv_bfloat16* dv; long lddv;
};

__device__ __forceinline__ uint4 ldg16(const __nv_bfloat16* p) { return *reinterpret_cast<const uint4*>(p); }

// A'(X)[(hl,t), f] tile for head group g from a [B*Lq, ld] matrix: zero-filled, then head hl's 32 features of row t.
// tile layout: 2 panels (64 features) x [128 rows x 128 B], SWIZZLE_128B.
__device__ __forceinline__ void build_masked_tile(unsigned char* tile, const __nv_bfloat16* x, long ld, int b, int g, int Lq,
                                                  int tid, int nthr) {
  for (int i = tid; i < TILE / 16; i += nthr) reinterpret_cast<uint4*>(tile)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  // 128 rows x 4 chunks of 16 B
  for (int i = tid; i < 128 * 4; i += nthr) {
    const int m = i >> 2, c = i & 3;
    const int hl = m >> 5, t = m & 31;
    if (t < Lq) {
      const uint4 v = ldg16(x + ((long)b * Lq + t) * ld + g * GF + hl * DH + c * 8);
      const int f = hl * DH + c * 8;                 // feature within the group
      *reinterpret_cast<uint4*>(tile + (f >> 6) * PANEL + sw128_offset(m, (f & 63) >> 3)) = v;
    }
  }
}

// Key chunks of one commit: chunk c = rows [row[c], row[c] + n[c]) of k / v, its keys are mask positions moff[c] + i.
struct Chunks { int nch; int row[MAX_CH]; int n[MAX_CH]; int moff[MAX_CH]; };

__device__ __forceinline__ void make_chunks(Chunks& ch, const int* ranges, int b, int Lk) {
  int n = 0;
  if (ranges) {
    const int s0 = ranges[4 * b], l0 = ranges[4 * b + 1], s1 = ranges[4 * b + 2], l1 = ranges[4 * b + 3];
    for (int o = 0; o < l0 && n < MAX_CH; o += KC, ++n) { ch.row[n] = s0 + o; ch.n[n] = min(KC, l0 - o); ch.moff[n] = o; }
    for (int o = 0; o < l1 && n < MAX_CH; o += KC, ++n) { ch.row[n] = s1 + o; ch.n[n] = min(KC, l1 - o); ch.moff[n] = l0 + o; }
  } else {
    for (int o = 0; o < Lk && n < MAX_CH; o += KC, ++n) { ch.row[n] = b * Lk + o; ch.n[n] = min(KC, Lk - o); ch.moff[n] = o; }
  }
  ch.nch = n;
}

// Key validity as bit masks, one word per 32-key group of a chunk:
//   exist[c*4+j] bit i : key j*32+i of chunk c is a key of this commit (below the chunk's key count)
//   bits [c*4+j] bit i : ... and its mask byte is set
// A chunk without a single valid key is DROPPED from the table when the commit has valid keys elsewhere (its
// probabilities and gradients are exactly zero: exp(-1e9 - max) == 0 in fp32); `rm` keeps the dropped chunks so that
// the backward can write their zero dK / dV rows.  A commit / row without any valid key keeps everything: every score
// is -1e9 there and the softmax is uniform over ALL keys, like the reference's masked_fill + softmax.
struct KeyBits { uint32_t bits[MAX_CH * 4]; uint32_t exist[MAX_CH * 4]; };

__device__ __forceinline__ void prepare_keys(Chunks& ch, Chunks& rm, KeyBits& kb, const unsigned char* s_mask, int causal,
                                             int warp, int lane) {
  if (warp == 0) {
    unsigned has = 0;
    for (int c = 0; c < ch.nch; ++c) {
      bool v = false;
      for (int i = lane; i < ch.n[c]; i += 32) v |= s_mask[ch.moff[c] + i] != 0;
      if (__any_sync(0xffffffffu, v)) has |= 1u << c;
    }
    if (lane == 0) {
      int k = 0, r = 0;
      const bool drop = has != 0 && !causal;
      for (int c = 0; c < ch.nch; ++c) {
        if (!drop || ((has >> c) & 1)) { ch.row[k] = ch.row[c]; ch.n[k] = ch.n[c]; ch.moff[k] = ch.moff[c]; ++k; }
        else { rm.row[r] = ch.row[c]; rm.n[r] = ch.n[c]; rm.moff[r] = ch.moff[c]; ++r; }
      }
      ch.nch = k; rm.nch = r;
    }
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < ch.nch * KC; idx += THREADS) {       // THREADS % 32 == 0: a warp covers one group
    const int c = idx >> 7, i = idx & 127;
    const bool ex = i < ch.n[c];
    const bool ok = ex && s_mask[ch.moff[c] + i] != 0;
    const unsigned bv = __ballot_sync(0xffffffffu, ok), be = __ballot_sync(0xffffffffu, ex);
    if (lane == 0) { kb.bits[idx >> 5] = bv; kb.exist[idx >> 5] = be; }
  }
  __syncthreads();
}

// valid keys of group j of chunk c for query row t
__device__ __forceinline__ uint32_t row_bits(const KeyBits& kb, const Chunks& ch, int c, int j, int t, int causal) {
  uint32_t v = kb.bits[c * 4 + j];
  if (causal) {                                     // key position <= t (causal attention has one chunk, moff = 0)
    const int lo = ch.moff[c] + j * 32;
    v &= t < lo ? 0u : (t - lo >= 31 ? 0xffffffffu : ((2u << (t - lo)) - 1u));
  }
  return v;
}

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
constexpr float kLog2e = 1.4426950408889634f;

// rows of this thread's accumulator fragments: mr[h] = tile row (hl, t), h = 0 / 1
struct FragRows { int mr[2], t[2]; int hl; };
__device__ __forceinline__ FragRows frag_rows(int warp, int lane) {
  FragRows f;
#pragma unroll
  for (int h = 0; h < 2; ++h) { f.mr[h] = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h; f.t[h] = f.mr[h] & 31; }
  f.hl = f.mr[0] >> 5;                               // both rows of a thread belong to the same head
  return f;
}
// bf16 pair (keys key, key + 1) into a P / dS tile: 2 panels of 64 keys x [128 rows x 128 B], SWIZZLE_128B
__device__ __forceinline__ uint32_t pair_off(int m, int key) {
  return (key >> 6) * PANEL + sw128_offset(m, (key & 63) >> 3) + (key & 7) * 2;
}

// S (64 rows of warpgroup wg x 128 keys of a chunk) = A'(Q) K^T
__device__ __forceinline__ void scores(float* s, uint32_t aq, uint32_t kt, int wg) {
#pragma unroll
  for (int i = 0; i < 64; ++i) s[i] = 0.f;
  wgmma_fence();
#pragma unroll
  for (int kb_ = 0; kb_ < 2; ++kb_)
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wgmma<128, 0, 0>(s, make_desc(aq + kb_ * PANEL + wg * 8192 + k * 32, 16, 1024), make_desc(kt + kb_ * PANEL + k * 32, 16, 1024));
  wgmma_commit();
  wgmma_wait<0>();
  reg_fence<64>(s);
}

// =================================================================================================== forward
// smem: A'(Q) 32 KB | K[3] 96 KB | V[2] 64 KB | P 32 KB   (V of chunk 2 reuses the V slot of chunk 0)
__global__ void __launch_bounds__(THREADS, 1)
attn_tc_fwd_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV, Args a) {
  extern __shared__ unsigned char smem_raw[];
  __shared__ __align__(8) unsigned long long k_full[MAX_CH], v_full[MAX_CH], v_free;
  __shared__ unsigned char s_mask[MAX_CH * KC];
  __shared__ Chunks ch, rm;
  __shared__ KeyBits kb;
  const uint32_t base = (smem_addr(smem_raw) + 1023u) & ~1023u;
  unsigned char* sm = smem_raw + (base - smem_addr(smem_raw));
  constexpr uint32_t OFF_AQ = 0, OFF_K = TILE, OFF_V = OFF_K + MAX_CH * TILE, OFF_P = OFF_V + 2 * TILE;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2, q4 = lane & 3;
  const int b = blockIdx.x >> 1, g = blockIdx.x & 1;

  if (threadIdx.x == 0) {
    for (int i = 0; i < MAX_CH; ++i) { mbar_init(smem_addr(&k_full[i]), 1); mbar_init(smem_addr(&v_full[i]), 1); }
    mbar_init(smem_addr(&v_free), THREADS);
    mbar_init_fence();
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
  }
  pdl_wait(); pdl_trigger();       // PDL: the prologue above overlapped the previous kernel's tail (common.cuh)
  if (threadIdx.x == 0) make_chunks(ch, a.ranges, b, a.Lk);
  for (int i = threadIdx.x; i < MAX_CH * KC; i += THREADS)
    s_mask[i] = i < a.Lk ? (a.key_mask ? a.key_mask[(long)b * a.Lk + i] : (unsigned char)1) : (unsigned char)0;
  __syncthreads();
  prepare_keys(ch, rm, kb, s_mask, a.causal, warp, lane);
  const int nch = ch.nch;
  auto load = [&](const CUtensorMap* map, uint32_t dst, int c, unsigned long long* bar) {
    mbar_expect_tx(smem_addr(bar), TILE);
    tma_load_2d(dst, map, g * GF, ch.row[c], smem_addr(bar));
    tma_load_2d(dst + PANEL, map, g * GF + 64, ch.row[c], smem_addr(bar));
  };
  if (threadIdx.x == 0) {                            // K and the first two V chunks fly while the A' tile is built
    for (int c = 0; c < nch; ++c) load(&tmK, base + OFF_K + c * TILE, c, &k_full[c]);
    for (int c = 0; c < nch && c < 2; ++c) load(&tmV, base + OFF_V + c * TILE, c, &v_full[c]);
  }
  build_masked_tile(sm + OFF_AQ, a.q, a.ldq, b, g, a.Lq, threadIdx.x, THREADS);
  fence_proxy_async();
  __syncthreads();

  const FragRows fr = frag_rows(warp, lane);
  bool live[2], rowfilled[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    live[h] = fr.t[h] < a.Lq;
    // does this row see any valid key at all?  (no: every score is -1e9 -> uniform over all existing keys)
    uint32_t any = 0;
    for (int c = 0; c < nch; ++c)
#pragma unroll
      for (int j = 0; j < 4; ++j) any |= row_bits(kb, ch, c, j, fr.t[h], a.causal);
    rowfilled[h] = any == 0;
  }
  float s[64];
  // pass A: row maximum of the raw scores over the valid keys (the scale is positive)
  float mraw[2] = {-INFINITY, -INFINITY};
  for (int c = 0; c < nch; ++c) {
    mbar_wait(smem_addr(&k_full[c]), 0);
    scores(s, base + OFF_AQ, base + OFF_K + c * TILE, wg);
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        const uint32_t vb = row_bits(kb, ch, c, jj >> 2, fr.t[h], a.causal) >> (8 * (jj & 3) + 2 * q4);
        if (vb & 1) mraw[h] = fmaxf(mraw[h], s[4 * jj + 2 * h]);
        if (vb & 2) mraw[h] = fmaxf(mraw[h], s[4 * jj + 2 * h + 1]);
      }
  }
  const float k2 = a.scale * kLog2e;
  float m2[2], sum[2] = {0.f, 0.f};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    mraw[h] = fmaxf(mraw[h], __shfl_xor_sync(0xffffffffu, mraw[h], 1));
    mraw[h] = fmaxf(mraw[h], __shfl_xor_sync(0xffffffffu, mraw[h], 2));
    m2[h] = mraw[h] * k2;
  }
  // pass B: scores again, P = bf16(exp) into shared memory, O' += P V
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  for (int c = 0; c < nch; ++c) {
    scores(s, base + OFF_AQ, base + OFF_K + c * TILE, wg);
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      const uint32_t eb = kb.exist[c * 4 + (jj >> 2)] >> (8 * (jj & 3) + 2 * q4);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t vb = row_bits(kb, ch, c, jj >> 2, fr.t[h], a.causal) >> (8 * (jj & 3) + 2 * q4);
        float e[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          // the MMA consumes bf16(e): sum the ROUNDED values so that P rows are normalised exactly
          const float x = rowfilled[h] ? (((eb >> i) & 1) ? 1.f : 0.f)
                                       : (((vb >> i) & 1) ? fast_exp2(fmaf(s[4 * jj + 2 * h + i], k2, -m2[h])) : 0.f);
          e[i] = live[h] ? __bfloat162float(__float2bfloat16_rn(x)) : 0.f;
          sum[h] += e[i];
        }
        *reinterpret_cast<__nv_bfloat162*>(sm + OFF_P + pair_off(fr.mr[h], 8 * jj + 2 * q4)) = __floats2bfloat162_rn(e[0], e[1]);
      }
    }
    fence_proxy_async();
    named_bar(2 + wg, 128);                          // the warpgroup's P rows are complete
    mbar_wait(smem_addr(&v_full[c]), 0);
    const uint32_t vt = base + OFF_V + (c & 1) * TILE;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 8; ++k)                      // 8 steps of 16 keys
      wgmma<128, 0, 1>(o, make_desc(base + OFF_P + (k >> 2) * PANEL + wg * 8192 + (k & 3) * 32, 16, 1024),
                       make_desc(vt + k * 2048, PANEL, 1024));
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<64>(o);
    if (c == 0 && nch == 3) {                        // V slot 0 is free: chunk 2's V goes there
      mbar_arrive(smem_addr(&v_free));
      if (threadIdx.x == 0) {
        mbar_wait(smem_addr(&v_free), 0);
        load(&tmV, base + OFF_V, 2, &v_full[2]);
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 1);
    sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 2);
    if (!live[h]) continue;
    const int t = fr.t[h];
    const float inv = 1.f / sum[h];
    __nv_bfloat16* dst = a.ctx + ((long)b * a.Lq + t) * a.ldo + g * GF;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj)                  // own head's 32 output columns
      if ((jj >> 2) == fr.hl)
        *reinterpret_cast<__nv_bfloat162*>(dst + 8 * jj + 2 * q4) =
            __floats2bfloat162_rn(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
    if (a.stats && q4 == 0) {
      float* st = a.stats + (((long)b * a.H + g * HG + fr.hl) * a.Lq + t) * 2;
      st[0] = rowfilled[h] ? kMaskFill : mraw[h] * a.scale;          // what the reference's softmax subtracts
      st[1] = sum[h];
    }
  }
}

// =================================================================================================== backward
// smem: A'(Q) | A'(dO) | K | V | P | dS  (6 x 32 KB)
__global__ void __launch_bounds__(THREADS, 1)
attn_tc_bwd_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV, Args a) {
  extern __shared__ unsigned char smem_raw[];
  __shared__ __align__(8) unsigned long long kv_full;
  __shared__ unsigned char s_mask[MAX_CH * KC];
  __shared__ Chunks ch, rm;
  __shared__ KeyBits kb;
  const uint32_t base = (smem_addr(smem_raw) + 1023u) & ~1023u;
  unsigned char* sm = smem_raw + (base - smem_addr(smem_raw));
  constexpr uint32_t OFF_AQ = 0, OFF_ADO = TILE, OFF_K = 2 * TILE, OFF_V = 3 * TILE, OFF_P = 4 * TILE, OFF_DS = 5 * TILE;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2, q4 = lane & 3;
  const int b = blockIdx.x >> 1, g = blockIdx.x & 1;

  if (threadIdx.x == 0) {
    rm.nch = 0;
    mbar_init(smem_addr(&kv_full), 1);
    mbar_init_fence();
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
  }
  pdl_wait(); pdl_trigger();       // PDL: the prologue above overlapped the previous kernel's tail (common.cuh)
  if (threadIdx.x == 0) make_chunks(ch, a.ranges, b, a.Lk);
  for (int i = threadIdx.x; i < MAX_CH * KC; i += THREADS)
    s_mask[i] = i < a.Lk ? (a.key_mask ? a.key_mask[(long)b * a.Lk + i] : (unsigned char)1) : (unsigned char)0;
  __syncthreads();
  prepare_keys(ch, rm, kb, s_mask, a.causal, warp, lane);
  const int nch = ch.nch;
  auto load_kv = [&](int c) {
    const uint32_t bar = smem_addr(&kv_full);
    mbar_expect_tx(bar, 2 * TILE);
    tma_load_2d(base + OFF_K, &tmK, g * GF, ch.row[c], bar);
    tma_load_2d(base + OFF_K + PANEL, &tmK, g * GF + 64, ch.row[c], bar);
    tma_load_2d(base + OFF_V, &tmV, g * GF, ch.row[c], bar);
    tma_load_2d(base + OFF_V + PANEL, &tmV, g * GF + 64, ch.row[c], bar);
  };
  if (threadIdx.x == 0 && nch > 0) load_kv(0);       // the first K / V chunk flies while the A' tiles are built
  // dropped chunks (no valid key, the commit has valid keys elsewhere): their dK / dV rows are exactly zero
  for (int c = 0; c < rm.nch; ++c)
    for (int i = threadIdx.x; i < rm.n[c] * (GF / 8); i += THREADS) {
      const int r = i / (GF / 8), q = i % (GF / 8);
      const uint4 z = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(a.dk + (long)(rm.row[c] + r) * a.lddk + g * GF + q * 8) = z;
      *reinterpret_cast<uint4*>(a.dv + (long)(rm.row[c] + r) * a.lddv + g * GF + q * 8) = z;
    }
  build_masked_tile(sm + OFF_AQ, a.q, a.ldq, b, g, a.Lq, threadIdx.x, THREADS);
  __syncthreads();
  build_masked_tile(sm + OFF_ADO, a.d_ctx, a.ldo, b, g, a.Lq, threadIdx.x, THREADS);
  fence_proxy_async();
  __syncthreads();

  const FragRows fr = frag_rows(warp, lane);
  bool live[2], rowfilled[2];
  // delta = dO . O over the own head's 32 features; row statistics
  float delta[2], m2[2], inv[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int t = fr.t[h];
    live[h] = t < a.Lq;
    uint32_t any = 0;
    for (int c = 0; c < nch; ++c)
#pragma unroll
      for (int j = 0; j < 4; ++j) any |= row_bits(kb, ch, c, j, t, a.causal);
    rowfilled[h] = any == 0;
    delta[h] = 0.f; m2[h] = 0.f; inv[h] = 0.f;
    if (live[h]) {
      const __nv_bfloat16* orow = a.ctx + ((long)b * a.Lq + t) * a.ldo + g * GF + fr.hl * DH;
      const __nv_bfloat16* grow = a.d_ctx + ((long)b * a.Lq + t) * a.ldo + g * GF + fr.hl * DH;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float o[8], d[8];
        Act<__nv_bfloat16>::load8(orow + q * 8, o);
        Act<__nv_bfloat16>::load8(grow + q * 8, d);
#pragma unroll
        for (int i = 0; i < 8; ++i) delta[h] = fmaf(o[i], d[i], delta[h]);
      }
      const float* st = a.stats + (((long)b * a.H + g * HG + fr.hl) * a.Lq + t) * 2;
      m2[h] = st[0] * kLog2e; inv[h] = 1.f / st[1];
    }
  }
  const float k2 = a.scale * kLog2e;
  float dq[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) dq[i] = 0.f;
  for (int c = 0; c < nch; ++c) {
    if (c >= 1 && threadIdx.x == 0) load_kv(c);      // every warpgroup is done with the previous chunk (barrier below)
    mbar_wait(smem_addr(&kv_full), c & 1);
    // ---- S and dP, 64 keys at a time -> P and dS (bf16) into shared memory
#pragma unroll 1
    for (int kh = 0; kh < 2; ++kh) {
      float sv[32], dp[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) { sv[i] = 0.f; dp[i] = 0.f; }
      wgmma_fence();
#pragma unroll
      for (int kb_ = 0; kb_ < 2; ++kb_)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma<64, 0, 0>(sv, make_desc(base + OFF_AQ + kb_ * PANEL + wg * 8192 + k * 32, 16, 1024),
                          make_desc(base + OFF_K + kb_ * PANEL + kh * 8192 + k * 32, 16, 1024));
          wgmma<64, 0, 0>(dp, make_desc(base + OFF_ADO + kb_ * PANEL + wg * 8192 + k * 32, 16, 1024),
                          make_desc(base + OFF_V + kb_ * PANEL + kh * 8192 + k * 32, 16, 1024));
        }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence<32>(sv);
      reg_fence<32>(dp);
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int key = kh * 64 + 8 * jj + 2 * q4, grp = key >> 5, sh = key & 31;
        const uint32_t eb = kb.exist[c * 4 + grp] >> sh;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t vb = row_bits(kb, ch, c, grp, fr.t[h], a.causal) >> sh;
          float pv[2], dsv[2];
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const bool ok = live[h] && !rowfilled[h] && ((vb >> i) & 1);
            const float p = ok ? fast_exp2(fmaf(sv[4 * jj + 2 * h + i], k2, -m2[h])) * inv[h]
                               : ((live[h] && rowfilled[h] && ((eb >> i) & 1)) ? inv[h] : 0.f);
            pv[i] = p;
            dsv[i] = ok ? p * (dp[4 * jj + 2 * h + i] - delta[h]) * a.scale : 0.f;      // masked_fill blocks the gradient
          }
          const uint32_t off = pair_off(fr.mr[h], key);
          *reinterpret_cast<__nv_bfloat162*>(sm + OFF_P + off) = __floats2bfloat162_rn(pv[0], pv[1]);
          *reinterpret_cast<__nv_bfloat162*>(sm + OFF_DS + off) = __floats2bfloat162_rn(dsv[0], dsv[1]);
        }
      }
    }
    fence_proxy_async();
    named_bar(1, THREADS);                           // all 128 rows of P / dS are in shared memory
    // ---- dQ' += dS K     A: dS K-major (k-block = k>>2, 32 B per step)      B: K tile MN-major (16 key rows per step)
    // ---- dK = dS^T A'(Q)  A: dS MN-major (M = this warpgroup's 64 keys, K = rows)   B: A'(Q) MN-major (K = rows, N = features)
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      wgmma<128, 0, 1>(dq, make_desc(base + OFF_DS + (k >> 2) * PANEL + wg * 8192 + (k & 3) * 32, 16, 1024),
                       make_desc(base + OFF_K + k * 2048, PANEL, 1024));
      wgmma<128, 1, 1>(acc, make_desc(base + OFF_DS + wg * PANEL + k * 2048, PANEL, 1024),
                       make_desc(base + OFF_AQ + k * 2048, PANEL, 1024));
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<64>(dq);
    reg_fence<64>(acc);
    // dK / dV rows of this chunk: fragment row = key of the chunk, 128 features of the group
    auto store_rows = [&](__nv_bfloat16* dst, long ld) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ki = fr.mr[h];
        if (ki < ch.n[c]) {
          __nv_bfloat16* row = dst + (long)(ch.row[c] + ki) * ld + g * GF;
#pragma unroll
          for (int jj = 0; jj < 16; ++jj)
            *reinterpret_cast<__nv_bfloat162*>(row + 8 * jj + 2 * q4) = __floats2bfloat162_rn(acc[4 * jj + 2 * h], acc[4 * jj + 2 * h + 1]);
        }
      }
    };
    store_rows(a.dk, a.lddk);
    // ---- dV = P^T A'(dO)
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 8; ++k)
      wgmma<128, 1, 1>(acc, make_desc(base + OFF_P + wg * PANEL + k * 2048, PANEL, 1024),
                       make_desc(base + OFF_ADO + k * 2048, PANEL, 1024));
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<64>(acc);
    store_rows(a.dv, a.lddv);
    named_bar(1, THREADS);                           // K / V / P / dS free for the next chunk
  }
  // ---- dQ: own head's 32 columns (the scale is already folded into dS)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!live[h]) continue;
    __nv_bfloat16* dst = a.dq + ((long)b * a.Lq + fr.t[h]) * a.lddq + g * GF;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj)
      if ((jj >> 2) == fr.hl)
        *reinterpret_cast<__nv_bfloat162*>(dst + 8 * jj + 2 * q4) = __floats2bfloat162_rn(dq[4 * jj + 2 * h], dq[4 * jj + 2 * h + 1]);
  }
}

// max_chunks: 128-key chunks a commit needs (padded batches ceil(Lk / 128); packed batches every range starts its own
// chunk, the caller passes the maximum over its commits); Lk = mask pitch
inline bool eligible(int B, int H, int Lq, int Lk, int d_head, long ldk, long ldv, int max_chunks) {
  return d_head == DH && H == 2 * HG && Lq >= 1 && Lq <= 32 && Lk >= 1 && Lk <= MAX_CH * KC && max_chunks <= MAX_CH &&
         (ldk % 8) == 0 && (ldv % 8) == 0;
}

}  // namespace attn_tc

// called by fira_attn_fwd / fira_attn_bwd (attention.cu) for the bf16 mode; returns FIRA_OK or an error code
int fira_attn_tc_fwd(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                     const unsigned char* key_mask, const int* ranges, long kv_rows, int causal, void* ctx, long ldo,
                     float* stats, int B, int H, int Lq, int Lk, void* stream) {
  using namespace attn_tc;
  CUtensorMap tk, tv;
  int rc = tc::make_map_bf16(&tk, k, kv_rows, 2 * GF, ldk, 64, KC, "attn_tc_fwd");
  if (rc) return rc;
  if ((rc = tc::make_map_bf16(&tv, v, kv_rows, 2 * GF, ldv, 64, KC, "attn_tc_fwd"))) return rc;
  Args a{};
  a.q = (const __nv_bfloat16*)q; a.ldq = ldq; a.key_mask = key_mask; a.ranges = ranges; a.causal = causal; a.B = B; a.H = H; a.Lq = Lq;
  a.Lk = Lk; a.scale = 1.f / sqrtf((float)DH); a.ctx = (__nv_bfloat16*)ctx; a.ldo = ldo; a.stats = stats;
  const size_t smem = (1 + MAX_CH + 2 + 1) * (size_t)TILE + 1024;
  cudaError_t e = cudaFuncSetAttribute(attn_tc_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { fira_set_error(FIRA_ERR_CUDA, "attn_tc_fwd attr: %s", cudaGetErrorString(e)); return FIRA_ERR_CUDA; }
  launch_k(attn_tc_fwd_kernel, dim3(B * 2), dim3(THREADS), smem, (cudaStream_t)stream, tk, tv, a);
  FIRA_CHECK_LAUNCH("fira_attn_fwd (wgmma)");
  return FIRA_OK;
}

int fira_attn_tc_bwd(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                     const unsigned char* key_mask, const int* ranges, long kv_rows, int causal, const void* ctx,
                     const void* d_ctx, long ldo, const float* stats, void* dq, long lddq, void* dk, long lddk, void* dv,
                     long lddv, int B, int H, int Lq, int Lk, void* stream) {
  using namespace attn_tc;
  CUtensorMap tk, tv;
  int rc = tc::make_map_bf16(&tk, k, kv_rows, 2 * GF, ldk, 64, KC, "attn_tc_bwd");
  if (rc) return rc;
  if ((rc = tc::make_map_bf16(&tv, v, kv_rows, 2 * GF, ldv, 64, KC, "attn_tc_bwd"))) return rc;
  Args a{};
  a.q = (const __nv_bfloat16*)q; a.ldq = ldq; a.key_mask = key_mask; a.ranges = ranges; a.causal = causal; a.B = B; a.H = H; a.Lq = Lq;
  a.Lk = Lk; a.scale = 1.f / sqrtf((float)DH); a.ctx = (__nv_bfloat16*)const_cast<void*>(ctx); a.ldo = ldo;
  a.stats = const_cast<float*>(stats); a.d_ctx = (const __nv_bfloat16*)d_ctx;
  a.dq = (__nv_bfloat16*)dq; a.lddq = lddq; a.dk = (__nv_bfloat16*)dk; a.lddk = lddk; a.dv = (__nv_bfloat16*)dv; a.lddv = lddv;
  const size_t smem = 6 * (size_t)TILE + 1024;
  cudaError_t e = cudaFuncSetAttribute(attn_tc_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { fira_set_error(FIRA_ERR_CUDA, "attn_tc_bwd attr: %s", cudaGetErrorString(e)); return FIRA_ERR_CUDA; }
  launch_k(attn_tc_bwd_kernel, dim3(B * 2), dim3(THREADS), smem, (cudaStream_t)stream, tk, tv, a);
  FIRA_CHECK_LAUNCH("fira_attn_bwd (wgmma)");
  return FIRA_OK;
}

bool fira_attn_tc_eligible(int B, int H, int Lq, int Lk, int d_head, long ldk, long ldv, int max_chunks) {
  return attn_tc::eligible(B, H, Lq, Lk, d_head, ldk, ldv, max_chunks);
}
