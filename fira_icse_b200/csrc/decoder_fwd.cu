// The whole bf16 decoder forward (gnn_transformer.py:108-122: embedding + PE, then per layer masked self-attention,
// cross-attention over the encoder memory and the feed-forward block, each closed by dropout + residual + post-LN) as
// ONE launch: a cluster of two CTAs per commit carries the commit's rows (padded to 32) through every layer in shared
// memory.  Nothing in the decoder mixes commits, so no grid-wide synchronisation is needed; the per-layer chain of 11
// launches on 15 row tiles becomes a chain of barriers inside one cluster.
//
// Why two CTAs: the kernel is bound by streaming the weights (11 MB per commit) from L2 into each SM.  The pair splits
// every product by output columns (128-column blocks, gcol()), so each SM pulls half of every weight matrix and 2 B SMs
// work instead of B; the halves both CTAs need next (attention context, Z, the FFN hidden tile) are written into the
// shared memory of both (DSMEM) before a cluster barrier.
//
//   products   mma.sync.m16n8k16, fp32 accumulators.  A = the commit's [32][K] activations in shared memory (row pitch
//              K + 32 bf16: the 16-B fragment loads of a quarter warp cover all 32 banks), B = the layer's bf16 weight
//              mirror [N][K] read straight from global memory (L2) into registers, 16 B per lane and k32 step, prefetched
//              PF steps ahead.  Every warp owns whole output columns over all 32 rows, so each weight byte is read once
//              per cluster.  Inside a k32 step the K order is permuted identically for A and B (lane quad q holds
//              k 8q..8q+7), which only reorders the fp32 sum.  Epilogue: + bias (relu for FFN1), rounded to bf16 once, as
//              gemm_tc.
//   attention  the attn_mma_fwd_kernel math (attn_mma.cuh) for the CTA's 4 heads: warp w < 8 takes head w/2 and query
//              rows 16 (w % 2) ..; the Q / K / V products write their epilogue straight into swizzled [32][32] head tiles.
//              Self-attention: one 32-key block, causal over tar_mask.  Cross-attention: the commit's compacted key list
//              (key_mask / ranges exactly as fira_attn_fwd / fira_attn_packed_fwd), 32-key blocks of the layer's K / V
//              slice of the hoisted KV product, double-buffered by cp.async per head (each warp pair syncs on its own
//              named barrier).
//   LayerNorm  Z (bf16) staged in shared memory, then ln_fwd_kernel's arithmetic row by row (warp per row, lane per
//              8 features, same Philox dropout key), so the statistics come from the bf16-rounded Z; both CTAs normalise
//              every row, each stores the rows of its parity.
// Every tensor the backward reads is written in the layouts of the per-layer launch sequence, one row per slot: with a
// live-row map (fira_target_rows) only the rows t < tlen[b] of commit b, to slots toff[b] + t, the pad slots zeroed;
// without one the slot is the row b T + t.  The rows are computed as without a map, so a live row's values do not depend
// on it.  The output (the head's input) keeps the rows b T + t, zero past tlen[b].
#include <string.h>
#include <cooperative_groups.h>
#include "attn_mma.cuh"
#include "common.cuh"
#include "fira_b200.h"

namespace {

namespace cg = cooperative_groups;
using namespace mma;
using bf16 = __nv_bfloat16;

constexpr int D = 256, F = 1024, NH = 8;
constexpr int TP = 32;                       // rows per commit on chip (T <= 32)
constexpr int NWARP = 16, NTHR = NWARP * 32;
constexpr int LDA = D + 32, LDF = F + 32;    // row pitches (bf16) of the [32][256] and [32][1024] activation tiles
constexpr int XT = TP * LDA * 2;             // bytes of one [32][256] tile
constexpr int HT = TP * ROWB;                // bytes of one [32][32] head tile
constexpr int CKB = 32;                      // cross-attention keys per block
constexpr int MAX_LAYERS = 8;

struct LayerW {
  const bf16* wqkv; const float* bqkv;                                   // self-attention q|k|v  [768, 256]
  const bf16* swo; const float* sbo; const float* slw; const float* slb;  // self-attention out + LayerNorm
  const bf16* cwq; const float* cbq;                                     // cross-attention q
  const bf16* cwo; const float* cbo; const float* clw; const float* clb;  // cross-attention out + LayerNorm
  const bf16* w1; const float* b1; const bf16* w2; const float* b2;      // feed-forward
  const float* flw; const float* flb;
};
static_assert(sizeof(LayerW) == 18 * sizeof(void*), "LayerW is the host's [L][18] pointer table");

struct DecParams {
  const int* tar; const float* emb; const float* pe; const unsigned char* tar_mask;
  const bf16* kv; long ldkv;                    // [Ms, L*512]: layer i's K at column 512 i, V at 512 i + 256
  const unsigned char* mem_mask; const int* ranges; int S;
  bf16* X;                                      // [L][R][256]: every layer's input
  bf16* out;                                    // [B*T][256]: the last layer's output
  bf16* qkv; bf16* ctx1; float* st1; bf16* z1; float* ls1; bf16* x1;
  bf16* q; bf16* ctx2; float* st2; bf16* z2; float* ls2; bf16* x2;
  bf16* hh; bf16* z3; float* ls3;
  const int* tlen; const int* toff;             // the live-row map, or NULL: slot = row
  long R;                                       // slots of the saved tensors
  int B, T, L;
  float scale, p_drop;
  uint64_t seed; const uint64_t* seed_ctr; uint32_t stream_id;
  LayerW w[MAX_LAYERS];
};

// shared memory: five [32][256] tiles, one region for the head tiles / K-V stages / the FFN hidden tile, key list
constexpr int OFF_X = 0, OFF_X1 = XT, OFF_X2 = 2 * XT, OFF_Y = 3 * XT, OFF_Z = 4 * XT, OFF_BIG = 5 * XT;
constexpr int BIG_BYTES = TP * LDF * 2;        // the FFN hidden tile [32][1024]
static_assert(BIG_BYTES >= 12 * HT && BIG_BYTES >= 4 * HT + 2 * 2 * 4 * CKB * ROWB,
              "the region also holds the q|k|v head tiles of four heads, and their q tiles + two K / V stages");
constexpr int SMEM_FIXED = OFF_BIG + BIG_BYTES;

__device__ __forceinline__ uint32_t word(const uint4& v, int i) { return i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w; }
__device__ __forceinline__ uint4 ldg16(const bf16* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void pair_bar(int h) { asm volatile("bar.sync %0, 64;" ::"r"(1 + h) : "memory"); }

// acc[mt][j] = rows 16 mt .., columns n0 + 8 j .. of A W^T: A = [32][K] tile (pitch K + 32), W = [N][K] global
template <int K, int NT8, int PF>
__device__ __forceinline__ void warp_mma(float (&acc)[2][NT8][4], const bf16* As, const bf16* __restrict__ W, int n0,
                                         int lane) {
  constexpr int lda = K + 32;
  const int g = lane >> 2, q = lane & 3;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int j = 0; j < NT8; ++j) acc[mt][j][0] = acc[mt][j][1] = acc[mt][j][2] = acc[mt][j][3] = 0.f;
  const bf16* wp = W + (long)(n0 + g) * K + 8 * q;
  const bf16* ap = As + g * lda + 8 * q;
  constexpr int nks = K / 32;
  uint4 bq[PF][NT8];
#pragma unroll
  for (int s = 0; s < PF; ++s)
#pragma unroll
    for (int j = 0; j < NT8; ++j) bq[s][j] = ldg16(wp + (long)8 * j * K + 32 * s);
  for (int k0 = 0; k0 < nks; k0 += PF) {
#pragma unroll
    for (int s = 0; s < PF; ++s) {
      const int ks = k0 + s;
      uint4 a[2][2], b[NT8];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) a[mt][hr] = *reinterpret_cast<const uint4*>(ap + (16 * mt + 8 * hr) * lda + 32 * ks);
#pragma unroll
      for (int j = 0; j < NT8; ++j) {
        b[j] = bq[s][j];
        if (ks + PF < nks) bq[s][j] = ldg16(wp + (long)8 * j * K + 32 * (ks + PF));
      }
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          const uint32_t af[4] = {word(a[mt][0], 2 * h), word(a[mt][1], 2 * h), word(a[mt][0], 2 * h + 1),
                                  word(a[mt][1], 2 * h + 1)};
#pragma unroll
          for (int j = 0; j < NT8; ++j) mma16816(acc[mt][j], af, word(b[j], 2 * h), word(b[j], 2 * h + 1));
        }
    }
  }
}

// the columns a CTA of the pair computes: the 128-column blocks of rank r out of every 256 (q | k | v blocks of its four
// heads, half of every other product)
__device__ __forceinline__ int gcol(int n, int rank) { return ((n >> 7) << 8) + rank * 128 + (n & 127); }

// out = A W^T + bias (relu), rounded to bf16, over this CTA's N / 2 columns (local n -> weight row gcol(n)), the warps
// taking groups of 8 NT8 columns; epi(t, n, c, v) receives the packed pair of columns (c, c + 1) = local (n, n + 1) of
// row t
template <int K, int NT8, int PF, bool RELU, typename Epi>
__device__ __forceinline__ void product(const bf16* As, const bf16* __restrict__ W, const float* __restrict__ bias, int N,
                                        int rank, int warp, int lane, Epi epi) {
  const int g = lane >> 2, q = lane & 3;
  for (int n0 = 8 * NT8 * warp; n0 < N / 2; n0 += 8 * NT8 * NWARP) {
    const int c0 = gcol(n0, rank);                   // 8 NT8 <= 128 columns: one block
    float acc[2][NT8][4];
    warp_mma<K, NT8, PF>(acc, As, W, c0, lane);
#pragma unroll
    for (int j = 0; j < NT8; ++j) {
      const int n = n0 + 8 * j + 2 * q, c = c0 + 8 * j + 2 * q;
      const float2 bb = *reinterpret_cast<const float2*>(bias + c);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          float v0 = acc[mt][j][2 * hr] + bb.x, v1 = acc[mt][j][2 * hr + 1] + bb.y;
          if (RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
          epi(16 * mt + 8 * hr + g, n, c, pack_bf16(v0, v1));
        }
    }
  }
}

// byte offset of (row t, local column n) in the head tiles of this CTA's columns of a q | k | v product
__device__ __forceinline__ uint32_t head_off(int t, int n) {
  return (n >> 5) * HT + swz(t, (n & 31) >> 3) + (n & 7) * 2;
}

// rows t < T, this CTA's N / 2 columns of an output of width N to the global [T][N] rows at dst, a warp per row;
// src(t, n) = the shared-memory address of (row t, local column n)
template <typename Src>
__device__ __forceinline__ void copy_out(bf16* __restrict__ dst, int N, int T, int rank, int warp, int lane, Src src) {
  for (int t = warp; t < T; t += NWARP)
    for (int n = 8 * lane; n < N / 2; n += 256)
      *reinterpret_cast<uint4*>(dst + (long)t * N + gcol(n, rank)) = *reinterpret_cast<const uint4*>(src(t, n));
}

// out = LN(dropout(Z) + resid) * gamma + beta over the commit's rows, two per warp: ln_fwd_kernel's arithmetic and
// dropout key (global row r0 + t, 8 features per lane).  Both CTAs of the pair compute every row (the same values); Z,
// out and the statistics of the rows of parity `rank` go to global memory, row t < n to slot s0 + t.  Rows >= T of the
// shared-memory out are zeroed.  out_rows: og takes rows r0 + t < r0 + T instead -- zero from tl on, NaN for a live row
// without a slot (t >= n), so that a live-row count above the slots shows as a NaN loss.
__device__ __forceinline__ void ln_rows(const unsigned char* sm, int off_z, int off_res, int off_out, const float* gamma,
                                        const float* beta, bf16* __restrict__ zg, bf16* __restrict__ og,
                                        float* __restrict__ stats, long rows, long r0, long s0, int T, int n, int tl,
                                        bool out_rows, float p_drop, uint64_t seed, const uint64_t* seed_ctr,
                                        uint32_t sid, int rank, int warp, int lane) {
  if (seed_ctr) seed += *seed_ctr;
  float g[8], bt[8];
  Act<float>::load8(gamma + lane * 8, g);
  Act<float>::load8(beta + lane * 8, bt);
  const float keep_scale = p_drop > 0.f ? 1.f / (1.f - p_drop) : 1.f;
  for (int t = 2 * warp; t < 2 * warp + 2; ++t) {
    const int o = (t * LDA + lane * 8) * 2;
    bf16* os = (bf16*)(sm + off_out + o);
    if (t >= T) { *reinterpret_cast<uint4*>(os) = make_uint4(0, 0, 0, 0); continue; }
    const long r = r0 + t, sl = s0 + t;
    const bool mine = (t & 1) == rank;
    const uint4 zraw = *reinterpret_cast<const uint4*>(sm + off_z + o);
    if (mine && t < n) *reinterpret_cast<uint4*>(zg + sl * D + lane * 8) = zraw;
    float y[8], x[8];
    Act<bf16>::load8((const bf16*)&zraw, y);
    Act<bf16>::load8((const bf16*)(sm + off_res + o), x);
    if (p_drop > 0.f) {
      uint32_t m = dropout_keep8(seed, sid, (uint64_t)r * 32 + lane, p_drop);
#pragma unroll
      for (int i = 0; i < 8; ++i) y[i] = ((m >> i) & 1) ? y[i] * keep_scale : 0.f;
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { y[i] += x[i]; s += y[i]; }
    const float mean = warp_sum(s) * (1.f / D);
    float qv = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { float d = y[i] - mean; qv += d * d; }
    const float rstd = rsqrtf(warp_sum(qv) * (1.f / D) + kLnEps);
#pragma unroll
    for (int i = 0; i < 8; ++i) y[i] = (y[i] - mean) * rstd * g[i] + bt[i];
    Act<bf16>::store8(os, y);
    if (mine) {
      if (out_rows) {
        const uint32_t fill = t < tl ? 0x7fc07fc0u : 0u;      // bf16 NaN pairs / zeros
        *reinterpret_cast<uint4*>(og + r * D + lane * 8) =
            t < n ? *reinterpret_cast<const uint4*>(os) : make_uint4(fill, fill, fill, fill);
      } else if (t < n) {
        *reinterpret_cast<uint4*>(og + sl * D + lane * 8) = *reinterpret_cast<const uint4*>(os);
      }
      if (lane == 0 && t < n) { stats[sl] = mean; stats[rows + sl] = rstd; }
    }
  }
}

// the warp's 16 query rows of head h against one block of keys: o, (m, l) as in attn_mma_fwd_kernel
struct AttnRows {
  int t[2];
  RowKeys rk[2];
  float m[2], l[2], o[4][4];
  uint32_t qa[2][4];
  __device__ __forceinline__ void init(const unsigned char* qtile, int r0, int lane) {
    ld_a(qtile, r0, lane, qa);
    m[0] = m[1] = -INFINITY;
    l[0] = l[1] = 0.f;
#pragma unroll
    for (int n = 0; n < 4; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
#pragma unroll
    for (int r = 0; r < 2; ++r) t[r] = r0 + (lane >> 2) + 8 * r;
  }
  __device__ __forceinline__ void block(const unsigned char* kt, const unsigned char* vt, int causal, int c0, int nv,
                                        float k2, int lane) {
    float s[4][4];
#pragma unroll
    for (int n = 0; n < 4; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
    mma_abt(s, qa, kt, lane);
    softmax_pv(s, rk, causal, c0, nv, k2, m, l, o, vt, lane);
  }
  // normalised context into the [32][256] tiles of both CTAs (columns of head h), statistics of rows < T to st
  __device__ __forceinline__ void finish(unsigned char* ytile, unsigned char* ytile_peer, int h, int T, float* st,
                                         int lane) {
    softmax_finish(o, l, m, rk, t, T, st, lane);
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        const int off = (t[r] * LDA + h * DH + 8 * n + 2 * (lane & 3)) * 2;
        const uint32_t v = pack_bf16(o[n][2 * r], o[n][2 * r + 1]);
        *reinterpret_cast<uint32_t*>(ytile + off) = v;
        *reinterpret_cast<uint32_t*>(ytile_peer + off) = v;
      }
  }
};

// A cluster of two CTAs per commit: CTA `rank` computes the 128-column blocks gcol(., rank) of every product -- so each
// streams half of every weight matrix from L2 -- and attention for heads 4 rank .. 4 rank + 3 (warps 0-7: head
// 4 rank + w/2, query rows 16 (w % 2) ..).  Attention context, Z and the FFN hidden tile are written into the shared
// memory of both CTAs (DSMEM), followed by a cluster barrier; LayerNorm runs on full rows in both.  A remote write to a
// tile always comes after the cluster barrier that follows the partner's last read of it.
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(NTHR, 1)
decoder_fwd_kernel(const __grid_constant__ DecParams p) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  extern __shared__ __align__(16) unsigned char sm[];
  __shared__ int nv_s, filled_s, s0_s, n_s, tl_s;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  unsigned char* peer = cluster.map_shared_rank(sm, rank ^ 1);
  // (few values stay live across the layer loop: the products need the registers)
  const int b = blockIdx.x >> 1, T = p.T;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, hl = (warp >> 1) & 3, r0q = 16 * (warp & 1);
  const long grow0 = (long)b * T, R = p.R;
  int* kidx = reinterpret_cast<int*>(sm + SMEM_FIXED);
  bf16* Xs = (bf16*)(sm + OFF_X);
  bf16* Ys = (bf16*)(sm + OFF_Y);
  unsigned char* big = sm + OFF_BIG;
  auto to_both = [&](int off, uint32_t v) {
    *reinterpret_cast<uint32_t*>(sm + off) = v;
    *reinterpret_cast<uint32_t*>(peer + off) = v;
  };

  if (threadIdx.x == 0) {
    s0_s = p.toff ? p.toff[b] : (int)grow0;
    n_s = p.toff ? p.toff[b + 1] - s0_s : T;
    tl_s = p.tlen ? p.tlen[b] : T;
  }
  // pad slots [toff[B], R) of every saved bf16 tensor are zeroed (the backward's products read all R slots); a slot's
  // 4,096 columns of one layer are one uint4 per thread
  if (p.toff) {
    const int c = 8 * threadIdx.x;
    for (long sl = p.toff[p.B] + blockIdx.x; sl < R; sl += gridDim.x)
      for (int i = 0; i < p.L; ++i) {
        const long ro = i * R + sl;
        bf16* dst;
        switch (c >> 8) {
          case 0: dst = p.X + ro * D + c; break;
          case 1: dst = p.ctx1 + ro * D + c - 256; break;
          case 2: dst = p.z1 + ro * D + c - 512; break;
          case 3: dst = p.x1 + ro * D + c - 768; break;
          case 4: dst = p.q + ro * D + c - 1024; break;
          case 5: dst = p.ctx2 + ro * D + c - 1280; break;
          case 6: dst = p.z2 + ro * D + c - 1536; break;
          case 7: dst = p.x2 + ro * D + c - 1792; break;
          case 8: dst = p.z3 + ro * D + c - 2048; break;
          case 9: case 10: case 11: dst = p.qkv + ro * 3 * D + c - 2304; break;
          default: dst = p.hh + ro * F + c - 3072; break;
        }
        *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
      }
  }
  // cross-attention keys of the commit (the same for every layer)
  compact_keys(p.mem_mask ? p.mem_mask + (long)b * p.S : nullptr, p.S, 0, kidx, &nv_s, &filled_s,
               p.ranges ? p.ranges + 4 * b : nullptr);

  // embedding: dec_emb[tar] + PE (embed_rows_kernel), rows >= T zero
  for (int t = warp; t < TP; t += NWARP) {
    float v[8];
    if (t < T) {
      float pe[8];
      Act<float>::load8(p.emb + (long)p.tar[grow0 + t] * D + lane * 8, v);
      Act<float>::load8(p.pe + (long)t * D + lane * 8, pe);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] += pe[i];
      if ((t & 1) == rank && t < n_s) Act<bf16>::store8(p.X + ((long)s0_s + t) * D + lane * 8, v);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = 0.f;
    }
    Act<bf16>::store8(Xs + t * LDA + lane * 8, v);
  }
  cluster.sync();                                  // both CTAs run: their shared memory may be written

  for (int i = 0; i < p.L; ++i) {
    const LayerW& w = p.w[i];
    const long o256 = i * R * D, s0 = s0_s;
    const int n = n_s;

    // ---- masked self-attention (gnn_transformer.py:117-119): q | k | v of this CTA's heads stay local
    product<D, 1, 8, false>(Xs, w.wqkv, w.bqkv, 3 * D, rank, warp, lane,
                            [&](int t, int n, int, uint32_t v) { *reinterpret_cast<uint32_t*>(big + head_off(t, n)) = v; });
    __syncthreads();
    copy_out(p.qkv + (i * R + s0) * 3 * D, 3 * D, n, rank, warp, lane, [&](int t, int n) { return big + head_off(t, n); });
    if (warp < 8) {
      // causal over tar_mask, identity key list of the T target rows
      AttnArgs sa{};
      sa.causal = 1;
      sa.Lk = T;
      const uint32_t mb = causal_mask_bits(sa, p.tar_mask + grow0, lane);
      AttnRows ar;
      ar.init(big + hl * HT, r0q, lane);
#pragma unroll
      for (int r = 0; r < 2; ++r) ar.rk[r] = row_keys(sa, mb, T, false, ar.t[r]);
      ar.block(big + (4 + hl) * HT, big + (8 + hl) * HT, 1, 0, T, p.scale * kLog2e, lane);
      const int h = 4 * rank + hl;
      ar.finish(sm + OFF_Y, peer + OFF_Y, h, T, p.st1 + (((long)i * p.B + b) * NH + h) * T * 2, lane);
    }
    cluster.sync();
    copy_out(p.ctx1 + o256 + s0 * D, D, n, rank, warp, lane, [&](int t, int n) { return Ys + t * LDA + gcol(n, rank); });
    product<D, 1, 8, false>(Ys, w.swo, w.sbo, D, rank, warp, lane,
                            [&](int t, int, int c, uint32_t v) { to_both(OFF_Z + (t * LDA + c) * 2, v); });
    cluster.sync();
    ln_rows(sm, OFF_Z, OFF_X, OFF_X1, w.slw, w.slb, p.z1 + o256, p.x1 + o256, p.ls1 + 2 * i * R, R, grow0, s0, T, n,
            T, false, p.p_drop, p.seed, p.seed_ctr, p.stream_id + 8 * i + 0, rank, warp, lane);
    __syncthreads();

    // ---- cross-attention over the encoder memory (gnn_transformer.py:120): q of this CTA's heads stays local
    product<D, 1, 8, false>((const bf16*)(sm + OFF_X1), w.cwq, w.cbq, D, rank, warp, lane,
                            [&](int t, int n, int, uint32_t v) { *reinterpret_cast<uint32_t*>(big + head_off(t, n)) = v; });
    __syncthreads();
    copy_out(p.q + o256 + s0 * D, D, n, rank, warp, lane, [&](int t, int n) { return big + head_off(t, n); });
    if (warp < 8) {
      const int h = 4 * rank + hl;
      const int nv = nv_s, nblk = (nv + CKB - 1) / CKB;
      const float k2 = p.scale * kLog2e;
      const long kvb = p.ranges ? 0 : (long)b * p.S;   // with ranges kidx holds global rows
      const bf16* kh = p.kv + kvb * p.ldkv + (long)i * 2 * D + h * DH;
      const bf16* vh = kh + D;
      unsigned char* stage = big + 4 * HT;           // [2 stages][K, V][local head][CKB][32]
      auto kt = [&](int s) { return stage + ((s * 2 + 0) * 4 + hl) * CKB * ROWB; };
      auto vt = [&](int s) { return stage + ((s * 2 + 1) * 4 + hl) * CKB * ROWB; };
      const int tid = threadIdx.x & 63;
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        if (s < nblk) stage_kv(kt(s), vt(s), kh, p.ldkv, vh, p.ldkv, kidx, s * CKB, min(CKB, nv - s * CKB), CKB, tid, 64);
        cp_async_commit();
      }
      AttnRows ar;
      ar.init(big + hl * HT, r0q, lane);
      ar.rk[0] = ar.rk[1] = RowKeys{0u, filled_s != 0};
      for (int blk = 0; blk < nblk; ++blk) {
        cp_async_wait<1>();
        pair_bar(hl);                                  // block blk of the head is in shared memory
        ar.block(kt(blk & 1), vt(blk & 1), 0, blk * CKB, nv, k2, lane);
        pair_bar(hl);                                  // its stage is free
        if (blk + 2 < nblk)
          stage_kv(kt(blk & 1), vt(blk & 1), kh, p.ldkv, vh, p.ldkv, kidx, (blk + 2) * CKB,
                   min(CKB, nv - (blk + 2) * CKB), CKB, tid, 64);
        cp_async_commit();
      }
      ar.finish(sm + OFF_Y, peer + OFF_Y, h, T, p.st2 + (((long)i * p.B + b) * NH + h) * T * 2, lane);
    }
    cluster.sync();
    copy_out(p.ctx2 + o256 + s0 * D, D, n, rank, warp, lane, [&](int t, int n) { return Ys + t * LDA + gcol(n, rank); });
    product<D, 1, 8, false>(Ys, w.cwo, w.cbo, D, rank, warp, lane,
                            [&](int t, int, int c, uint32_t v) { to_both(OFF_Z + (t * LDA + c) * 2, v); });
    cluster.sync();
    ln_rows(sm, OFF_Z, OFF_X1, OFF_X2, w.clw, w.clb, p.z2 + o256, p.x2 + o256, p.ls2 + 2 * i * R, R, grow0, s0, T, n,
            T, false, p.p_drop, p.seed, p.seed_ctr, p.stream_id + 8 * i + 1, rank, warp, lane);
    __syncthreads();

    // ---- feed-forward (gnn_transformer.py:170-174)
    bf16* Hs = (bf16*)big;
    product<D, 2, 4, true>((const bf16*)(sm + OFF_X2), w.w1, w.b1, F, rank, warp, lane,
                           [&](int t, int, int c, uint32_t v) { to_both(OFF_BIG + (t * LDF + c) * 2, v); });
    cluster.sync();
    copy_out(p.hh + (i * R + s0) * F, F, n, rank, warp, lane, [&](int t, int n) { return Hs + t * LDF + gcol(n, rank); });
    product<F, 1, 8, false>(Hs, w.w2, w.b2, D, rank, warp, lane,
                            [&](int t, int, int c, uint32_t v) { to_both(OFF_Z + (t * LDA + c) * 2, v); });
    cluster.sync();
    const bool last = i == p.L - 1;
    ln_rows(sm, OFF_Z, OFF_X2, OFF_X, w.flw, w.flb, p.z3 + o256, last ? p.out : p.X + o256 + R * D, p.ls3 + 2 * i * R, R,
            grow0, s0, T, n, tl_s, last, p.p_drop, p.seed, p.seed_ctr, p.stream_id + 8 * i + 2, rank, warp, lane);
    __syncthreads();
  }
}

}  // namespace

extern "C" int fira_decoder_fwd_rows(const int* tar, const float* dec_emb, const float* pos_table,
                                     const unsigned char* tar_mask, const void* kv, long ldkv,
                                     const unsigned char* mem_mask, const int* ranges, int S,
                                     const void* const* layer_ptrs, int L, void* X, void* out, void* qkv, void* ctx1,
                                     float* st1, void* z1, float* ls1, void* x1, void* q, void* ctx2, float* st2,
                                     void* z2, float* ls2, void* x2, void* hh, void* z3, float* ls3, const int* tlen,
                                     const int* toff, long R, int B, int T, float p_drop, uint64_t seed,
                                     const uint64_t* seed_ctr, uint32_t stream_id, void* stream) {
  FIRA_CHECK_ARG(B > 0 && T > 0 && T <= TP, FIRA_ERR_SHAPE, "decoder_fwd: B %d, T %d (T <= 32)", B, T);
  FIRA_CHECK_ARG(L > 0 && L <= MAX_LAYERS, FIRA_ERR_SHAPE, "decoder_fwd: %d layers (1..%d)", L, MAX_LAYERS);
  FIRA_CHECK_ARG(S > 0, FIRA_ERR_SHAPE, "decoder_fwd: S %d", S);
  FIRA_CHECK_ARG(!tlen == !toff && (toff ? R > 0 && R <= (long)B * T : R == (long)B * T), FIRA_ERR_ARG,
                 "decoder_fwd: tlen and toff both or neither, 0 < R <= B*T (R = B*T without them)");
  FIRA_CHECK_ARG(mem_mask || ranges, FIRA_ERR_ARG, "decoder_fwd: mem_mask may only be NULL with ranges");
  FIRA_CHECK_ARG(layer_ptrs && tar && dec_emb && pos_table && tar_mask && kv, FIRA_ERR_ARG, "decoder_fwd: null input");
  FIRA_CHECK_ARG(fira_aligned16(kv) && ldkv % 8 == 0 && ldkv >= (long)L * 2 * D, FIRA_ERR_ALIGN,
                 "decoder_fwd: kv must be 16-B aligned with ldkv a multiple of 8 and >= L*512");
  void* outs[] = {X, out, qkv, ctx1, z1, x1, q, ctx2, z2, x2, hh, z3};
  for (void* o : outs) FIRA_CHECK_ARG(o && fira_aligned16(o), FIRA_ERR_ALIGN, "decoder_fwd: outputs must be 16-B aligned");
  FIRA_CHECK_ARG(st1 && ls1 && st2 && ls2 && ls3, FIRA_ERR_ARG, "decoder_fwd: null statistics");
  DecParams p{tar, dec_emb, pos_table, tar_mask, (const bf16*)kv, ldkv, mem_mask, ranges, S,
              (bf16*)X, (bf16*)out, (bf16*)qkv, (bf16*)ctx1, st1, (bf16*)z1, ls1, (bf16*)x1,
              (bf16*)q, (bf16*)ctx2, st2, (bf16*)z2, ls2, (bf16*)x2, (bf16*)hh, (bf16*)z3, ls3, tlen, toff, R,
              B, T, L, 1.f / sqrtf((float)DH), p_drop, seed, seed_ctr, stream_id, {}};
  for (int i = 0; i < L; ++i) {
    const void* const* t = layer_ptrs + 18 * i;
    for (int j = 0; j < 18; ++j)
      FIRA_CHECK_ARG(t[j] && fira_aligned16(t[j]), FIRA_ERR_ALIGN, "decoder_fwd: layer %d pointer %d null or unaligned", i, j);
    memcpy(&p.w[i], t, sizeof(LayerW));
  }
  const size_t smem = SMEM_FIXED + sizeof(int) * (size_t)S;
  FIRA_CHECK_ARG(smem <= 227 * 1024, FIRA_ERR_SHAPE, "decoder_fwd: S %d needs %zu B shared memory", S, smem);
  cudaError_t e = cudaFuncSetAttribute(decoder_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { fira_set_error(FIRA_ERR_CUDA, "decoder_fwd: %s", cudaGetErrorString(e)); return FIRA_ERR_CUDA; }
  launch_k(decoder_fwd_kernel, dim3(2 * B), dim3(NTHR), smem, (cudaStream_t)stream, p);
  FIRA_CHECK_LAUNCH("fira_decoder_fwd");
  return FIRA_OK;
}

extern "C" int fira_decoder_fwd(const int* tar, const float* dec_emb, const float* pos_table,
                                const unsigned char* tar_mask, const void* kv, long ldkv, const unsigned char* mem_mask,
                                const int* ranges, int S, const void* const* layer_ptrs, int L, void* X, void* qkv,
                                void* ctx1, float* st1, void* z1, float* ls1, void* x1, void* q, void* ctx2, float* st2,
                                void* z2, float* ls2, void* x2, void* hh, void* z3, float* ls3, int B, int T,
                                float p_drop, uint64_t seed, const uint64_t* seed_ctr, uint32_t stream_id,
                                void* stream) {
  FIRA_CHECK_ARG(X && L > 0 && B > 0 && T > 0, FIRA_ERR_ARG, "decoder_fwd: arguments");
  void* out = (bf16*)X + (long)L * B * T * D;
  return fira_decoder_fwd_rows(tar, dec_emb, pos_table, tar_mask, kv, ldkv, mem_mask, ranges, S, layer_ptrs, L, X, out,
                               qkv, ctx1, st1, z1, ls1, x1, q, ctx2, st2, z2, ls2, x2, hh, z3, ls3, nullptr, nullptr,
                               (long)B * T, B, T, p_drop, seed, seed_ctr, stream_id, stream);
}
