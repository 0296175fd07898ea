// Multi-head attention core (gnn_transformer.py:144-156), one CTA per (commit, head):
//     S = Q K^T / sqrt(d_head);  S[mask == 0] = -1e9;  P = softmax(S);  ctx = P V
// mask = key padding (and causal for decoder self-attention, gnn_transformer.py:117); no dropout on P.
//
// The problem is tiny (Lq = 30, Lk <= 370, d_head = 32) and mostly padding: on the DataSet only ~127 of the
// 370 memory rows are real.  exp(-1e9 - max) is exactly 0 in fp32, so masked keys contribute nothing --
// the kernels COMPACT the valid keys first (ballot scan into a shared index list) and only load / multiply
// those (3x less work on real data, bit-for-bit the same sums).  A fully masked row (all keys padded)
// keeps the reference's behaviour: uniform P over all keys, no gradient to the scores.
// Each warp handles two query rows at a time so every K / V shared-memory read feeds two rows.
// Forward saves (row max, row sum); backward recomputes P from them, gets delta = rowsum(P * dP) as
// dO . O (so keys can be processed in chunks of 64 with a small shared-memory footprint, 5 CTAs/SM)
// and writes zero gradients for the masked keys.
//
// bf16 activations run on the tensor cores (attn_mma_fwd/bwd_kernel below): the same key compaction, then warp-level
// mma.sync.m16n8k16 on register fragments.
#include <stdlib.h>
#include "attn_mma.cuh"
#include "common.cuh"
#include "fira_b200.h"

namespace {

// bf16 activations go to the tensor-core kernels unless FIRA_ATTN_TC=0 (A/B runs against the FFMA kernels below)
bool use_tc(int dtype) {
  if (dtype != FIRA_BF16) return false;
  const char* e = getenv("FIRA_ATTN_TC");      // read per call: an A/B switch, not cached process state
  return e ? atoi(e) != 0 : true;
}

constexpr int KPAD = DH + 1;     // conflict-free column reads of K/V tiles
constexpr int NWARPS = 8;
constexpr int NTHR = NWARPS * 32;
constexpr int KC = 128;          // keys per forward chunk
constexpr int KCB = 64;          // keys per backward chunk (42 KB shared memory -> 5 CTAs per SM)

// 16-byte loads of a 32-wide head slice; row index taken from `rows_idx` (compacted keys) or identity
template <typename T>
__device__ __forceinline__ void load_rows(float* dst, const T* src, long ld, const int* rows_idx, int row0, int nrows) {
  constexpr int EPV = 16 / sizeof(T);
  constexpr int VPR = DH / EPV;
#pragma unroll 4
  for (int idx = threadIdx.x; idx < nrows * VPR; idx += NTHR) {
    const int j = idx / VPR, c = idx % VPR;
    const int r = rows_idx ? rows_idx[row0 + j] : row0 + j;
    const uint4 raw = *reinterpret_cast<const uint4*>(src + (long)r * ld + c * EPV);
    float* o = dst + j * KPAD + c * EPV;
    if constexpr (sizeof(T) == 4) {
      o[0] = __uint_as_float(raw.x); o[1] = __uint_as_float(raw.y);
      o[2] = __uint_as_float(raw.z); o[3] = __uint_as_float(raw.w);
    } else {
      const __nv_bfloat162* hh = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
      for (int q = 0; q < 4; ++q) { const float2 f = __bfloat1622float2(hh[q]); o[2 * q] = f.x; o[2 * q + 1] = f.y; }
    }
  }
}

// ------------------------------------------------------------------------------------------------ forward
// Keys are consumed in chunks of KC with a running (max, sum, output) per query row (online softmax), so the
// shared-memory footprint is ~48 KB whatever Lk is: 4 CTAs per SM instead of 1 for Lk = 370.
constexpr int PAIRS_MAX = (LQ_MAX / 2 + NWARPS - 1) / NWARPS;      // query-row pairs per warp (2)

template <typename T>
__global__ void __launch_bounds__(NTHR) attn_fwd_kernel(AttnArgs a, T* __restrict__ ctx, long ldo,
                                                        float* __restrict__ stats /* [B,H,Lq,2] */) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  extern __shared__ float smem[];
  __shared__ int nv_s, filled_s;
  const int b = blockIdx.x / a.H, h = blockIdx.x % a.H;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* Ks = smem;                          // [KC][KPAD]
  float* Vs = Ks + KC * KPAD;                // [KC][KPAD]
  float* Qs = Vs + KC * KPAD;                // [Lq][KPAD]
  float* Ps = Qs + a.Lq * KPAD;              // [NWARPS][2][KC]
  int* kidx = reinterpret_cast<int*>(Ps + NWARPS * 2 * KC);   // [Lk]
  const unsigned char* km = a.key_mask ? a.key_mask + (long)b * a.Lk : nullptr;
  const int* rg = a.ranges ? a.ranges + 4 * b : nullptr;
  const long kvb = rg ? 0 : (long)b * a.Lk;                    // with ranges kidx holds global rows
  compact_keys(km, a.Lk, a.causal, kidx, &nv_s, &filled_s, rg);
  const int nv = nv_s;
  const bool filled = filled_s != 0;
  load_rows(Qs, (const T*)a.q + (long)b * a.Lq * a.ldq + h * DH, a.ldq, nullptr, 0, a.Lq);
  float* P0 = Ps + (warp * 2 + 0) * KC;
  float* P1 = Ps + (warp * 2 + 1) * KC;
  float m0[PAIRS_MAX], m1[PAIRS_MAX], l0[PAIRS_MAX], l1[PAIRS_MAX], o0[PAIRS_MAX], o1[PAIRS_MAX];
#pragma unroll
  for (int i = 0; i < PAIRS_MAX; ++i) { m0[i] = m1[i] = -INFINITY; l0[i] = l1[i] = 0.f; o0[i] = o1[i] = 0.f; }

  for (int c0 = 0; c0 < nv; c0 += KC) {
    const int nc = min(KC, nv - c0);
    __syncthreads();                                       // previous chunk consumed; Qs visible
    load_rows(Ks, (const T*)a.k + kvb * a.ldk + h * DH, a.ldk, kidx, c0, nc);
    load_rows(Vs, (const T*)a.v + kvb * a.ldv + h * DH, a.ldv, kidx, c0, nc);
    __syncthreads();
#pragma unroll
    for (int i = 0; i < PAIRS_MAX; ++i) {
      const int t0 = (warp + i * NWARPS) * 2;
      if (t0 < a.Lq) {
        const int t1 = min(t0 + 1, a.Lq - 1);              // odd Lq: row duplicated, second result dropped
        float q0[DH], q1[DH];
#pragma unroll
        for (int d = 0; d < DH; ++d) { q0[d] = Qs[t0 * KPAD + d]; q1[d] = Qs[t1 * KPAD + d]; }
        float cm0 = -INFINITY, cm1 = -INFINITY;
        for (int j = lane; j < nc; j += 32) {
          float s0 = 0.f, s1 = 0.f;
#pragma unroll
          for (int d = 0; d < DH; ++d) { const float kd = Ks[j * KPAD + d]; s0 = fmaf(q0[d], kd, s0); s1 = fmaf(q1[d], kd, s1); }
          const int ko = kidx[c0 + j];
          const bool pad = filled || (a.causal && km[ko] == 0);
          s0 = (pad || (a.causal && ko > t0)) ? kMaskFill : s0 * a.scale;
          s1 = (pad || (a.causal && ko > t1)) ? kMaskFill : s1 * a.scale;
          P0[j] = s0; P1[j] = s1;
          cm0 = fmaxf(cm0, s0); cm1 = fmaxf(cm1, s1);
        }
        const float nm0 = fmaxf(m0[i], warp_max(cm0)), nm1 = fmaxf(m1[i], warp_max(cm1));
        const float r0 = expf(m0[i] - nm0), r1 = expf(m1[i] - nm1);     // exp(-inf) = 0 on the first chunk
        float sum0 = 0.f, sum1 = 0.f;
        for (int j = lane; j < nc; j += 32) {
          const float e0 = expf(P0[j] - nm0), e1 = expf(P1[j] - nm1);
          P0[j] = e0; P1[j] = e1; sum0 += e0; sum1 += e1;
        }
        l0[i] = l0[i] * r0 + warp_sum(sum0);
        l1[i] = l1[i] * r1 + warp_sum(sum1);
        m0[i] = nm0; m1[i] = nm1;
        __syncwarp();
        float a0 = o0[i] * r0, a1 = o1[i] * r1;
        for (int j = 0; j < nc; ++j) { const float vv = Vs[j * KPAD + lane]; a0 = fmaf(P0[j], vv, a0); a1 = fmaf(P1[j], vv, a1); }
        o0[i] = a0; o1[i] = a1;
        __syncwarp();
      }
    }
  }
#pragma unroll
  for (int i = 0; i < PAIRS_MAX; ++i) {
    const int t0 = (warp + i * NWARPS) * 2;
    if (t0 < a.Lq) {
      const int t1 = min(t0 + 1, a.Lq - 1);
      Act<T>::st(ctx + ((long)b * a.Lq + t0) * ldo + h * DH + lane, o0[i] / l0[i]);
      if (t1 != t0) Act<T>::st(ctx + ((long)b * a.Lq + t1) * ldo + h * DH + lane, o1[i] / l1[i]);
      if (lane == 0 && stats) {
        float* st = stats + (((long)b * a.H + h) * a.Lq + t0) * 2;
        st[0] = m0[i]; st[1] = l0[i];
        if (t1 != t0) { st[2] = m1[i]; st[3] = l1[i]; }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward
// dV = P^T dO, dP = dO V^T, dS = P * (dP - delta), delta = dO . O, dQ = scale dS K, dK = scale dS^T Q.
template <typename T>
__global__ void __launch_bounds__(NTHR) attn_bwd_kernel(AttnArgs a, const T* __restrict__ out, const T* __restrict__ d_ctx,
                                                        long ldo, const float* __restrict__ stats, T* __restrict__ dq,
                                                        long lddq, T* __restrict__ dk, long lddk, T* __restrict__ dv,
                                                        long lddv) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  extern __shared__ float smem[];
  __shared__ int nv_s, filled_s;
  __shared__ float delta_s[LQ_MAX], mx_s[LQ_MAX], inv_s[LQ_MAX];
  const int b = blockIdx.x / a.H, h = blockIdx.x % a.H;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int PP = KCB + 1;
  float* Ks = smem;                          // [KCB][KPAD]
  float* Vs = Ks + KCB * KPAD;                // [KCB][KPAD]
  float* Qs = Vs + KCB * KPAD;                // [Lq][KPAD]
  float* Os = Qs + a.Lq * KPAD;              // [Lq][KPAD]  dO
  float* Pm = Os + a.Lq * KPAD;              // [Lq][PP]    P
  float* Sm = Pm + a.Lq * PP;                // [Lq][PP]    dS
  int* kidx = reinterpret_cast<int*>(Sm + a.Lq * PP);   // [Lk]
  const unsigned char* km = a.key_mask ? a.key_mask + (long)b * a.Lk : nullptr;
  const int* rg = a.ranges ? a.ranges + 4 * b : nullptr;
  const long kvb = rg ? 0 : (long)b * a.Lk;
  compact_keys(km, a.Lk, a.causal, kidx, &nv_s, &filled_s, rg);
  const int nv = nv_s;
  const bool filled = filled_s != 0;
  // delta_t = dO_t . O_t  (== sum_s P dP), row statistics
  load_rows(Qs, out + (long)b * a.Lq * ldo + h * DH, ldo, nullptr, 0, a.Lq);       // O, temporarily in Qs
  load_rows(Os, d_ctx + (long)b * a.Lq * ldo + h * DH, ldo, nullptr, 0, a.Lq);
  __syncthreads();
  for (int t = warp; t < a.Lq; t += NWARPS) {
    const float x = warp_sum(Qs[t * KPAD + lane] * Os[t * KPAD + lane]);
    if (lane == 0) {
      delta_s[t] = x;
      const float* st = stats + (((long)b * a.H + h) * a.Lq + t) * 2;
      mx_s[t] = st[0]; inv_s[t] = 1.f / st[1];
    }
  }
  __syncthreads();
  load_rows(Qs, (const T*)a.q + (long)b * a.Lq * a.ldq + h * DH, a.ldq, nullptr, 0, a.Lq);
  float dqa[(LQ_MAX + NWARPS - 1) / NWARPS];   // dQ[t][lane] for this warp's rows t = warp + 8*i
#pragma unroll
  for (int i = 0; i < (LQ_MAX + NWARPS - 1) / NWARPS; ++i) dqa[i] = 0.f;

  for (int c0 = 0; c0 < nv; c0 += KCB) {
    const int nc = min(KCB, nv - c0);
    __syncthreads();                                     // previous chunk fully consumed (and Qs loaded)
    load_rows(Ks, (const T*)a.k + kvb * a.ldk + h * DH, a.ldk, kidx, c0, nc);
    load_rows(Vs, (const T*)a.v + kvb * a.ldv + h * DH, a.ldv, kidx, c0, nc);
    __syncthreads();
    // ---- phase A: P, dS for the warp's query rows; dQ accumulation
#pragma unroll
    for (int i = 0; i < (LQ_MAX + NWARPS - 1) / NWARPS; ++i) {
      const int t = warp + i * NWARPS;
      if (t < a.Lq) {
        float qr[DH], orr[DH];
#pragma unroll
        for (int d = 0; d < DH; ++d) { qr[d] = Qs[t * KPAD + d]; orr[d] = Os[t * KPAD + d]; }
        const float mx = mx_s[t], inv = inv_s[t], dl = delta_s[t];
        for (int j = lane; j < nc; j += 32) {
          float sc = 0.f, dp = 0.f;
#pragma unroll
          for (int d = 0; d < DH; ++d) { sc = fmaf(qr[d], Ks[j * KPAD + d], sc); dp = fmaf(orr[d], Vs[j * KPAD + d], dp); }
          const bool masked = filled || (a.causal && (kidx[c0 + j] > t || km[kidx[c0 + j]] == 0));
          sc = masked ? kMaskFill : sc * a.scale;
          const float pr = expf(sc - mx) * inv;
          Pm[t * PP + j] = pr;
          Sm[t * PP + j] = masked ? 0.f : pr * (dp - dl);      // masked_fill blocks the gradient
        }
        __syncwarp();
        float g = 0.f;
        for (int j = 0; j < nc; ++j) g = fmaf(Sm[t * PP + j], Ks[j * KPAD + lane], g);
        dqa[i] += g;
      }
    }
    __syncthreads();
    // ---- phase B: dK, dV rows of this chunk (written at the keys' original positions)
    for (int j = warp; j < nc; j += NWARPS) {
      float gk = 0.f, gv = 0.f;
      for (int t = 0; t < a.Lq; ++t) {
        gk = fmaf(Sm[t * PP + j], Qs[t * KPAD + lane], gk);
        gv = fmaf(Pm[t * PP + j], Os[t * KPAD + lane], gv);
      }
      const long row = kvb + kidx[c0 + j];
      Act<T>::st(dk + row * lddk + h * DH + lane, gk * a.scale);
      Act<T>::st(dv + row * lddv + h * DH + lane, gv);
    }
  }
#pragma unroll
  for (int i = 0; i < (LQ_MAX + NWARPS - 1) / NWARPS; ++i) {
    const int t = warp + i * NWARPS;
    if (t < a.Lq) Act<T>::st(dq + ((long)b * a.Lq + t) * lddq + h * DH + lane, dqa[i] * a.scale);
  }
  // masked keys receive exactly zero gradient
  if (!filled && !a.causal && km) {
    const int L = rg ? rg[1] + rg[3] : a.Lk;
    for (int s = warp; s < L; s += NWARPS) {
      if (km[s] == 0) {
        const long row = rg ? (s < rg[1] ? rg[0] + s : rg[2] + (s - rg[1])) : (long)b * a.Lk + s;
        Act<T>::st(dk + row * lddk + h * DH + lane, 0.f);
        Act<T>::st(dv + row * lddv + h * DH + lane, 0.f);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ bf16 tensor cores
// One CTA per (commit, head) on the compacted key list, warp-level mma.sync.m16n8k16 (bf16 in, fp32 accumulate;
// the helpers are in attn_mma.cuh).
//   forward:  warp w = query rows [16 w, 16 w + 16); 64-key blocks, double-buffered by cp.async; online softmax
//             (ex2.approx) on the fragments; the row sum adds the bf16-rounded P that the P V product consumes.
//   backward: warp w = key blocks w, w + 3, ... of 32 keys, all query rows; S and dP recomputed, P from the saved
//             statistics, dS = P (dP - delta) scale; dQ += dS K into the warp's fp32 partial in shared memory (summed
//             over the warps at the end), dK = dS^T Q and dV = P^T dO from P / dS written to the warp's shared memory.
// Every key of a block is valid (compaction), except in causal self-attention (identity list, Lk <= 32) and in a
// commit without valid keys (every key of the list, uniform P) -- the same rules as the FFMA kernels.
namespace mma {

constexpr int FWARPS_MAX = LQ_MAX / 16;
constexpr int FKB = 64;          // forward keys per block
constexpr int FST = 2;           // forward K / V stages
constexpr int BWARPS = 3;
constexpr int BKB = 32;          // backward keys per warp block
constexpr int BWARP_SMEM = 4 * BKB * ROWB + LQ_MAX * DH * 4;   // K, V, P, dS, fp32 dQ partial of one warp
static_assert(LQ_MAX == 32 && BKB == 32, "tile shapes");

// float index of (row r, column f) of a [32][32] fp32 tile, float2 pairs XOR-swizzled by the row so that the
// accumulator fragment stores of a half warp (rows g, g + 1, .., 4 columns) hit distinct banks
__device__ __forceinline__ int swz_f32(int r, int f) { return r * DH + 2 * ((f >> 1) ^ ((r & 3) << 2)) + (f & 1); }

__global__ void __launch_bounds__(FWARPS_MAX * 32)
attn_mma_fwd_kernel(AttnArgs a, __nv_bfloat16* __restrict__ ctx, long ldo, float* __restrict__ stats /* [B,H,Lq,2] */) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  extern __shared__ __align__(16) unsigned char mma_smem[];
  __shared__ int nv_s, filled_s;
  unsigned char* Ks = mma_smem;                          // [FST][FKB][32]
  unsigned char* Vs = Ks + FST * FKB * ROWB;             // [FST][FKB][32]
  int* kidx = reinterpret_cast<int*>(Vs + FST * FKB * ROWB);
  const int b = blockIdx.x / a.H, h = blockIdx.x % a.H;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, q = lane & 3;
  const unsigned char* km = a.key_mask ? a.key_mask + (long)b * a.Lk : nullptr;
  const int* rg = a.ranges ? a.ranges + 4 * b : nullptr;
  const long kvb = rg ? 0 : (long)b * a.Lk;
  const __nv_bfloat16* kh = (const __nv_bfloat16*)a.k + kvb * a.ldk + h * DH;
  const __nv_bfloat16* vh = (const __nv_bfloat16*)a.v + kvb * a.ldv + h * DH;
  compact_keys(km, a.Lk, a.causal, kidx, &nv_s, &filled_s, rg);
  const int nv = nv_s;
  const int nblk = (nv + FKB - 1) / FKB;
#pragma unroll
  for (int s = 0; s < FST; ++s) {
    if (s < nblk)
      stage_kv(Ks + s * FKB * ROWB, Vs + s * FKB * ROWB, kh, a.ldk, vh, a.ldv, kidx, s * FKB, min(FKB, nv - s * FKB), FKB,
               threadIdx.x, blockDim.x);
    cp_async_commit();
  }
  // the warp's 16 query rows as A fragments, straight from global memory (rows >= Lq are zero)
  int t[2];
  uint32_t qa[2][4];
  RowKeys rk[2];
  const uint32_t mb = causal_mask_bits(a, km, lane);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    t[r] = 16 * warp + (lane >> 2) + 8 * r;
    const uint32_t* qr = reinterpret_cast<const uint32_t*>((const __nv_bfloat16*)a.q + ((long)b * a.Lq + t[r]) * a.ldq + h * DH);
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      qa[kk][r] = t[r] < a.Lq ? qr[8 * kk + q] : 0u;
      qa[kk][2 + r] = t[r] < a.Lq ? qr[8 * kk + 4 + q] : 0u;
    }
    rk[r] = row_keys(a, mb, nv, filled_s != 0, t[r]);
  }
  const float k2 = a.scale * kLog2e;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[4][4];
#pragma unroll
  for (int n = 0; n < 4; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;

  for (int i = 0; i < nblk; ++i) {
    cp_async_wait<FST - 1>();
    __syncthreads();                                     // block i is in shared memory for every warp
    const unsigned char* kt = Ks + (i % FST) * FKB * ROWB;
    const unsigned char* vt = Vs + (i % FST) * FKB * ROWB;
    const int c0 = i * FKB;
    float s[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
    mma_abt(s, qa, kt, lane);
    softmax_pv(s, rk, a.causal, c0, nv, k2, m, l, o, vt, lane);
    __syncthreads();                                     // stage i % FST is free
    if (i + FST < nblk)
      stage_kv(Ks + (i % FST) * FKB * ROWB, Vs + (i % FST) * FKB * ROWB, kh, a.ldk, vh, a.ldv, kidx, (i + FST) * FKB,
               min(FKB, nv - (i + FST) * FKB), FKB, threadIdx.x, blockDim.x);
    cp_async_commit();
  }
  softmax_finish(o, l, m, rk, t, a.Lq, stats ? stats + ((long)b * a.H + h) * a.Lq * 2 : nullptr, lane);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (t[r] >= a.Lq) continue;
    __nv_bfloat16* dst = ctx + ((long)b * a.Lq + t[r]) * ldo + h * DH + 2 * q;
#pragma unroll
    for (int n = 0; n < 4; ++n)
      *reinterpret_cast<__nv_bfloat162*>(dst + 8 * n) = __floats2bfloat162_rn(o[n][2 * r], o[n][2 * r + 1]);
  }
}

// Three warps of <= 152 registers and ~42 KB shared memory: 4 CTAs per SM, so the B * H = 512 CTAs of the bench step
// run in one wave on 132 SMs (four warps fit only 3 CTAs per SM, or spill at 128 registers).
__global__ void __launch_bounds__(BWARPS * 32, 1)
attn_mma_bwd_kernel(AttnArgs a, const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ d_ctx, long ldo,
                    const float* __restrict__ stats, __nv_bfloat16* __restrict__ dq, long lddq,
                    __nv_bfloat16* __restrict__ dk, long lddk, __nv_bfloat16* __restrict__ dv, long lddv) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  // with qoff, a.Lq / a.Lk become the commit's query rows (and causal keys) from here on; sp / kp keep the pitches
  const int sp = a.Lq, kp = a.Lk;
  const long qb = a.qoff ? (long)a.qoff[blockIdx.x / a.H] : (long)(blockIdx.x / a.H) * sp;
  if (a.qoff) {
    a.Lq = a.qoff[blockIdx.x / a.H + 1] - (int)qb;
    if (a.causal) a.Lk = a.Lq;
    if (blockIdx.x / a.H == a.B - 1) {           // the last commit's CTAs zero the head's columns of the pad rows
      const int h = blockIdx.x % a.H;
      const long p0 = a.qoff[a.B];
      for (long i = threadIdx.x; i < (a.qrows - p0) * 4; i += blockDim.x) {
        const long r = p0 + (i >> 2);
        const int c = (int)(i & 3) * 8 + h * DH;
        *reinterpret_cast<uint4*>(dq + r * lddq + c) = make_uint4(0, 0, 0, 0);
        if (a.causal) {
          *reinterpret_cast<uint4*>(dk + r * lddk + c) = make_uint4(0, 0, 0, 0);
          *reinterpret_cast<uint4*>(dv + r * lddv + c) = make_uint4(0, 0, 0, 0);
        }
      }
    }
  }
  extern __shared__ __align__(16) unsigned char mma_smem[];
  __shared__ int nv_s, filled_s;
  __shared__ float delta_s[LQ_MAX], m2_s[LQ_MAX], inv_s[LQ_MAX];
  unsigned char* Qs = mma_smem;                          // [32][32]
  unsigned char* Os = Qs + LQ_MAX * ROWB;                // [32][32] dO
  unsigned char* Ws = Os + LQ_MAX * ROWB;                // per warp: K, V [BKB][32]; P, dS [32 rows][BKB keys]; dQ
  int* kidx = reinterpret_cast<int*>(Ws + BWARPS * BWARP_SMEM);
  const int b = blockIdx.x / a.H, h = blockIdx.x % a.H;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, q = lane & 3;
  const unsigned char* km = a.key_mask ? a.key_mask + (long)b * kp : nullptr;
  const int* rg = a.ranges ? a.ranges + 4 * b : nullptr;
  const long kvb = rg ? 0 : a.qoff && a.causal ? qb : (long)b * kp;
  const __nv_bfloat16* kh = (const __nv_bfloat16*)a.k + kvb * a.ldk + h * DH;
  const __nv_bfloat16* vh = (const __nv_bfloat16*)a.v + kvb * a.ldv + h * DH;
  unsigned char* Kw = Ws + warp * BWARP_SMEM;
  unsigned char* Vw = Kw + BKB * ROWB;
  unsigned char* Pw = Vw + BKB * ROWB;
  unsigned char* Sw = Pw + LQ_MAX * ROWB;
  float* dQw = reinterpret_cast<float*>(Sw + LQ_MAX * ROWB);   // [32][32] fp32, swz_f32
  compact_keys(km, a.Lk, a.causal, kidx, &nv_s, &filled_s, rg);
  const int nv = nv_s;
  const bool filled = filled_s != 0;
  if (warp * BKB < nv) stage_kv(Kw, Vw, kh, a.ldk, vh, a.ldv, kidx, warp * BKB, min(BKB, nv - warp * BKB), BKB, lane, 32);
  for (int i = threadIdx.x; i < 2 * LQ_MAX * 4; i += blockDim.x) {
    const int which = i / (LQ_MAX * 4), r = (i >> 2) & (LQ_MAX - 1), c = i & 3;
    unsigned char* dst = (which ? Os : Qs) + swz(r, c);
    if (r < a.Lq) cp_async16(su32(dst), which ? d_ctx + (qb + r) * ldo + h * DH + c * 8
                                              : (const __nv_bfloat16*)a.q + (qb + r) * a.ldq + h * DH + c * 8);
    else *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
  }
  cp_async_commit();
  // delta_t = dO_t . O_t over the head's 32 features; row statistics
  if (threadIdx.x < a.Lq) {
    const int t = threadIdx.x;
    const __nv_bfloat16* orow = out + (qb + t) * ldo + h * DH;
    const __nv_bfloat16* grow = d_ctx + (qb + t) * ldo + h * DH;
    float d = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float ov[8], gv[8];
      Act<__nv_bfloat16>::load8(orow + c * 8, ov);
      Act<__nv_bfloat16>::load8(grow + c * 8, gv);
#pragma unroll
      for (int e = 0; e < 8; ++e) d = fmaf(ov[e], gv[e], d);
    }
    const float* st = stats + (((long)b * a.H + h) * sp + t) * 2;
    delta_s[t] = d; m2_s[t] = st[0] * kLog2e; inv_s[t] = 1.f / st[1];
  }
  // masked keys receive exactly zero gradient (the mask bytes of 32 keys per ballot, then one row per lane group)
  if (!filled && !a.causal && km) {
    const int L = rg ? rg[1] + rg[3] : a.Lk;
    for (int s0 = 32 * warp; s0 < L; s0 += 32 * BWARPS) {
      uint32_t dead = __ballot_sync(0xffffffffu, s0 + lane < L && km[s0 + lane] == 0);
      while (dead) {
        const int s = s0 + __ffs(dead) - 1;
        dead &= dead - 1;
        const long row = rg ? (s < rg[1] ? rg[0] + s : rg[2] + (s - rg[1])) : (long)b * a.Lk + s;
        dk[row * lddk + h * DH + lane] = __float2bfloat16_rn(0.f);
        dv[row * lddv + h * DH + lane] = __float2bfloat16_rn(0.f);
      }
    }
  }
  cp_async_wait<0>();
  __syncthreads();

  const float k2 = a.scale * kLog2e;
  const uint32_t mb = causal_mask_bits(a, km, lane);
  for (int i = lane; i < LQ_MAX * DH / 4; i += 32) reinterpret_cast<float4*>(dQw)[i] = make_float4(0.f, 0.f, 0.f, 0.f);

  for (int blk = warp; blk * BKB < nv; blk += BWARPS) {
    const int c0 = blk * BKB, nc = min(BKB, nv - c0);
    if (blk != warp) {
      __syncwarp();                                      // the previous block's tiles are consumed
      stage_kv(Kw, Vw, kh, a.ldk, vh, a.ldv, kidx, c0, nc, BKB, lane, 32);
      cp_async_commit();
      cp_async_wait<0>();
    }
    __syncwarp();
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      if (16 * mt < a.Lq) {
        // S = Q K^T -> P (kept in s) ; dP = dO V^T -> dS = P (dP - delta) scale (in s)
        uint32_t fa[2][4];
        float s[4][4], dp[4][4];
#pragma unroll
        for (int n = 0; n < 4; ++n)
#pragma unroll
          for (int e = 0; e < 4; ++e) s[n][e] = dp[n][e] = 0.f;
        ld_a(Qs, 16 * mt, lane, fa);
        mma_abt(s, fa, Kw, lane);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int t = 16 * mt + (lane >> 2) + 8 * r;
          const bool live = t < a.Lq;
          const float m2 = live ? m2_s[t] : 0.f, inv = live ? inv_s[t] : 0.f;
          const RowKeys k = row_keys(a, mb, nv, filled, t);
#pragma unroll
          for (int n = 0; n < 4; ++n) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const bool ok = live && key_ok(k, a.causal, c0 + 8 * n + 2 * q + e, nv);
              float& x = s[n][2 * r + e];
              x = !ok ? 0.f : (k.fill ? inv : ex2(fmaf(x, k2, -m2)) * inv);
            }
            *reinterpret_cast<uint32_t*>(Pw + swz(t, n) + 4 * q) = pack_bf16(s[n][2 * r], s[n][2 * r + 1]);
          }
        }
        ld_a(Os, 16 * mt, lane, fa);
        mma_abt(dp, fa, Vw, lane);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int t = 16 * mt + (lane >> 2) + 8 * r;
          const float dl = t < a.Lq ? delta_s[t] : 0.f;
          const bool fill = row_keys(a, mb, nv, filled, t).fill;        // masked_fill blocks the gradient
#pragma unroll
          for (int n = 0; n < 4; ++n) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float& x = s[n][2 * r + e];                 // P = 0 where the key is not valid for the row
              x = fill ? 0.f : x * (dp[n][2 * r + e] - dl) * a.scale;
            }
            *reinterpret_cast<uint32_t*>(Sw + swz(t, n) + 4 * q) = pack_bf16(s[n][2 * r], s[n][2 * r + 1]);
          }
        }
        // dQ += dS K (each lane owns its fragment's elements of the warp's dQ partial)
        float dqa[4][4];
#pragma unroll
        for (int n = 0; n < 4; ++n) dqa[n][0] = dqa[n][1] = dqa[n][2] = dqa[n][3] = 0.f;
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
          uint32_t da[4];
          acc_to_a(s, kk, da);
          mma_ax(dqa, da, Kw, kk, lane);
        }
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
          for (int n = 0; n < 4; ++n) {
            float2& d = *reinterpret_cast<float2*>(dQw + swz_f32(16 * mt + (lane >> 2) + 8 * r, 8 * n + 2 * q));
            d.x += dqa[n][2 * r];
            d.y += dqa[n][2 * r + 1];
          }
      }
    }
    __syncwarp();                                        // P / dS of the block are in shared memory
    // dK = dS^T Q, dV = P^T dO: M = the block's keys, K = query rows, N = features
#pragma unroll 1
    for (int which = 0; which < 2; ++which) {
      const unsigned char* At = which ? Pw : Sw;
      const unsigned char* Bt = which ? Os : Qs;
      float acc[2][4][4];
#pragma unroll
      for (int mk = 0; mk < 2; ++mk)
#pragma unroll
        for (int n = 0; n < 4; ++n) acc[mk][n][0] = acc[mk][n][1] = acc[mk][n][2] = acc[mk][n][3] = 0.f;
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        if (16 * kk >= a.Lq) break;
#pragma unroll
        for (int mk = 0; mk < 2; ++mk) {
          uint32_t at[4];
          ldsm4_t(su32(At + swz(16 * kk + (lane & 7) + (lane >> 4) * 8, 2 * mk + ((lane >> 3) & 1))), at);
          mma_ax(acc[mk], at, Bt, kk, lane);
        }
      }
      __nv_bfloat16* dst = which ? dv : dk;
      const long ld = which ? lddv : lddk;
#pragma unroll
      for (int mk = 0; mk < 2; ++mk)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int j = 16 * mk + (lane >> 2) + 8 * r;
          if (j < nc) {
            __nv_bfloat16* row = dst + (kvb + kidx[c0 + j]) * ld + h * DH + 2 * q;
#pragma unroll
            for (int n = 0; n < 4; ++n)
              *reinterpret_cast<__nv_bfloat162*>(row + 8 * n) = __floats2bfloat162_rn(acc[mk][n][2 * r], acc[mk][n][2 * r + 1]);
          }
        }
    }
  }
  // dQ: the sum of the warps' partials
  __syncthreads();
  for (int i = threadIdx.x; i < a.Lq * DH; i += blockDim.x) {
    const int t = i / DH, f = i % DH;
    float x = 0.f;
#pragma unroll
    for (int w = 0; w < BWARPS; ++w)
      x += reinterpret_cast<const float*>(Ws + w * BWARP_SMEM + 4 * BKB * ROWB)[swz_f32(t, f)];
    dq[(qb + t) * lddq + h * DH + f] = __float2bfloat16_rn(x);
  }
}

size_t fwd_smem(int Lk) { return (size_t)2 * FST * FKB * ROWB + sizeof(int) * (size_t)Lk; }
size_t bwd_smem(int Lk) { return (size_t)2 * LQ_MAX * ROWB + (size_t)BWARPS * BWARP_SMEM + sizeof(int) * (size_t)Lk; }

}  // namespace mma

size_t fwd_smem(int Lq, int Lk) {
  return sizeof(float) * ((size_t)2 * KC * KPAD + (size_t)Lq * KPAD + (size_t)NWARPS * 2 * KC) + sizeof(int) * (size_t)Lk;
}
size_t bwd_smem(int Lq, int Lk) {
  return sizeof(float) * ((size_t)2 * KCB * KPAD + (size_t)2 * Lq * KPAD + (size_t)2 * Lq * (KCB + 1)) +
         sizeof(int) * (size_t)Lk;
}

template <typename K>
int set_smem(K kernel, size_t bytes, const char* name) {
  if (bytes > 227 * 1024) {
    fira_set_error(FIRA_ERR_SHAPE, "%s: needs %zu B shared memory (> 227 KB)", name, bytes);
    return FIRA_ERR_SHAPE;
  }
  if (bytes > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) { fira_set_error(FIRA_ERR_CUDA, "%s: %s", name, cudaGetErrorString(e)); return FIRA_ERR_CUDA; }
  }
  return FIRA_OK;
}

int check_layout(const char* name, const void* p, long ld, int dtype) {
  const long esz = dtype == FIRA_F32 ? 4 : 2;
  if ((reinterpret_cast<uintptr_t>(p) & 15) != 0 || (ld * esz) % 16 != 0) {
    fira_set_error(FIRA_ERR_ALIGN, "%s: operands must be 16-B aligned with 16-B row pitch", name);
    return FIRA_ERR_ALIGN;
  }
  return FIRA_OK;
}

}  // namespace

namespace {

int attn_fwd_impl(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                  const unsigned char* key_mask, const int* ranges, int causal, void* ctx, long ldo, float* stats, int B, int H, int Lq, int Lk, int d_head, int dtype, void* stream) {
  FIRA_CHECK_ARG(d_head == DH, FIRA_ERR_SHAPE, "attn_fwd: d_head %d != 32", d_head);
  FIRA_CHECK_ARG(B > 0 && H > 0 && Lq > 0 && Lk > 0 && Lq <= LQ_MAX, FIRA_ERR_SHAPE, "attn_fwd: shape (Lq <= 32)");
  FIRA_CHECK_ARG(!causal || (Lq == Lk && !ranges), FIRA_ERR_SHAPE, "attn_fwd: causal needs Lq == Lk and no ranges");
  FIRA_CHECK_ARG(key_mask || ranges, FIRA_ERR_ARG, "attn_fwd: key_mask may only be NULL with ranges");
  FIRA_CHECK_ARG(dtype == FIRA_F32 || dtype == FIRA_BF16, FIRA_ERR_DTYPE, "attn_fwd: dtype %d", dtype);
  int rc;
  if ((rc = check_layout("attn_fwd", q, ldq, dtype)) || (rc = check_layout("attn_fwd", k, ldk, dtype)) ||
      (rc = check_layout("attn_fwd", v, ldv, dtype)))
    return rc;
  AttnArgs a{q, ldq, k, ldk, v, ldv, key_mask, ranges, causal, B, H, Lq, Lk, 1.f / sqrtf((float)d_head)};
  if (use_tc(dtype)) {
    const size_t smem = mma::fwd_smem(Lk);
    if ((rc = set_smem(mma::attn_mma_fwd_kernel, smem, "attn_fwd"))) return rc;
    launch_k(mma::attn_mma_fwd_kernel, dim3(B * H), dim3(32 * ((Lq + 15) / 16)), smem, (cudaStream_t)stream, a,
             (__nv_bfloat16*)ctx, ldo, stats);
    FIRA_CHECK_LAUNCH("fira_attn_fwd (mma)");
    return FIRA_OK;
  }
  const size_t smem = fwd_smem(Lq, Lk);
  if (dtype == FIRA_F32) {
    if ((rc = set_smem(attn_fwd_kernel<float>, smem, "attn_fwd"))) return rc;
    launch_k(attn_fwd_kernel<float>, dim3(B * H), dim3(NTHR), smem, (cudaStream_t)stream, a, (float*)ctx, ldo, stats);
  } else {
    if ((rc = set_smem(attn_fwd_kernel<__nv_bfloat16>, smem, "attn_fwd"))) return rc;
    launch_k(attn_fwd_kernel<__nv_bfloat16>, dim3(B * H), dim3(NTHR), smem, (cudaStream_t)stream, a, (__nv_bfloat16*)ctx, ldo, stats);
  }
  FIRA_CHECK_LAUNCH("fira_attn_fwd");
  return FIRA_OK;
}

int attn_bwd_impl(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                  const unsigned char* key_mask, const int* ranges, int causal, const void* ctx, const void* d_ctx, long ldo, const float* stats, void* dq, long lddq, void* dk,
                  long lddk, void* dv, long lddv, int B, int H, int Lq, int Lk, int d_head, int dtype, void* stream,
                  const int* qoff = nullptr, long qrows = 0) {
  FIRA_CHECK_ARG(d_head == DH, FIRA_ERR_SHAPE, "attn_bwd: d_head %d != 32", d_head);
  FIRA_CHECK_ARG(B > 0 && H > 0 && Lq > 0 && Lk > 0 && Lq <= LQ_MAX, FIRA_ERR_SHAPE, "attn_bwd: shape (Lq <= 32)");
  FIRA_CHECK_ARG(key_mask || ranges, FIRA_ERR_ARG, "attn_bwd: key_mask may only be NULL with ranges");
  FIRA_CHECK_ARG(dtype == FIRA_F32 || dtype == FIRA_BF16, FIRA_ERR_DTYPE, "attn_bwd: dtype %d", dtype);
  int rc;
  if ((rc = check_layout("attn_bwd", q, ldq, dtype)) || (rc = check_layout("attn_bwd", k, ldk, dtype)) ||
      (rc = check_layout("attn_bwd", v, ldv, dtype)) || (rc = check_layout("attn_bwd", ctx, ldo, dtype)) ||
      (rc = check_layout("attn_bwd", d_ctx, ldo, dtype)))
    return rc;
  AttnArgs a{q, ldq, k, ldk, v, ldv, key_mask, ranges, causal, B, H, Lq, Lk, 1.f / sqrtf((float)d_head), qoff, qrows};
  FIRA_CHECK_ARG(!qoff || (dtype == FIRA_BF16 && (lddk % 8) == 0 && (lddv % 8) == 0 && (lddq % 8) == 0 &&
                           (!causal || (Lq == Lk && !ranges))),
                 FIRA_ERR_ARG, "attn_bwd_rows: bf16, 16-B gradient pitches, causal with Lq == Lk and no ranges");
  if (qoff || (use_tc(dtype) && (lddk % 8) == 0 && (lddv % 8) == 0 && (lddq % 8) == 0)) {
    const size_t smem = mma::bwd_smem(Lk);
    if ((rc = set_smem(mma::attn_mma_bwd_kernel, smem, "attn_bwd"))) return rc;
    launch_k(mma::attn_mma_bwd_kernel, dim3(B * H), dim3(mma::BWARPS * 32), smem, (cudaStream_t)stream, a,
             (const __nv_bfloat16*)ctx, (const __nv_bfloat16*)d_ctx, ldo, stats, (__nv_bfloat16*)dq, lddq,
             (__nv_bfloat16*)dk, lddk, (__nv_bfloat16*)dv, lddv);
    FIRA_CHECK_LAUNCH("fira_attn_bwd (mma)");
    return FIRA_OK;
  }
  const size_t smem = bwd_smem(Lq, Lk);
  if (dtype == FIRA_F32) {
    if ((rc = set_smem(attn_bwd_kernel<float>, smem, "attn_bwd"))) return rc;
    launch_k(attn_bwd_kernel<float>, dim3(B * H), dim3(NTHR), smem, (cudaStream_t)stream, 
        a, (const float*)ctx, (const float*)d_ctx, ldo, stats, (float*)dq, lddq, (float*)dk, lddk, (float*)dv, lddv);
  } else {
    if ((rc = set_smem(attn_bwd_kernel<__nv_bfloat16>, smem, "attn_bwd"))) return rc;
    launch_k(attn_bwd_kernel<__nv_bfloat16>, dim3(B * H), dim3(NTHR), smem, (cudaStream_t)stream, 
        a, (const __nv_bfloat16*)ctx, (const __nv_bfloat16*)d_ctx, ldo, stats, (__nv_bfloat16*)dq, lddq,
        (__nv_bfloat16*)dk, lddk, (__nv_bfloat16*)dv, lddv);
  }
  FIRA_CHECK_LAUNCH("fira_attn_bwd");
  return FIRA_OK;
}

}  // namespace

extern "C" {

int fira_attn_fwd(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                  const unsigned char* key_mask, int causal, void* ctx, long ldo, float* stats, int B, int H, int Lq,
                  int Lk, int d_head, int dtype, void* stream) {
  FIRA_CHECK_ARG(key_mask, FIRA_ERR_ARG, "attn_fwd: null key_mask");
  return attn_fwd_impl(q, ldq, k, ldk, v, ldv, key_mask, nullptr, causal, ctx, ldo, stats,
                       B, H, Lq, Lk, d_head, dtype, stream);
}

int fira_attn_bwd(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                  const unsigned char* key_mask, int causal, const void* ctx, const void* d_ctx, long ldo,
                  const float* stats, void* dq, long lddq, void* dk, long lddk, void* dv, long lddv, int B, int H,
                  int Lq, int Lk, int d_head, int dtype, void* stream) {
  FIRA_CHECK_ARG(key_mask, FIRA_ERR_ARG, "attn_bwd: null key_mask");
  return attn_bwd_impl(q, ldq, k, ldk, v, ldv, key_mask, nullptr, causal, ctx, d_ctx, ldo,
                       stats, dq, lddq, dk, lddk, dv, lddv, B, H, Lq, Lk, d_head, dtype, stream);
}

int fira_attn_packed_fwd(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv, const int* ranges,
                         long kv_rows, const unsigned char* key_mask, int mask_pitch, int max_chunks, void* ctx, long ldo,
                         float* stats, int B, int H, int Lq, int d_head, int dtype, void* stream) {
  FIRA_CHECK_ARG(ranges && kv_rows > 0, FIRA_ERR_ARG, "attn_packed_fwd: ranges / kv_rows");
  return attn_fwd_impl(q, ldq, k, ldk, v, ldv, key_mask, ranges, 0, ctx, ldo, stats, B, H, Lq,
                       mask_pitch, d_head, dtype, stream);
}

int fira_attn_packed_bwd(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv, const int* ranges,
                         long kv_rows, const unsigned char* key_mask, int mask_pitch, int max_chunks, const void* ctx,
                         const void* d_ctx, long ldo, const float* stats, void* dq, long lddq, void* dk, long lddk,
                         void* dv, long lddv, int B, int H, int Lq, int d_head, int dtype, void* stream) {
  FIRA_CHECK_ARG(ranges && kv_rows > 0, FIRA_ERR_ARG, "attn_packed_bwd: ranges / kv_rows");
  return attn_bwd_impl(q, ldq, k, ldk, v, ldv, key_mask, ranges, 0, ctx, d_ctx, ldo, stats, dq, lddq,
                       dk, lddk, dv, lddv, B, H, Lq, mask_pitch, d_head, dtype, stream);
}

int fira_attn_bwd_rows(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv, const int* ranges,
                       const unsigned char* key_mask, int mask_pitch, int causal, const int* qoff, long rows,
                       const void* ctx, const void* d_ctx, long ldo, const float* stats, void* dq, long lddq, void* dk,
                       long lddk, void* dv, long lddv, int B, int H, int Lq, int d_head, int dtype, void* stream) {
  FIRA_CHECK_ARG(qoff && rows > 0, FIRA_ERR_ARG, "attn_bwd_rows: null qoff or no rows");
  return attn_bwd_impl(q, ldq, k, ldk, v, ldv, key_mask, ranges, causal, ctx, d_ctx, ldo, stats, dq, lddq, dk, lddk,
                       dv, lddv, B, H, Lq, mask_pitch, d_head, dtype, stream, qoff, rows);
}

}  // extern "C"
