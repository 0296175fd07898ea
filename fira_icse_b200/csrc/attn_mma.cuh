// Attention pieces shared by the attention kernels (attention.cu) and the fused decoder forward (decoder_fwd.cu):
// the key-list arguments, valid-key compaction, and the warp-level mma.sync.m16n8k16 helpers of the bf16 kernels --
// swizzled [rows][32] head tiles, ldmatrix fragment loads, K / V staging by cp.async, the per-row key rules and the
// online-softmax step on score fragments.
#pragma once
#include "common.cuh"

namespace {

constexpr int DH = 32;           // head dim (256 / 8)
constexpr int LQ_MAX = 32;       // tar_len 30 (run_model.py:32)

struct AttnArgs {
  const void* q; long ldq;       // row (b*Lq + t), head h at column h*32
  const void* k; long ldk;       // row (b*Lk + s)
  const void* v; long ldv;
  const unsigned char* key_mask; // [B, Lk], 1 = attend (may be NULL with ranges: all keys valid)
  const int* ranges;             // NULL, or [B][4] = {first row, rows, first row, rows} of k / v (packed batches)
  int causal;
  int B, H, Lq, Lk;
  float scale;
  // NULL, or [B+1] (attn_mma_bwd_kernel): the query rows of commit b are rows qoff[b] .. qoff[b+1] - 1 (at most Lq; Lq
  // stays the pitch of stats); causal: so are its keys, and key_mask keeps the pitch Lk
  const int* qoff = nullptr;
  long qrows = 0;                // with qoff: rows of q / dq (causal: of k / v too); rows qoff[B] .. qrows - 1 are pad
};

// valid-key compaction by warp 0: kidx[0..nv) = original indices of keys with mask == 1 (ascending).
// nv == 0 (every key padded): identity list of all keys and *filled = 1 (scores are all -1e9 -> uniform P).
// causal (self-attention, Lk = 30): no compaction -- a row whose every permitted key is padding must stay
// uniform over ALL keys like the reference, so padding is handled by the score mask instead.
__device__ __forceinline__ void compact_keys(const unsigned char* km, int Lk, int causal, int* kidx, int* nv_out,
                                             int* filled, const int* rg = nullptr) {
  // rg != NULL (packed batches): key position m of the commit lives in global row
  //   m < rg[1] ? rg[0] + m : rg[2] + (m - rg[1]),   m < rg[1] + rg[3];   kidx then holds GLOBAL rows
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    const int L = rg ? rg[1] + rg[3] : Lk;
    int n = 0;
    for (int s0 = 0; s0 < L && !causal; s0 += 32) {
      const int s = s0 + lane;
      const bool ok = s < L && (km == nullptr || km[s] != 0);
      const unsigned bal = __ballot_sync(0xffffffffu, ok);
      if (ok) kidx[n + __popc(bal & ((1u << lane) - 1u))] = rg ? (s < rg[1] ? rg[0] + s : rg[2] + (s - rg[1])) : s;
      n += __popc(bal);
    }
    if (n == 0) {
      for (int s = lane; s < L; s += 32) kidx[s] = rg ? (s < rg[1] ? rg[0] + s : rg[2] + (s - rg[1])) : s;
      n = L;
      if (lane == 0) *filled = causal ? 0 : 1;
    } else if (lane == 0) *filled = 0;
    if (lane == 0) *nv_out = n;
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------ bf16 tensor cores
// A warp holds 16 query rows x 8 keys per accumulator fragment; the fragment of a score tile IS, register for
// register, the A operand of the product that consumes it (P V, dS K), so P and dS never leave the registers there.
// K / V / Q / dO / P / dS tiles in shared memory are [rows][32] bf16, read with ldmatrix (.trans for the operands
// whose reduction dimension is the tile's row).
namespace mma {

constexpr int ROWB = DH * 2;     // bytes per row of a [rows][32] bf16 tile
constexpr float kLog2e = 1.4426950408889634f;

// byte offset of 16-B chunk c (8 bf16) of row r in a [rows][32] bf16 tile: the XOR spreads the 8 rows of an ldmatrix
// 8x8 matrix (and the 4-B fragment stores of P / dS) over all 32 banks
__device__ __forceinline__ uint32_t swz(int r, int c) { return r * ROWB + ((c ^ ((r >> 1) & 3)) << 4); }
__device__ __forceinline__ uint32_t su32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void ldsm4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ void ldsm4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
// d += a b   (m16n8k16, a row-major 16x16, b column-major 16x8)
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float round_bf16(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// A fragments (16 rows from r0 x 32 features = two k16 steps) of a [rows][32] tile
__device__ __forceinline__ void ld_a(const unsigned char* tile, int r0, int lane, uint32_t (&a)[2][4]) {
#pragma unroll
  for (int kk = 0; kk < 2; ++kk)
    ldsm4(su32(tile + swz(r0 + (lane & 7) + ((lane >> 3) & 1) * 8, 2 * kk + (lane >> 4))), a[kk]);
}
// s[n] += A X^T for 8-row groups n of the [rows][32] tile x (X rows = the N dimension, 32 features = K)
template <int NT>
__device__ __forceinline__ void mma_abt(float (&s)[NT][4], const uint32_t (&a)[2][4], const unsigned char* x, int lane) {
#pragma unroll
  for (int n = 0; n < NT; ++n) {
    uint32_t b[4];
    ldsm4(su32(x + swz(8 * n + (lane & 7), lane >> 3)), b);
    mma16816(s[n], a[0], b[0], b[1]);
    mma16816(s[n], a[1], b[2], b[3]);
  }
}
// o[n] += A X over k16 step kk: X = rows [16 kk, 16 kk + 16) of a [rows][32] tile (rows = K, 32 features = N)
__device__ __forceinline__ void mma_ax(float (&o)[4][4], const uint32_t (&a)[4], const unsigned char* x, int kk, int lane) {
#pragma unroll
  for (int np = 0; np < 2; ++np) {
    uint32_t b[4];
    ldsm4_t(su32(x + swz(16 * kk + (lane & 7) + ((lane >> 3) & 1) * 8, 2 * np + (lane >> 4))), b);
    mma16816(o[2 * np], a, b[0], b[1]);
    mma16816(o[2 * np + 1], a, b[2], b[3]);
  }
}
// A fragment of a k16 step from score-layout accumulators (keys 16 kk .. 16 kk + 15)
template <int NT>
__device__ __forceinline__ void acc_to_a(const float (&s)[NT][4], int kk, uint32_t (&a)[4]) {
  a[0] = pack_bf16(s[2 * kk][0], s[2 * kk][1]);
  a[1] = pack_bf16(s[2 * kk][2], s[2 * kk][3]);
  a[2] = pack_bf16(s[2 * kk + 1][0], s[2 * kk + 1][1]);
  a[3] = pack_bf16(s[2 * kk + 1][2], s[2 * kk + 1][3]);
}

// K and V rows of compacted keys [c0, c0 + n) into [nk][32] tiles (rows >= n zeroed: P = 0 there must not meet NaN)
__device__ __forceinline__ void stage_kv(unsigned char* ks, unsigned char* vs, const __nv_bfloat16* kh, long ldk,
                                         const __nv_bfloat16* vh, long ldv, const int* kidx, int c0, int n, int nk,
                                         int tid, int nthr) {
  for (int i = tid; i < nk * 4; i += nthr) {
    const int j = i >> 2, c = i & 3;
    const uint32_t off = swz(j, c);
    if (j < n) {
      const long r = kidx[c0 + j];
      cp_async16(su32(ks + off), kh + r * ldk + c * 8);
      cp_async16(su32(vs + off), vh + r * ldv + c * 8);
    } else {
      *reinterpret_cast<uint4*>(ks + off) = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(vs + off) = make_uint4(0, 0, 0, 0);
    }
  }
}

// Keys valid for query row t.  Causal (identity list, Lk <= 32): key m <= t with its mask byte set; a row without one
// is uniform over every key of the list (`fill`).  Otherwise every listed key is valid, and `fill` is the commit's.
// mb = causal_mask_bits(): bit m = mask byte of key m.
struct RowKeys { uint32_t causal_bits; bool fill; };
__device__ __forceinline__ uint32_t causal_mask_bits(const AttnArgs& a, const unsigned char* km, int lane) {
  return a.causal ? __ballot_sync(0xffffffffu, lane < a.Lk && km[lane] != 0) : 0u;
}
__device__ __forceinline__ RowKeys row_keys(const AttnArgs& a, uint32_t mb, int nv, bool filled, int t) {
  RowKeys r{0u, filled};
  if (a.causal) {
    const uint32_t w = mb & ((2u << min(t, 31)) - 1u);
    r.fill = w == 0;
    r.causal_bits = r.fill ? (nv >= 32 ? 0xffffffffu : (1u << nv) - 1u) : w;
  }
  return r;
}
__device__ __forceinline__ bool key_ok(const RowKeys& r, int causal, int key, int nv) {
  return causal ? key < 32 && ((r.causal_bits >> key) & 1u) : key < nv;
}

// One key block of the forward: s = the block's raw scores Q K^T (NT 8-key groups, keys c0 ..) for the warp's rows
// (lane >> 2) + 8 r.  Log2-domain scores of the valid keys (-inf elsewhere), online max / rescale of (m, l, o),
// P = bf16(exp) -- the row sum adds the bf16-rounded P that the P V product consumes -- then o += P V (vt: the block's
// [keys][32] V tile).
template <int NT>
__device__ __forceinline__ void softmax_pv(float (&s)[NT][4], const RowKeys (&rk)[2], int causal, int c0, int nv,
                                           float k2, float (&m)[2], float (&l)[2], float (&o)[4][4],
                                           const unsigned char* vt, int lane) {
  const int q = lane & 3;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float mx = -INFINITY;
#pragma unroll
    for (int n = 0; n < NT; ++n)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float& x = s[n][2 * r + e];
        x = key_ok(rk[r], causal, c0 + 8 * n + 2 * q + e, nv) ? (rk[r].fill ? 0.f : x * k2) : -INFINITY;
        mx = fmaxf(mx, x);
      }
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float mn = fmaxf(m[r], mx);
    const float mu = mn == -INFINITY ? 0.f : mn;       // nothing valid yet: keep everything at exactly 0
    const float corr = ex2(m[r] - mu);
    m[r] = mn;
    l[r] *= corr;
#pragma unroll
    for (int n = 0; n < 4; ++n) { o[n][2 * r] *= corr; o[n][2 * r + 1] *= corr; }
#pragma unroll
    for (int n = 0; n < NT; ++n)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float p = round_bf16(ex2(s[n][2 * r + e] - mu));   // the MMA consumes bf16(p): sum the rounded value
        s[n][2 * r + e] = p;
        l[r] += p;
      }
  }
#pragma unroll
  for (int kk = 0; kk < NT / 2; ++kk) {
    uint32_t pa[4];
    acc_to_a(s, kk, pa);
    mma_ax(o, pa, vt, kk, lane);
  }
}

// End of the forward for the warp's rows t[r]: l summed over the lane quad, o scaled by 1 / l, and the statistics of
// rows t < Lq written to st (the (commit, head)'s [Lq][2] rows; may be NULL): (max in natural-log units, or kMaskFill
// for a fill row -- what the reference's softmax subtracts; l).
__device__ __forceinline__ void softmax_finish(float (&o)[4][4], float (&l)[2], const float (&m)[2],
                                               const RowKeys (&rk)[2], const int (&t)[2], int Lq, float* st, int lane) {
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    const float inv = l[r] > 0.f ? 1.f / l[r] : 0.f;
#pragma unroll
    for (int n = 0; n < 4; ++n) { o[n][2 * r] *= inv; o[n][2 * r + 1] *= inv; }
    if (st && (lane & 3) == 0 && t[r] < Lq) {
      st[2 * t[r]] = rk[r].fill ? kMaskFill : m[r] / kLog2e;
      st[2 * t[r] + 1] = l[r];
    }
  }
}

}  // namespace mma
}  // namespace
