// Row-wise bandwidth kernels (D = 256 features per row, one warp per row, 8 features per lane):
//   embeddings (+position table), dropout+residual+LayerNorm fwd/bwd, Combination gate fwd/bwd,
//   column sums (bias gradients), encoder-memory pack/unpack.
// All are HBM-bound: every lane moves 32 B (fp32) / 16 B (bf16) per row access, a warp moves one
// whole contiguous row, grids are sized as multiples of the SM count.
#include "common.cuh"
#include "fira_b200.h"

namespace {

constexpr int D = 256;          // embedding_dim (run_model.py:38); checked at every entry point
constexpr int ROWS_PER_CTA = 8; // 8 warps
constexpr int CTA = ROWS_PER_CTA * kWarp;

__host__ inline int row_grid(long rows) {
  long g = (rows + ROWS_PER_CTA - 1) / ROWS_PER_CTA;
  const long cap = (long)fira_num_sms() * 16;   // grid-stride beyond 16 CTAs/SM
  return (int)(g < cap ? (g > 0 ? g : 1) : cap);
}

// ------------------------------------------------------------------ embeddings
// Encoder node rows, segment-major order (DESIGN.md "node buffer"):
//   rows [0, B*n_code)                code tokens   emb[sou] + PE[pos]      -> out_code[r]
//   rows [B*n_code, B*(n_code+n_sub)) sub-tokens    emb[sub_token]          -> out_rest[r]
//   rows [.., B*(n_code+n_sub+n_ast)) AST/edit      ast_emb[ast_change]     -> out_rest[r]
// gnn_transformer.py:46-52 (the torch.cat of :58 disappears: the three segments are written in place).
template <typename T>
__global__ void embed_nodes_kernel(const int* __restrict__ sou, const int* __restrict__ sub, const int* __restrict__ ast,
                                   const float* __restrict__ emb, const float* __restrict__ ast_emb,
                                   const float* __restrict__ pe, const int* __restrict__ pos_idx,
                                   T* __restrict__ out_code, T* __restrict__ out_rest, int B, int n_code, int n_sub,
                                   int n_ast) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const long R = (long)B * (n_code + n_sub + n_ast);
  const int lane = threadIdx.x & 31;
  for (long r = (long)blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5); r < R; r += (long)gridDim.x * ROWS_PER_CTA) {
    const float* src; const float* pos = nullptr; T* dst;
    if (r < (long)B * n_code) {
      // pos_idx (packed batches): position of the token inside its commit; padded batches: the column index
      src = emb + (long)sou[r] * D; pos = pe + (long)(pos_idx ? pos_idx[r] : (int)(r % n_code)) * D; dst = out_code + r * D;
    } else if (r < (long)B * (n_code + n_sub)) {
      src = emb + (long)sub[r - (long)B * n_code] * D; dst = out_rest + r * D;
    } else {
      src = ast_emb + (long)ast[r - (long)B * (n_code + n_sub)] * D; dst = out_rest + r * D;
    }
    float v[8];
    Act<float>::load8(src + lane * 8, v);
    if (pos) {
      float q[8];
      Act<float>::load8(pos + lane * 8, q);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] += q[i];
    }
    Act<T>::store8(dst + lane * 8, v);
  }
}

// grad of the above into the two dense tables (nn.Embedding default dense grads); id 0 is padding_idx
// in both encoder tables (gnn_transformer.py:32-35) and gets no gradient.
template <typename T>
__global__ void embed_nodes_bwd_kernel(const int* __restrict__ sou, const int* __restrict__ sub,
                                       const int* __restrict__ ast, const T* __restrict__ d_code,
                                       const T* __restrict__ d_rest, float* __restrict__ d_emb,
                                       float* __restrict__ d_ast_emb, int B, int n_code, int n_sub, int n_ast) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const long R = (long)B * (n_code + n_sub + n_ast);
  const int lane = threadIdx.x & 31;
  for (long r = (long)blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5); r < R; r += (long)gridDim.x * ROWS_PER_CTA) {
    int id; float* dst; const T* g;
    if (r < (long)B * n_code) { id = sou[r]; dst = d_emb; g = d_code + r * D; }
    else if (r < (long)B * (n_code + n_sub)) { id = sub[r - (long)B * n_code]; dst = d_emb; g = d_rest + r * D; }
    else { id = ast[r - (long)B * (n_code + n_sub)]; dst = d_ast_emb; g = d_rest + r * D; }
    if (id == 0) continue;
    float v[8];
    Act<T>::load8(g + lane * 8, v);
    float* o = dst + (long)id * D + lane * 8;
    // two 16-byte vector reductions per lane (red.global.add.v4.f32, sm_90+) instead of eight scalar ones
    atomicAdd(reinterpret_cast<float4*>(o), make_float4(v[0], v[1], v[2], v[3]));
    atomicAdd(reinterpret_cast<float4*>(o + 4), make_float4(v[4], v[5], v[6], v[7]));
  }
}

// Decoder input rows: dec_emb[tar] + PE[t]  (gnn_transformer.py:110-113); no padding_idx on this table.
template <typename T>
__global__ void embed_rows_kernel(const int* __restrict__ ids, const float* __restrict__ emb,
                                  const float* __restrict__ pe, T* __restrict__ out, long rows, int period) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const int lane = threadIdx.x & 31;
  for (long r = (long)blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5); r < rows; r += (long)gridDim.x * ROWS_PER_CTA) {
    float v[8], q[8];
    Act<float>::load8(emb + (long)ids[r] * D + lane * 8, v);
    Act<float>::load8(pe + (r % period) * D + lane * 8, q);
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] += q[i];
    Act<T>::store8(out + r * D + lane * 8, v);
  }
}
// rmap (may be NULL): row r of g is row rmap[r] of ids, -1 = no row
template <typename T>
__global__ void embed_rows_bwd_kernel(const int* __restrict__ ids, const int* __restrict__ rmap, const T* __restrict__ g,
                                      float* __restrict__ d_emb, long rows) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const int lane = threadIdx.x & 31;
  for (long r = (long)blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5); r < rows; r += (long)gridDim.x * ROWS_PER_CTA) {
    const long src = rmap ? rmap[r] : r;
    if (src < 0) continue;
    float v[8];
    Act<T>::load8(g + r * D + lane * 8, v);
    // rows whose gradient is exactly zero (padded target positions: no loss, masked as keys) add nothing; skipping
    // them avoids ~1,000 rows of atomics serialising on the <pad> row of the table
    bool nz = false;
#pragma unroll
    for (int i = 0; i < 8; ++i) nz |= v[i] != 0.f;
    if (!__any_sync(0xffffffffu, nz)) continue;
    float* o = d_emb + (long)ids[src] * D + lane * 8;
    // two 16-byte vector reductions per lane (red.global.add.v4.f32, sm_90+) instead of eight scalar ones
    atomicAdd(reinterpret_cast<float4*>(o), make_float4(v[0], v[1], v[2], v[3]));
    atomicAdd(reinterpret_cast<float4*>(o + 4), make_float4(v[4], v[5], v[6], v[7]));
  }
}

// ------------------------------------------------------------------ dropout + residual + LayerNorm
// out = LN(dropout_p(z) + resid) * gamma + beta, eps 1e-5, post-LN
// (gnn_transformer.py:83,161,174,205).  Rows < split go to outA[r], the others to outB[r].
template <typename T>
__global__ void ln_fwd_kernel(const T* __restrict__ z, const T* __restrict__ resid, const float* __restrict__ gamma,
                              const float* __restrict__ beta, T* __restrict__ outA, T* __restrict__ outB, long split,
                              float* __restrict__ mean_out, float* __restrict__ rstd_out, long rows, float p_drop,
                              uint64_t seed, const uint64_t* __restrict__ seed_ctr, uint32_t stream_id) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  if (seed_ctr) seed += *seed_ctr;
  const int lane = threadIdx.x & 31;
  float g[8], bt[8];
  Act<float>::load8(gamma + lane * 8, g);
  Act<float>::load8(beta + lane * 8, bt);
  const float keep_scale = p_drop > 0.f ? 1.f / (1.f - p_drop) : 1.f;
  for (long r = (long)blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5); r < rows; r += (long)gridDim.x * ROWS_PER_CTA) {
    float y[8], x[8];
    Act<T>::load8(z + r * D + lane * 8, y);
    Act<T>::load8(resid + r * D + lane * 8, x);
    if (p_drop > 0.f) {
      uint32_t m = dropout_keep8(seed, stream_id, (uint64_t)r * 32 + lane, p_drop);
#pragma unroll
      for (int i = 0; i < 8; ++i) y[i] = ((m >> i) & 1) ? y[i] * keep_scale : 0.f;
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { y[i] += x[i]; s += y[i]; }
    const float mean = warp_sum(s) * (1.f / D);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { float d = y[i] - mean; q += d * d; }
    const float rstd = rsqrtf(warp_sum(q) * (1.f / D) + kLnEps);
#pragma unroll
    for (int i = 0; i < 8; ++i) y[i] = (y[i] - mean) * rstd * g[i] + bt[i];
    T* dst = (r < split ? outA : outB) + r * D + lane * 8;
    Act<T>::store8(dst, y);
    if (lane == 0 && mean_out) { mean_out[r] = mean; rstd_out[r] = rstd; }
  }
}

// Backward of the block above.  Recomputes y = dropout(z) + resid and xhat from the saved
// (mean, rstd); writes d_z (dropout mask applied) and d_resid, accumulates d_gamma / d_beta.
// d_resid_accum != 0: d_resid += dy (used when the residual input also feeds another branch).
template <typename T>
__global__ void ln_bwd_kernel(const T* __restrict__ doutA, const T* __restrict__ doutB, long split,
                              const T* __restrict__ z, const T* __restrict__ resid, const float* __restrict__ mean_in,
                              const float* __restrict__ rstd_in, const float* __restrict__ gamma, T* __restrict__ d_z,
                              T* __restrict__ d_resid, int d_resid_accum, float* __restrict__ d_gamma,
                              float* __restrict__ d_beta, long rows, float p_drop, uint64_t seed,
                              const uint64_t* __restrict__ seed_ctr, uint32_t stream_id, const int* __restrict__ rmap) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  if (seed_ctr) seed += *seed_ctr;
  __shared__ __align__(16) float red[2][ROWS_PER_CTA][D];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float g[8], dg[8], db[8];
  Act<float>::load8(gamma + lane * 8, g);
#pragma unroll
  for (int i = 0; i < 8; ++i) { dg[i] = 0.f; db[i] = 0.f; }
  const float keep_scale = p_drop > 0.f ? 1.f / (1.f - p_drop) : 1.f;
  for (long r = (long)blockIdx.x * ROWS_PER_CTA + warp; r < rows; r += (long)gridDim.x * ROWS_PER_CTA) {
    const long pr = rmap ? rmap[r] : r;            // the row the forward's dropout mask was drawn for
    float y[8], x[8], go[8];
    if (pr < 0) {                                  // pad slot: zero gradients, nothing to d_gamma / d_beta
#pragma unroll
      for (int i = 0; i < 8; ++i) y[i] = 0.f;
      Act<T>::store8(d_z + r * D + lane * 8, y);
      if (d_resid && !d_resid_accum) Act<T>::store8(d_resid + r * D + lane * 8, y);
      continue;
    }
    Act<T>::load8(z + r * D + lane * 8, y);
    Act<T>::load8(resid + r * D + lane * 8, x);
    Act<T>::load8((r < split ? doutA : doutB) + r * D + lane * 8, go);
    uint32_t m = 0xffu;
    if (p_drop > 0.f) {
      m = dropout_keep8(seed, stream_id, (uint64_t)pr * 32 + lane, p_drop);
#pragma unroll
      for (int i = 0; i < 8; ++i) y[i] = ((m >> i) & 1) ? y[i] * keep_scale : 0.f;
    }
    const float mean = mean_in[r], rstd = rstd_in[r];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float xh = (y[i] + x[i] - mean) * rstd;
      float dxh = go[i] * g[i];
      dg[i] += go[i] * xh; db[i] += go[i];
      s1 += dxh; s2 += dxh * xh;
      y[i] = xh; x[i] = dxh;   // reuse: y = xhat, x = dxhat
    }
    s1 = warp_sum(s1) * (1.f / D);
    s2 = warp_sum(s2) * (1.f / D);
    float dy[8], dz[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      dy[i] = rstd * (x[i] - s1 - y[i] * s2);
      dz[i] = ((m >> i) & 1) ? dy[i] * keep_scale : 0.f;
    }
    Act<T>::store8(d_z + r * D + lane * 8, dz);
    if (d_resid) {
      if (d_resid_accum) {
        float old[8];
        Act<T>::load8(d_resid + r * D + lane * 8, old);
#pragma unroll
        for (int i = 0; i < 8; ++i) dy[i] += old[i];
      }
      Act<T>::store8(d_resid + r * D + lane * 8, dy);
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) { red[0][warp][lane * 8 + i] = dg[i]; red[1][warp][lane * 8 + i] = db[i]; }
  __syncthreads();
  // 2 x 256 column sums of this CTA -> global: 128 threads, four columns each, one 16-byte vector reduction per thread
  // (red.global.add.v4.f32) instead of 512 scalar ones per CTA
  if (threadIdx.x < 2 * D / 4) {
    const int which = threadIdx.x / (D / 4), col = (threadIdx.x % (D / 4)) * 4;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int w = 0; w < ROWS_PER_CTA; ++w) {
      const float4 v = *reinterpret_cast<const float4*>(&red[which][w][col]);
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    float* dst = (which ? d_beta : d_gamma) + col;
    if ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0) {
      atomicAdd(reinterpret_cast<float4*>(dst), s);
    } else {
      atomicAdd(dst, s.x); atomicAdd(dst + 1, s.y); atomicAdd(dst + 2, s.z); atomicAdd(dst + 3, s.w);
    }
  }
}

// ------------------------------------------------------------------ Combination gate
// combination_layer.py:7-17 with heads folded away (the op is element-wise; d_k only sets the scale):
//   c = w_k*k + w_v*v,  (w_k, w_v) = softmax([q*k, q*v] / sqrt(d_k))  ==>  c = v + sigmoid(s*q*(k-v))*(k-v)
// `value` is Linear(mark_embedding[mark]) and mark has 4 classes, so v comes from a 4 x D table.
template <typename T>
__global__ void comb_gate_fwd_kernel(const T* __restrict__ qk, long ld_qk, const float* __restrict__ vtab,
                                     const int* __restrict__ mark, T* __restrict__ out, long rows, float scale,
                                     float p_drop, uint64_t seed, const uint64_t* __restrict__ seed_ctr,
                                     uint32_t stream_id) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  if (seed_ctr) seed += *seed_ctr;
  const int lane = threadIdx.x & 31;
  const float keep_scale = p_drop > 0.f ? 1.f / (1.f - p_drop) : 1.f;
  for (long r = (long)blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5); r < rows; r += (long)gridDim.x * ROWS_PER_CTA) {
    float q[8], k[8], v[8], c[8];
    Act<T>::load8(qk + r * ld_qk + lane * 8, q);
    Act<T>::load8(qk + r * ld_qk + D + lane * 8, k);
    Act<float>::load8(vtab + (long)mark[r] * D + lane * 8, v);
    uint32_t m = 0xffu;
    if (p_drop > 0.f) m = dropout_keep8(seed, stream_id, (uint64_t)r * 32 + lane, p_drop);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float e = k[i] - v[i];
      float gte = 1.f / (1.f + expf(-scale * q[i] * e));
      float x = fmaf(gte, e, v[i]);
      c[i] = ((m >> i) & 1) ? x * keep_scale : 0.f;
    }
    Act<T>::store8(out + r * D + lane * 8, c);
  }
}

template <typename T>
__global__ void comb_gate_bwd_kernel(const T* __restrict__ qk, long ld_qk, const float* __restrict__ vtab,
                                     const int* __restrict__ mark, const T* __restrict__ d_out, T* __restrict__ d_qk,
                                     float* __restrict__ d_vtab, long rows, float scale, float p_drop, uint64_t seed,
                                     const uint64_t* __restrict__ seed_ctr, uint32_t stream_id) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  if (seed_ctr) seed += *seed_ctr;
  __shared__ __align__(16) float red[ROWS_PER_CTA][4][D + 8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float dv[4][8];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int i = 0; i < 8; ++i) dv[c][i] = 0.f;
  const float keep_scale = p_drop > 0.f ? 1.f / (1.f - p_drop) : 1.f;
  for (long r = (long)blockIdx.x * ROWS_PER_CTA + warp; r < rows; r += (long)gridDim.x * ROWS_PER_CTA) {
    float q[8], k[8], v[8], go[8], dq[8], dk[8];
    const int cls = mark[r];
    Act<T>::load8(qk + r * ld_qk + lane * 8, q);
    Act<T>::load8(qk + r * ld_qk + D + lane * 8, k);
    Act<float>::load8(vtab + (long)cls * D + lane * 8, v);
    Act<T>::load8(d_out + r * D + lane * 8, go);
    uint32_t m = 0xffu;
    if (p_drop > 0.f) m = dropout_keep8(seed, stream_id, (uint64_t)r * 32 + lane, p_drop);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float dc = ((m >> i) & 1) ? go[i] * keep_scale : 0.f;
      float e = k[i] - v[i];
      float gte = 1.f / (1.f + expf(-scale * q[i] * e));
      float da = dc * e * gte * (1.f - gte);
      dq[i] = da * scale * e;
      float de = dc * gte + da * scale * q[i];
      dk[i] = de;
      float dvi = dc - de;
#pragma unroll
      for (int c = 0; c < 4; ++c) dv[c][i] += (c == cls) ? dvi : 0.f;
    }
    Act<T>::store8(d_qk + r * ld_qk + lane * 8, dq);
    Act<T>::store8(d_qk + r * ld_qk + D + lane * 8, dk);
  }
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int i = 0; i < 8; ++i) red[warp][c][lane * 8 + i] = dv[c][i];
  __syncthreads();
  {   // 4 x 256 sums of this CTA -> global: one 16-byte vector reduction per thread (256 threads x 4 columns)
    const int c = threadIdx.x / (D / 4), col = (threadIdx.x % (D / 4)) * 4;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int w = 0; w < ROWS_PER_CTA; ++w) {
      const float4 v = *reinterpret_cast<const float4*>(&red[w][c][col]);
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    float* dst = d_vtab + c * D + col;
    if ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0) {
      atomicAdd(reinterpret_cast<float4*>(dst), s);
    } else {
      atomicAdd(dst, s.x); atomicAdd(dst + 1, s.y); atomicAdd(dst + 2, s.z); atomicAdd(dst + 3, s.w);
    }
  }
}

// General-value form of the same gate for the stand-alone Combination / CombinationLayer modules
// (combination_layer.py:7-17 with an arbitrary `value` tensor instead of the 4-row mark table): q, k, v, out [rows, D].
template <typename T>
__global__ void comb_gate3_fwd_kernel(const T* __restrict__ qp, const T* __restrict__ kp, const T* __restrict__ vp,
                                      T* __restrict__ out, long rows, float scale, float p_drop, uint64_t seed,
                                      const uint64_t* __restrict__ seed_ctr, uint32_t stream_id) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  if (seed_ctr) seed += *seed_ctr;
  const int lane = threadIdx.x & 31;
  const float keep_scale = p_drop > 0.f ? 1.f / (1.f - p_drop) : 1.f;
  for (long r = (long)blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5); r < rows; r += (long)gridDim.x * ROWS_PER_CTA) {
    float q[8], k[8], v[8], c[8];
    Act<T>::load8(qp + r * D + lane * 8, q);
    Act<T>::load8(kp + r * D + lane * 8, k);
    Act<T>::load8(vp + r * D + lane * 8, v);
    uint32_t m = 0xffu;
    if (p_drop > 0.f) m = dropout_keep8(seed, stream_id, (uint64_t)r * 32 + lane, p_drop);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float e = k[i] - v[i];
      float gte = 1.f / (1.f + expf(-scale * q[i] * e));
      float x = fmaf(gte, e, v[i]);
      c[i] = ((m >> i) & 1) ? x * keep_scale : 0.f;
    }
    Act<T>::store8(out + r * D + lane * 8, c);
  }
}

template <typename T>
__global__ void comb_gate3_bwd_kernel(const T* __restrict__ qp, const T* __restrict__ kp, const T* __restrict__ vp,
                                      const T* __restrict__ d_out, T* __restrict__ dqp, T* __restrict__ dkp,
                                      T* __restrict__ dvp, long rows, float scale, float p_drop, uint64_t seed,
                                      const uint64_t* __restrict__ seed_ctr, uint32_t stream_id) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  if (seed_ctr) seed += *seed_ctr;
  const int lane = threadIdx.x & 31;
  const float keep_scale = p_drop > 0.f ? 1.f / (1.f - p_drop) : 1.f;
  for (long r = (long)blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5); r < rows; r += (long)gridDim.x * ROWS_PER_CTA) {
    float q[8], k[8], v[8], go[8], dq[8], dk[8], dv[8];
    Act<T>::load8(qp + r * D + lane * 8, q);
    Act<T>::load8(kp + r * D + lane * 8, k);
    Act<T>::load8(vp + r * D + lane * 8, v);
    Act<T>::load8(d_out + r * D + lane * 8, go);
    uint32_t m = 0xffu;
    if (p_drop > 0.f) m = dropout_keep8(seed, stream_id, (uint64_t)r * 32 + lane, p_drop);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float dc = ((m >> i) & 1) ? go[i] * keep_scale : 0.f;
      float e = k[i] - v[i];
      float gte = 1.f / (1.f + expf(-scale * q[i] * e));
      float da = dc * e * gte * (1.f - gte);
      dq[i] = da * scale * e;
      float de = dc * gte + da * scale * q[i];
      dk[i] = de;
      dv[i] = dc - de;
    }
    Act<T>::store8(dqp + r * D + lane * 8, dq);
    Act<T>::store8(dkp + r * D + lane * 8, dk);
    Act<T>::store8(dvp + r * D + lane * 8, dv);
  }
}

// rows [off[0][B], Rc) and [Rc + off[1][B], Rc + Rs) of a packed batch's memory-row matrices are segment padding: no
// kernel writes them, the GEMMs that follow read every row -> zero them (off = the packed batch's [3][B+1] row offsets).
template <typename T>
__global__ void zero_pad_rows_kernel(T* __restrict__ x, long ld, int width, const int* __restrict__ off, int B, int Rc,
                                     int Rs) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const int lo0 = off[B], lo1 = Rc + off[(B + 1) + B];
  const long n0 = Rc - lo0, n1 = (long)Rc + Rs - lo1;
  const int vec = width / 8;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < (n0 + n1) * vec; i += (long)gridDim.x * blockDim.x) {
    const long r = i / vec; const int c = (int)(i % vec);
    const long row = r < n0 ? lo0 + r : lo1 + (r - n0);
    float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    Act<T>::store8(x + row * ld + c * 8, z);
  }
}

// ------------------------------------------------------------------ column sums (bias gradients)
// out[n] += sum_m x[m, n]; one warp covers 32 columns x a strided set of rows.
template <typename T>
__global__ void colsum_kernel(const T* __restrict__ x, long ld, long M, int N, float* __restrict__ out) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ float red[8][33];
  const int col = blockIdx.x * 32 + (threadIdx.x & 31);
  const int wy = threadIdx.x >> 5;
  float s = 0.f;
  if (col < N)
    for (long m = (long)blockIdx.y * 8 + wy; m < M; m += (long)gridDim.y * 8) s += Act<T>::ld(x + m * ld + col);
  red[wy][threadIdx.x & 31] = s;
  __syncthreads();
  if (wy == 0 && col < N) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w][threadIdx.x & 31];
    atomicAdd(out + col, t);
  }
}

// weighted variant: out[n] += sum_m w[m] * x[m, n]   (GCN: d(W2*b1) = sum_i rowsum(A)_i * dZ_i)
template <typename T>
__global__ void colsum_weighted_kernel(const T* __restrict__ x, long ld, const float* __restrict__ w, long M, int N,
                                       float* __restrict__ out) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ float red[8][33];
  const int col = blockIdx.x * 32 + (threadIdx.x & 31);
  const int wy = threadIdx.x >> 5;
  float s = 0.f;
  if (col < N)
    for (long m = (long)blockIdx.y * 8 + wy; m < M; m += (long)gridDim.y * 8) s += w[m] * Act<T>::ld(x + m * ld + col);
  red[wy][threadIdx.x & 31] = s;
  __syncthreads();
  if (wy == 0 && col < N) {
    float t = 0.f;
#pragma unroll
    for (int w8 = 0; w8 < 8; ++w8) t += red[w8][threadIdx.x & 31];
    atomicAdd(out + col, t);
  }
}

// ------------------------------------------------------------------ encoder memory pack / unpack
// memory[b, s, :] = s < n_code ? code[b*n_code + s] : rest[B*n_code + b*n_sub + (s - n_code)]
// (Model.py:48 torch.cat((sou_embedding, sub_token_embedding), 1)); unpack is its adjoint and also
// zero-fills the AST/edit rows, which the encoder drops (gnn_transformer.py:62).
template <typename T>
__global__ void pack_memory_kernel(const T* __restrict__ code, const T* __restrict__ rest, T* __restrict__ mem, int B,
                                   int n_code, int n_sub) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const int S = n_code + n_sub;
  const long rows = (long)B * S;
  const int lane = threadIdx.x & 31;
  for (long r = (long)blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5); r < rows; r += (long)gridDim.x * ROWS_PER_CTA) {
    const long b = r / S; const int s = (int)(r % S);
    const T* src = s < n_code ? code + (b * n_code + s) * D : rest + ((long)B * n_code + b * n_sub + (s - n_code)) * D;
    *reinterpret_cast<uint4*>(mem + r * D + lane * 8) = *reinterpret_cast<const uint4*>(src + lane * 8);
    if (sizeof(T) == 4)
      *reinterpret_cast<uint4*>(reinterpret_cast<char*>(mem + r * D + lane * 8) + 16) =
          *reinterpret_cast<const uint4*>(reinterpret_cast<const char*>(src + lane * 8) + 16);
  }
}
template <typename T>
__global__ void unpack_memory_kernel(const T* __restrict__ d_mem, T* __restrict__ d_code, T* __restrict__ d_rest, int B,
                                     int n_code, int n_sub, int n_ast) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const long R = (long)B * (n_code + n_sub + n_ast);
  const int S = n_code + n_sub;
  const int lane = threadIdx.x & 31;
  for (long r = (long)blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5); r < R; r += (long)gridDim.x * ROWS_PER_CTA) {
    float v[8];
    T* dst;
    if (r < (long)B * n_code) {
      const long b = r / n_code; const int s = (int)(r % n_code);
      Act<T>::load8(d_mem + (b * S + s) * D + lane * 8, v);
      dst = d_code + r * D;
    } else if (r < (long)B * S) {
      const long q = r - (long)B * n_code; const long b = q / n_sub; const int s = (int)(q % n_sub);
      Act<T>::load8(d_mem + (b * S + n_code + s) * D + lane * 8, v);
      dst = d_rest + r * D;
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = 0.f;
      dst = d_rest + r * D;
    }
    Act<T>::store8(dst + lane * 8, v);
  }
}

// d = (h > 0) ? d : 0, 8 elements per thread (n % 8 == 0)
template <typename T>
__global__ void relu_bwd_kernel(const T* __restrict__ h, T* __restrict__ d, long n8) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long)gridDim.x * blockDim.x) {
    float a[8], g[8];
    Act<T>::load8(h + i * 8, a);
    Act<T>::load8(d + i * 8, g);
#pragma unroll
    for (int k = 0; k < 8; ++k) g[k] = a[k] > 0.f ? g[k] : 0.f;
    Act<T>::store8(d + i * 8, g);
  }
}

}  // namespace

#define DISPATCH_T(dtype, ...)                                                            \
  if ((dtype) == FIRA_F32) { using T = float; __VA_ARGS__ }                               \
  else if ((dtype) == FIRA_BF16) { using T = __nv_bfloat16; __VA_ARGS__ }                 \
  else { fira_set_error(FIRA_ERR_DTYPE, "unknown dtype %d", (int)(dtype)); return FIRA_ERR_DTYPE; }

extern "C" {

int fira_embed_nodes_fwd(const int* sou, const int* sub_token, const int* ast_change, const float* emb,
                         const float* ast_emb, const float* pos_table, void* out_code, void* out_rest, int B,
                         int n_code, int n_sub, int n_ast, int dim, int dtype, void* stream) {
  return fira_embed_nodes_pos_fwd(sou, nullptr, sub_token, ast_change, emb, ast_emb, pos_table, out_code, out_rest, B,
                                  n_code, n_sub, n_ast, dim, dtype, stream);
}

int fira_embed_nodes_pos_fwd(const int* sou, const int* pos, const int* sub_token, const int* ast_change,
                             const float* emb, const float* ast_emb, const float* pos_table, void* out_code,
                             void* out_rest, int B, int n_code, int n_sub, int n_ast, int dim, int dtype, void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "embed_nodes: dim %d != 256", dim);
  FIRA_CHECK_ARG(fira_aligned16(out_code) && fira_aligned16(out_rest) && fira_aligned16(emb), FIRA_ERR_ALIGN,
                 "embed_nodes: 16-B alignment");
  const long R = (long)B * (n_code + n_sub + n_ast);
  DISPATCH_T(dtype, launch_k(embed_nodes_kernel<T>, dim3(row_grid(R)), dim3(CTA), 0, (cudaStream_t)stream, 
      sou, sub_token, ast_change, emb, ast_emb, pos_table, pos, (T*)out_code, (T*)out_rest, B, n_code, n_sub, n_ast);)
  FIRA_CHECK_LAUNCH("fira_embed_nodes_fwd");
  return FIRA_OK;
}

int fira_zero_pad_rows(void* x, long ld, int width, const int* off, int B, int Rc, int Rs, int dtype, void* stream) {
  FIRA_CHECK_ARG(x && off && B > 0 && width > 0 && width % 8 == 0 && ld >= width, FIRA_ERR_ARG, "zero_pad_rows: arguments");
  FIRA_CHECK_ARG(fira_aligned16(x) && (ld % 8) == 0, FIRA_ERR_ALIGN, "zero_pad_rows: 16-B alignment");
  DISPATCH_T(dtype, launch_k(zero_pad_rows_kernel<T>, dim3(fira_num_sms()), dim3(256), 0, (cudaStream_t)stream, (T*)x, ld, width, off, B, Rc, Rs);)
  FIRA_CHECK_LAUNCH("fira_zero_pad_rows");
  return FIRA_OK;
}

int fira_embed_nodes_bwd(const int* sou, const int* sub_token, const int* ast_change, const void* d_code,
                         const void* d_rest, float* d_emb, float* d_ast_emb, int B, int n_code, int n_sub, int n_ast,
                         int dim, int dtype, void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "embed_nodes_bwd: dim %d != 256", dim);
  const long R = (long)B * (n_code + n_sub + n_ast);
  DISPATCH_T(dtype, launch_k(embed_nodes_bwd_kernel<T>, dim3(row_grid(R)), dim3(CTA), 0, (cudaStream_t)stream, 
      sou, sub_token, ast_change, (const T*)d_code, (const T*)d_rest, d_emb, d_ast_emb, B, n_code, n_sub, n_ast);)
  FIRA_CHECK_LAUNCH("fira_embed_nodes_bwd");
  return FIRA_OK;
}

int fira_embed_rows_fwd(const int* ids, const float* emb, const float* pos_table, void* out, long rows, int period,
                        int dim, int dtype, void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "embed_rows: dim %d != 256", dim);
  FIRA_CHECK_ARG(period > 0, FIRA_ERR_SHAPE, "embed_rows: period");
  DISPATCH_T(dtype, launch_k(embed_rows_kernel<T>, dim3(row_grid(rows)), dim3(CTA), 0, (cudaStream_t)stream, ids, emb, pos_table,
                                                                                         (T*)out, rows, period);)
  FIRA_CHECK_LAUNCH("fira_embed_rows_fwd");
  return FIRA_OK;
}

int fira_embed_rows_bwd(const int* ids, const void* d_out, float* d_emb, long rows, int dim, int dtype, void* stream) {
  return fira_embed_rows_bwd_rows(ids, nullptr, d_out, d_emb, rows, dim, dtype, stream);
}

int fira_embed_rows_bwd_rows(const int* ids, const int* rows_map, const void* d_out, float* d_emb, long rows, int dim,
                             int dtype, void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "embed_rows_bwd: dim %d != 256", dim);
  if (rows == 0) return FIRA_OK;
  DISPATCH_T(dtype, launch_k(embed_rows_bwd_kernel<T>, dim3(row_grid(rows)), dim3(CTA), 0, (cudaStream_t)stream, ids,
                             rows_map, (const T*)d_out, d_emb, rows);)
  FIRA_CHECK_LAUNCH("fira_embed_rows_bwd");
  return FIRA_OK;
}

int fira_ln_residual_fwd(const void* z, const void* resid, const float* gamma, const float* beta, void* outA,
                         void* outB, long split, float* mean, float* rstd, long rows, int dim, float p_drop,
                         uint64_t seed, const uint64_t* seed_ctr, uint32_t stream_id, int dtype, void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "ln_residual_fwd: dim %d != 256", dim);
  FIRA_CHECK_ARG(p_drop >= 0.f && p_drop < 1.f, FIRA_ERR_ARG, "ln_residual_fwd: p_drop %f", p_drop);
  FIRA_CHECK_ARG(fira_aligned16(z) && fira_aligned16(resid) && fira_aligned16(outA) && fira_aligned16(outB),
                 FIRA_ERR_ALIGN, "ln_residual_fwd: 16-B alignment");
  if (rows == 0) return FIRA_OK;
  DISPATCH_T(dtype, launch_k(ln_fwd_kernel<T>, dim3(row_grid(rows)), dim3(CTA), 0, (cudaStream_t)stream, 
      (const T*)z, (const T*)resid, gamma, beta, (T*)outA, (T*)outB, split, mean, rstd, rows, p_drop, seed, seed_ctr, stream_id);)
  FIRA_CHECK_LAUNCH("fira_ln_residual_fwd");
  return FIRA_OK;
}

int fira_ln_residual_bwd(const void* d_outA, const void* d_outB, long split, const void* z, const void* resid,
                         const float* mean, const float* rstd, const float* gamma, void* d_z, void* d_resid,
                         int d_resid_accum, float* d_gamma, float* d_beta, long rows, int dim, float p_drop,
                         uint64_t seed, const uint64_t* seed_ctr, uint32_t stream_id, int dtype, void* stream) {
  return fira_ln_residual_bwd_rows(d_outA, d_outB, split, z, resid, mean, rstd, gamma, d_z, d_resid, d_resid_accum,
                                   d_gamma, d_beta, nullptr, rows, dim, p_drop, seed, seed_ctr, stream_id, dtype, stream);
}

int fira_ln_residual_bwd_rows(const void* d_outA, const void* d_outB, long split, const void* z, const void* resid,
                              const float* mean, const float* rstd, const float* gamma, void* d_z, void* d_resid,
                              int d_resid_accum, float* d_gamma, float* d_beta, const int* rows_map, long rows, int dim,
                              float p_drop, uint64_t seed, const uint64_t* seed_ctr, uint32_t stream_id, int dtype,
                              void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "ln_residual_bwd: dim %d != 256", dim);
  if (rows == 0) return FIRA_OK;
  long g = (rows + ROWS_PER_CTA - 1) / ROWS_PER_CTA;
  int grid = (int)(g < (long)fira_num_sms() * 4 ? g : (long)fira_num_sms() * 4);   // few CTAs -> few d_gamma/d_beta atomics
  DISPATCH_T(dtype, launch_k(ln_bwd_kernel<T>, dim3(grid), dim3(CTA), 0, (cudaStream_t)stream, 
      (const T*)d_outA, (const T*)d_outB, split, (const T*)z, (const T*)resid, mean, rstd, gamma, (T*)d_z,
      (T*)d_resid, d_resid_accum, d_gamma, d_beta, rows, p_drop, seed, seed_ctr, stream_id, rows_map);)
  FIRA_CHECK_LAUNCH("fira_ln_residual_bwd");
  return FIRA_OK;
}

int fira_comb_gate_fwd(const void* qk, long ld_qk, const float* vtab, const int* mark, void* out, long rows, int dim,
                       int d_head, float p_drop, uint64_t seed, const uint64_t* seed_ctr, uint32_t stream_id, int dtype, void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "comb_gate_fwd: dim %d != 256", dim);
  FIRA_CHECK_ARG(ld_qk >= 2 * D && (ld_qk % 8) == 0, FIRA_ERR_SHAPE, "comb_gate_fwd: ld_qk %ld", ld_qk);
  if (rows == 0) return FIRA_OK;
  const float scale = 1.f / sqrtf((float)d_head);
  DISPATCH_T(dtype, launch_k(comb_gate_fwd_kernel<T>, dim3(row_grid(rows)), dim3(CTA), 0, (cudaStream_t)stream, 
      (const T*)qk, ld_qk, vtab, mark, (T*)out, rows, scale, p_drop, seed, seed_ctr, stream_id);)
  FIRA_CHECK_LAUNCH("fira_comb_gate_fwd");
  return FIRA_OK;
}

int fira_comb_gate_bwd(const void* qk, long ld_qk, const float* vtab, const int* mark, const void* d_out, void* d_qk,
                       float* d_vtab, long rows, int dim, int d_head, float p_drop, uint64_t seed, const uint64_t* seed_ctr,
                       uint32_t stream_id, int dtype, void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "comb_gate_bwd: dim %d != 256", dim);
  if (rows == 0) return FIRA_OK;
  const float scale = 1.f / sqrtf((float)d_head);
  long g = (rows + ROWS_PER_CTA - 1) / ROWS_PER_CTA;
  int grid = (int)(g < (long)fira_num_sms() * 4 ? g : (long)fira_num_sms() * 4);
  DISPATCH_T(dtype, launch_k(comb_gate_bwd_kernel<T>, dim3(grid), dim3(CTA), 0, (cudaStream_t)stream, 
      (const T*)qk, ld_qk, vtab, mark, (const T*)d_out, (T*)d_qk, d_vtab, rows, scale, p_drop, seed, seed_ctr, stream_id);)
  FIRA_CHECK_LAUNCH("fira_comb_gate_bwd");
  return FIRA_OK;
}

int fira_comb_gate3_fwd(const void* q, const void* k, const void* v, void* out, long rows, int dim, int d_head,
                        float p_drop, uint64_t seed, const uint64_t* seed_ctr, uint32_t stream_id, int dtype, void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "comb_gate3_fwd: dim %d != 256", dim);
  FIRA_CHECK_ARG(d_head > 0, FIRA_ERR_SHAPE, "comb_gate3_fwd: d_head %d", d_head);
  if (rows == 0) return FIRA_OK;
  const float scale = 1.f / sqrtf((float)d_head);
  DISPATCH_T(dtype, launch_k(comb_gate3_fwd_kernel<T>, dim3(row_grid(rows)), dim3(CTA), 0, (cudaStream_t)stream, 
      (const T*)q, (const T*)k, (const T*)v, (T*)out, rows, scale, p_drop, seed, seed_ctr, stream_id);)
  FIRA_CHECK_LAUNCH("fira_comb_gate3_fwd");
  return FIRA_OK;
}

int fira_comb_gate3_bwd(const void* q, const void* k, const void* v, const void* d_out, void* d_q, void* d_k, void* d_v,
                        long rows, int dim, int d_head, float p_drop, uint64_t seed, const uint64_t* seed_ctr,
                        uint32_t stream_id, int dtype, void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "comb_gate3_bwd: dim %d != 256", dim);
  FIRA_CHECK_ARG(d_head > 0, FIRA_ERR_SHAPE, "comb_gate3_bwd: d_head %d", d_head);
  if (rows == 0) return FIRA_OK;
  const float scale = 1.f / sqrtf((float)d_head);
  DISPATCH_T(dtype, launch_k(comb_gate3_bwd_kernel<T>, dim3(row_grid(rows)), dim3(CTA), 0, (cudaStream_t)stream, 
      (const T*)q, (const T*)k, (const T*)v, (const T*)d_out, (T*)d_q, (T*)d_k, (T*)d_v, rows, scale, p_drop, seed,
      seed_ctr, stream_id);)
  FIRA_CHECK_LAUNCH("fira_comb_gate3_bwd");
  return FIRA_OK;
}

int fira_colsum(const void* x, long ld, long M, int N, const float* row_weight, float* out, int dtype, void* stream) {
  if (M == 0 || N == 0) return FIRA_OK;
  long gy = (M + 63) / 64;
  if (gy > 64) gy = 64;
  dim3 grid((N + 31) / 32, (unsigned)gy);
  if (row_weight) {
    DISPATCH_T(dtype, launch_k(colsum_weighted_kernel<T>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, (const T*)x, ld, row_weight,
                                                                                         M, N, out);)
  } else {
    DISPATCH_T(dtype, launch_k(colsum_kernel<T>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, (const T*)x, ld, M, N, out);)
  }
  FIRA_CHECK_LAUNCH("fira_colsum");
  return FIRA_OK;
}

int fira_relu_bwd(const void* h, void* d, long n, int dtype, void* stream) {
  FIRA_CHECK_ARG(n % 8 == 0, FIRA_ERR_SHAPE, "relu_bwd: n %ld not a multiple of 8", n);
  if (n == 0) return FIRA_OK;
  long blocks = (n / 8 + 255) / 256;
  if (blocks > (long)fira_num_sms() * 16) blocks = (long)fira_num_sms() * 16;
  DISPATCH_T(dtype, launch_k(relu_bwd_kernel<T>, dim3((int)blocks), dim3(256), 0, (cudaStream_t)stream, (const T*)h, (T*)d, n / 8);)
  FIRA_CHECK_LAUNCH("fira_relu_bwd");
  return FIRA_OK;
}

int fira_pack_memory(const void* code, const void* rest, void* mem, int B, int n_code, int n_sub, int dim, int dtype,
                     void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "pack_memory: dim %d != 256", dim);
  DISPATCH_T(dtype, launch_k(pack_memory_kernel<T>, dim3(row_grid((long)B * (n_code + n_sub))), dim3(CTA), 0, (cudaStream_t)stream, 
      (const T*)code, (const T*)rest, (T*)mem, B, n_code, n_sub);)
  FIRA_CHECK_LAUNCH("fira_pack_memory");
  return FIRA_OK;
}

int fira_unpack_memory(const void* d_mem, void* d_code, void* d_rest, int B, int n_code, int n_sub, int n_ast, int dim,
                       int dtype, void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "unpack_memory: dim %d != 256", dim);
  DISPATCH_T(dtype, launch_k(unpack_memory_kernel<T>, dim3(row_grid((long)B * (n_code + n_sub + n_ast))), dim3(CTA), 0, (cudaStream_t)stream, (const T*)d_mem, (T*)d_code, (T*)d_rest, B,
                                                                      n_code, n_sub, n_ast);)
  FIRA_CHECK_LAUNCH("fira_unpack_memory");
  return FIRA_OK;
}

}  // extern "C"
