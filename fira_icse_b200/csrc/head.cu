// Output head: CopyNet pointer scores (Model.py:15-20) and the dual-copy mixture / loss / argmax
// (Model.py:54-86).  Both are bandwidth/SFU kernels (no contraction worth a tensor core):
//   copy scores : sc[b,t,s] = b_res + sum_d w_res[d] * tanh(src[b,s,d] + tgt[b,t,d])
//                 the reference materialises the [B,30,370,256] tanh tensor (1.9 GB at B=170); here the
//                 30 target rows of a commit sit in shared memory and each warp streams source rows.
//   mixture     : p = [g0 * softmax(vocab logits) || g1 * softmax(masked copy scores)],
//                 logp = log(clamp(p, 1e-10, 1)), nll at the shifted label, argmax for 'dev'/'test'.
//                 Row-wise max/sum are warp/CTA reductions; the 25,020-wide distribution is never stored.
#include "common.cuh"
#include "fira_b200.h"

namespace {

constexpr int D = 256;
constexpr int TMAX = 32;   // tar_len 30 (run_model.py:32) padded

// source row of (commit b, memory position s): padded batches b*S + s; packed batches (ranges[b] = {first code row,
// code rows, first sub-token row, sub-token rows}) the s-th row of the two ranges, -1 beyond them
__device__ __forceinline__ long src_row(const int* __restrict__ ranges, int b, int S, int s) {
  if (!ranges) return (long)b * S + s;
  const int* r = ranges + 4 * b;
  if (s < r[1]) return r[0] + s;
  s -= r[1];
  return s < r[3] ? (long)(r[2] + s) : -1;
}

// ------------------------------------------------------------------ copy scores forward
template <typename T>
__global__ void __launch_bounds__(256) copy_scores_fwd_kernel(const T* __restrict__ src, const T* __restrict__ tgt,
                                                              const float* __restrict__ w_res,
                                                              const float* __restrict__ b_res_p,
                                                              const unsigned char* __restrict__ src_mask,
                                                              const unsigned char* __restrict__ row_mask,
                                                              const int* __restrict__ ranges,
                                                              float* __restrict__ sc, int B, int Tn, int S) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  // src_mask / row_mask (optional): padded source positions are overwritten with -1e9 by the mixture kernel
  // (Model.py:61) and target rows without a label never reach the loss -- both are skipped (score 0 written).
  const float b_res = *b_res_p;
  __shared__ __align__(16) float tg[TMAX][D];
  __shared__ __align__(16) float wr[D];
  __shared__ int active_t[TMAX];
  __shared__ int n_active;
  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int rows_per_cta = 32;
  const int s0 = blockIdx.x * rows_per_cta;
  const int s_end = min(S, s0 + rows_per_cta);
  // target rows that need scores (training: only rows whose label is a copy label).  The others get their zeros by
  // ROW segments (one 128-byte store per warp and row) instead of one scattered 4-byte store per (source row, target row)
  // out of the compute loop -- ~27 of 30 target rows of a commit are inactive.
  if (threadIdx.x == 0) {
    int n = 0;
    for (int t = 0; t < Tn; ++t) if (!row_mask || row_mask[(long)b * Tn + t]) active_t[n++] = t;
    n_active = n;
  }
  for (int idx = threadIdx.x; idx < D; idx += blockDim.x) wr[idx] = w_res[idx];
  __syncthreads();
  const int na = n_active;
  for (int idx = threadIdx.x; idx < na * D; idx += blockDim.x) {
    const int t = active_t[idx / D];
    tg[t][idx % D] = Act<T>::ld(tgt + ((long)b * Tn + t) * D + idx % D);
  }
  if (row_mask)
    for (int t = warp; t < Tn; t += 8)
      if (row_mask[(long)b * Tn + t] == 0 && s0 + lane < s_end) sc[((long)b * Tn + t) * S + s0 + lane] = 0.f;
  __syncthreads();
  float w[8];
  Act<float>::load8(wr + lane * 8, w);
  for (int s = s0 + warp; s < s_end; s += 8) {
    const long srow = src_row(ranges, b, S, s);
    if (srow < 0 || (src_mask && src_mask[(long)b * S + s] == 0)) {
      for (int a = lane; a < na; a += 32) sc[((long)b * Tn + active_t[a]) * S + s] = 0.f;
      continue;
    }
    float x[8];
    Act<T>::load8(src + srow * D + lane * 8, x);
    for (int a = 0; a < na; ++a) {
      const int t = active_t[a];
      float y[8];
      Act<float>::load8(&tg[t][lane * 8], y);
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) acc = fmaf(w[i], tanhf(x[i] + y[i]), acc);
      acc = warp_sum(acc);
      if (lane == 0) sc[((long)b * Tn + t) * S + s] = acc + b_res;
    }
  }
}

// backward: only (b,t) rows flagged active carry gradient (rows whose label is a copy label).
//   d_src[b,s,:] = sum_t g[b,t,s] w (1 - th^2),  d_tgt[b,t,:] = sum_s (same),  d_w = sum g th,  d_b = sum g
template <typename T>
__global__ void __launch_bounds__(256) copy_scores_bwd_kernel(const T* __restrict__ src, const T* __restrict__ tgt,
                                                              const float* __restrict__ w_res,
                                                              const float* __restrict__ d_sc,
                                                              const unsigned char* __restrict__ row_active,
                                                              const int* __restrict__ ranges,
                                                              T* __restrict__ d_src, float* __restrict__ d_tgt,
                                                              float* __restrict__ d_w, float* __restrict__ d_b, int B,
                                                              int Tn, int S) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  extern __shared__ __align__(16) float dyn_smem[];
  float (*tg)[D] = reinterpret_cast<float (*)[D]>(dyn_smem);                    // [TMAX][D]
  float (*dtg)[D] = reinterpret_cast<float (*)[D]>(dyn_smem + TMAX * D);        // [TMAX][D]
  float* wr = dyn_smem + 2 * TMAX * D;                                          // [D]
  float (*red_w)[D] = reinterpret_cast<float (*)[D]>(dyn_smem + 2 * TMAX * D + D);  // [8][D]
  __shared__ int active_t[TMAX];
  __shared__ int n_active;
  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    int n = 0;
    for (int t = 0; t < Tn; ++t) if (row_active[(long)b * Tn + t]) active_t[n++] = t;
    n_active = n;
  }
  for (int idx = threadIdx.x; idx < Tn * D; idx += blockDim.x) {
    tg[idx / D][idx % D] = Act<T>::ld(tgt + (long)b * Tn * D + idx);
    dtg[idx / D][idx % D] = 0.f;
  }
  for (int idx = threadIdx.x; idx < D; idx += blockDim.x) wr[idx] = w_res[idx];
  __syncthreads();
  const int na = n_active;
  float w[8], dw[8];
  Act<float>::load8(wr + lane * 8, w);
#pragma unroll
  for (int i = 0; i < 8; ++i) dw[i] = 0.f;
  float dbias = 0.f;
  const int rows_per_cta = 32;
  const int s_end = min(S, (int)(blockIdx.x + 1) * rows_per_cta);
  for (int s = blockIdx.x * rows_per_cta + warp; s < s_end; s += 8) {
    const long srow = src_row(ranges, b, S, s);
    if (srow < 0) continue;                            // beyond the commit's memory rows (packed batches)
    float x[8], dx[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) dx[i] = 0.f;
    if (na > 0) Act<T>::load8(src + srow * D + lane * 8, x);
    for (int a = 0; a < na; ++a) {
      const int t = active_t[a];
      const float g = d_sc[((long)b * Tn + t) * S + s];
      if (g == 0.f) continue;      // warp-uniform
      float y[8];
      Act<float>::load8(&tg[t][lane * 8], y);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float th = tanhf(x[i] + y[i]);
        const float term = g * w[i] * (1.f - th * th);
        dx[i] += term;
        dw[i] = fmaf(g, th, dw[i]);
        atomicAdd(&dtg[t][lane * 8 + i], term);
      }
      dbias += g;
    }
    Act<T>::store8(d_src + srow * D + lane * 8, dx);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) red_w[warp][lane * 8 + i] = dw[i];
  __syncthreads();
  if (na > 0) {
    for (int idx = threadIdx.x; idx < D; idx += blockDim.x) {
      float sacc = 0.f;
#pragma unroll
      for (int q = 0; q < 8; ++q) sacc += red_w[q][idx];
      atomicAdd(d_w + idx, sacc);
    }
    for (int a = 0; a < na; ++a) {
      const int t = active_t[a];
      for (int idx = threadIdx.x; idx < D; idx += blockDim.x) atomicAdd(d_tgt + ((long)b * Tn + t) * D + idx, dtg[t][idx]);
    }
    if (lane == 0 && dbias != 0.f) atomicAdd(d_b, dbias);
  }
}

// ------------------------------------------------------------------ mixture / loss / argmax
struct MaxSum { float m, s; };
__device__ __forceinline__ MaxSum ms_merge(MaxSum a, MaxSum b) {
  const float m = fmaxf(a.m, b.m);
  MaxSum r;
  r.m = m;
  r.s = (a.s == 0.f ? 0.f : a.s * expf(a.m - m)) + (b.s == 0.f ? 0.f : b.s * expf(b.m - m));
  return r;
}
__device__ __forceinline__ MaxSum ms_warp(MaxSum v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    MaxSum u;
    u.m = __shfl_xor_sync(0xffffffffu, v.m, o);
    u.s = __shfl_xor_sync(0xffffffffu, v.s, o);
    v = ms_merge(v, u);
  }
  return v;
}
struct ArgMax { float v; int i; };
__device__ __forceinline__ ArgMax am_better(ArgMax a, ArgMax b) {   // larger value, then smaller index
  return (b.v > a.v || (b.v == a.v && b.i < a.i)) ? b : a;
}

// The mixture of one row, defined once: every kernel that forms P_j or log clamp(P_j) goes through these, so the
// log-probability a decoding step emits for label j is bit for bit -nll of fira_pointer_mix_nll_fwd for that label.
// Row statistics: vocab max / sum-exp (online, 8 logits per 16-byte (bf16) / 32-byte (fp32) load, the running (max, sum)
// rescaled once per group), copy max / sum-exp with the -1e9 fill (Model.py:61), gates.  Block-wide: every thread of
// the 256 calls it.  vocab == false skips the vocabulary pass without reading lrow and records vmax = 0, vsum = 1.
struct MixRow {
  float vmax, vsum, cmax, csum, g0, g1;
  __device__ __forceinline__ float pv(float x) const { return g0 * (expf(x - vmax) / vsum); }   // P of logit x
  __device__ __forceinline__ float pc(float c) const { return g1 * (expf(c - cmax) / csum); }   // P of copy score c
};
template <typename T>
__device__ __forceinline__ MixRow mix_row_stats(const T* __restrict__ lrow, const float* __restrict__ srow,
                                                const unsigned char* __restrict__ mrow, const float* __restrict__ gl,
                                                int V, int S, MaxSum* sh_ms, float* bc, bool vocab = true) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  MaxSum v{-INFINITY, 0.f};
  if (vocab) {
    const int V8 = V >> 3;
    for (int g = threadIdx.x; g < V8; g += blockDim.x) {
      float x[8];
      Act<T>::load8(lrow + (long)g * 8, x);
      float m8 = x[0];
#pragma unroll
      for (int i = 1; i < 8; ++i) m8 = fmaxf(m8, x[i]);
      if (m8 > v.m) { v.s *= expf(v.m - m8); v.m = m8; }
#pragma unroll
      for (int i = 0; i < 8; ++i) v.s += expf(x[i] - v.m);
    }
    for (int j = V8 * 8 + threadIdx.x; j < V; j += blockDim.x) { MaxSum u{Act<T>::ld(lrow + j), 1.f}; v = ms_merge(v, u); }
  } else if (threadIdx.x == 0) v = MaxSum{0.f, 1.f};
  v = ms_warp(v);
  if (lane == 0) sh_ms[warp] = v;
  __syncthreads();
  if (warp == 0) { MaxSum u = lane < 8 ? sh_ms[lane] : MaxSum{-INFINITY, 0.f}; u = ms_warp(u); if (lane == 0) { bc[0] = u.m; bc[1] = u.s; } }
  __syncthreads();
  MaxSum c{-INFINITY, 0.f};
  for (int j = threadIdx.x; j < S; j += blockDim.x) { MaxSum u{mrow[j] ? srow[j] : kMaskFill, 1.f}; c = ms_merge(c, u); }
  c = ms_warp(c);
  if (lane == 0) sh_ms[warp] = c;
  __syncthreads();
  if (warp == 0) { MaxSum u = lane < 8 ? sh_ms[lane] : MaxSum{-INFINITY, 0.f}; u = ms_warp(u); if (lane == 0) { bc[2] = u.m; bc[3] = u.s; } }
  __syncthreads();
  const float vmax = bc[0], vsum = bc[1], cmax = bc[2], csum = bc[3];
  const float gl0 = gl[0], gl1 = gl[1];
  const float gm = fmaxf(gl0, gl1);
  const float e0 = expf(gl0 - gm), e1 = expf(gl1 - gm);
  const float g0 = e0 / (e0 + e1), g1 = e1 / (e0 + e1);
  return MixRow{vmax, vsum, cmax, csum, g0, g1};
}
// P_j, the probability of label j < V + S
template <typename T>
__device__ __forceinline__ float mix_prob(const MixRow& ms, const T* __restrict__ lrow, const float* __restrict__ srow,
                                          const unsigned char* __restrict__ mrow, int V, int j) {
  if (j < V) return ms.pv(Act<T>::ld(lrow + j));
  const int s = j - V;
  return ms.pc(mrow[s] ? srow[s] : kMaskFill);
}
// log(clamp(p, 1e-10, 1)): the label's log-probability, -nll (Model.py:69,81-82)
__device__ __forceinline__ float mix_lp(float p) { return logf(fminf(fmaxf(p, 1e-10f), 1.f)); }

// Vocabulary-label rows of a training batch (label in (0, V)) in row order: vslot[row] = the row's compact slot or -1,
// vrows[slot] = its row, -1 in the slots [count, cap).  One CTA; each thread takes a contiguous run of rows.
constexpr int kRowsThreads = 1024;
__global__ void __launch_bounds__(kRowsThreads) vocab_rows_kernel(const int* __restrict__ label, long rows, int V,
                                                                  int* __restrict__ vslot, int* __restrict__ vrows,
                                                                  int cap) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ int warp_sum_s[kRowsThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long per = (rows + kRowsThreads - 1) / kRowsThreads;
  const long r0 = min(rows, (long)threadIdx.x * per), r1 = min(rows, r0 + per);
  int n = 0;
  for (long r = r0; r < r1; ++r) n += (label[r] != 0 && label[r] < V);
  int incl = n;                                   // inclusive scan over the warp, then over the warps
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
  if (lane == 31) warp_sum_s[warp] = incl;
  for (int s = threadIdx.x; s < cap; s += kRowsThreads) vrows[s] = -1;
  __syncthreads();
  int slot = incl - n;
  for (int w = 0; w < warp; ++w) slot += warp_sum_s[w];
  for (long r = r0; r < r1; ++r) {
    // count <= cap is the caller's bound; rows past it get no slot, and head_fwd_kernel gives them a NaN loss
    const bool v = label[r] != 0 && label[r] < V && slot < cap;
    vslot[r] = v ? slot : -1;
    if (v) vrows[slot++] = (int)r;
  }
}

// Live target rows of a training batch, the rows before each commit's last non-zero shifted label: tlen[b] = 1 + that
// t (0 without one); toff[b] = the commit's first slot, slots in row order; trows[slot] = b T + t, -1 in the slots past
// the count.  A commit past cap gets the slots left (toff clamps to cap), so toff[b + 1] - toff[b] < tlen[b] flags it.
// One CTA, one thread per commit.
__global__ void __launch_bounds__(kRowsThreads) target_rows_kernel(const int* __restrict__ label, int B, int T,
                                                                   int* __restrict__ tlen, int* __restrict__ toff,
                                                                   int* __restrict__ trows, int cap) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ int warp_sum_s[kRowsThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, b = threadIdx.x;
  int n = 0;
  if (b < B)
    for (int t = T - 1; t >= 0; --t)
      if (label[(long)b * T + t] != 0) { n = t + 1; break; }
  int incl = n;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
  if (lane == 31) warp_sum_s[warp] = incl;
  for (int s = threadIdx.x; s < cap; s += kRowsThreads) trows[s] = -1;
  __syncthreads();
  int off = incl - n;
  for (int w = 0; w < warp; ++w) off += warp_sum_s[w];
  if (b < B) {
    const int s0 = min(off, cap), s1 = min(off + n, cap);
    tlen[b] = n;
    toff[b] = s0;
    if (b == B - 1) toff[B] = s1;
    for (int s = s0; s < s1; ++s) trows[s] = b * T + (s - off);
  }
}

// dst[i] = idx[i] >= 0 ? src[idx[i]] : 0 over rows of `width` elements (width % 8 == 0); one warp per row
template <typename T>
__global__ void __launch_bounds__(256) gather_rows_kernel(const T* __restrict__ src, long ld_src,
                                                          const int* __restrict__ idx, T* __restrict__ dst, long ld_dst,
                                                          long n, int width) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const int lane = threadIdx.x & 31;
  for (long i = (long)blockIdx.x * 8 + (threadIdx.x >> 5); i < n; i += (long)gridDim.x * 8) {
    const int r = idx[i];
    for (int c = lane * 8; c < width; c += 256) {
      float x[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (r >= 0) Act<T>::load8(src + (long)r * ld_src + c, x);
      Act<T>::store8(dst + i * ld_dst + c, x);
    }
  }
}

// stats row layout (8 floats): vmax, vsum, cmax, csum, g0, g1, p_label, unused
// vslot (may be NULL): the logits of row r are row vslot[r] of `logits` (vocabulary-label rows only, training)
template <typename T>
__global__ void __launch_bounds__(256) head_fwd_kernel(const T* __restrict__ logits, long ldl,
                                                       const float* __restrict__ sc, const float* __restrict__ gate_logit,
                                                       const unsigned char* __restrict__ mem_mask,
                                                       const int* __restrict__ label, const int* __restrict__ vslot,
                                                       float* __restrict__ stats, float* __restrict__ nll,
                                                       int* __restrict__ argmax_out, int Tn, int V, int S) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ MaxSum sh_ms[8];
  __shared__ ArgMax sh_am[8];
  __shared__ float bc[8];
  const long row = blockIdx.x;
  const int b = (int)(row / Tn);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long lslot = vslot ? (long)vslot[row] : row;       // -1: the row has no logits
  const T* lrow = logits + lslot * ldl;
  const float* srow = sc + row * S;
  const unsigned char* mrow = mem_mask + (long)b * S;

  // pass 1: the row statistics.  Training (no argmax wanted): a row's loss only needs the softmax its label lives in,
  // so rows whose label is padding or a copy label skip the 24,650-wide pass (and copy-label rows are the only ones
  // that need `sc`).
  const int lab = label[row];
  const bool need_vocab = argmax_out != nullptr || (lab != 0 && lab < V && lslot >= 0);
  const MixRow ms = mix_row_stats(lrow, srow, mrow, gate_logit + row * 2, V, S, sh_ms, bc, need_vocab);

  if (threadIdx.x == 0) {
    float p = 1.f;
    // a vocabulary-label row left without a slot (a caller's cap below the row count) reports NaN, not a plausible loss
    const bool no_slot = lab != 0 && lab < V && lslot < 0;
    if (lab != 0) {
      // a copy label beyond the (possibly loader-trimmed) source is never read out of bounds: it gets p = 0 -> the
      // clamp floor, no gradient -- what the reference computes for a label on a padded (masked) source position
      // (Model.py:61,69); beyond V+370 the reference's nll_loss raises instead (Model.py:81)
      if (no_slot) p = NAN;
      else p = lab - V < S ? mix_prob(ms, lrow, srow, mrow, V, lab) : 0.f;
    }
    float* st = stats + row * 8;
    st[0] = ms.vmax; st[1] = ms.vsum; st[2] = ms.cmax; st[3] = ms.csum; st[4] = ms.g0; st[5] = ms.g1; st[6] = p;
    st[7] = 0.f;
    // loss = -log(clamp(p, 1e-10, 1)), zeroed where label == 0
    nll[row] = no_slot ? NAN : (lab != 0 ? -mix_lp(p) : 0.f);
  }
  if (argmax_out) {
    // argmax over log(clamp(p)) of the concatenation, first index wins ties (Model.py:86)
    ArgMax best{-INFINITY, 0x7fffffff};
    const float iv = 1.f / ms.vsum, ic = 1.f / ms.csum;
    for (int j = threadIdx.x; j < V + S; j += blockDim.x) {
      float p;
      if (j < V) p = ms.g0 * (expf(Act<T>::ld(lrow + j) - ms.vmax) * iv);
      else { const int s = j - V; p = ms.g1 * (expf((mrow[s] ? srow[s] : kMaskFill) - ms.cmax) * ic); }
      ArgMax cand{mix_lp(p), j};
      best = am_better(best, cand);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ArgMax u{__shfl_xor_sync(0xffffffffu, best.v, o), __shfl_xor_sync(0xffffffffu, best.i, o)};
      best = am_better(best, u);
    }
    if (lane == 0) sh_am[warp] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
      ArgMax r = sh_am[0];
      for (int q = 1; q < 8; ++q) r = am_better(r, sh_am[q]);
      argmax_out[row] = r.i;
    }
  }
}

// d(loss_sum)/d(logits, copy scores, gate logits); `upstream` is d(loss_sum) (a device scalar).
// Exactly one of the two softmaxes receives gradient per row (the picked element decides), rows with
// label == 0 or p outside [1e-10, 1] (clamp) receive none.
// seq_weight (may be NULL = all 1): loss_sum = sum_row seq_weight[row / Tn] * nll[row], so row `row` takes upstream
// *upstream * seq_weight[row / Tn]; a row of weight exactly 0 receives nothing, like a label-0 row.
// vslot / vrows (may be NULL, then logits / d_logits have one row per row): logits and d_logits hold the slots of the
// vocabulary-label rows; d_logits is written for those slots only, and CTA s < cap also zeroes slot s if it is unused.
template <typename T>
__global__ void __launch_bounds__(256) head_bwd_kernel(const T* __restrict__ logits, long ldl,
                                                       const float* __restrict__ sc,
                                                       const unsigned char* __restrict__ mem_mask,
                                                       const int* __restrict__ label, const int* __restrict__ vslot,
                                                       const int* __restrict__ vrows, int cap,
                                                       const float* __restrict__ stats,
                                                       const float* __restrict__ upstream, T* __restrict__ d_logits,
                                                       float* __restrict__ d_sc, float* __restrict__ d_gate_logit,
                                                       unsigned char* __restrict__ row_active, int Tn, int V, int S,
                                                       const float* __restrict__ seq_weight) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const long row = blockIdx.x;
  const int b = (int)(row / Tn);
  const float* st = stats + row * 8;
  const float vmax = st[0], vsum = st[1], cmax = st[2], csum = st[3], g0 = st[4], g1 = st[5], p = st[6];
  const int lab = label[row];
  const float w = seq_weight ? seq_weight[b] : 1.f;
  const float up = seq_weight ? *upstream * w : *upstream;
  const bool live = lab != 0 && w != 0.f && p >= 1e-10f && p <= 1.f;
  const long lslot = vslot ? (long)vslot[row] : row;      // -1: the row has no logits
  const bool vocab = live && lab < V && lslot >= 0;
  const bool copy = live && lab >= V;
  T* drow = d_logits + lslot * ldl;
  const T* lrow = logits + lslot * ldl;
  const int V8 = V >> 3;                         // 8 logits per vector load / store, scalar tail
  const float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (vslot && row < cap && vrows[row] < 0) {    // an unused slot: the products over the slots read it
    T* prow = d_logits + row * ldl;
    for (int g = threadIdx.x; g < V8; g += blockDim.x) Act<T>::store8(prow + (long)g * 8, z);
    for (int j = V8 * 8 + threadIdx.x; j < V; j += blockDim.x) Act<T>::st(prow + j, 0.f);
  }
  if (vocab) {
    const float iv = 1.f / vsum;
    for (int g = threadIdx.x; g < V8; g += blockDim.x) {
      float x[8];
      Act<T>::load8(lrow + (long)g * 8, x);
#pragma unroll
      for (int i = 0; i < 8; ++i) x[i] = up * (expf(x[i] - vmax) * iv - (g * 8 + i == lab ? 1.f : 0.f));
      Act<T>::store8(drow + (long)g * 8, x);
    }
    for (int j = V8 * 8 + threadIdx.x; j < V; j += blockDim.x) {
      float pv = expf(Act<T>::ld(lrow + j) - vmax) * iv;
      Act<T>::st(drow + j, up * (pv - (j == lab ? 1.f : 0.f)));
    }
  } else if (lslot >= 0) {
    for (int g = threadIdx.x; g < V8; g += blockDim.x) Act<T>::store8(drow + (long)g * 8, z);
    for (int j = V8 * 8 + threadIdx.x; j < V; j += blockDim.x) Act<T>::st(drow + j, 0.f);
  }
  const float* srow = sc + row * S;
  const unsigned char* mrow = mem_mask + (long)b * S;
  float* dsrow = d_sc + row * S;
  if (copy) {
    const float ic = 1.f / csum;
    for (int j = threadIdx.x; j < S; j += blockDim.x) {
      float pc = expf((mrow[j] ? srow[j] : kMaskFill) - cmax) * ic;
      // masked positions were overwritten by masked_fill -> no gradient reaches the raw score
      dsrow[j] = mrow[j] ? up * (pc - (j == lab - V ? 1.f : 0.f)) : 0.f;
    }
  } else {
    for (int j = threadIdx.x; j < S; j += blockDim.x) dsrow[j] = 0.f;
  }
  if (threadIdx.x == 0) {
    float d0 = 0.f, d1 = 0.f;
    if (vocab) { d0 = up * (g0 - 1.f); d1 = up * g1; }
    if (copy) { d0 = up * g0; d1 = up * (g1 - 1.f); }
    d_gate_logit[row * 2] = d0; d_gate_logit[row * 2 + 1] = d1;
    row_active[row] = copy ? 1 : 0;
  }
}

// ------------------------------------------------------------------ seeded sampling from the mixture
// One CTA per row (commit b, sample n).  Candidates are the j of [vocab || copy positions] with mem_mask set and
// P_j > 0 in fp32; s_j = log P_j / T.  The rank order (s descending, then index ascending) is a strict total order,
// encoded as a 47-bit key (32 order-preserving bits of s, 15 bits of 0x7fff - j), so every cut is "key >= threshold":
//   top-k: the largest threshold that still keeps k candidates; top-p: the largest threshold whose kept weight
//   sum(exp(s - s_max)) reaches p times the weight left after top-k.  Both are bisections over the key with
//   fixed-order block reductions (integer counts / fp32 sums), so a row's draw is a pure function of its inputs.
// Draw: u * Z against the kept weights in index order.  The scores are staged once in dynamic shared memory.
constexpr int kSampleThreads = 256;                   // = head_fwd_kernel's block: the same row statistics, bit for bit
constexpr uint32_t kSampleStream = 0x53414D50u;       // Philox stream id of the draw; dropout sites use ids < 256
constexpr uint64_t kKeyEnd = 1ull << 47;

__device__ __forceinline__ bool is_cand(float s) { return s == s; }          // NaN marks a non-candidate
__device__ __forceinline__ uint32_t order_bits(float s) {      // unsigned order = float order (no NaN)
  const uint32_t b = __float_as_uint(s);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ uint64_t rank_key(float s, int j) {
  return ((uint64_t)order_bits(s) << 15) | (uint32_t)(0x7FFF - j);
}

// fixed-order reduction: xor butterfly inside each warp, then the 8 warp results in warp order (every thread gets it)
template <typename V, typename Op>
__device__ __forceinline__ V block_reduce(V v, V* sh, Op op) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();                                    // `sh` may still be read by the previous reduction
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  V r = sh[0];
#pragma unroll
  for (int w = 1; w < kSampleThreads / 32; ++w) r = op(r, sh[w]);
  return r;
}
// the candidates among this thread's staged scores s[j0, j1) with rank_key(s_j, j) >= th, counted over the block
__device__ __forceinline__ unsigned count_key_ge(const float* s, int j0, int j1, uint64_t th, unsigned* shu) {
  unsigned k = 0;
  for (int j = j0; j < j1; ++j) { const float v = s[j]; k += (is_cand(v) && rank_key(v, j) >= th) ? 1u : 0u; }
  return block_reduce(k, shu, [](unsigned a, unsigned x) { return a + x; });
}
// for k below the candidate count: the largest cut with count_ge(cut) >= k.  Keys are distinct, so the candidates with
// rank_key >= cut are exactly the k best.
template <typename Count>
__device__ __forceinline__ uint64_t key_cut(unsigned k, Count&& count_ge) {
  uint64_t lo = 1, hi = kKeyEnd;                      // count_ge(lo) >= k, count_ge(hi) < k
  while (hi - lo > 1) { const uint64_t mid = lo + (hi - lo) / 2; if (count_ge(mid) >= k) lo = mid; else hi = mid; }
  return lo;
}

// n-gram repeat blocking and minimum length (the _rules entry points).  The words of a live row at position `pos` are
// its history hist[1..pos] (hist[0] is <start>; a copy's word is already copy_src there).  Label j with word w is banned
// at column pos + 1 when appending w repeats an n-gram of the history (n = no_repeat >= 1) or when w is eos_id and the
// row has fewer than min_len words (pos < min_len).  Banned words go into a list s_ban[0..nb): s_ban[0] is eos_id or
// -1, s_ban[i] (1 <= i <= pos - n + 1) is words[i + n - 1] when words[i .. i + n - 2] == words[pos - n + 2 .. pos], else
// -1 (no word is negative).  nb = 0 when both rules are off.
__device__ __forceinline__ int ban_count(int pos, int no_repeat, int min_len) {
  if (!no_repeat && !min_len) return 0;
  return 1 + (no_repeat ? max(0, pos - no_repeat + 1) : 0);
}
// threads 0..pos copy the history into shared memory; a __syncthreads must follow before ban_build
__device__ __forceinline__ void ban_load(const int* __restrict__ hist, int pos, int nb, int* s_hist) {
  if (nb && (int)threadIdx.x <= pos) s_hist[threadIdx.x] = hist[threadIdx.x];
}
// threads 0..nb-1 write one entry each; a __syncthreads must follow before the list is read
__device__ __forceinline__ void ban_build(const int* s_hist, int pos, int no_repeat, int min_len, int eos_id, int nb,
                                          int* s_ban) {
  const int i = threadIdx.x;
  if (i >= nb) return;
  int w = -1;
  if (i == 0) {
    if (pos < min_len) w = eos_id;
  } else {                                            // nb > 1: no_repeat >= 1 and i + no_repeat - 1 <= pos
    bool same = true;
    for (int k = 0; k + 1 < no_repeat; ++k) same &= s_hist[i + k] == s_hist[pos - no_repeat + 2 + k];
    if (same) w = s_hist[i + no_repeat - 1];
  }
  s_ban[i] = w;
}
__device__ __forceinline__ bool is_banned(const int* s_ban, int nb, int w) {
  bool hit = false;
  for (int e = 0; e < nb; ++e) hit |= s_ban[e] == w;
  return hit;
}

template <typename T>
__global__ void __launch_bounds__(kSampleThreads) pointer_mix_sample_kernel(
    const T* __restrict__ logits, long ldl, const float* __restrict__ sc, const float* __restrict__ gate_logit,
    const unsigned char* __restrict__ mem_mask, const int* __restrict__ copy_src, const uint64_t* __restrict__ seed_p,
    const int* __restrict__ first_index_p, const float* __restrict__ uniforms, float temp, int top_k, float top_p,
    int eos_id, int pad_id, int* __restrict__ next_tok, int* __restrict__ seq, int* __restrict__ raw,
    float* __restrict__ tok_lp, unsigned char* __restrict__ tok_mask, long ld_out, int pos,
    unsigned char* __restrict__ finished, int* __restrict__ length, float* __restrict__ lp_sum,
    const int* __restrict__ prefix, int ld_prefix, const int* __restrict__ prefix_len, int no_repeat, int min_len,
    int N, int V, int S) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  extern __shared__ float s_sc[];                     // [V + S] tempered scores, NaN = not a candidate
  __shared__ int s_hist[TMAX], s_ban[TMAX];           // the row's history and banned words (ban_build)
  __shared__ MaxSum sh_ms[8];
  __shared__ float bc[4];
  __shared__ float shf[8];
  __shared__ unsigned shu[8];
  __shared__ int shi[8];
  __shared__ float part[kSampleThreads];
  __shared__ float sh_target;
  __shared__ int sh_pick;
  const long row = blockIdx.x;
  const int b = (int)(row / N), n = (int)(row % N);
  const long o = row * ld_out + pos + 1;
  if (finished[row]) {                                // after <eos>: pad, no log-probability, length kept
    if (threadIdx.x == 0) { next_tok[row] = pad_id; seq[o] = pad_id; raw[o] = pad_id; tok_lp[o] = 0.f; tok_mask[o] = 0; }
    return;
  }
  const T* lrow = logits + row * ldl;
  const float* srow = sc + row * S;
  const unsigned char* mrow = mem_mask + (long)b * S;

  const MixRow ms = mix_row_stats(lrow, srow, mrow, gate_logit + row * 2, V, S, sh_ms, bc);
  // thread 0: label j becomes the row's token at column pos + 1, with the loop bookkeeping
  auto emit = [&](int j) {
    const float lp = mix_lp(mix_prob(ms, lrow, srow, mrow, V, j));
    const int tok = j < V ? j : copy_src[(long)b * S + (j - V)];
    next_tok[row] = tok; seq[o] = tok; raw[o] = j; tok_lp[o] = lp; tok_mask[o] = tok != pad_id;
    length[row] += 1;
    lp_sum[row] += lp;
    if (tok == eos_id) finished[row] = 1;
  };
  if (prefix && pos < prefix_len[b]) {                // inside the commit's prefix: its label, no cut and no draw
    if (threadIdx.x == 0) emit(prefix[(long)b * ld_prefix + pos]);
    return;
  }

  const int nb = ban_count(pos, no_repeat, min_len);
  ban_load(seq + row * ld_out, pos, nb, s_hist);
  const int C = V + S;
  for (int j = threadIdx.x; j < C; j += blockDim.x) {
    const float p = mix_prob(ms, lrow, srow, mrow, V, j);
    s_sc[j] = ((j < V || mrow[j - V]) && p > 0.f) ? logf(fminf(p, 1.f)) / temp : __int_as_float(0x7fffffff);
  }
  __syncthreads();
  if (nb) {                                           // banned labels stop being candidates (before the cuts)
    ban_build(s_hist, pos, no_repeat, min_len, eos_id, nb, s_ban);
    __syncthreads();
    if ((int)threadIdx.x < nb) { const int w = s_ban[threadIdx.x]; if (w >= 0 && w < V) s_sc[w] = __int_as_float(0x7fffffff); }
    const int* crow = copy_src + (long)b * S;
    for (int s = threadIdx.x; s < S; s += blockDim.x)
      if (is_cand(s_sc[V + s]) && is_banned(s_ban, nb, crow[s])) s_sc[V + s] = __int_as_float(0x7fffffff);
    __syncthreads();
  }

  // every pass below walks a contiguous index range per thread (index order is what the draw needs)
  const int chunk = (C + kSampleThreads - 1) / kSampleThreads;
  const int j0 = min(C, (int)threadIdx.x * chunk), j1 = min(C, j0 + chunk);
  auto add_u = [](unsigned a, unsigned x) { return a + x; };
  auto add_f = [](float a, float x) { return a + x; };
  float smax = -INFINITY;
  unsigned cnt = 0;
  for (int j = j0; j < j1; ++j) { const float s = s_sc[j]; if (is_cand(s)) { smax = fmaxf(smax, s); ++cnt; } }
  smax = block_reduce(smax, shf, [](float a, float x) { return fmaxf(a, x); });
  const unsigned n_cand = block_reduce(cnt, shu, add_u);
  auto weight = [&](float s) { return s == smax ? 1.f : expf(s - smax); };
  auto count_ge = [&](uint64_t th) { return count_key_ge(s_sc, j0, j1, th, shu); };
  auto weight_ge = [&](uint64_t th) {
    float a = 0.f;
    for (int j = j0; j < j1; ++j) { const float s = s_sc[j]; if (is_cand(s) && rank_key(s, j) >= th) a += weight(s); }
    return block_reduce(a, shf, add_f);
  };
  uint64_t cut = 1;                                   // kept <=> candidate with rank_key >= cut
  if (top_k > 0 && (unsigned)top_k < n_cand) cut = key_cut((unsigned)top_k, count_ge);
  if (top_p < 1.f && n_cand > 1) {
    const float target = top_p * weight_ge(cut);
    uint64_t lo = cut, hi = kKeyEnd;                  // the top candidate alone has weight 1 > 0: lo stays at or below it
    while (hi - lo > 1) { const uint64_t mid = lo + (hi - lo) / 2; if (weight_ge(mid) >= target) lo = mid; else hi = mid; }
    cut = lo;
  }

  // draw: prefix sums of the kept weights in index order (one fixed-order scan of the per-thread sums)
  float a = 0.f;
  int last = -1;
  for (int j = j0; j < j1; ++j) {
    const float s = s_sc[j];
    if (is_cand(s) && rank_key(s, j) >= cut) { const float w = weight(s); a += w; if (w > 0.f) last = j; }
  }
  last = block_reduce(last, shi, [](int x, int y) { return max(x, y); });   // fallback when u * Z rounds to Z
  part[threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    float acc = 0.f;
    for (int i = 0; i < kSampleThreads; ++i) { acc += part[i]; part[i] = acc; }
    float u;
    if (uniforms) {
      u = uniforms[row];
    } else {
      const uint64_t seed = *seed_p;
      const uint4 r = philox4((uint32_t)(*first_index_p + b), (uint32_t)n, kSampleStream, (uint32_t)pos,
                              (uint32_t)seed, (uint32_t)(seed >> 32));
      u = (float)(r.x >> 8) * 0x1p-24f;
    }
    sh_target = u * acc;
    sh_pick = last >= 0 ? last : 0;
  }
  __syncthreads();
  const float target = sh_target;
  const float excl = threadIdx.x ? part[threadIdx.x - 1] : 0.f;
  if (excl <= target && target < part[threadIdx.x]) {   // at most one thread: the one whose range crosses u * Z
    float r = excl;
    int pick = -1;
    for (int j = j0; j < j1; ++j) {
      const float s = s_sc[j];
      if (!is_cand(s) || rank_key(s, j) < cut) continue;
      const float w = weight(s);
      if (w > 0.f) { r += w; pick = j; if (r > target) break; }
    }
    sh_pick = pick;
  }
  __syncthreads();
  if (threadIdx.x == 0) emit(sh_pick);
}

// ------------------------------------------------------------------ one n-best beam step from the mixture
// Slot rows r = b * K + k.  The slot state is double-buffered ([2][B*K] scalars, [2][B*K][T] histories): position
// `pos` reads half pos & 1 and writes the other half, since a new slot's history is copied from a parent row that
// another CTA may be rewriting.  status: 0 live, 1 finished (its token was <eos>), 2 inactive (before position 0).
//   row stage     one CTA per live slot row: lp_j = log(clamp(P_j, 1e-10, 1)) of every vocabulary entry and unmasked
//                 copy position; the row's K best by rank_key(lp, j) (lp descending, then j ascending) -> workspace.
//                 Each thread keeps a sorted top K in registers over its strided indices, then K fixed-order block
//                 maxima pop the heads, so the result is a pure function of the row.
//   select stage  one CTA per commit: live slot i proposes its K row winners (i, j) with L = L_i + lp and n = n_i + 1,
//                 finished slot i proposes itself once as j = C = V + S; score = L / powf((5 + n) / 6, alpha); the K
//                 best by (score descending, then i * (C + 1) + j ascending) become new slots 0..K-1 in that order.
// Within one parent row the score rises with lp (n is the same for every extension), so every winner of the select
// stage is among its parent's row top K.
constexpr int kBeamThreads = 256;   // = head_fwd_kernel's block (the same row statistics); >= kMaxBeam^2 candidates
constexpr int kMaxBeam = 16;

__device__ __forceinline__ float key_lp(uint64_t key) {          // inverse of rank_key's score bits
  const uint32_t b = (uint32_t)(key >> 15);
  return __uint_as_float((b & 0x80000000u) ? (b & 0x7FFFFFFFu) : ~b);
}
__device__ __forceinline__ int key_index(uint64_t key) { return 0x7FFF - (int)(key & 0x7FFFu); }
__device__ __forceinline__ uint64_t key_max(uint64_t a, uint64_t b) { return a > b ? a : b; }
__device__ __forceinline__ uint64_t key_min(uint64_t a, uint64_t b) { return a < b ? a : b; }
// insert `x` into the descending list top[0..K) (entries from K on stay 0) -> the new top[K - 1]
__device__ __forceinline__ uint64_t topk_insert(uint64_t (&top)[kMaxBeam], uint64_t x, int K) {
  uint64_t last = ~0ull;                              // min over top[0..K) = top[K - 1], without a dynamic index
#pragma unroll
  for (int i = 0; i < kMaxBeam; ++i)
    if (i < K) { const uint64_t hi = key_max(top[i], x); x = key_min(top[i], x); top[i] = hi; last = key_min(last, hi); }
  return last;
}
// offer(P_j, j) for every vocabulary entry and unmasked copy position j of the row, this thread's strided share:
// 8 logits per vector load, the scalar tail, then the copy positions
template <typename T, typename Offer>
__device__ __forceinline__ void mix_scan(const MixRow& ms, const T* __restrict__ lrow, const float* __restrict__ srow,
                                         const unsigned char* __restrict__ mrow, int V, int S, Offer&& offer) {
  const int V8 = V >> 3;
  for (int g = threadIdx.x; g < V8; g += blockDim.x) {
    float x[8];
    Act<T>::load8(lrow + (long)g * 8, x);
#pragma unroll
    for (int i = 0; i < 8; ++i) offer(ms.pv(x[i]), g * 8 + i);
  }
  for (int j = V8 * 8 + threadIdx.x; j < V; j += blockDim.x) offer(ms.pv(Act<T>::ld(lrow + j)), j);
  for (int s = threadIdx.x; s < S; s += blockDim.x)
    if (mrow[s]) offer(ms.pc(srow[s]), V + s);
}
// block top K of the threads' descending lists: K fixed-order maxima over the list heads; keys are distinct, so exactly
// one thread owns each maximum and pops it.  Every thread calls emit(k, m) with the k-th best key m (0 = none left).
template <typename Emit>
__device__ __forceinline__ void topk_pop(uint64_t (&top)[kMaxBeam], int K, uint64_t* shk, Emit&& emit) {
  for (int k = 0; k < K; ++k) {
    const uint64_t m = block_reduce(top[0], shk, key_max);
    if (m != 0 && top[0] == m) {
#pragma unroll
      for (int i = 0; i + 1 < kMaxBeam; ++i) top[i] = top[i + 1];
      top[kMaxBeam - 1] = 0;
    }
    emit(k, m);
  }
}

// Lexically constrained n-best (LEX = true, fira_pointer_mix_beam_step_lexical; dynamic beam allocation, Post & Vilar,
// 2018).  Commit b has up to kPhrases phrases of up to kPhraseLen words, constraints[b][p][m] (0 = padding, no gaps),
// Tc words in all.  The words of a row are its history hist[1..pos] (copies as their words, prefix words included).
// Per phrase c of length L: prog_c(h) = L when c occurs contiguously in h, else the largest m < L with h ending in
// c_1..c_m (0 if none).  A row's progress is the sum over its phrases; it meets its constraints when progress = Tc.
// A live, non-forced row bans <eos> while its progress is below Tc and proposes
//   (a) its K best allowed labels (the plain row stage), and
//   (b) per unmet phrase, in phrase order, the best label by rank_key among j = w and the unmasked copies of w, where
//       w = c_{prog_c + 1}; skipped when w is banned, when an earlier phrase proposed w, or when the label is in (a).
// Every proposal (a forced row's one label too) carries its bank, the progress of the history with its word appended,
// in key bits kBankShift.. (rank_key uses bits 0..46; key_lp and key_index ignore the bank).  Phrase state from the
// history: occ (c occurs) and ends (bit m: h ends with c_1..c_m; bit 0 always); appending w gives L when occ, else the
// largest m <= L with ends bit m - 1 and c_m == w (0 if none).
constexpr int kPhrases = 4, kPhraseLen = 4, kMaxConstraintWords = kPhrases * kPhraseLen;
constexpr int kBankShift = 48;

struct Phrases { int con[kMaxConstraintWords], len[kPhrases], occ[kPhrases], ends[kPhrases], prog[kPhrases]; };

__device__ __forceinline__ int constraint_words(const int* __restrict__ con) {     // Tc of one commit
  int tc = 0;
  for (int e = 0; e < kMaxConstraintWords; ++e) tc += con[e] != 0;
  return tc;
}
// threads 0..kPhrases-1 fill phrase threadIdx.x's state from s_hist[1..pos]; a __syncthreads must follow
__device__ __forceinline__ void phrase_state(const int* __restrict__ con, const int* s_hist, int pos, Phrases& ph) {
  const int p = threadIdx.x;
  if (p >= kPhrases) return;
  const int* c = con + p * kPhraseLen;
  int L = 0;
  for (int m = 0; m < kPhraseLen; ++m) { ph.con[p * kPhraseLen + m] = c[m]; L += c[m] != 0; }
  const int* h = s_hist + 1;                          // the pos words
  bool occ = false;
  for (int a = 0; L && a + L <= pos && !occ; ++a) {
    bool same = true;
    for (int m = 0; m < L; ++m) same &= h[a + m] == c[m];
    occ = same;
  }
  int ends = 1, prog = 0;
  for (int m = 1; m < L && m <= pos; ++m) {
    bool same = true;
    for (int e = 0; e < m; ++e) same &= h[pos - m + e] == c[e];
    if (same) { ends |= 1 << m; prog = m; }
  }
  ph.len[p] = L; ph.occ[p] = occ; ph.ends[p] = ends; ph.prog[p] = occ ? L : prog;
}
// the progress of the row's words with w appended
__device__ __forceinline__ int phrase_bank(const Phrases& ph, int w) {
  int bank = 0;
  for (int p = 0; p < kPhrases; ++p) {
    const int L = ph.len[p];
    int best = ph.occ[p] ? L : 0;
    for (int m = 1; m <= L && !ph.occ[p]; ++m)
      if (((ph.ends[p] >> (m - 1)) & 1) && ph.con[p * kPhraseLen + m - 1] == w) best = m;
    bank += best;
  }
  return bank;
}

// LEX = false: the plain row stage (K entries per row); LEX = true: K + kPhrases entries per row, (a) then (b)
template <typename T, bool LEX>
__global__ void __launch_bounds__(kBeamThreads, 1) beam_row_kernel(
    const T* __restrict__ logits, long ldl, const float* __restrict__ sc, const float* __restrict__ gate_logit,
    const unsigned char* __restrict__ mem_mask, const int* __restrict__ copy_src, const unsigned char* __restrict__ status,
    const int* __restrict__ seq, int Tn, uint64_t* __restrict__ row_top, const int* __restrict__ prefix, int ld_prefix,
    const int* __restrict__ prefix_len, int no_repeat, int min_len, int eos_id, int pos, int K, int V, int S,
    const int* __restrict__ constraints) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ MaxSum sh_ms[8];
  __shared__ float bc[4];
  __shared__ uint64_t shk[8];
  __shared__ int s_hist[TMAX], s_ban[TMAX];           // the row's history and banned words (ban_build)
  const long row = blockIdx.x;
  if (status[row] != 0) return;                       // finished or inactive: the select stage reads nothing of it
  const int b = (int)(row / K);
  const int W = LEX ? K + kPhrases : K;               // row_top entries per row
  const T* lrow = logits + row * ldl;
  const float* srow = sc + row * S;
  const unsigned char* mrow = mem_mask + (long)b * S;
  const int nb = ban_count(pos, no_repeat, min_len);
  const int* con = LEX ? constraints + (long)b * kMaxConstraintWords : nullptr;
  const int tc = LEX ? constraint_words(con) : 0;
  ban_load(seq + row * Tn, pos, nb | tc, s_hist);
  const MixRow ms = mix_row_stats(lrow, srow, mrow, gate_logit + row * 2, V, S, sh_ms, bc);   // syncs s_hist too
  __shared__ Phrases ph;
  if constexpr (LEX) {
    if (tc) {
      phrase_state(con, s_hist, pos, ph);
      __syncthreads();
    }
  }
  auto with_bank = [&](uint64_t key) -> uint64_t {   // a proposal's key with its bank (LEX, Tc > 0)
    if (!LEX || !tc || key == 0) return key;
    const int j = key_index(key);
    return key | ((uint64_t)phrase_bank(ph, j < V ? j : copy_src[(long)b * S + (j - V)]) << kBankShift);
  };
  if (prefix && pos < prefix_len[b]) {                // inside the commit's prefix: its label is the row's one winner
    if (threadIdx.x == 0) {
      const int j = prefix[(long)b * ld_prefix + pos];
      row_top[row * W] = with_bank(rank_key(mix_lp(mix_prob(ms, lrow, srow, mrow, V, j)), j));
      for (int k = 1; k < W; ++k) row_top[row * W + k] = 0;
    }
    return;
  }
  int nbx = nb;                                       // nb + the <eos> entry of the constraints (LEX, Tc > 0)
  if constexpr (LEX) {
    if (tc) {
      int prog = 0;
      for (int p = 0; p < kPhrases; ++p) prog += ph.prog[p];
      if ((int)threadIdx.x == nb) s_ban[nb] = prog < tc ? eos_id : -1;
      nbx = nb + 1;
    }
  }
  if (nbx) {
    ban_build(s_hist, pos, no_repeat, min_len, eos_id, nb, s_ban);
    __syncthreads();
  }
  const int* crow = copy_src + (long)b * S;

  uint64_t top[kMaxBeam];                             // this thread's best keys, descending; 0 = empty
#pragma unroll
  for (int i = 0; i < kMaxBeam; ++i) top[i] = 0;
  uint64_t thr = 0;                                   // top[K - 1]: the key a candidate has to beat
  mix_scan(ms, lrow, srow, mrow, V, S, [&](float p, int j) {
    const uint64_t key = rank_key(mix_lp(p), j);
    if (key <= thr) return;
    if (nbx && is_banned(s_ban, nbx, j < V ? j : crow[j - V])) return;     // only entries that would enter the top K
    thr = topk_insert(top, key, K);
  });
  topk_pop(top, K, shk, [&](int k, uint64_t m) { if (threadIdx.x == 0) row_top[row * W + k] = with_bank(m); });
  if constexpr (LEX) {                                // (b): one block-wide best label per unmet phrase
    int nx = K;                                       // thread 0: the next free entry
    for (int p = 0; tc && p < kPhrases; ++p) {        // shared state only: uniform across the block
      if (ph.prog[p] == ph.len[p]) continue;
      const int w = ph.con[p * kPhraseLen + ph.prog[p]];
      bool skip = is_banned(s_ban, nbx, w);
      for (int q = 0; q < p; ++q) skip |= ph.prog[q] < ph.len[q] && ph.con[q * kPhraseLen + ph.prog[q]] == w;
      if (skip) continue;
      uint64_t best = threadIdx.x == 0 ? rank_key(mix_lp(mix_prob(ms, lrow, srow, mrow, V, w)), w) : 0;
      for (int s = threadIdx.x; s < S; s += blockDim.x)
        if (mrow[s] && crow[s] == w) best = key_max(best, rank_key(mix_lp(ms.pc(srow[s])), V + s));
      best = block_reduce(best, shk, key_max);
      if (threadIdx.x == 0) {
        bool in_a = false;                            // (a) as written above by this thread, without the banks
        for (int k = 0; k < K; ++k) in_a |= (row_top[row * W + k] & (kKeyEnd - 1)) == best;
        if (!in_a) row_top[row * W + nx++] = with_bank(best);
      }
    }
    if (threadIdx.x == 0) for (; nx < W; ++nx) row_top[row * W + nx] = 0;
  }
}

// Every select stage: new slot k0 + k (k < n) continues slot s_from[k] (j = s_j[k], C: carried unchanged) -> the written
// half of the slot state, parent, next_tok, chosen (may be NULL: the token it grew with, -1 when carried) and the
// histories (a grown slot gets its new token at column pos + 1)
__device__ __forceinline__ void beam_write_slots(const int* s_from, const int* s_j, const int* s_tok, const float* s_lp,
                                                 const float* s_L, const float* s_score, int eos_id, int pad_id,
                                                 int* __restrict__ seq, int* __restrict__ raw, float* __restrict__ tok_lp,
                                                 int* __restrict__ length, float* __restrict__ lp_sum,
                                                 float* __restrict__ score, unsigned char* __restrict__ status,
                                                 long* __restrict__ parent, int* __restrict__ next_tok,
                                                 int* __restrict__ chosen, int Tn, int pos, long in, long out, long base,
                                                 int k0, int n, int C) {
  if (threadIdx.x < n) {
    const int k = threadIdx.x;
    const long pr = in + base + s_from[k], slot = base + k0 + k, nr = out + slot;
    parent[slot] = base + s_from[k];
    if (s_j[k] == C) {                                // a finished (or inactive) slot carried unchanged
      length[nr] = length[pr]; lp_sum[nr] = lp_sum[pr]; score[nr] = score[pr]; status[nr] = status[pr];
      next_tok[slot] = pad_id;
      if (chosen) chosen[slot] = -1;
    } else {
      length[nr] = length[pr] + 1; lp_sum[nr] = s_L[k]; score[nr] = s_score[k];
      status[nr] = s_tok[k] == eos_id ? 1 : 0;
      next_tok[slot] = s_tok[k];
      if (chosen) chosen[slot] = s_tok[k];
    }
  }
  for (int e = threadIdx.x; e < n * Tn; e += blockDim.x) {
    const int k = e / Tn, c = e % Tn;
    const long src = (in + base + s_from[k]) * Tn + c, dst = (out + base + k0 + k) * Tn + c;
    const bool grow = s_j[k] != C && c == pos + 1;
    seq[dst] = grow ? s_tok[k] : seq[src];
    raw[dst] = grow ? s_j[k] : raw[src];
    tok_lp[dst] = grow ? s_lp[k] : tok_lp[src];
  }
}

// Select stage, plain and lexical: one CTA per commit, candidate threadIdx.x = i * W + q (W = K plain, K + kPhrases
// lexical: the row stage's entries per row): the q-th row entry of live slot i (lexical: its bank in key bits
// kBankShift..), or (q = 0) finished slot i itself; L = L_i + lp, n = n_i + 1, score = L / powf((5 + n) / 6, alpha).
// Tc = 0 (always without constraints): one bank, the K best by (score descending, i * (C + 1) + j ascending).
// Tc > 0: the carried finished slots first, best score first; then the live candidates striped over the banks: rank r
// within the candidate's bank by (score, index) as above, then the order (r ascending, bank descending), which is
// total since two candidates of one bank never share r.  Every order counts the larger keys.
constexpr int kSelectThreads = kMaxBeam * (kMaxBeam + kPhrases);     // 320 candidates at K = 16
__global__ void __launch_bounds__(kSelectThreads) beam_select_kernel(
    const uint64_t* __restrict__ row_top, int W, const int* __restrict__ constraints, const int* __restrict__ copy_src,
    float alpha, int eos_id, int pad_id, int* __restrict__ seq, int* __restrict__ raw, float* __restrict__ tok_lp,
    int* __restrict__ length, float* __restrict__ lp_sum, float* __restrict__ score, unsigned char* __restrict__ status,
    long* __restrict__ parent, int* __restrict__ next_tok, int Tn, int pos, int B, int K, int V, int S) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ uint64_t sh_key[kSelectThreads];
  __shared__ int sh_cls[kSelectThreads], sh_bank[kSelectThreads], sh_r[kSelectThreads];
  __shared__ int s_from[kMaxBeam], s_j[kMaxBeam], s_tok[kMaxBeam];
  __shared__ float s_lp[kMaxBeam], s_L[kMaxBeam], s_score[kMaxBeam];
  const int b = blockIdx.x, C = V + S, n_cand = K * W;
  const long R = (long)B * K;
  const long in = (pos & 1) ? R : 0, out = (pos & 1) ? 0 : R;     // row offsets of the read and the written half
  const long base = (long)b * K;
  const int tc = constraints ? constraint_words(constraints + (long)b * kMaxConstraintWords) : 0;
  if (threadIdx.x < K) { s_from[threadIdx.x] = threadIdx.x; s_j[threadIdx.x] = C; }   // unfilled slot: keeps itself

  uint64_t mine = 0;
  int i = 0, j = C, bank = 0, cls = 0;                // cls: 0 none, 1 live candidate, 2 carried finished slot
  float lp = 0.f, L = 0.f, sco = 0.f;
  if ((int)threadIdx.x < n_cand) {
    i = threadIdx.x / W;
    const int q = threadIdx.x % W;
    const long pr = in + base + i;
    if (status[pr] == 0) {
      const uint64_t c = row_top[(base + i) * W + q];
      if (c != 0) {
        lp = key_lp(c);
        j = key_index(c);
        bank = (int)(c >> kBankShift);
        L = lp_sum[pr] + lp;
        const int n = length[pr];                     // tokens generated with this one: (length - 1) + 1
        sco = L / powf((5.f + (float)n) / 6.f, alpha) + 0.f;           // + 0: -0 and +0 rank as one value
        cls = 1;
      }
    } else if (status[pr] == 1 && q == 0) {
      L = lp_sum[pr];
      sco = score[pr] + 0.f;
      cls = 2;
    }
    if (cls) mine = ((uint64_t)order_bits(sco) << 32) | (0xFFFFFFFFu - (uint32_t)(i * (C + 1) + j));
  }
  if ((int)threadIdx.x < n_cand) { sh_key[threadIdx.x] = mine; sh_cls[threadIdx.x] = cls; sh_bank[threadIdx.x] = bank; }
  __syncthreads();
  int rank = 0, r = 0;
  if (cls && tc == 0) {
    for (int u = 0; u < n_cand; ++u) rank += sh_key[u] > mine ? 1 : 0;
  } else if (cls == 2) {
    for (int u = 0; u < n_cand; ++u) rank += sh_cls[u] == 2 && sh_key[u] > mine ? 1 : 0;
  } else if (cls == 1) {
    for (int u = 0; u < n_cand; ++u) r += sh_cls[u] == 1 && sh_bank[u] == bank && sh_key[u] > mine ? 1 : 0;
  }
  if ((int)threadIdx.x < n_cand) sh_r[threadIdx.x] = r;
  __syncthreads();
  if (cls == 1 && tc) {
    for (int u = 0; u < n_cand; ++u)
      rank += sh_cls[u] == 2 || (sh_cls[u] == 1 && (sh_r[u] < r || (sh_r[u] == r && sh_bank[u] > bank))) ? 1 : 0;
  }
  if (cls && rank < K) {
    s_from[rank] = i; s_j[rank] = j; s_lp[rank] = lp; s_L[rank] = L; s_score[rank] = sco;
    s_tok[rank] = j < V ? j : (j < C ? copy_src[(long)b * S + (j - V)] : pad_id);
  }
  __syncthreads();
  beam_write_slots(s_from, s_j, s_tok, s_lp, s_L, s_score, eos_id, pad_id, seq, raw, tok_lp, length, lp_sum, score,
                   status, parent, next_tok, nullptr, Tn, pos, in, out, base, 0, K, C);
}

// ------------------------------------------------------------------ one diverse n-best beam step (beam groups)
// The K slots of a commit form G groups of Kg = K / G; group g owns slots g * Kg .. (g + 1) * Kg - 1 and the groups
// choose in order.  A live slot i of group g proposes (i, j) with the n-best score, ranked by
//   value = score - diversity * h,   h = how many slots of groups 0..g-1 grew at this position with j's token
// (a copy's token is copy_src[b, j - V], so a copy and the vocabulary entry spelling the same word count alike); a
// finished slot proposes itself with its stored score.  The Kg best by (value descending, then i * (C + 1) + j
// ascending) become the group's slots, parents always inside the group.  The penalty only ranks: lp, L and score are
// the n-best quantities.  Per group two launches: a row stage (one CTA per slot of the group) keeping each row's Kg
// best by value, then a select stage (one CTA per commit) merging the group's <= Kg^2 candidates and writing `chosen`
// (the token each new slot grew with, -1 when carried or empty) for the later groups.
// Both stages rank by the same fp32 value from diverse_value (explicit _rn operations: no contraction can make them
// disagree), so a select winner is always among its row's Kg best and the row prefilter is exact.
__device__ __forceinline__ float beam_norm(int n, float alpha) { return powf((5.f + (float)n) / 6.f, alpha); }
// -> the rank value; *score = (L_i + lp) / norm, the n-best score of the candidate
__device__ __forceinline__ float diverse_value(float L_i, float lp, float norm, float diversity, int h, float* score) {
  *score = __fdiv_rn(__fadd_rn(L_i, lp), norm);
  return __fsub_rn(*score, __fmul_rn(diversity, (float)h)) + 0.f;     // + 0: -0 and +0 rank as one value
}
__device__ __forceinline__ int count_token(const int* s_prev, int n_prev, int tok) {
  int h = 0;
  for (int e = 0; e < n_prev; ++e) h += s_prev[e] == tok ? 1 : 0;
  return h;
}

template <typename T>
__global__ void __launch_bounds__(kBeamThreads, 1) diverse_row_kernel(
    const T* __restrict__ logits, long ldl, const float* __restrict__ sc, const float* __restrict__ gate_logit,
    const unsigned char* __restrict__ mem_mask, const int* __restrict__ copy_src, const unsigned char* __restrict__ status,
    const float* __restrict__ lp_sum, const int* __restrict__ length, const int* __restrict__ chosen, float alpha,
    float diversity, uint64_t* __restrict__ row_top, float* __restrict__ row_lp, const int* __restrict__ seq, int Tn,
    const int* __restrict__ prefix, int ld_prefix, const int* __restrict__ prefix_len, int no_repeat, int min_len,
    int eos_id, int pos, int g, int Kg, int K, int V, int S) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ MaxSum sh_ms[8];
  __shared__ float bc[4];
  __shared__ uint64_t shk[8];
  __shared__ int s_prev[kMaxBeam];                    // tokens the earlier groups' slots grew with at this position
  __shared__ int s_hist[TMAX], s_ban[TMAX];           // the row's history and banned words (ban_build)
  const int b = blockIdx.x / Kg;
  const long row = (long)b * K + g * Kg + blockIdx.x % Kg;     // slot row (status / state are of the read half)
  if (status[row] != 0) return;                       // finished or inactive: the select stage reads nothing of it
  const int n_prev = g * Kg;
  if (threadIdx.x < n_prev) s_prev[threadIdx.x] = chosen[(long)b * K + threadIdx.x];
  const int nb = ban_count(pos, no_repeat, min_len);
  ban_load(seq + row * Tn, pos, nb, s_hist);
  const T* lrow = logits + row * ldl;
  const float* srow = sc + row * S;
  const unsigned char* mrow = mem_mask + (long)b * S;
  const int* crow = copy_src + (long)b * S;
  const MixRow ms = mix_row_stats(lrow, srow, mrow, gate_logit + row * 2, V, S, sh_ms, bc);   // syncs s_prev, s_hist
  const float L_i = lp_sum[row], norm = beam_norm(length[row], alpha);
  if (prefix && pos < prefix_len[b]) {                // inside the commit's prefix: its label is the row's one winner
    if (threadIdx.x == 0) {
      const int j = prefix[(long)b * ld_prefix + pos];
      const float lp = mix_lp(mix_prob(ms, lrow, srow, mrow, V, j));
      const int h = n_prev ? count_token(s_prev, n_prev, j < V ? j : crow[j - V]) : 0;
      float score;
      row_top[row * Kg] = rank_key(diverse_value(L_i, lp, norm, diversity, h, &score), j);
      row_lp[row * Kg] = lp;
      for (int k = 1; k < Kg; ++k) { row_top[row * Kg + k] = 0; row_lp[row * Kg + k] = 0.f; }
    }
    return;
  }
  if (nb) {
    ban_build(s_hist, pos, no_repeat, min_len, eos_id, nb, s_ban);
    __syncthreads();
  }

  uint64_t top[kMaxBeam];                             // this thread's best keys, descending; 0 = empty
#pragma unroll
  for (int i = 0; i < kMaxBeam; ++i) top[i] = 0;
  uint64_t thr = 0;                                   // top[Kg - 1]: the key a candidate has to beat
  mix_scan(ms, lrow, srow, mrow, V, S, [&](float p, int j) {
    const float lp = mix_lp(p);
    float score;
    const float v0 = diverse_value(L_i, lp, norm, diversity, 0, &score);
    if (rank_key(v0, j) <= thr) return;               // the penalty only lowers the value
    const int w = j < V ? j : crow[j - V];
    if (nb && is_banned(s_ban, nb, w)) return;        // only entries that would enter the top Kg
    const int h = n_prev ? count_token(s_prev, n_prev, w) : 0;
    const uint64_t key = h ? rank_key(diverse_value(L_i, lp, norm, diversity, h, &score), j) : rank_key(v0, j);
    if (key > thr) thr = topk_insert(top, key, Kg);
  });
  // the winner's lp is formed again from its index, so it is the lp its value was ranked with
  topk_pop(top, Kg, shk, [&](int k, uint64_t m) {
    if (threadIdx.x == 0) {
      row_top[row * Kg + k] = m;
      row_lp[row * Kg + k] = m != 0 ? mix_lp(mix_prob(ms, lrow, srow, mrow, V, key_index(m))) : 0.f;
    }
  });
}

__global__ void __launch_bounds__(kBeamThreads) diverse_select_kernel(
    const uint64_t* __restrict__ row_top, const float* __restrict__ row_lp, const int* __restrict__ copy_src,
    float alpha, float diversity, int eos_id, int pad_id, int* __restrict__ seq, int* __restrict__ raw,
    float* __restrict__ tok_lp, int* __restrict__ length, float* __restrict__ lp_sum, float* __restrict__ score,
    unsigned char* __restrict__ status, long* __restrict__ parent, int* __restrict__ next_tok,
    int* __restrict__ chosen, int Tn, int pos, int B, int g, int Kg, int K, int V, int S) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ uint64_t sh_key[kBeamThreads];
  __shared__ int s_from[kMaxBeam], s_j[kMaxBeam], s_tok[kMaxBeam], s_prev[kMaxBeam];
  __shared__ float s_lp[kMaxBeam], s_L[kMaxBeam], s_score[kMaxBeam];
  const int b = blockIdx.x, C = V + S;
  const long R = (long)B * K;
  const long in = (pos & 1) ? R : 0, out = (pos & 1) ? 0 : R;     // row offsets of the read and the written half
  const long base = (long)b * K;
  const int g0 = g * Kg, n_prev = g0;                 // the group's first slot; earlier groups' slots precede it
  if (threadIdx.x < Kg) { s_from[threadIdx.x] = g0 + threadIdx.x; s_j[threadIdx.x] = C; }   // unfilled: keeps itself
  if (threadIdx.x < n_prev) s_prev[threadIdx.x] = chosen[base + threadIdx.x];
  __syncthreads();

  // candidate threadIdx.x = il * Kg + q: the q-th row winner of live slot i = g0 + il, or (q = 0) finished slot i
  uint64_t mine = 0;
  int i = 0, j = C, tok = pad_id;
  float lp = 0.f, L = 0.f, sco = 0.f;
  if (threadIdx.x < Kg * Kg) {
    i = g0 + threadIdx.x / Kg;
    const int q = threadIdx.x % Kg;
    const long pr = in + base + i;
    float value = 0.f;
    if (status[pr] == 0) {
      const uint64_t c = row_top[(base + i) * Kg + q];
      if (c != 0) {
        lp = row_lp[(base + i) * Kg + q];
        j = key_index(c);
        tok = j < V ? j : copy_src[(long)b * S + (j - V)];
        L = __fadd_rn(lp_sum[pr], lp);
        value = diverse_value(lp_sum[pr], lp, beam_norm(length[pr], alpha), diversity,
                              count_token(s_prev, n_prev, tok), &sco);
        sco += 0.f;
        mine = 1;
      }
    } else if (status[pr] == 1 && q == 0) {
      L = lp_sum[pr];
      sco = score[pr] + 0.f;
      value = sco;
      mine = 1;
    }
    if (mine) mine = ((uint64_t)order_bits(value) << 32) | (0xFFFFFFFFu - (uint32_t)(i * (C + 1) + j));
  }
  sh_key[threadIdx.x] = mine;
  __syncthreads();
  if (mine) {
    int rank = 0;
    for (int u = 0; u < Kg * Kg; ++u) rank += sh_key[u] > mine ? 1 : 0;
    if (rank < Kg) { s_from[rank] = i; s_j[rank] = j; s_lp[rank] = lp; s_L[rank] = L; s_score[rank] = sco; s_tok[rank] = tok; }
  }
  __syncthreads();
  beam_write_slots(s_from, s_j, s_tok, s_lp, s_L, s_score, eos_id, pad_id, seq, raw, tok_lp, length, lp_sum, score,
                   status, parent, next_tok, chosen, Tn, pos, in, out, base, g0, Kg, C);
}

// ------------------------------------------------------------------ ensemble combine
// M members' (logits, copy scores, gate logits) -> one fp32 triple whose mixture (Model.py:54-86, as the step kernels
// form it) is the weighted average sum_m w_m P^m.  With member m's row statistics from mix_row_stats (bit for bit those
// its own step kernel would form) and G0 = sum_m w_m g0^m, G1 = sum_m w_m g1^m:
//   x'_j = LSE over m with w_m g0^m > 0 of [log(w_m g0^m / G0) + x^m_j - vmax^m - log vsum^m]
//   c'_s = LSE over m with w_m g1^m > 0 of [log(w_m g1^m / G1) + c^m_s - cmax^m - log csum^m]   (masked s: kMaskFill)
//   gl'  = (log G0, log G1)
// softmax(x') sums to 1, so g0' softmax(x')_j = G0 * sum_m (w_m g0^m / G0) softmax(x^m)_j.  G0 == 0 (every member's gate
// saturated to the copy side) uses log w_m as the offsets: x' stays finite and gl'_0 = -inf makes g0' exactly 0; the
// same for G1.  The log domain keeps x' and c' finite where every member's probability underflows in fp32.
constexpr int kMaxMembers = 8;
constexpr int kEnsThreads = 256;                      // = the step kernels' block: mix_row_stats' reduction order
struct Members {                                      // by value: a captured launch bakes the pointers in
  const void* logits[kMaxMembers];
  const float* sc[kMaxMembers];
  const float* gl[kMaxMembers];
};

// running log-sum-exp (mx, s): one expf per term
__device__ __forceinline__ void lse_add(float& mx, float& s, float y) {
  if (y > mx) { s = s * expf(mx - y) + 1.f; mx = y; }
  else s += expf(y - mx);
}

template <typename T>
__global__ void __launch_bounds__(kEnsThreads) pointer_mix_ensemble_kernel(
    Members mem, int M, long ldl, const float* __restrict__ log_w, const unsigned char* __restrict__ mem_mask,
    float* __restrict__ logits_out, long ld_out, float* __restrict__ sc_out, float* __restrict__ gl_out, int N, int V,
    int S) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ MaxSum sh_ms[8];
  __shared__ float bc[4];
  __shared__ const T* s_l[kMaxMembers];
  __shared__ const float* s_c[kMaxMembers];
  __shared__ const float* s_gl[kMaxMembers];
  __shared__ float s_g0[kMaxMembers], s_g1[kMaxMembers], s_ov[kMaxMembers], s_oc[kMaxMembers];
  __shared__ float s_gate[2];
  const long row = blockIdx.x;
  const int b = (int)(row / N);
  const unsigned char* mrow = mem_mask + (long)b * S;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int m = 0; m < kMaxMembers; ++m) {           // static indices: the parameter struct stays in constant space
      s_l[m] = (const T*)mem.logits[m] + row * ldl;
      s_c[m] = mem.sc[m] + row * S;
      s_gl[m] = mem.gl[m] + row * 2;
    }
  }
  __syncthreads();
  // pass 1 per member: its row statistics (vocab max / sum, copy max / sum, gates)
  for (int m = 0; m < M; ++m) {
    const MixRow ms = mix_row_stats(s_l[m], s_c[m], mrow, s_gl[m], V, S, sh_ms, bc);
    if (threadIdx.x == 0) {
      s_g0[m] = ms.g0; s_g1[m] = ms.g1;
      s_ov[m] = -ms.vmax - logf(ms.vsum);
      s_oc[m] = -ms.cmax - logf(ms.csum);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float G0 = 0.f, G1 = 0.f;
    for (int m = 0; m < M; ++m) { const float w = expf(log_w[m]); G0 += w * s_g0[m]; G1 += w * s_g1[m]; }
    const float lG0 = logf(G0), lG1 = logf(G1);
    for (int m = 0; m < M; ++m) {
      const float w = expf(log_w[m]);
      const float a0 = w * s_g0[m], a1 = w * s_g1[m];
      // -inf drops a member whose weighted gate is 0; with G == 0 every member keeps log w_m
      s_ov[m] += G0 > 0.f ? (a0 > 0.f ? logf(a0) - lG0 : -INFINITY) : log_w[m];
      s_oc[m] += G1 > 0.f ? (a1 > 0.f ? logf(a1) - lG1 : -INFINITY) : log_w[m];
    }
    s_gate[0] = lG0; s_gate[1] = lG1;
  }
  __syncthreads();
  // pass 2: vocabulary entries, 8 per vector load / store (the step kernels' load8), scalar tail
  float* orow = logits_out + row * ld_out;
  const int V8 = V >> 3;
  for (int g = threadIdx.x; g < V8; g += blockDim.x) {
    float mx[8], s[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { mx[i] = -INFINITY; s[i] = 0.f; }
    for (int m = 0; m < M; ++m) {
      const float o = s_ov[m];
      if (o == -INFINITY) continue;
      float x[8];
      Act<T>::load8(s_l[m] + (long)g * 8, x);
#pragma unroll
      for (int i = 0; i < 8; ++i) lse_add(mx[i], s[i], o + x[i]);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) mx[i] += logf(s[i]);
    Act<float>::store8(orow + (long)g * 8, mx);
  }
  for (int j = V8 * 8 + threadIdx.x; j < V; j += blockDim.x) {
    float mx = -INFINITY, s = 0.f;
    for (int m = 0; m < M; ++m)
      if (s_ov[m] != -INFINITY) lse_add(mx, s, s_ov[m] + Act<T>::ld(s_l[m] + j));
    orow[j] = mx + logf(s);
  }
  // copy positions
  float* crow = sc_out + row * S;
  for (int j = threadIdx.x; j < S; j += blockDim.x) {
    float r = kMaskFill;
    if (mrow[j]) {
      float mx = -INFINITY, s = 0.f;
      for (int m = 0; m < M; ++m)
        if (s_oc[m] != -INFINITY) lse_add(mx, s, s_oc[m] + s_c[m][j]);
      r = mx + logf(s);
    }
    crow[j] = r;
  }
  if (threadIdx.x == 0) { gl_out[row * 2] = s_gate[0]; gl_out[row * 2 + 1] = s_gate[1]; }
}

// ------------------------------------------------------------------ nearest-neighbour combine
// One row's (logits, copy scores, gate logits) and its k neighbours from fira_knn_search -> one fp32 triple whose
// mixture is P'_j = (1 - lam) P_j + lam q_j (j < V), P'_{V+s} = (1 - lam) P_{V+s}.  P's row statistics come from
// mix_row_stats (bit for bit the step kernels'); q_w = sum over neighbours i with word w of e_i / Z, e_i =
// exp(-(d_i - d_1) / tau), Z = sum_i e_i in neighbour order.  With a0 = (1 - lam) g0, a1 = (1 - lam) g1, G0 = a0 + lam:
//   gl'  = (log G0, log a1)                                           (a1 == 0: -inf, the copy side is exactly 0)
//   x'_j = o + x_j,  o = log a0 - log G0 - vmax - log vsum            (a0 == 0: kMaskFill)
//   x'_w = LSE(o + x_w, log(lam q_w) - log G0)                       for each neighbour word w
//   c'_s = c_s                                                        (masked s: kMaskFill)
// exp(gl'_0) + exp(gl'_1) = 1 and sum_j exp(x'_j) = 1 up to rounding, so the step kernels' g0' softmax(x')_j is P'_j.
constexpr int kKnnMaxK = 64;

__device__ __forceinline__ float lse2(float a, float b) {
  const float mx = fmaxf(a, b), mn = fminf(a, b);
  return mn == -INFINITY ? mx : mx + log1pf(expf(mn - mx));
}

template <typename T>
__global__ void __launch_bounds__(kEnsThreads) pointer_mix_knn_kernel(
    const T* __restrict__ logits, long ldl, const float* __restrict__ sc, const float* __restrict__ gl,
    const unsigned char* __restrict__ mem_mask, const int* __restrict__ nb_idx, const float* __restrict__ nb_dist,
    const int* __restrict__ words, int k, const float* __restrict__ params, float* __restrict__ logits_out,
    long ld_out, float* __restrict__ sc_out, float* __restrict__ gl_out, int N, int V, int S) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ MaxSum sh_ms[8];
  __shared__ float bc[4];
  __shared__ int s_w[kKnnMaxK];
  __shared__ float s_e[kKnnMaxK];
  __shared__ float s_o[3];                            // o, log G0, Z
  const long row = blockIdx.x;
  const int b = (int)(row / N);
  const T* lrow = logits + row * ldl;
  const float* srow = sc + row * S;
  const unsigned char* mrow = mem_mask + (long)b * S;
  const MixRow ms = mix_row_stats(lrow, srow, mrow, gl + row * 2, V, S, sh_ms, bc);
  const float lam = params[0], tau = params[1];
  if ((int)threadIdx.x < k) {
    const long i = row * k + threadIdx.x;
    s_w[threadIdx.x] = words[nb_idx[i]];
    s_e[threadIdx.x] = expf(-(nb_dist[i] - nb_dist[row * k]) / tau);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float Z = 0.f;
    for (int i = 0; i < k; ++i) Z += s_e[i];
    const float a0 = (1.f - lam) * ms.g0, a1 = (1.f - lam) * ms.g1, lG0 = logf(a0 + lam);
    s_o[0] = a0 > 0.f ? logf(a0) - lG0 - ms.vmax - logf(ms.vsum) : -INFINITY;
    s_o[1] = lG0;
    s_o[2] = Z;
    gl_out[row * 2] = lG0;
    gl_out[row * 2 + 1] = a1 > 0.f ? logf(a1) : -INFINITY;
  }
  __syncthreads();
  const float o = s_o[0];
  float* orow = logits_out + row * ld_out;
  const int V8 = V >> 3;
  for (int g = threadIdx.x; g < V8; g += blockDim.x) {
    float x[8];
    Act<T>::load8(lrow + (long)g * 8, x);
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = o == -INFINITY ? kMaskFill : o + x[i];
    Act<float>::store8(orow + (long)g * 8, x);
  }
  for (int j = V8 * 8 + threadIdx.x; j < V; j += blockDim.x)
    orow[j] = o == -INFINITY ? kMaskFill : o + Act<T>::ld(lrow + j);
  float* crow = sc_out + row * S;
  for (int j = threadIdx.x; j < S; j += blockDim.x) crow[j] = mrow[j] ? srow[j] : kMaskFill;
  __syncthreads();                                    // the plain entries are written; the neighbour words follow
  if ((int)threadIdx.x < k) {
    const int i = threadIdx.x, w = s_w[i];
    bool first = w >= 0 && w < V;                     // the datastore holds vocabulary ids only
    for (int j = 0; j < i && first; ++j) first = s_w[j] != w;
    if (first) {                                      // the first neighbour with word w writes x'_w
      float e = 0.f;
      for (int j = i; j < k; ++j) e += s_w[j] == w ? s_e[j] : 0.f;
      const float nb = logf(lam * (e / s_o[2])) - s_o[1];
      const float x = o == -INFINITY ? nb : lse2(o + Act<T>::ld(lrow + w), nb);
      orow[w] = x == -INFINITY ? kMaskFill : x;       // lam q_w underflowed with a0 == 0: P'_w is 0, as masked
    }
  }
}

// ------------------------------------------------------------------ knowledge distillation loss
// Row r with shifted label y != 0: the student's mixture P (head_fwd_kernel's expressions) against the teacher's t (the
// same expressions on the teacher's fp32 triple, fira_pointer_mix_ensemble's output):
//   nll = -log clamp(P_y, 1e-10, 1),  kd = -sum_j t_j log clamp(P_j, 1e-10, 1),  loss = (1 - alpha) nll + alpha kd
//   a_j = [(1 - alpha) [j == y] + alpha t_j] live_j  (live_j: 1e-10 <= P_j <= 1),  A_V = sum_{j<V} a_j,  A_C = the rest
// The clamp needs the final row statistics before any term, so the forward walks both rows twice: statistics, then kd,
// A_V and A_C.  The backward reads A_V / A_C from the stats row and walks both rows once.
// stats row (16 floats): student vmax vsum cmax csum g0 g1, p_label, 0, teacher vmax vsum cmax csum g0 g1, A_V, A_C
constexpr int kKdThreads = 256;                       // = head_fwd_kernel's block: the same student statistics
constexpr int kKdStats = 16;

struct KdRow {
  float vmax, iv, g0, lv;            // student vocabulary side: P_j = g0 (e^(x_j - vmax) iv), log P_j = x_j + lv
  float cmax, ic, g1, lc;            // student copy side
  float tvmax, tiv, tg0, tcmax, tic, tg1;
  float p_lab, lp_lab, hard, alpha;  // P_y as head_fwd_kernel forms it, log clamp(P_y), 1 - alpha, alpha
  int y;
};
// the student's fields from st[0..6] (both stats layouts start with them); kd_row adds the teacher's
__device__ __forceinline__ KdRow kd_student(const float* st, float alpha, int y) {
  KdRow k;
  k.vmax = st[0]; k.iv = 1.f / st[1]; k.g0 = st[4]; k.lv = logf(st[4]) - st[0] - logf(st[1]);
  k.cmax = st[2]; k.ic = 1.f / st[3]; k.g1 = st[5]; k.lc = logf(st[5]) - st[2] - logf(st[3]);
  k.tvmax = k.tiv = k.tg0 = k.tcmax = k.tic = k.tg1 = 0.f;
  k.p_lab = st[6]; k.lp_lab = mix_lp(st[6]);
  k.hard = 1.f - alpha; k.alpha = alpha; k.y = y;
  return k;
}
__device__ __forceinline__ KdRow kd_row(const float* st, float alpha, int y) {
  KdRow k = kd_student(st, alpha, y);
  k.tvmax = st[8]; k.tiv = 1.f / st[9]; k.tcmax = st[10]; k.tic = 1.f / st[11]; k.tg0 = st[12]; k.tg1 = st[13];
  return k;
}
// a_j of entry j from the student's P_j and the teacher's t_j (forward and backward form it the same way)
__device__ __forceinline__ float kd_weight(const KdRow& k, int j, float p, float t) {
  return (p >= 1e-10f && p <= 1.f) ? fmaf(k.alpha, t, j == k.y ? k.hard : 0.f) : 0.f;
}
// forward term of entry j: a_j into `acc`, -t_j log clamp(P_j) into `kd` (t_j == 0 adds nothing; lp: log P_j if live)
__device__ __forceinline__ void kd_term(const KdRow& k, int j, float p, float t, float lp, float& kd, float& acc) {
  acc += kd_weight(k, j, p, t);
  if (t > 0.f) {
    const float l = j == k.y ? k.lp_lab : (p >= 1e-10f && p <= 1.f) ? lp : (p < 1e-10f ? logf(1e-10f) : 0.f);
    kd = fmaf(-t, l, kd);
  }
}

template <typename T>
__global__ void __launch_bounds__(kKdThreads) pointer_mix_kd_fwd_kernel(
    const T* __restrict__ logits, long ldl, const float* __restrict__ sc, const float* __restrict__ gate_logit,
    const unsigned char* __restrict__ mem_mask, const int* __restrict__ label, const float* __restrict__ t_logits,
    long ldt, const float* __restrict__ t_sc, const float* __restrict__ t_gate_logit, float alpha,
    float* __restrict__ stats, float* __restrict__ nll, float* __restrict__ kd, float* __restrict__ loss, int Tn, int V,
    int S) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ MaxSum sh_ms[2][8];
  __shared__ float bc[8];
  __shared__ float shf[8];
  __shared__ float s_st[kKdStats];
  const long row = blockIdx.x;
  const int y = label[row];
  float* st = stats + row * kKdStats;
  if (y == 0) {                                       // no loss: neither row is read
    if (threadIdx.x < kKdStats) st[threadIdx.x] = 0.f;
    if (threadIdx.x == 0) { nll[row] = 0.f; kd[row] = 0.f; loss[row] = 0.f; }
    return;
  }
  const int b = (int)(row / Tn);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const T* lrow = logits + row * ldl;
  const float* srow = sc + row * S;
  const float* trow = t_logits + row * ldt;
  const float* tsrow = t_sc + row * S;
  const unsigned char* mrow = mem_mask + (long)b * S;

  // pass 1: both rows' statistics, student and teacher in the same loops.  The student's arithmetic and reduction order
  // are mix_row_stats' (= head_fwd_kernel's), so its P_y and nll are fira_pointer_mix_nll_fwd's bit for bit.
  MaxSum v{-INFINITY, 0.f}, u{-INFINITY, 0.f};
  const int V8 = V >> 3;
  for (int g = threadIdx.x; g < V8; g += blockDim.x) {
    float x[8], z[8];
    Act<T>::load8(lrow + (long)g * 8, x);
    Act<float>::load8(trow + (long)g * 8, z);
    float m8 = x[0], n8 = z[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) { m8 = fmaxf(m8, x[i]); n8 = fmaxf(n8, z[i]); }
    if (m8 > v.m) { v.s *= expf(v.m - m8); v.m = m8; }
    if (n8 > u.m) { u.s *= expf(u.m - n8); u.m = n8; }
#pragma unroll
    for (int i = 0; i < 8; ++i) { v.s += expf(x[i] - v.m); u.s += expf(z[i] - u.m); }
  }
  for (int j = V8 * 8 + threadIdx.x; j < V; j += blockDim.x) {
    v = ms_merge(v, MaxSum{Act<T>::ld(lrow + j), 1.f});
    u = ms_merge(u, MaxSum{trow[j], 1.f});
  }
  v = ms_warp(v); u = ms_warp(u);
  if (lane == 0) { sh_ms[0][warp] = v; sh_ms[1][warp] = u; }
  __syncthreads();
  if (warp < 2) {
    MaxSum w = lane < 8 ? sh_ms[warp][lane] : MaxSum{-INFINITY, 0.f};
    w = ms_warp(w);
    if (lane == 0) { bc[4 * warp] = w.m; bc[4 * warp + 1] = w.s; }
  }
  __syncthreads();
  MaxSum c{-INFINITY, 0.f}, d{-INFINITY, 0.f};
  for (int j = threadIdx.x; j < S; j += blockDim.x) {
    const bool m = mrow[j];
    c = ms_merge(c, MaxSum{m ? srow[j] : kMaskFill, 1.f});
    d = ms_merge(d, MaxSum{m ? tsrow[j] : kMaskFill, 1.f});
  }
  c = ms_warp(c); d = ms_warp(d);
  if (lane == 0) { sh_ms[0][warp] = c; sh_ms[1][warp] = d; }
  __syncthreads();
  if (warp < 2) {
    MaxSum w = lane < 8 ? sh_ms[warp][lane] : MaxSum{-INFINITY, 0.f};
    w = ms_warp(w);
    if (lane == 0) { bc[4 * warp + 2] = w.m; bc[4 * warp + 3] = w.s; }
  }
  __syncthreads();
  if (threadIdx.x < 2) {                              // thread 0: the student's gates, thread 1: the teacher's
    const float* gl = (threadIdx.x ? t_gate_logit : gate_logit) + row * 2;
    const float gl0 = gl[0], gl1 = gl[1];
    const float gm = fmaxf(gl0, gl1);
    const float e0 = expf(gl0 - gm), e1 = expf(gl1 - gm);
    float* o = s_st + 8 * threadIdx.x;
    o[0] = bc[4 * threadIdx.x]; o[1] = bc[4 * threadIdx.x + 1]; o[2] = bc[4 * threadIdx.x + 2];
    o[3] = bc[4 * threadIdx.x + 3]; o[4] = e0 / (e0 + e1); o[5] = e1 / (e0 + e1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {                             // P_y; a copy label beyond S: p = 0, the clamp floor, no gradient
    const MixRow ms{s_st[0], s_st[1], s_st[2], s_st[3], s_st[4], s_st[5]};
    s_st[6] = y - V < S ? mix_prob(ms, lrow, srow, mrow, V, y) : 0.f;
    s_st[7] = 0.f;
  }
  __syncthreads();

  // pass 2: kd, A_V and A_C in fixed order (per-thread sums, then block_reduce)
  const KdRow k = kd_row(s_st, alpha, y);
  float kdp = 0.f, av = 0.f, ac = 0.f;
  for (int g = threadIdx.x; g < V8; g += blockDim.x) {
    float x[8], z[8];
    Act<T>::load8(lrow + (long)g * 8, x);
    Act<float>::load8(trow + (long)g * 8, z);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int j = g * 8 + i;
      const float p = j == y ? k.p_lab : k.g0 * (expf(x[i] - k.vmax) * k.iv);
      kd_term(k, j, p, k.tg0 * (expf(z[i] - k.tvmax) * k.tiv), x[i] + k.lv, kdp, av);
    }
  }
  for (int j = V8 * 8 + threadIdx.x; j < V; j += blockDim.x) {
    const float x = Act<T>::ld(lrow + j);
    const float p = j == y ? k.p_lab : k.g0 * (expf(x - k.vmax) * k.iv);
    kd_term(k, j, p, k.tg0 * (expf(trow[j] - k.tvmax) * k.tiv), x + k.lv, kdp, av);
  }
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    const bool m = mrow[s];
    const float x = m ? srow[s] : kMaskFill;
    const float p = V + s == y ? k.p_lab : k.g1 * (expf(x - k.cmax) * k.ic);
    kd_term(k, V + s, p, m ? k.tg1 * (expf(tsrow[s] - k.tcmax) * k.tic) : 0.f, x + k.lc, kdp, ac);
  }
  auto add = [](float a, float x) { return a + x; };
  kdp = block_reduce(kdp, shf, add);
  av = block_reduce(av, shf, add);
  ac = block_reduce(ac, shf, add);
  if (threadIdx.x < kKdStats) st[threadIdx.x] = threadIdx.x == 14 ? av : threadIdx.x == 15 ? ac : s_st[threadIdx.x];
  if (threadIdx.x == 0) {
    const float h = -k.lp_lab;                        // = fira_pointer_mix_nll_fwd's nll
    nll[row] = h;
    kd[row] = kdp;
    loss[row] = fmaf(alpha, kdp, k.hard * h);
  }
}

// d(sum_r upstream * loss_r) / d(logits, copy scores, gate logits) from the forward's stats rows:
//   dx_k = u (p_k A_V - a_k),  dc_s = u (q_s A_C - a_{V+s}) (0 at a masked s),  dgl = u (g (A_V + A_C) - (A_V, A_C))
// with p, q the two softmaxes.  A side whose A is 0 is written as zeros without reading the rows.
template <typename T>
__global__ void __launch_bounds__(kKdThreads) pointer_mix_kd_bwd_kernel(
    const T* __restrict__ logits, long ldl, const float* __restrict__ sc, const unsigned char* __restrict__ mem_mask,
    const int* __restrict__ label, const float* __restrict__ t_logits, long ldt, const float* __restrict__ t_sc,
    float alpha, const float* __restrict__ stats, const float* __restrict__ upstream, T* __restrict__ d_logits,
    float* __restrict__ d_sc, float* __restrict__ d_gate_logit, unsigned char* __restrict__ row_active, int Tn, int V,
    int S) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const long row = blockIdx.x;
  const int b = (int)(row / Tn);
  const int y = label[row];
  const float* st = stats + row * kKdStats;
  const float A_V = y ? st[14] : 0.f, A_C = y ? st[15] : 0.f;
  const float up = *upstream;
  const KdRow k = kd_row(st, alpha, y);
  const T* lrow = logits + row * ldl;
  const float* trow = t_logits + row * ldt;
  T* drow = d_logits + row * ldl;
  const int V8 = V >> 3;                              // 8 logits per vector load / store, scalar tail
  if (A_V != 0.f) {
    const float sv = k.iv * A_V;
    for (int g = threadIdx.x; g < V8; g += blockDim.x) {
      float x[8], z[8];
      Act<T>::load8(lrow + (long)g * 8, x);
      Act<float>::load8(trow + (long)g * 8, z);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int j = g * 8 + i;
        const float e = expf(x[i] - k.vmax);
        const float a = kd_weight(k, j, j == y ? k.p_lab : k.g0 * (e * k.iv), k.tg0 * (expf(z[i] - k.tvmax) * k.tiv));
        x[i] = up * (e * sv - a);
      }
      Act<T>::store8(drow + (long)g * 8, x);
    }
    for (int j = V8 * 8 + threadIdx.x; j < V; j += blockDim.x) {
      const float e = expf(Act<T>::ld(lrow + j) - k.vmax);
      const float a = kd_weight(k, j, j == y ? k.p_lab : k.g0 * (e * k.iv), k.tg0 * (expf(trow[j] - k.tvmax) * k.tiv));
      Act<T>::st(drow + j, up * (e * sv - a));
    }
  } else {
    const float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int g = threadIdx.x; g < V8; g += blockDim.x) Act<T>::store8(drow + (long)g * 8, z);
    for (int j = V8 * 8 + threadIdx.x; j < V; j += blockDim.x) Act<T>::st(drow + j, 0.f);
  }
  const float* srow = sc + row * S;
  const float* tsrow = t_sc + row * S;
  const unsigned char* mrow = mem_mask + (long)b * S;
  float* dsrow = d_sc + row * S;
  if (A_C != 0.f) {
    const float scc = k.ic * A_C;
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
      float r = 0.f;                                  // a masked position takes no gradient (masked_fill)
      if (mrow[s]) {
        const int j = V + s;
        const float e = expf(srow[s] - k.cmax);
        const float a = kd_weight(k, j, j == y ? k.p_lab : k.g1 * (e * k.ic), k.tg1 * (expf(tsrow[s] - k.tcmax) * k.tic));
        r = up * (e * scc - a);
      }
      dsrow[s] = r;
    }
  } else {
    for (int s = threadIdx.x; s < S; s += blockDim.x) dsrow[s] = 0.f;
  }
  if (threadIdx.x == 0) {
    const float A = A_V + A_C;
    d_gate_logit[row * 2] = y ? up * (k.g0 * A - A_V) : 0.f;
    d_gate_logit[row * 2 + 1] = y ? up * (k.g1 * A - A_C) : 0.f;
    row_active[row] = A_C != 0.f ? 1 : 0;
  }
}

// ------------------------------------------------------------------ offline distillation: top-k teacher targets
// fira_pointer_mix_topk keeps, per loss row, the teacher's k candidates (every vocabulary entry and unmasked copy
// position with P_j > 0 in fp32, P from mix_row_stats / mix_prob) with the largest rank_key(P_j, j): P descending, then
// j ascending, the sampler's key taken on P itself.  mass = the kept P summed in key order; stored t~_i = P_i / mass.
// The sparse loss kernels then read the student row as fira_pointer_mix_kd_fwd / _bwd do against the dense vector that
// holds t~ at the kept labels and 0 elsewhere:
//   forward   mix_row_stats once, then the <= k + 1 weighted entries (the kept labels and y), one per thread, summed by
//             block_reduce in entry order
//   backward  one dense write pass of u (softmax A - a) without the a term, then, after a __syncthreads, the <= k + 1
//             columns with a != 0 rewritten from the whole expression (one rounding, as the dense kernel's)
// stats row (kKdSparseStats floats): student vmax vsum cmax csum g0 g1, p_label, 0, A_V, A_C
constexpr int kKdMaxTopk = 64;
constexpr int kKdSparseStats = 10;

// P_j (P_y: the forward's p_label) and log P_j of entry j < V + S; log P_j is what kd_term reads for a live P_j
template <typename T>
__device__ __forceinline__ float kd_entry(const MixRow& ms, const KdRow& k, const T* __restrict__ lrow,
                                          const float* __restrict__ srow, const unsigned char* __restrict__ mrow, int V,
                                          int j, float& lp) {
  if (j < V) lp = Act<T>::ld(lrow + j) + k.lv;
  else lp = (mrow[j - V] ? srow[j - V] : kMaskFill) + k.lc;
  return j == k.y ? k.p_lab : mix_prob(ms, lrow, srow, mrow, V, j);
}
// thread i's entry: the kept label i < K with its t~, or y (t = 0) at i == K unless y is a kept label; -1: none.
// Block-wide (a __syncthreads_or).
__device__ __forceinline__ int kd_sparse_entry(const int* __restrict__ lab, const float* __restrict__ prob, int K, int y,
                                               int V, int S, float& t) {
  const int i = threadIdx.x;
  int j = i < K ? lab[i] : (i == K ? y : -1);
  t = i < K ? prob[i] : 0.f;
  const bool y_kept = __syncthreads_or(i < K && j == y);
  if (j < 0 || j >= V + S || (i == K && y_kept)) j = -1;
  return j;
}

__global__ void __launch_bounds__(kSampleThreads) pointer_mix_topk_kernel(
    const float* __restrict__ t_logits, long ldt, const float* __restrict__ t_sc, const float* __restrict__ t_gl,
    const unsigned char* __restrict__ mem_mask, const int* __restrict__ label, int K, int* __restrict__ t_label,
    float* __restrict__ t_prob, float* __restrict__ mass, int Tn, int V, int S) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  extern __shared__ float s_p[];                      // [V + S] P_j, NaN = not a candidate
  __shared__ MaxSum sh_ms[8];
  __shared__ float bc[4];
  __shared__ unsigned shu[8];
  __shared__ unsigned s_n;
  __shared__ uint64_t s_key[kKdMaxTopk], s_sorted[kKdMaxTopk];
  __shared__ float s_mass;
  const long row = blockIdx.x;
  int* lo = t_label + row * K;
  float* po = t_prob + row * K;
  if (label[row] == 0) {                              // no loss: nothing is read
    if ((int)threadIdx.x < K) { lo[threadIdx.x] = -1; po[threadIdx.x] = 0.f; }
    if (threadIdx.x == 0) mass[row] = 0.f;
    return;
  }
  const int b = (int)(row / Tn);
  const float* lrow = t_logits + row * ldt;
  const float* srow = t_sc + row * S;
  const unsigned char* mrow = mem_mask + (long)b * S;
  const MixRow ms = mix_row_stats(lrow, srow, mrow, t_gl + row * 2, V, S, sh_ms, bc);
  const float nan = __int_as_float(0x7fffffff);
  for (int s = threadIdx.x; s < S; s += blockDim.x)
    if (!mrow[s]) s_p[V + s] = nan;                   // mix_scan does not offer masked copies
  mix_scan(ms, lrow, srow, mrow, V, S, [&](float p, int j) { s_p[j] = p > 0.f ? p : nan; });
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();

  const int C = V + S;
  const int chunk = (C + kSampleThreads - 1) / kSampleThreads;
  const int j0 = min(C, (int)threadIdx.x * chunk), j1 = min(C, j0 + chunk);
  unsigned cnt = 0;
  for (int j = j0; j < j1; ++j) cnt += is_cand(s_p[j]) ? 1u : 0u;
  const unsigned n_cand = block_reduce(cnt, shu, [](unsigned a, unsigned x) { return a + x; });
  uint64_t cut = 1;
  if ((unsigned)K < n_cand) cut = key_cut((unsigned)K, [&](uint64_t th) { return count_key_ge(s_p, j0, j1, th, shu); });
  // the kept keys (min(K, n_cand) of them) in arrival order, then each placed at its rank: keys are distinct
  for (int j = j0; j < j1; ++j) {
    const float p = s_p[j];
    if (is_cand(p)) { const uint64_t key = rank_key(p, j); if (key >= cut) s_key[atomicAdd(&s_n, 1u)] = key; }
  }
  __syncthreads();
  const int n = (int)s_n;
  if ((int)threadIdx.x < n) {
    const uint64_t key = s_key[threadIdx.x];
    int r = 0;
    for (int q = 0; q < n; ++q) r += s_key[q] > key;
    s_sorted[r] = key;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = 0.f;
    for (int i = 0; i < n; ++i) m += s_p[key_index(s_sorted[i])];
    s_mass = m;
    mass[row] = m;
  }
  __syncthreads();
  if ((int)threadIdx.x < K) {
    const int i = threadIdx.x;
    const int j = i < n ? key_index(s_sorted[i]) : -1;
    lo[i] = j;
    po[i] = i < n ? s_p[j] / s_mass : 0.f;
  }
}

template <typename T>
__global__ void __launch_bounds__(kKdThreads) pointer_mix_kd_sparse_fwd_kernel(
    const T* __restrict__ logits, long ldl, const float* __restrict__ sc, const float* __restrict__ gate_logit,
    const unsigned char* __restrict__ mem_mask, const int* __restrict__ label, const int* __restrict__ t_label,
    const float* __restrict__ t_prob, int K, float alpha, float* __restrict__ stats, float* __restrict__ nll,
    float* __restrict__ kd, float* __restrict__ loss, int Tn, int V, int S) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ MaxSum sh_ms[8];
  __shared__ float bc[4];
  __shared__ float shf[8];
  __shared__ float s_st[8];
  const long row = blockIdx.x;
  const int y = label[row];
  float* st = stats + row * kKdSparseStats;
  if (y == 0) {                                       // no loss: neither the row nor its targets are read
    if (threadIdx.x < kKdSparseStats) st[threadIdx.x] = 0.f;
    if (threadIdx.x == 0) { nll[row] = 0.f; kd[row] = 0.f; loss[row] = 0.f; }
    return;
  }
  const int b = (int)(row / Tn);
  const T* lrow = logits + row * ldl;
  const float* srow = sc + row * S;
  const unsigned char* mrow = mem_mask + (long)b * S;
  // the student's statistics and P_y: fira_pointer_mix_nll_fwd's, bit for bit
  const MixRow ms = mix_row_stats(lrow, srow, mrow, gate_logit + row * 2, V, S, sh_ms, bc);
  if (threadIdx.x == 0) {                             // a copy label beyond S: p = 0, the clamp floor, no gradient
    s_st[0] = ms.vmax; s_st[1] = ms.vsum; s_st[2] = ms.cmax; s_st[3] = ms.csum; s_st[4] = ms.g0; s_st[5] = ms.g1;
    s_st[6] = y - V < S ? mix_prob(ms, lrow, srow, mrow, V, y) : 0.f;
    s_st[7] = 0.f;
  }
  __syncthreads();
  const KdRow k = kd_student(s_st, alpha, y);
  float t;
  const int j = kd_sparse_entry(t_label + row * K, t_prob + row * K, K, y, V, S, t);
  float kdp = 0.f, acc = 0.f;
  if (j >= 0) {
    float lp;
    const float p = kd_entry(ms, k, lrow, srow, mrow, V, j, lp);
    kd_term(k, j, p, t, lp, kdp, acc);
  }
  float av = j < V ? acc : 0.f, ac = j < V ? 0.f : acc;
  auto add = [](float a, float x) { return a + x; };
  kdp = block_reduce(kdp, shf, add);
  av = block_reduce(av, shf, add);
  ac = block_reduce(ac, shf, add);
  if (threadIdx.x < kKdSparseStats) st[threadIdx.x] = threadIdx.x == 8 ? av : threadIdx.x == 9 ? ac : s_st[threadIdx.x];
  if (threadIdx.x == 0) {
    const float h = -k.lp_lab;                        // = fira_pointer_mix_nll_fwd's nll
    nll[row] = h;
    kd[row] = kdp;
    loss[row] = fmaf(alpha, kdp, k.hard * h);
  }
}

template <typename T>
__global__ void __launch_bounds__(kKdThreads) pointer_mix_kd_sparse_bwd_kernel(
    const T* __restrict__ logits, long ldl, const float* __restrict__ sc, const unsigned char* __restrict__ mem_mask,
    const int* __restrict__ label, const int* __restrict__ t_label, const float* __restrict__ t_prob, int K,
    float alpha, const float* __restrict__ stats, const float* __restrict__ upstream, T* __restrict__ d_logits,
    float* __restrict__ d_sc, float* __restrict__ d_gate_logit, unsigned char* __restrict__ row_active, int Tn, int V,
    int S) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  const long row = blockIdx.x;
  const int b = (int)(row / Tn);
  const int y = label[row];
  const float* st = stats + row * kKdSparseStats;
  const float A_V = y ? st[8] : 0.f, A_C = y ? st[9] : 0.f;
  const float up = *upstream;
  const KdRow k = kd_student(st, alpha, y);
  const T* lrow = logits + row * ldl;
  const float* srow = sc + row * S;
  const unsigned char* mrow = mem_mask + (long)b * S;
  T* drow = d_logits + row * ldl;
  float* dsrow = d_sc + row * S;
  // this thread's entry and its a_j, as the forward formed them (a != 0 implies its side's A != 0)
  float t, a = 0.f;
  const int j = y ? kd_sparse_entry(t_label + row * K, t_prob + row * K, K, y, V, S, t) : -1;
  if (j >= 0) {
    const MixRow ms{st[0], st[1], st[2], st[3], st[4], st[5]};
    float lp;
    a = kd_weight(k, j, kd_entry(ms, k, lrow, srow, mrow, V, j, lp), t);
  }
  const int V8 = V >> 3;                              // 8 logits per vector load / store, scalar tail
  const float sv = k.iv * A_V, scc = k.ic * A_C;
  if (A_V != 0.f) {
    for (int g = threadIdx.x; g < V8; g += blockDim.x) {
      float x[8];
      Act<T>::load8(lrow + (long)g * 8, x);
#pragma unroll
      for (int i = 0; i < 8; ++i) x[i] = up * (expf(x[i] - k.vmax) * sv);
      Act<T>::store8(drow + (long)g * 8, x);
    }
    for (int q = V8 * 8 + threadIdx.x; q < V; q += blockDim.x)
      Act<T>::st(drow + q, up * (expf(Act<T>::ld(lrow + q) - k.vmax) * sv));
  } else {
    const float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int g = threadIdx.x; g < V8; g += blockDim.x) Act<T>::store8(drow + (long)g * 8, z);
    for (int q = V8 * 8 + threadIdx.x; q < V; q += blockDim.x) Act<T>::st(drow + q, 0.f);
  }
  if (A_C != 0.f) {
    for (int s = threadIdx.x; s < S; s += blockDim.x)   // a masked position takes no gradient (masked_fill)
      dsrow[s] = mrow[s] ? up * (expf(srow[s] - k.cmax) * scc) : 0.f;
  } else {
    for (int s = threadIdx.x; s < S; s += blockDim.x) dsrow[s] = 0.f;
  }
  __syncthreads();                                    // the dense pass is written; the weighted columns follow
  if (a != 0.f) {
    if (j < V) {
      Act<T>::st(drow + j, up * (expf(Act<T>::ld(lrow + j) - k.vmax) * sv - a));
    } else if (mrow[j - V]) {
      dsrow[j - V] = up * (expf(srow[j - V] - k.cmax) * scc - a);
    }
  }
  if (threadIdx.x == 0) {
    const float A = A_V + A_C;
    d_gate_logit[row * 2] = y ? up * (k.g0 * A - A_V) : 0.f;
    d_gate_logit[row * 2 + 1] = y ? up * (k.g1 * A - A_C) : 0.f;
    row_active[row] = A_C != 0.f ? 1 : 0;
  }
}

}  // namespace

#define DISPATCH_T(dtype, ...)                                                            \
  if ((dtype) == FIRA_F32) { using T = float; __VA_ARGS__ }                               \
  else if ((dtype) == FIRA_BF16) { using T = __nv_bfloat16; __VA_ARGS__ }                 \
  else { fira_set_error(FIRA_ERR_DTYPE, "unknown dtype %d", (int)(dtype)); return FIRA_ERR_DTYPE; }

extern "C" {

static int copy_scores_fwd_impl(const void* src_proj, const void* tgt_proj, const float* w_res, const float* b_res,
                                const unsigned char* src_mask, const unsigned char* row_mask, const int* ranges,
                                float* scores, int B, int T_len, int S, int dim, int dtype, void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "copy_scores_fwd: dim %d != 256", dim);
  FIRA_CHECK_ARG(T_len > 0 && T_len <= TMAX, FIRA_ERR_SHAPE, "copy_scores_fwd: T_len %d > %d", T_len, TMAX);
  if (B == 0 || S == 0) return FIRA_OK;
  dim3 grid((S + 31) / 32, B);
  DISPATCH_T(dtype, launch_k(copy_scores_fwd_kernel<T>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, 
      (const T*)src_proj, (const T*)tgt_proj, w_res, b_res, src_mask, row_mask, ranges, scores, B, T_len, S);)
  FIRA_CHECK_LAUNCH("fira_copy_scores_fwd");
  return FIRA_OK;
}

static int copy_scores_bwd_impl(const void* src_proj, const void* tgt_proj, const float* w_res, const float* d_scores,
                                const unsigned char* row_active, const int* ranges, void* d_src_proj, float* d_tgt_proj,
                                float* d_w_res, float* d_b_res, int B, int T_len, int S, int dim, int dtype, void* stream) {
  FIRA_CHECK_ARG(dim == D, FIRA_ERR_SHAPE, "copy_scores_bwd: dim %d != 256", dim);
  FIRA_CHECK_ARG(T_len > 0 && T_len <= TMAX, FIRA_ERR_SHAPE, "copy_scores_bwd: T_len %d > %d", T_len, TMAX);
  if (B == 0 || S == 0) return FIRA_OK;
  dim3 grid((S + 31) / 32, B);
  const int smem = (int)sizeof(float) * (2 * TMAX * D + D + 8 * D);
  cudaError_t e = dtype == FIRA_F32
      ? cudaFuncSetAttribute(copy_scores_bwd_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)
      : cudaFuncSetAttribute(copy_scores_bwd_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) { fira_set_error(FIRA_ERR_CUDA, "copy_scores_bwd attr: %s", cudaGetErrorString(e)); return FIRA_ERR_CUDA; }
  DISPATCH_T(dtype, launch_k(copy_scores_bwd_kernel<T>, dim3(grid), dim3(256), smem, (cudaStream_t)stream, 
      (const T*)src_proj, (const T*)tgt_proj, w_res, d_scores, row_active, ranges, (T*)d_src_proj, d_tgt_proj, d_w_res,
      d_b_res, B, T_len, S);)
  FIRA_CHECK_LAUNCH("fira_copy_scores_bwd");
  return FIRA_OK;
}

int fira_copy_scores_fwd(const void* src_proj, const void* tgt_proj, const float* w_res, const float* b_res,
                         const unsigned char* src_mask, const unsigned char* row_mask, float* scores,
                         int B, int T_len, int S, int dim, int dtype, void* stream) {
  return copy_scores_fwd_impl(src_proj, tgt_proj, w_res, b_res, src_mask, row_mask, nullptr, scores, B, T_len, S, dim,
                              dtype, stream);
}

int fira_copy_scores_bwd(const void* src_proj, const void* tgt_proj, const float* w_res, const float* d_scores,
                         const unsigned char* row_active, void* d_src_proj, float* d_tgt_proj, float* d_w_res,
                         float* d_b_res, int B, int T_len, int S, int dim, int dtype, void* stream) {
  return copy_scores_bwd_impl(src_proj, tgt_proj, w_res, d_scores, row_active, nullptr, d_src_proj, d_tgt_proj, d_w_res,
                              d_b_res, B, T_len, S, dim, dtype, stream);
}

int fira_copy_scores_packed_fwd(const void* src_proj, const void* tgt_proj, const float* w_res, const float* b_res,
                                const int* ranges, const unsigned char* src_mask, const unsigned char* row_mask,
                                float* scores, int B, int T_len, int S, int dim, int dtype, void* stream) {
  FIRA_CHECK_ARG(ranges, FIRA_ERR_ARG, "copy_scores_packed_fwd: null ranges");
  return copy_scores_fwd_impl(src_proj, tgt_proj, w_res, b_res, src_mask, row_mask, ranges, scores, B, T_len, S, dim,
                              dtype, stream);
}

int fira_copy_scores_packed_bwd(const void* src_proj, const void* tgt_proj, const float* w_res, const float* d_scores,
                                const unsigned char* row_active, const int* ranges, void* d_src_proj, float* d_tgt_proj,
                                float* d_w_res, float* d_b_res, int B, int T_len, int S, int dim, int dtype, void* stream) {
  FIRA_CHECK_ARG(ranges, FIRA_ERR_ARG, "copy_scores_packed_bwd: null ranges");
  return copy_scores_bwd_impl(src_proj, tgt_proj, w_res, d_scores, row_active, ranges, d_src_proj, d_tgt_proj, d_w_res,
                              d_b_res, B, T_len, S, dim, dtype, stream);
}

int fira_vocab_rows(const int* label, long rows, int V, int* vslot, int* vrows, int cap, void* stream) {
  FIRA_CHECK_ARG(label && vslot && vrows && rows >= 0 && V > 0 && cap >= 0, FIRA_ERR_ARG, "vocab_rows: arguments");
  launch_k(vocab_rows_kernel, dim3(1), dim3(kRowsThreads), 0, (cudaStream_t)stream, label, rows, V, vslot, vrows, cap);
  FIRA_CHECK_LAUNCH("fira_vocab_rows");
  return FIRA_OK;
}

int fira_target_rows(const int* label, int B, int T, int* tlen, int* toff, int* trows, int cap, void* stream) {
  FIRA_CHECK_ARG(label && tlen && toff && trows && B > 0 && B <= kRowsThreads && T > 0 && cap >= 0, FIRA_ERR_ARG,
                 "target_rows: arguments (B <= %d)", kRowsThreads);
  launch_k(target_rows_kernel, dim3(1), dim3(kRowsThreads), 0, (cudaStream_t)stream, label, B, T, tlen, toff, trows, cap);
  FIRA_CHECK_LAUNCH("fira_target_rows");
  return FIRA_OK;
}

int fira_gather_rows(const void* src, long ld_src, const int* idx, void* dst, long ld_dst, long n, int width, int dtype,
                     void* stream) {
  FIRA_CHECK_ARG(idx && n >= 0 && width > 0 && width % 8 == 0 && ld_src >= width && ld_dst >= width, FIRA_ERR_ARG,
                 "gather_rows: arguments");
  FIRA_CHECK_ARG(fira_aligned16(src) && fira_aligned16(dst) && ld_src % 8 == 0 && ld_dst % 8 == 0, FIRA_ERR_ALIGN,
                 "gather_rows: 16-B alignment");
  if (n == 0) return FIRA_OK;
  const long g = (n + 7) / 8, gmax = (long)fira_num_sms() * 16;
  DISPATCH_T(dtype, launch_k(gather_rows_kernel<T>, dim3((unsigned)(g < gmax ? g : gmax)), dim3(256), 0,
      (cudaStream_t)stream, (const T*)src, ld_src, idx, (T*)dst, ld_dst, n, width);)
  FIRA_CHECK_LAUNCH("fira_gather_rows");
  return FIRA_OK;
}

int fira_pointer_mix_nll_fwd_rows(const void* logits, long ld_logits, const float* copy_scores, const float* gate_logits,
                                  const unsigned char* mem_mask, const int* label, const int* vslot, float* stats,
                                  float* nll, int* argmax_out, long rows, int T_len, int V, int S, int dtype,
                                  void* stream) {
  FIRA_CHECK_ARG(rows >= 0 && T_len > 0 && V > 0 && S > 0, FIRA_ERR_SHAPE, "pointer_mix_nll_fwd: shape");
  FIRA_CHECK_ARG(fira_aligned16(logits) && ld_logits % 8 == 0, FIRA_ERR_ALIGN,
                 "pointer_mix_nll_fwd: logits must be 16-byte aligned with a leading dimension that is a multiple of 8");
  FIRA_CHECK_ARG(!(vslot && argmax_out), FIRA_ERR_ARG, "pointer_mix_nll_fwd: the argmax needs the logits of every row");
  if (rows == 0) return FIRA_OK;
  DISPATCH_T(dtype, launch_k(head_fwd_kernel<T>, dim3((unsigned)rows), dim3(256), 0, (cudaStream_t)stream,
      (const T*)logits, ld_logits, copy_scores, gate_logits, mem_mask, label, vslot, stats, nll, argmax_out, T_len, V,
      S);)
  FIRA_CHECK_LAUNCH("fira_pointer_mix_nll_fwd");
  return FIRA_OK;
}

int fira_pointer_mix_nll_fwd(const void* logits, long ld_logits, const float* copy_scores, const float* gate_logits,
                             const unsigned char* mem_mask, const int* label, float* stats, float* nll,
                             int* argmax_out, long rows, int T_len, int V, int S, int dtype, void* stream) {
  return fira_pointer_mix_nll_fwd_rows(logits, ld_logits, copy_scores, gate_logits, mem_mask, label, nullptr, stats, nll,
                                       argmax_out, rows, T_len, V, S, dtype, stream);
}

static int nll_bwd_impl(const void* logits, long ld_logits, const float* copy_scores, const unsigned char* mem_mask,
                        const int* label, const int* vslot, const int* vrows, int cap, const float* stats,
                        const float* upstream, const float* seq_weight, void* d_logits, float* d_copy_scores,
                        float* d_gate_logits, unsigned char* row_active, long rows, int T_len, int V, int S, int dtype,
                        void* stream) {
  FIRA_CHECK_ARG(rows >= 0 && T_len > 0 && V > 0 && S > 0, FIRA_ERR_SHAPE, "pointer_mix_nll_bwd: shape");
  FIRA_CHECK_ARG(fira_aligned16(logits) && fira_aligned16(d_logits) && ld_logits % 8 == 0, FIRA_ERR_ALIGN,
                 "pointer_mix_nll_bwd: logits / d_logits must be 16-byte aligned with a leading dimension that is a multiple of 8");
  FIRA_CHECK_ARG(!vslot || (vrows && cap >= 0 && cap <= rows), FIRA_ERR_ARG, "pointer_mix_nll_bwd: vrows / cap");
  if (rows == 0) return FIRA_OK;
  DISPATCH_T(dtype, launch_k(head_bwd_kernel<T>, dim3((unsigned)rows), dim3(256), 0, (cudaStream_t)stream,
      (const T*)logits, ld_logits, copy_scores, mem_mask, label, vslot, vrows, cap, stats, upstream, (T*)d_logits,
      d_copy_scores, d_gate_logits, row_active, T_len, V, S, seq_weight);)
  FIRA_CHECK_LAUNCH("fira_pointer_mix_nll_bwd");
  return FIRA_OK;
}

int fira_pointer_mix_nll_bwd_rows(const void* logits, long ld_logits, const float* copy_scores,
                                  const unsigned char* mem_mask, const int* label, const int* vslot, const int* vrows,
                                  int cap, const float* stats, const float* upstream, void* d_logits,
                                  float* d_copy_scores, float* d_gate_logits, unsigned char* row_active, long rows,
                                  int T_len, int V, int S, int dtype, void* stream) {
  return nll_bwd_impl(logits, ld_logits, copy_scores, mem_mask, label, vslot, vrows, cap, stats, upstream, nullptr,
                      d_logits, d_copy_scores, d_gate_logits, row_active, rows, T_len, V, S, dtype, stream);
}

int fira_pointer_mix_nll_bwd_rows_weighted(const void* logits, long ld_logits, const float* copy_scores,
                                           const unsigned char* mem_mask, const int* label, const int* vslot,
                                           const int* vrows, int cap, const float* stats, const float* upstream,
                                           void* d_logits, float* d_copy_scores, float* d_gate_logits,
                                           unsigned char* row_active, long rows, int T_len, int V, int S, int dtype,
                                           void* stream, const float* seq_weight) {
  FIRA_CHECK_ARG(seq_weight, FIRA_ERR_ARG, "pointer_mix_nll_bwd_rows_weighted: null seq_weight");
  return nll_bwd_impl(logits, ld_logits, copy_scores, mem_mask, label, vslot, vrows, cap, stats, upstream, seq_weight,
                      d_logits, d_copy_scores, d_gate_logits, row_active, rows, T_len, V, S, dtype, stream);
}

int fira_pointer_mix_nll_bwd(const void* logits, long ld_logits, const float* copy_scores,
                             const unsigned char* mem_mask, const int* label, const float* stats,
                             const float* upstream, void* d_logits, float* d_copy_scores, float* d_gate_logits,
                             unsigned char* row_active, long rows, int T_len, int V, int S, int dtype, void* stream) {
  return fira_pointer_mix_nll_bwd_rows(logits, ld_logits, copy_scores, mem_mask, label, nullptr, nullptr, 0, stats,
                                       upstream, d_logits, d_copy_scores, d_gate_logits, row_active, rows, T_len, V, S,
                                       dtype, stream);
}

// The checks every decoding step makes; `who` is the entry point's name without its _prefix / _rules suffix, `hist` the
// width of the token histories (its name in the messages: `hist_name`)
static int step_check(const char* who, const void* logits, long ld_logits, long hist, const char* hist_name, int pos,
                      const int* prefix, int ld_prefix, const int* prefix_len, int no_repeat, int min_len) {
  FIRA_CHECK_ARG(!prefix || (prefix_len && ld_prefix > pos), FIRA_ERR_ARG,
                 "%s_prefix: null prefix_len or ld_prefix %d <= pos %d", who, ld_prefix, pos);
  FIRA_CHECK_ARG(no_repeat >= 0 && min_len >= 0, FIRA_ERR_ARG,
                 "%s_rules: no_repeat_ngram %d / min_length %d < 0", who, no_repeat, min_len);
  FIRA_CHECK_ARG((!no_repeat && !min_len) || hist <= TMAX, FIRA_ERR_SHAPE, "%s_rules: %s %ld > %d", who, hist_name,
                 hist, TMAX);
  FIRA_CHECK_ARG(pos >= 0 && hist >= pos + 2, FIRA_ERR_SHAPE, "%s: pos %d, %s %ld", who, pos, hist_name, hist);
  FIRA_CHECK_ARG(fira_aligned16(logits) && ld_logits % 8 == 0, FIRA_ERR_ALIGN,
                 "%s: logits must be 16-byte aligned with a leading dimension that is a multiple of 8", who);
  return FIRA_OK;
}

static int sample_impl(const void* logits, long ld_logits, const float* copy_scores, const float* gate_logits,
                       const unsigned char* mem_mask, const int* copy_src, const uint64_t* seed, const int* first_index,
                       const float* uniforms, float temperature, int top_k, float top_p, int eos_id, int pad_id,
                       int* next_tok, int* seq, int* raw, float* token_logprob, unsigned char* tok_mask, long ld_out,
                       int pos, unsigned char* finished, int* length, float* logprob, int B, int N, int V, int S,
                       const int* prefix, int ld_prefix, const int* prefix_len, int no_repeat, int min_len, int dtype,
                       void* stream) {
  const int rc = step_check("pointer_mix_sample", logits, ld_logits, ld_out, "ld_out", pos, prefix, ld_prefix,
                            prefix_len, no_repeat, min_len);
  if (rc != FIRA_OK) return rc;
  FIRA_CHECK_ARG(B >= 0 && N > 0 && V > 0 && S > 0 && V + S <= 0x7FFF, FIRA_ERR_SHAPE,
                 "pointer_mix_sample: shape (B %d, N %d, V %d, S %d; V + S must be <= 32767)", B, N, V, S);
  FIRA_CHECK_ARG(temperature > 0.f && temperature <= 3.4e38f, FIRA_ERR_ARG, "pointer_mix_sample: temperature %g",
                 (double)temperature);
  FIRA_CHECK_ARG(top_k >= 0, FIRA_ERR_ARG, "pointer_mix_sample: top_k %d < 0", top_k);
  FIRA_CHECK_ARG(top_p > 0.f && top_p <= 1.f, FIRA_ERR_ARG, "pointer_mix_sample: top_p %g not in (0, 1]", (double)top_p);
  FIRA_CHECK_ARG(uniforms || (seed && first_index), FIRA_ERR_ARG, "pointer_mix_sample: seed / first_index missing");
  if (B == 0) return FIRA_OK;
  const int smem = (int)sizeof(float) * (V + S);
  cudaError_t e = dtype == FIRA_F32
      ? cudaFuncSetAttribute(pointer_mix_sample_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)
      : cudaFuncSetAttribute(pointer_mix_sample_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) { fira_set_error(FIRA_ERR_CUDA, "pointer_mix_sample attr: %s", cudaGetErrorString(e)); return FIRA_ERR_CUDA; }
  DISPATCH_T(dtype, launch_k(pointer_mix_sample_kernel<T>, dim3((unsigned)(B * N)), dim3(kSampleThreads), smem,
      (cudaStream_t)stream, (const T*)logits, ld_logits, copy_scores, gate_logits, mem_mask, copy_src, seed, first_index,
      uniforms, temperature, top_k, top_p, eos_id, pad_id, next_tok, seq, raw, token_logprob, tok_mask, ld_out, pos,
      finished, length, logprob, prefix, ld_prefix, prefix_len, no_repeat, min_len, N, V, S);)
  FIRA_CHECK_LAUNCH("fira_pointer_mix_sample");
  return FIRA_OK;
}

int fira_pointer_mix_sample(const void* logits, long ld_logits, const float* copy_scores, const float* gate_logits,
                            const unsigned char* mem_mask, const int* copy_src, const uint64_t* seed,
                            const int* first_index, const float* uniforms, float temperature, int top_k, float top_p,
                            int eos_id, int pad_id, int* next_tok, int* seq, int* raw, float* token_logprob,
                            unsigned char* tok_mask, long ld_out, int pos, unsigned char* finished, int* length,
                            float* logprob, int B, int N, int V, int S, int dtype, void* stream) {
  return sample_impl(logits, ld_logits, copy_scores, gate_logits, mem_mask, copy_src, seed, first_index, uniforms,
                     temperature, top_k, top_p, eos_id, pad_id, next_tok, seq, raw, token_logprob, tok_mask, ld_out, pos,
                     finished, length, logprob, B, N, V, S, nullptr, 0, nullptr, 0, 0, dtype, stream);
}

int fira_pointer_mix_sample_prefix(const void* logits, long ld_logits, const float* copy_scores,
                                   const float* gate_logits, const unsigned char* mem_mask, const int* copy_src,
                                   const uint64_t* seed, const int* first_index, const float* uniforms,
                                   float temperature, int top_k, float top_p, int eos_id, int pad_id, int* next_tok,
                                   int* seq, int* raw, float* token_logprob, unsigned char* tok_mask, long ld_out,
                                   int pos, unsigned char* finished, int* length, float* logprob, int B, int N, int V,
                                   int S, int dtype, void* stream, const int* prefix, int ld_prefix,
                                   const int* prefix_len) {
  return sample_impl(logits, ld_logits, copy_scores, gate_logits, mem_mask, copy_src, seed, first_index, uniforms,
                     temperature, top_k, top_p, eos_id, pad_id, next_tok, seq, raw, token_logprob, tok_mask, ld_out, pos,
                     finished, length, logprob, B, N, V, S, prefix, ld_prefix, prefix_len, 0, 0, dtype, stream);
}

int fira_pointer_mix_sample_rules(const void* logits, long ld_logits, const float* copy_scores,
                                  const float* gate_logits, const unsigned char* mem_mask, const int* copy_src,
                                  const uint64_t* seed, const int* first_index, const float* uniforms,
                                  float temperature, int top_k, float top_p, int eos_id, int pad_id, int* next_tok,
                                  int* seq, int* raw, float* token_logprob, unsigned char* tok_mask, long ld_out,
                                  int pos, unsigned char* finished, int* length, float* logprob, int B, int N, int V,
                                  int S, int dtype, void* stream, const int* prefix, int ld_prefix,
                                  const int* prefix_len, int no_repeat_ngram, int min_length) {
  return sample_impl(logits, ld_logits, copy_scores, gate_logits, mem_mask, copy_src, seed, first_index, uniforms,
                     temperature, top_k, top_p, eos_id, pad_id, next_tok, seq, raw, token_logprob, tok_mask, ld_out, pos,
                     finished, length, logprob, B, N, V, S, prefix, ld_prefix, prefix_len, no_repeat_ngram, min_length,
                     dtype, stream);
}

static int beam_step_impl(const void* logits, long ld_logits, const float* copy_scores, const float* gate_logits,
                          const unsigned char* mem_mask, const int* copy_src, float length_penalty, int eos_id,
                          int pad_id, uint64_t* workspace, int* seq, int* raw, float* token_logprob, int* length,
                          float* logprob, float* score, unsigned char* status, long* parent, int* next_tok, int T_len,
                          int pos, int B, int K, int V, int S, const int* prefix, int ld_prefix, const int* prefix_len,
                          int no_repeat, int min_len, int dtype, void* stream, const int* constraints = nullptr) {
  const int rc = step_check("pointer_mix_beam_step", logits, ld_logits, T_len, "T_len", pos, prefix, ld_prefix,
                            prefix_len, no_repeat, min_len);
  if (rc != FIRA_OK) return rc;
  FIRA_CHECK_ARG(!constraints || T_len <= TMAX, FIRA_ERR_SHAPE, "pointer_mix_beam_step_lexical: T_len %d > %d", T_len,
                 TMAX);
  FIRA_CHECK_ARG(B >= 0 && K >= 1 && K <= kMaxBeam && V >= K && S > 0 && V + S <= 0x7FFF, FIRA_ERR_SHAPE,
                 "pointer_mix_beam_step: shape (B %d, K %d, V %d, S %d; 1 <= K <= 16, K <= V, V + S <= 32767)",
                 B, K, V, S);
  FIRA_CHECK_ARG(length_penalty >= 0.f && length_penalty <= 3.4e38f, FIRA_ERR_ARG,
                 "pointer_mix_beam_step: length_penalty %g", (double)length_penalty);
  if (B == 0) return FIRA_OK;
  const unsigned char* st_in = status + (pos & 1) * (long)B * K;
  const int* seq_in = seq + (pos & 1) * (long)B * K * T_len;
  if (constraints) {
    DISPATCH_T(dtype, launch_k(beam_row_kernel<T, true>, dim3((unsigned)(B * K)), dim3(kBeamThreads), 0,
        (cudaStream_t)stream, (const T*)logits, ld_logits, copy_scores, gate_logits, mem_mask, copy_src, st_in, seq_in,
        T_len, workspace, prefix, ld_prefix, prefix_len, no_repeat, min_len, eos_id, pos, K, V, S, constraints);)
    FIRA_CHECK_LAUNCH("fira_pointer_mix_beam_step_lexical (rows)");
  } else {
    DISPATCH_T(dtype, launch_k(beam_row_kernel<T, false>, dim3((unsigned)(B * K)), dim3(kBeamThreads), 0,
        (cudaStream_t)stream, (const T*)logits, ld_logits, copy_scores, gate_logits, mem_mask, copy_src, st_in, seq_in,
        T_len, workspace, prefix, ld_prefix, prefix_len, no_repeat, min_len, eos_id, pos, K, V, S, nullptr);)
    FIRA_CHECK_LAUNCH("fira_pointer_mix_beam_step (rows)");
  }
  const int W = constraints ? K + kPhrases : K;       // row_top entries per row (beam_row_kernel)
  launch_k(beam_select_kernel, dim3((unsigned)B), dim3(kSelectThreads), 0, (cudaStream_t)stream,
           (const uint64_t*)workspace, W, constraints, copy_src, length_penalty, eos_id, pad_id, seq, raw, token_logprob,
           length, logprob, score, status, parent, next_tok, T_len, pos, B, K, V, S);
  FIRA_CHECK_LAUNCH(constraints ? "fira_pointer_mix_beam_step_lexical (select)" : "fira_pointer_mix_beam_step (select)");
  return FIRA_OK;
}

int fira_pointer_mix_beam_step(const void* logits, long ld_logits, const float* copy_scores, const float* gate_logits,
                               const unsigned char* mem_mask, const int* copy_src, float length_penalty, int eos_id,
                               int pad_id, uint64_t* workspace, int* seq, int* raw, float* token_logprob, int* length,
                               float* logprob, float* score, unsigned char* status, long* parent, int* next_tok,
                               int T_len, int pos, int B, int K, int V, int S, int dtype, void* stream) {
  return beam_step_impl(logits, ld_logits, copy_scores, gate_logits, mem_mask, copy_src, length_penalty, eos_id, pad_id,
                        workspace, seq, raw, token_logprob, length, logprob, score, status, parent, next_tok, T_len, pos,
                        B, K, V, S, nullptr, 0, nullptr, 0, 0, dtype, stream);
}

int fira_pointer_mix_beam_step_prefix(const void* logits, long ld_logits, const float* copy_scores,
                                      const float* gate_logits, const unsigned char* mem_mask, const int* copy_src,
                                      float length_penalty, int eos_id, int pad_id, uint64_t* workspace, int* seq,
                                      int* raw, float* token_logprob, int* length, float* logprob, float* score,
                                      unsigned char* status, long* parent, int* next_tok, int T_len, int pos, int B,
                                      int K, int V, int S, int dtype, void* stream, const int* prefix, int ld_prefix,
                                      const int* prefix_len) {
  return beam_step_impl(logits, ld_logits, copy_scores, gate_logits, mem_mask, copy_src, length_penalty, eos_id, pad_id,
                        workspace, seq, raw, token_logprob, length, logprob, score, status, parent, next_tok, T_len, pos,
                        B, K, V, S, prefix, ld_prefix, prefix_len, 0, 0, dtype, stream);
}

int fira_pointer_mix_beam_step_rules(const void* logits, long ld_logits, const float* copy_scores,
                                     const float* gate_logits, const unsigned char* mem_mask, const int* copy_src,
                                     float length_penalty, int eos_id, int pad_id, uint64_t* workspace, int* seq,
                                     int* raw, float* token_logprob, int* length, float* logprob, float* score,
                                     unsigned char* status, long* parent, int* next_tok, int T_len, int pos, int B,
                                     int K, int V, int S, int dtype, void* stream, const int* prefix, int ld_prefix,
                                     const int* prefix_len, int no_repeat_ngram, int min_length) {
  return beam_step_impl(logits, ld_logits, copy_scores, gate_logits, mem_mask, copy_src, length_penalty, eos_id, pad_id,
                        workspace, seq, raw, token_logprob, length, logprob, score, status, parent, next_tok, T_len, pos,
                        B, K, V, S, prefix, ld_prefix, prefix_len, no_repeat_ngram, min_length, dtype, stream);
}

int fira_pointer_mix_beam_step_lexical(const void* logits, long ld_logits, const float* copy_scores,
                                       const float* gate_logits, const unsigned char* mem_mask, const int* copy_src,
                                       float length_penalty, int eos_id, int pad_id, uint64_t* workspace, int* seq,
                                       int* raw, float* token_logprob, int* length, float* logprob, float* score,
                                       unsigned char* status, long* parent, int* next_tok, int T_len, int pos, int B,
                                       int K, int V, int S, int dtype, void* stream, const int* prefix, int ld_prefix,
                                       const int* prefix_len, int no_repeat_ngram, int min_length,
                                       const int* constraints) {
  FIRA_CHECK_ARG(constraints && workspace, FIRA_ERR_ARG, "pointer_mix_beam_step_lexical: null constraints / workspace");
  return beam_step_impl(logits, ld_logits, copy_scores, gate_logits, mem_mask, copy_src, length_penalty, eos_id, pad_id,
                        workspace, seq, raw, token_logprob, length, logprob, score, status, parent, next_tok, T_len, pos,
                        B, K, V, S, prefix, ld_prefix, prefix_len, no_repeat_ngram, min_length, dtype, stream,
                        constraints);
}

static int diverse_beam_step_impl(const void* logits, long ld_logits, const float* copy_scores,
                                  const float* gate_logits, const unsigned char* mem_mask, const int* copy_src,
                                  float length_penalty, int eos_id, int pad_id, uint64_t* workspace, int* seq, int* raw,
                                  float* token_logprob, int* length, float* logprob, float* score,
                                  unsigned char* status, long* parent, int* next_tok, int T_len, int pos, int B, int K,
                                  int V, int S, int groups, float diversity, int* chosen, float* lp_workspace,
                                  const int* prefix, int ld_prefix, const int* prefix_len, int no_repeat, int min_len,
                                  int dtype, void* stream) {
  const int rc = step_check("pointer_mix_diverse_beam_step", logits, ld_logits, T_len, "T_len", pos, prefix, ld_prefix,
                            prefix_len, no_repeat, min_len);
  if (rc != FIRA_OK) return rc;
  FIRA_CHECK_ARG(B >= 0 && K >= 1 && K <= kMaxBeam && V >= K && S > 0 && V + S <= 0x7FFF, FIRA_ERR_SHAPE,
                 "pointer_mix_diverse_beam_step: shape (B %d, K %d, V %d, S %d; 1 <= K <= 16, K <= V, V + S <= 32767)",
                 B, K, V, S);
  FIRA_CHECK_ARG(groups >= 1 && groups <= K && K % groups == 0, FIRA_ERR_ARG,
                 "pointer_mix_diverse_beam_step: groups %d must divide K %d", groups, K);
  FIRA_CHECK_ARG(length_penalty >= 0.f && length_penalty <= 3.4e38f, FIRA_ERR_ARG,
                 "pointer_mix_diverse_beam_step: length_penalty %g", (double)length_penalty);
  FIRA_CHECK_ARG(diversity >= 0.f && diversity <= 3.4e38f, FIRA_ERR_ARG,
                 "pointer_mix_diverse_beam_step: diversity %g", (double)diversity);
  FIRA_CHECK_ARG(workspace && lp_workspace && chosen, FIRA_ERR_ARG,
                 "pointer_mix_diverse_beam_step: null workspace / lp_workspace / chosen");
  if (B == 0) return FIRA_OK;
  const int Kg = K / groups;
  const long in = (pos & 1) * (long)B * K;            // the read half of the slot state
  for (int g = 0; g < groups; ++g) {
    DISPATCH_T(dtype, launch_k(diverse_row_kernel<T>, dim3((unsigned)(B * Kg)), dim3(kBeamThreads), 0,
        (cudaStream_t)stream, (const T*)logits, ld_logits, copy_scores, gate_logits, mem_mask, copy_src,
        (const unsigned char*)status + in, (const float*)logprob + in, (const int*)length + in, (const int*)chosen,
        length_penalty, diversity, workspace, lp_workspace, (const int*)seq + in * T_len, T_len, prefix, ld_prefix,
        prefix_len, no_repeat, min_len, eos_id, pos, g, Kg, K, V, S);)
    FIRA_CHECK_LAUNCH("fira_pointer_mix_diverse_beam_step (rows)");
    launch_k(diverse_select_kernel, dim3((unsigned)B), dim3(kBeamThreads), 0, (cudaStream_t)stream,
             (const uint64_t*)workspace, (const float*)lp_workspace, copy_src, length_penalty, diversity, eos_id,
             pad_id, seq, raw, token_logprob, length, logprob, score, status, parent, next_tok, chosen, T_len, pos, B,
             g, Kg, K, V, S);
    FIRA_CHECK_LAUNCH("fira_pointer_mix_diverse_beam_step (select)");
  }
  return FIRA_OK;
}

int fira_pointer_mix_diverse_beam_step(const void* logits, long ld_logits, const float* copy_scores,
                                       const float* gate_logits, const unsigned char* mem_mask, const int* copy_src,
                                       float length_penalty, int eos_id, int pad_id, uint64_t* workspace, int* seq,
                                       int* raw, float* token_logprob, int* length, float* logprob, float* score,
                                       unsigned char* status, long* parent, int* next_tok, int T_len, int pos, int B,
                                       int K, int V, int S, int groups, float diversity, int* chosen,
                                       float* lp_workspace, int dtype, void* stream) {
  return diverse_beam_step_impl(logits, ld_logits, copy_scores, gate_logits, mem_mask, copy_src, length_penalty, eos_id,
                                pad_id, workspace, seq, raw, token_logprob, length, logprob, score, status, parent,
                                next_tok, T_len, pos, B, K, V, S, groups, diversity, chosen, lp_workspace, nullptr, 0,
                                nullptr, 0, 0, dtype, stream);
}

int fira_pointer_mix_diverse_beam_step_prefix(const void* logits, long ld_logits, const float* copy_scores,
                                              const float* gate_logits, const unsigned char* mem_mask,
                                              const int* copy_src, float length_penalty, int eos_id, int pad_id,
                                              uint64_t* workspace, int* seq, int* raw, float* token_logprob,
                                              int* length, float* logprob, float* score, unsigned char* status,
                                              long* parent, int* next_tok, int T_len, int pos, int B, int K, int V,
                                              int S, int groups, float diversity, int* chosen, float* lp_workspace,
                                              int dtype, void* stream, const int* prefix, int ld_prefix,
                                              const int* prefix_len) {
  return diverse_beam_step_impl(logits, ld_logits, copy_scores, gate_logits, mem_mask, copy_src, length_penalty, eos_id,
                                pad_id, workspace, seq, raw, token_logprob, length, logprob, score, status, parent,
                                next_tok, T_len, pos, B, K, V, S, groups, diversity, chosen, lp_workspace, prefix,
                                ld_prefix, prefix_len, 0, 0, dtype, stream);
}

int fira_pointer_mix_diverse_beam_step_rules(const void* logits, long ld_logits, const float* copy_scores,
                                             const float* gate_logits, const unsigned char* mem_mask,
                                             const int* copy_src, float length_penalty, int eos_id, int pad_id,
                                             uint64_t* workspace, int* seq, int* raw, float* token_logprob,
                                             int* length, float* logprob, float* score, unsigned char* status,
                                             long* parent, int* next_tok, int T_len, int pos, int B, int K, int V,
                                             int S, int groups, float diversity, int* chosen, float* lp_workspace,
                                             int dtype, void* stream, const int* prefix, int ld_prefix,
                                             const int* prefix_len, int no_repeat_ngram, int min_length) {
  return diverse_beam_step_impl(logits, ld_logits, copy_scores, gate_logits, mem_mask, copy_src, length_penalty, eos_id,
                                pad_id, workspace, seq, raw, token_logprob, length, logprob, score, status, parent,
                                next_tok, T_len, pos, B, K, V, S, groups, diversity, chosen, lp_workspace, prefix,
                                ld_prefix, prefix_len, no_repeat_ngram, min_length, dtype, stream);
}

int fira_pointer_mix_ensemble(const void* const* logits, long ld_logits, const float* const* copy_scores,
                              const float* const* gate_logits, int M, const float* log_weights,
                              const unsigned char* mem_mask, float* logits_out, long ld_out, float* copy_out,
                              float* gate_out, int B, int N, int V, int S, int dtype, void* stream) {
  FIRA_CHECK_ARG(M >= 1 && M <= kMaxMembers, FIRA_ERR_ARG, "pointer_mix_ensemble: M %d not in [1, %d]", M, kMaxMembers);
  FIRA_CHECK_ARG(logits && copy_scores && gate_logits && log_weights && mem_mask && logits_out && copy_out && gate_out,
                 FIRA_ERR_ARG, "pointer_mix_ensemble: null pointer");
  Members mem = {};
  for (int m = 0; m < M; ++m) {
    FIRA_CHECK_ARG(logits[m] && copy_scores[m] && gate_logits[m], FIRA_ERR_ARG,
                   "pointer_mix_ensemble: null pointer of member %d", m);
    FIRA_CHECK_ARG(fira_aligned16(logits[m]), FIRA_ERR_ALIGN,
                   "pointer_mix_ensemble: logits of member %d must be 16-byte aligned", m);
    mem.logits[m] = logits[m]; mem.sc[m] = copy_scores[m]; mem.gl[m] = gate_logits[m];
  }
  FIRA_CHECK_ARG(fira_aligned16(logits_out) && ld_logits % 8 == 0 && ld_out % 8 == 0, FIRA_ERR_ALIGN,
                 "pointer_mix_ensemble: logits_out must be 16-byte aligned, ld_logits %ld and ld_out %ld multiples of 8",
                 ld_logits, ld_out);
  FIRA_CHECK_ARG(B >= 0 && N > 0 && V > 0 && S > 0 && V + S <= 0x7FFF && ld_logits >= V && ld_out >= V, FIRA_ERR_SHAPE,
                 "pointer_mix_ensemble: shape (B %d, N %d, V %d, S %d, ld_logits %ld, ld_out %ld; V + S must be <= 32767)",
                 B, N, V, S, ld_logits, ld_out);
  if (B == 0) return FIRA_OK;
  DISPATCH_T(dtype, launch_k(pointer_mix_ensemble_kernel<T>, dim3((unsigned)(B * N)), dim3(kEnsThreads), 0,
      (cudaStream_t)stream, mem, M, ld_logits, log_weights, mem_mask, logits_out, ld_out, copy_out, gate_out, N, V, S);)
  FIRA_CHECK_LAUNCH("fira_pointer_mix_ensemble");
  return FIRA_OK;
}

int fira_pointer_mix_knn(const void* logits, long ld_logits, const float* copy_scores, const float* gate_logits,
                         const unsigned char* mem_mask, const int* nb_idx, const float* nb_dist, const int* words,
                         int k, const float* params, float* logits_out, long ld_out, float* copy_out, float* gate_out,
                         int B, int N, int V, int S, int dtype, void* stream) {
  FIRA_CHECK_ARG(k >= 1 && k <= kKnnMaxK, FIRA_ERR_ARG, "pointer_mix_knn: k %d not in [1, %d]", k, kKnnMaxK);
  FIRA_CHECK_ARG(logits && copy_scores && gate_logits && mem_mask && nb_idx && nb_dist && words && params &&
                 logits_out && copy_out && gate_out, FIRA_ERR_ARG, "pointer_mix_knn: null pointer");
  FIRA_CHECK_ARG(fira_aligned16(logits) && fira_aligned16(logits_out) && ld_logits % 8 == 0 && ld_out % 8 == 0,
                 FIRA_ERR_ALIGN, "pointer_mix_knn: logits / logits_out must be 16-byte aligned, ld_logits %ld and "
                 "ld_out %ld multiples of 8", ld_logits, ld_out);
  FIRA_CHECK_ARG(B >= 0 && N > 0 && V > 0 && S > 0 && V + S <= 0x7FFF && ld_logits >= V && ld_out >= V, FIRA_ERR_SHAPE,
                 "pointer_mix_knn: shape (B %d, N %d, V %d, S %d, ld_logits %ld, ld_out %ld; V + S must be <= 32767)",
                 B, N, V, S, ld_logits, ld_out);
  if (B == 0) return FIRA_OK;
  DISPATCH_T(dtype, launch_k(pointer_mix_knn_kernel<T>, dim3((unsigned)(B * N)), dim3(kEnsThreads), 0,
      (cudaStream_t)stream, (const T*)logits, ld_logits, copy_scores, gate_logits, mem_mask, nb_idx, nb_dist, words, k,
      params, logits_out, ld_out, copy_out, gate_out, N, V, S);)
  FIRA_CHECK_LAUNCH("fira_pointer_mix_knn");
  return FIRA_OK;
}

static int kd_check(const char* who, const void* logits, long ld_logits, const float* t_logits, long ld_t, float alpha,
                    long rows, int T_len, int V, int S) {
  FIRA_CHECK_ARG(alpha >= 0.f && alpha <= 1.f, FIRA_ERR_ARG, "%s: alpha %g not in [0, 1]", who, (double)alpha);
  FIRA_CHECK_ARG(rows >= 0 && T_len > 0 && V > 0 && S > 0 && V + S <= 0x7FFF && ld_logits >= V && ld_t >= V,
                 FIRA_ERR_SHAPE, "%s: shape (rows %ld, T_len %d, V %d, S %d, ld_logits %ld, ld_t %ld; V + S must be <= 32767)",
                 who, rows, T_len, V, S, ld_logits, ld_t);
  FIRA_CHECK_ARG(fira_aligned16(logits) && fira_aligned16(t_logits) && ld_logits % 8 == 0 && ld_t % 8 == 0,
                 FIRA_ERR_ALIGN, "%s: logits / teacher logits must be 16-byte aligned with leading dimensions that are "
                 "multiples of 8", who);
  return FIRA_OK;
}

int fira_pointer_mix_kd_fwd(const void* logits, long ld_logits, const float* copy_scores, const float* gate_logits,
                            const unsigned char* mem_mask, const int* label, const float* t_logits, long ld_t,
                            const float* t_copy_scores, const float* t_gate_logits, float alpha, float* stats,
                            float* nll, float* kd, float* loss, long rows, int T_len, int V, int S, int dtype,
                            void* stream) {
  FIRA_CHECK_ARG(logits && copy_scores && gate_logits && mem_mask && label && t_logits && t_copy_scores && t_gate_logits
                 && stats && nll && kd && loss, FIRA_ERR_ARG, "pointer_mix_kd_fwd: null pointer");
  const int rc = kd_check("pointer_mix_kd_fwd", logits, ld_logits, t_logits, ld_t, alpha, rows, T_len, V, S);
  if (rc != FIRA_OK) return rc;
  if (rows == 0) return FIRA_OK;
  DISPATCH_T(dtype, launch_k(pointer_mix_kd_fwd_kernel<T>, dim3((unsigned)rows), dim3(kKdThreads), 0,
      (cudaStream_t)stream, (const T*)logits, ld_logits, copy_scores, gate_logits, mem_mask, label, t_logits, ld_t,
      t_copy_scores, t_gate_logits, alpha, stats, nll, kd, loss, T_len, V, S);)
  FIRA_CHECK_LAUNCH("fira_pointer_mix_kd_fwd");
  return FIRA_OK;
}

int fira_pointer_mix_kd_bwd(const void* logits, long ld_logits, const float* copy_scores,
                            const unsigned char* mem_mask, const int* label, const float* t_logits, long ld_t,
                            const float* t_copy_scores, float alpha, const float* stats, const float* upstream,
                            void* d_logits, float* d_copy_scores, float* d_gate_logits, unsigned char* row_active,
                            long rows, int T_len, int V, int S, int dtype, void* stream) {
  FIRA_CHECK_ARG(logits && copy_scores && mem_mask && label && t_logits && t_copy_scores && stats && upstream && d_logits
                 && d_copy_scores && d_gate_logits && row_active, FIRA_ERR_ARG, "pointer_mix_kd_bwd: null pointer");
  const int rc = kd_check("pointer_mix_kd_bwd", logits, ld_logits, t_logits, ld_t, alpha, rows, T_len, V, S);
  if (rc != FIRA_OK) return rc;
  FIRA_CHECK_ARG(fira_aligned16(d_logits), FIRA_ERR_ALIGN, "pointer_mix_kd_bwd: d_logits must be 16-byte aligned");
  if (rows == 0) return FIRA_OK;
  DISPATCH_T(dtype, launch_k(pointer_mix_kd_bwd_kernel<T>, dim3((unsigned)rows), dim3(kKdThreads), 0,
      (cudaStream_t)stream, (const T*)logits, ld_logits, copy_scores, mem_mask, label, t_logits, ld_t, t_copy_scores,
      alpha, stats, upstream, (T*)d_logits, d_copy_scores, d_gate_logits, row_active, T_len, V, S);)
  FIRA_CHECK_LAUNCH("fira_pointer_mix_kd_bwd");
  return FIRA_OK;
}

int fira_pointer_mix_topk(const float* t_logits, long ld_t, const float* t_copy_scores, const float* t_gate_logits,
                          const unsigned char* mem_mask, const int* label, int k, int* t_label, float* t_prob,
                          float* mass, long rows, int T_len, int V, int S, void* stream) {
  FIRA_CHECK_ARG(k >= 1 && k <= kKdMaxTopk, FIRA_ERR_ARG, "pointer_mix_topk: k %d not in [1, %d]", k, kKdMaxTopk);
  FIRA_CHECK_ARG(t_logits && t_copy_scores && t_gate_logits && mem_mask && label && t_label && t_prob && mass,
                 FIRA_ERR_ARG, "pointer_mix_topk: null pointer");
  FIRA_CHECK_ARG(rows >= 0 && T_len > 0 && V > 0 && S > 0 && V + S <= 0x7FFF && ld_t >= V, FIRA_ERR_SHAPE,
                 "pointer_mix_topk: shape (rows %ld, T_len %d, V %d, S %d, ld_t %ld; V + S must be <= 32767)", rows,
                 T_len, V, S, ld_t);
  FIRA_CHECK_ARG(fira_aligned16(t_logits) && ld_t % 8 == 0, FIRA_ERR_ALIGN,
                 "pointer_mix_topk: t_logits must be 16-byte aligned, ld_t %ld a multiple of 8", ld_t);
  if (rows == 0) return FIRA_OK;
  const size_t smem = (size_t)(V + S) * sizeof(float);
  const cudaError_t e = cudaFuncSetAttribute(pointer_mix_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)smem);
  if (e != cudaSuccess) { fira_set_error(FIRA_ERR_CUDA, "pointer_mix_topk attr: %s", cudaGetErrorString(e)); return FIRA_ERR_CUDA; }
  launch_k(pointer_mix_topk_kernel, dim3((unsigned)rows), dim3(kSampleThreads), smem, (cudaStream_t)stream, t_logits,
           ld_t, t_copy_scores, t_gate_logits, mem_mask, label, k, t_label, t_prob, mass, T_len, V, S);
  FIRA_CHECK_LAUNCH("fira_pointer_mix_topk");
  return FIRA_OK;
}

static int kd_sparse_check(const char* who, const void* logits, long ld_logits, int k, float alpha, long rows,
                           int T_len, int V, int S) {
  FIRA_CHECK_ARG(alpha >= 0.f && alpha <= 1.f, FIRA_ERR_ARG, "%s: alpha %g not in [0, 1]", who, (double)alpha);
  FIRA_CHECK_ARG(k >= 1 && k <= kKdMaxTopk, FIRA_ERR_ARG, "%s: k %d not in [1, %d]", who, k, kKdMaxTopk);
  FIRA_CHECK_ARG(rows >= 0 && T_len > 0 && V > 0 && S > 0 && V + S <= 0x7FFF && ld_logits >= V, FIRA_ERR_SHAPE,
                 "%s: shape (rows %ld, T_len %d, V %d, S %d, ld_logits %ld; V + S must be <= 32767)", who, rows, T_len,
                 V, S, ld_logits);
  FIRA_CHECK_ARG(fira_aligned16(logits) && ld_logits % 8 == 0, FIRA_ERR_ALIGN,
                 "%s: logits must be 16-byte aligned with a leading dimension that is a multiple of 8", who);
  return FIRA_OK;
}

int fira_pointer_mix_kd_sparse_fwd(const void* logits, long ld_logits, const float* copy_scores,
                                   const float* gate_logits, const unsigned char* mem_mask, const int* label,
                                   const int* t_label, const float* t_prob, int k, float alpha, float* stats,
                                   float* nll, float* kd, float* loss, long rows, int T_len, int V, int S, int dtype,
                                   void* stream) {
  FIRA_CHECK_ARG(logits && copy_scores && gate_logits && mem_mask && label && t_label && t_prob && stats && nll && kd
                 && loss, FIRA_ERR_ARG, "pointer_mix_kd_sparse_fwd: null pointer");
  const int rc = kd_sparse_check("pointer_mix_kd_sparse_fwd", logits, ld_logits, k, alpha, rows, T_len, V, S);
  if (rc != FIRA_OK) return rc;
  if (rows == 0) return FIRA_OK;
  DISPATCH_T(dtype, launch_k(pointer_mix_kd_sparse_fwd_kernel<T>, dim3((unsigned)rows), dim3(kKdThreads), 0,
      (cudaStream_t)stream, (const T*)logits, ld_logits, copy_scores, gate_logits, mem_mask, label, t_label, t_prob, k,
      alpha, stats, nll, kd, loss, T_len, V, S);)
  FIRA_CHECK_LAUNCH("fira_pointer_mix_kd_sparse_fwd");
  return FIRA_OK;
}

int fira_pointer_mix_kd_sparse_bwd(const void* logits, long ld_logits, const float* copy_scores,
                                   const unsigned char* mem_mask, const int* label, const int* t_label,
                                   const float* t_prob, int k, float alpha, const float* stats, const float* upstream,
                                   void* d_logits, float* d_copy_scores, float* d_gate_logits,
                                   unsigned char* row_active, long rows, int T_len, int V, int S, int dtype,
                                   void* stream) {
  FIRA_CHECK_ARG(logits && copy_scores && mem_mask && label && t_label && t_prob && stats && upstream && d_logits &&
                 d_copy_scores && d_gate_logits && row_active, FIRA_ERR_ARG, "pointer_mix_kd_sparse_bwd: null pointer");
  const int rc = kd_sparse_check("pointer_mix_kd_sparse_bwd", logits, ld_logits, k, alpha, rows, T_len, V, S);
  if (rc != FIRA_OK) return rc;
  FIRA_CHECK_ARG(fira_aligned16(d_logits), FIRA_ERR_ALIGN, "pointer_mix_kd_sparse_bwd: d_logits must be 16-byte aligned");
  if (rows == 0) return FIRA_OK;
  DISPATCH_T(dtype, launch_k(pointer_mix_kd_sparse_bwd_kernel<T>, dim3((unsigned)rows), dim3(kKdThreads), 0,
      (cudaStream_t)stream, (const T*)logits, ld_logits, copy_scores, mem_mask, label, t_label, t_prob, k, alpha, stats,
      upstream, (T*)d_logits, d_copy_scores, d_gate_logits, row_active, T_len, V, S);)
  FIRA_CHECK_LAUNCH("fira_pointer_mix_kd_sparse_bwd");
  return FIRA_OK;
}

}  // extern "C"
