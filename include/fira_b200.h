/* libfira_b200 -- C ABI of the H100-native (sm_90a) FIRA hot path.
 *
 * The reference (DJjjjhao/FIRA-ICSE) has no FFI of its own: its hot path is PyTorch library
 * calls issued from Model.py / gnn_transformer.py / combination_layer.py.  The drop-in boundary
 * is therefore the nn.Module surface (kept by fira_icse_b200/), and THIS header is the thin
 * C ABI those modules call instead of torch ops.  Each entry point names the reference
 * statement(s) it replaces (paths relative to the reference repository root).
 *
 * Conventions (SURVEY.md section 8b)
 *   - plain pointers + sizes; every pointer is DEVICE memory owned by the caller (PyTorch caching
 *     allocator); the library never allocates, frees or retains a pointer;
 *   - tensors are contiguous row-major unless a leading dimension (ld*) is given, 16-byte aligned;
 *   - ids / indices are int32; masks are uint8 (1 = keep);
 *   - `dtype` selects the ACTIVATION storage type: FIRA_F32 (parity mode) or FIRA_BF16 (throughput
 *     mode); parameters, statistics and gradients of parameters are always fp32;
 *   - `stream` is a cudaStream_t passed as void*; launches are asynchronous, no implicit sync;
 *   - return 0 on success, a FIRA_ERR_* code otherwise; fira_last_error_string() describes the last
 *     failure on the calling thread; nothing throws or aborts across the boundary;
 *   - re-entrant, no hidden global state besides the per-thread error string;
 *   - dropout masks are a pure function of (seed [+ *seed_ctr], stream_id, element index): backward
 *     recomputes them; seed_ctr (device uint64, may be NULL) lets a captured CUDA graph draw fresh masks
 *     on every replay by bumping the counter on the device.
 */
#ifndef FIRA_B200_H_
#define FIRA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FIRA_F32 0
#define FIRA_BF16 1
#define FIRA_EDGE_F32 0
#define FIRA_EDGE_BF16 1
#define FIRA_EDGE_F64 2

int fira_version(void);                    /* ABI version, bumped on any signature change */
const char* fira_last_error_string(void);
int fira_built_arch(void);                 /* 90 when compiled for sm_90a */
int fira_num_sms(void);                    /* SMs of the current device; every launch shape is sized from it */
/* Launch mode of every kernel of the library (the one process-wide switch, atomic): on = programmatic dependent
 * launch -- a kernel's CTAs are scheduled while the previous kernel of the stream drains and block in
 * griddepcontrol.wait before their first global-memory access (results are identical).
 * Default: on (FIRA_PDL=0 in the environment turns it off). */
int fira_set_pdl(int on);
int fira_get_pdl(void);

/* ---- generic fp32 Linear pieces (every nn.Linear of the path; e.g. gnn_transformer.py:78,82,
 *      141-143,158,171-173,200-204; Model.py:16-19,54).
 *      C[M,N] = A(MxK) * B(KxN) + bias[n] + rs[m]*rc[n], optional relu.
 *      A(m,k) = a_kcontig ? A[m*lda+k] : A[k*lda+m];  B(k,n) = b_kcontig ? B[n*ldb+k] : B[k*ldb+n].
 *      accumulate: C += result.  splits>1: K is split across CTAs, partials are atomically added
 *      (the library zero-fills C first unless accumulate). */
int fira_gemm_f32(const float* A, long lda, int a_kcontig, const float* B, long ldb, int b_kcontig, float* C,
                  long ldc, int M, int N, int K, const float* bias, const float* rs, const float* rc, int relu,
                  int accumulate, int splits, void* stream);

/* ---- bf16 tensor-core Linear (throughput mode): wgmma with register accumulators, TMA-staged
 *      operands.  Same contraction as fira_gemm_f32 on bf16 operands (fp32 accumulate):
 *      A(m,k) = a_kmajor ? A[m*lda+k] : A[k*lda+m];  B(k,n) = b_kmajor ? B[n*ldb+k] : B[k*ldb+n];
 *      lda/ldb multiples of 8; C fp32 or bf16 (c_is_bf16), columns >= N of C never written;
 *      accumulate: C += result, relu included
 *      (C += relu(A B + bias + rs rc)), a bf16 C rounded once after the add;
 *      splits>1 = split-K with fp32 atomics (C zero-filled first unless accumulate; bias and rs/rc added by the first
 *      split only). */
int fira_gemm_bf16_tc(const void* A, long lda, int a_kmajor, const void* B, long ldb, int b_kmajor, void* C,
                      long ldc, int c_is_bf16, int M, int N, int K, const float* bias, const float* rs,
                      const float* rc, int relu, int accumulate, int splits, void* stream);

/* Weight-gradient form with the bias gradient folded in (every `dW = dY^T X`, `db = colsum(dY)` pair of the backward
 * pass, e.g. gnn_transformer.py:141-143,158,171-173 under autograd): A = dY read MN-major (A(m,k) = A[k*lda+m]),
 * C[M,N] = A B as above, and d_bias[m] += sum_k A(m,k), accumulated atomically into a zero-filled buffer from the A
 * tiles while they sit in shared memory -- no separate column-sum pass over dY. */
int fira_gemm_bf16_tc_dbias(const void* A, long lda, const void* B, long ldb, int b_kmajor, void* C, long ldc,
                            int c_is_bf16, int M, int N, int K, int accumulate, int splits, float* d_bias, void* stream);

/* Input gradient through a relu (gnn_transformer.py:172 under autograd): dx[m,n] = h[m,n] > 0 ? sum_k dy[m,k] W[k,n] : 0
 * with W the nn.Linear weight [K = out, N = in] as it lies in memory and h the forward activations (bf16, same shape and
 * leading dimension as dx): the relu backward folded into the epilogue of the input-gradient product (bf16 throughput mode). */
int fira_gemm_bf16_tc_dx_relu(const void* dy, long lddy, const void* W, long ldw, void* dx, long lddx, const void* h,
                              int M, int N, int K, void* stream);

/* Debugging aid (tools/gemm_probe.py): with a device buffer of >= 16 uint64 set, CTA (0,0,0) of every following
 * fira_gemm_bf16_tc launch stamps %globaltimer at its phase boundaries (entry, prologue, dependency wait, TMA issued,
 * first stage landed, MMAs issued, accumulator ready, stores issued, exit); NULL switches it off (the default). */
int fira_debug_set_probe(void* probe);

/* ---- embeddings -------------------------------------------------------------------------------
 * Encoder node features in segment-major order (all code rows, all sub-token rows, all AST/edit
 * rows): emb[sou]+PE | emb[sub_token] | ast_emb[ast_change]     (gnn_transformer.py:46-52,58).
 * out_code holds rows [0, B*n_code); out_rest is indexed by the GLOBAL row (rows >= B*n_code). */
int fira_embed_nodes_fwd(const int* sou, const int* sub_token, const int* ast_change, const float* emb,
                         const float* ast_emb, const float* pos_table, void* out_code, void* out_rest, int B,
                         int n_code, int n_sub, int n_ast, int dim, int dtype, void* stream);
/* The same with an explicit position per code row (packed batches, fira_icse_b200/packed.py: `pos` = index of the token
 * inside its commit; B = 1, n_code / n_sub / n_ast = the padded row counts of the three segments). */
int fira_embed_nodes_pos_fwd(const int* sou, const int* pos, const int* sub_token, const int* ast_change,
                             const float* emb, const float* ast_emb, const float* pos_table, void* out_code,
                             void* out_rest, int B, int n_code, int n_sub, int n_ast, int dim, int dtype, void* stream);
/* Zero the segment-padding rows of a packed batch's [Rc + Rs, ld] memory-row matrix (off = its [3][B+1] row offsets). */
int fira_zero_pad_rows(void* x, long ld, int width, const int* off, int B, int Rc, int Rs, int dtype, void* stream);
int fira_embed_nodes_bwd(const int* sou, const int* sub_token, const int* ast_change, const void* d_code,
                         const void* d_rest, float* d_emb, float* d_ast_emb, int B, int n_code, int n_sub, int n_ast,
                         int dim, int dtype, void* stream);
/* Decoder input: dec_emb[tar] + PE[t]  (gnn_transformer.py:110-113). */
int fira_embed_rows_fwd(const int* ids, const float* emb, const float* pos_table, void* out, long rows, int period,
                        int dim, int dtype, void* stream);
int fira_embed_rows_bwd(const int* ids, const void* d_out, float* d_emb, long rows, int dim, int dtype, void* stream);
/* The same with d_out in slots (fira_target_rows): slot r is row rows_map[r] of ids, -1 = none (rows = slots). */
int fira_embed_rows_bwd_rows(const int* ids, const int* rows_map, const void* d_out, float* d_emb, long rows, int dim,
                             int dtype, void* stream);

/* ---- LN(dropout(z) + resid)  (gnn_transformer.py:83,161,174,205) -------------------------------
 * rows < split are written to outA[row], the others to outB[row] (lets a GCN layer hand its code
 * rows to the next Combination without a torch.cat / slice copy). */
int fira_ln_residual_fwd(const void* z, const void* resid, const float* gamma, const float* beta, void* outA,
                         void* outB, long split, float* mean, float* rstd, long rows, int dim, float p_drop,
                         uint64_t seed, const uint64_t* seed_ctr, uint32_t stream_id, int dtype, void* stream);
int fira_ln_residual_bwd(const void* d_outA, const void* d_outB, long split, const void* z, const void* resid,
                         const float* mean, const float* rstd, const float* gamma, void* d_z, void* d_resid,
                         int d_resid_accum, float* d_gamma, float* d_beta, long rows, int dim, float p_drop,
                         uint64_t seed, const uint64_t* seed_ctr, uint32_t stream_id, int dtype, void* stream);
/* The same over slots (fira_target_rows): the dropout mask of slot r is the one drawn for row rows_map[r]; a slot with
 * rows_map[r] < 0 writes zeros to d_z (and d_resid unless d_resid_accum) and adds nothing to d_gamma / d_beta.
 * rows_map NULL: fira_ln_residual_bwd. */
int fira_ln_residual_bwd_rows(const void* d_outA, const void* d_outB, long split, const void* z, const void* resid,
                              const float* mean, const float* rstd, const float* gamma, void* d_z, void* d_resid,
                              int d_resid_accum, float* d_gamma, float* d_beta, const int* rows_map, long rows, int dim,
                              float p_drop, uint64_t seed, const uint64_t* seed_ctr, uint32_t stream_id, int dtype,
                              void* stream);

/* ---- Combination gate (combination_layer.py:7-17): c = v + sigmoid(q*(k-v)/sqrt(d_head))*(k-v),
 *      dropout; qk = [q | k] per row, v = vtab[mark[row]] (4 x dim table = Linear(mark_embedding)). */
int fira_comb_gate_fwd(const void* qk, long ld_qk, const float* vtab, const int* mark, void* out, long rows, int dim,
                       int d_head, float p_drop, uint64_t seed, const uint64_t* seed_ctr, uint32_t stream_id, int dtype, void* stream);
int fira_comb_gate_bwd(const void* qk, long ld_qk, const float* vtab, const int* mark, const void* d_out, void* d_qk,
                       float* d_vtab, long rows, int dim, int d_head, float p_drop, uint64_t seed, const uint64_t* seed_ctr,
                       uint32_t stream_id, int dtype, void* stream);

/* The same gate with an arbitrary per-row `value` tensor (the stand-alone Combination.forward(query, key, value) /
 * CombinationLayer.forward of gnn_transformer.py:192-205, combination_layer.py:7-17): q, k, v, out are [rows, dim]. */
int fira_comb_gate3_fwd(const void* q, const void* k, const void* v, void* out, long rows, int dim, int d_head,
                        float p_drop, uint64_t seed, const uint64_t* seed_ctr, uint32_t stream_id, int dtype, void* stream);
int fira_comb_gate3_bwd(const void* q, const void* k, const void* v, const void* d_out, void* d_q, void* d_k, void* d_v,
                        long rows, int dim, int d_head, float p_drop, uint64_t seed, const uint64_t* seed_ctr,
                        uint32_t stream_id, int dtype, void* stream);

/* d[i] = h[i] > 0 ? d[i] : 0  (backward of the FeedForward relu, gnn_transformer.py:172). */
int fira_relu_bwd(const void* h, void* d, long n, int dtype, void* stream);
/* out[n] += sum_m w[m] * x[m,n]  (w == NULL -> 1): bias gradients. */
int fira_colsum(const void* x, long ld, long M, int N, const float* row_weight, float* out, int dtype, void* stream);

/* ---- optimizer step (run_model.py:101-109: `optimizer.step()` of torch.optim.Adam(lr), no weight decay / amsgrad) over
 *      ONE flat fp32 parameter buffer (fira_icse_b200/optim.py re-homes the model's parameters in it), one launch:
 *        g' = g / *grad_scale (grad_scale NULL -> 1);  m = b1 m + (1-b1) g';  v = b2 v + (1-b2) g'^2;
 *        p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps),  t = *step (device fp32 scalar, the caller has
 *        already incremented it);  p_bf16 (may be NULL) receives the bf16 copy of the updated parameters (the GEMM
 *        operands of the throughput mode).  n: multiple of 8; all buffers 16-byte aligned. */
int fira_adam_flat(float* p, const float* g, float* m, float* v, void* p_bf16, long n, float lr, float beta1, float beta2,
                   float eps, const float* step, const float* grad_scale, void* stream);
/* y = bf16(x), n a multiple of 8 (refresh of the bf16 parameter mirror after parameters were set from outside). */
int fira_cast_bf16(const float* x, void* y, long n, void* stream);

/* memory = cat(code rows, sub-token rows) per commit (Model.py:48) and its adjoint. */
int fira_pack_memory(const void* code, const void* rest, void* mem, int B, int n_code, int n_sub, int dim, int dtype,
                     void* stream);
int fira_unpack_memory(const void* d_mem, void* d_code, void* d_rest, int B, int n_code, int n_sub, int n_ast, int dim,
                       int dtype, void* stream);

/* ---- graph: dense [B,N,N] adjacency (Dataset.py:340 toarray(), any strides) -> packed CSR.
 * Two calls because the caller owns the buffers: count (+ exclusive scan into rowptr[B*N+1]),
 * read rowptr[B*N] to size col/val, then fill. */
int fira_csr_count_dense(const void* edge, int edge_dtype, long stride_b, long stride_i, long stride_j, int B, int N,
                         int* counts, int* rowptr, void* stream);
int fira_csr_fill_dense(const void* edge, int edge_dtype, long stride_b, long stride_i, long stride_j, int B, int N,
                        const int* rowptr, int* col, float* val, void* stream);
int fira_csr_rowsum(const int* rowptr, const float* val, int B, int n_code, int n_sub, int n_ast, float* out,
                    void* stream);
/* The GNN scatter: y = A x (+ addend), replacing torch.bmm(edge.float(), x) (gnn_transformer.py:80). */
int fira_gcn_aggregate(const int* rowptr, const int* col, const float* val, const void* x, const void* addend,
                       void* y, int B, int n_code, int n_sub, int n_ast, int dim, int dtype, void* stream);

/* ---- fused GCN layer, bf16 throughput mode (gnn_transformer.py:74-86 as ONE kernel per direction): gather the
 *      neighbour rows into the shared-memory A tile -> wgmma with the merged weight -> epilogue on the register accumulators.
 *      The CSR is in BUFFER order: rowptr_rows[r] indexes the rows of the node buffer, col_rows are buffer rows
 *      (fira_csr_to_rows converts the (graph, node)-ordered CSR; counts is an int32[rows] workspace).
 *   fwd:  z = (A h) w_merged^T + rowsum(A) (x) c1 + bias ;  out = LN(dropout(z) + h)   (w_merged = fc2.W fc1.W [out,in]
 *         bf16, c1 = fc2.W fc1.b, bias = fc2.b; rows < split -> outA[row], the others -> outB[row]; mean/rstd for
 *         fira_ln_residual_bwd; the dropout mask is the one fira_ln_residual_fwd/bwd draw for (seed, stream_id)).
 *   bwd:  agg_dz = A^T dz (kept: d(w_merged) = agg_dz^T h, d(c1) = colsum(agg_dz)) ;  d_h = agg_dz w_merged + d_resid
 *         (w_merged_t = w_merged^T as a row-major [in,out] bf16 matrix; rowptr/col/val of A^T, = A when symmetric). */
int fira_csr_to_rows(const int* rowptr, const int* col, const float* val, int B, int n_code, int n_sub, int n_ast,
                     int* counts, int* rowptr_rows, int* col_rows, float* val_rows, void* stream);
int fira_gcn_layer_fwd(const int* rowptr_rows, const int* col_rows, const float* val_rows, const void* h,
                       const void* w_merged, const float* bias, const float* c1, const float* gamma, const float* beta,
                       void* z, void* outA, void* outB, long split, float* mean, float* rstd, long rows, int dim,
                       float p_drop, uint64_t seed, const uint64_t* seed_ctr, uint32_t stream_id, void* stream);
int fira_gcn_layer_bwd(const int* rowptr_rows_t, const int* col_rows_t, const float* val_rows_t, const void* d_z,
                       const void* w_merged_t, const void* d_resid, void* agg_dz, void* d_h, long rows, int dim,
                       void* stream);

/* ---- attention core (gnn_transformer.py:144-156); stats = (row max, row sum) [B,H,Lq,2];
 *      backward also takes the forward output `ctx` (same layout as d_ctx): delta = dO . O. */
int fira_attn_fwd(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                  const unsigned char* key_mask, int causal, void* ctx, long ldo, float* stats, int B, int H, int Lq,
                  int Lk, int d_head, int dtype, void* stream);
int fira_attn_bwd(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv,
                  const unsigned char* key_mask, int causal, const void* ctx, const void* d_ctx, long ldo,
                  const float* stats, void* dq, long lddq, void* dk, long lddk, void* dv, long lddv, int B, int H,
                  int Lq, int Lk, int d_head, int dtype, void* stream);

/* Cross-attention of a PACKED batch (fira_icse_b200/packed.py): the keys / values of commit b are two row ranges of
 * k / v, ranges[b] = {first row, rows, first row, rows} (code rows, sub-token rows; GLOBAL row ids, kv_rows = rows of
 * k / v), key_mask [B, mask_pitch] over the commit's own key positions (NULL: all valid), mask_pitch >= rows of any
 * commit; max_chunks is not used (any number of keys per commit is supported).  Rows of dk / dv outside every range
 * are not written (fira_zero_pad_rows clears the segment padding).  Results equal fira_attn_fwd / _bwd bit for bit on
 * the same keys laid out padded (mask 0 beyond the commit's rows), except for a commit without a valid key: it attends
 * uniformly over its own rows, the padded entry points over all Lk positions. */
int fira_attn_packed_fwd(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv, const int* ranges,
                         long kv_rows, const unsigned char* key_mask, int mask_pitch, int max_chunks, void* ctx, long ldo,
                         float* stats, int B, int H, int Lq, int d_head, int dtype, void* stream);
int fira_attn_packed_bwd(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv, const int* ranges,
                         long kv_rows, const unsigned char* key_mask, int mask_pitch, int max_chunks, const void* ctx,
                         const void* d_ctx, long ldo, const float* stats, void* dq, long lddq, void* dk, long lddk,
                         void* dv, long lddv, int B, int H, int Lq, int d_head, int dtype, void* stream);
/* Backward over per-commit query-row ranges (bf16 only): the query rows of commit b (q, ctx, d_ctx, dq) are rows
 * qoff[b] .. qoff[b+1] - 1 (at most Lq; stats keep the [B,H,Lq,2] layout, rows past the count unread); dq has `rows`
 * rows, and its pad rows qoff[B] .. rows - 1 are zeroed (causal: those of dk / dv too).  Keys as
 * fira_attn_packed_bwd (ranges != NULL) or fira_attn_bwd (key_mask [B, mask_pitch], rows b*mask_pitch + s); causal
 * (self-attention, ranges NULL, mask_pitch = Lq): the keys are the commit's query rows, masked by its first key_mask
 * bytes.  A commit without query rows writes zero gradients to its keys (causal: it has none). */
int fira_attn_bwd_rows(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv, const int* ranges,
                       const unsigned char* key_mask, int mask_pitch, int causal, const int* qoff, long rows,
                       const void* ctx, const void* d_ctx, long ldo, const float* stats, void* dq, long lddq, void* dk,
                       long lddk, void* dv, long lddv, int B, int H, int Lq, int d_head, int dtype, void* stream);

/* ---- the whole decoder forward, bf16 throughput mode (gnn_transformer.py:108-122), ONE launch of B two-CTA clusters: embedding +
 *      PE, then L x [causal self-attention over tar_mask [B,T], cross-attention, feed-forward], each closed by
 *      LN(dropout(z) + resid).  T <= 32, 8 heads of 32, D = 256, FFN width 1024.
 *   kv        [Ms, ldkv] bf16: layer i's cross-attention K at column 512 i, V at 512 i + 256 (the hoisted K/V product);
 *             keys of commit b as fira_attn_fwd (mem_mask [B,S], rows b*S + s; ranges NULL) or fira_attn_packed_fwd
 *             (ranges [B][4], mem_mask [B,S] over the commit's key positions or NULL)
 *   layer_ptrs HOST array [L][18] of device pointers, per layer: Wqkv (bf16 [768,256]), bqkv, Wo, bo, ln w, ln b of the
 *             self-attention; Wq, bq, Wo, bo, ln w, ln b of the cross-attention; W1 (bf16 [1024,256]), b1, W2 (bf16
 *             [256,1024]), b2, ln w, ln b of the feed-forward (weights bf16 [out,in], the rest fp32; copied into the
 *             launch's parameters)
 *   outputs   (bf16 unless noted, rows b*T + t, t >= T never written): X [L+1][B*T,256] (each layer's input, then the
 *             output); per layer i (leading dimension L): qkv [B*T,768], ctx1, z1, x1, q, ctx2, z2, x2 [B*T,256],
 *             hh [B*T,1024], z3 [B*T,256]; st1 / st2 fp32 [B,8,T,2] (fira_attn_fwd's statistics); ls1 / ls2 / ls3 fp32
 *             [2][B*T] (mean, rstd).  Products are rounded to bf16 once from fp32 + bias, as fira_gemm_bf16_tc;
 *             LayerNorm and its dropout masks are fira_ln_residual_fwd's on the stored z, site i of stream_id being
 *             stream_id + 8 i + {0, 1, 2}. */
int fira_decoder_fwd(const int* tar, const float* dec_emb, const float* pos_table, const unsigned char* tar_mask,
                     const void* kv, long ldkv, const unsigned char* mem_mask, const int* ranges, int S,
                     const void* const* layer_ptrs, int L, void* X, void* qkv, void* ctx1, float* st1, void* z1,
                     float* ls1, void* x1, void* q, void* ctx2, float* st2, void* z2, float* ls2, void* x2, void* hh,
                     void* z3, float* ls3, int B, int T, float p_drop, uint64_t seed, const uint64_t* seed_ctr,
                     uint32_t stream_id, void* stream);
/* The same with a live-row map (fira_target_rows; tlen and toff both NULL: slot = row b*T + t, R = B*T, which is
 * fira_decoder_fwd with out = X + L*B*T*256).  X [L][R,256] holds each layer's input and every per-layer output
 * above has R slot rows: row t < toff[b+1] - toff[b] of commit b in slot toff[b] + t, the slots from toff[B] on zero;
 * st1 / st2 and the dropout masks keep the rows b*T + t.  out [B*T,256] is the last layer's output: rows t >= tlen[b]
 * zero, a live row without a slot NaN.  Every row is computed as without the map, so the live rows' values are the
 * same. */
int fira_decoder_fwd_rows(const int* tar, const float* dec_emb, const float* pos_table, const unsigned char* tar_mask,
                          const void* kv, long ldkv, const unsigned char* mem_mask, const int* ranges, int S,
                          const void* const* layer_ptrs, int L, void* X, void* out, void* qkv, void* ctx1, float* st1,
                          void* z1, float* ls1, void* x1, void* q, void* ctx2, float* st2, void* z2, float* ls2,
                          void* x2, void* hh, void* z3, float* ls3, const int* tlen, const int* toff, long R, int B,
                          int T, float p_drop, uint64_t seed, const uint64_t* seed_ctr, uint32_t stream_id,
                          void* stream);

/* ---- CopyNet scores (Model.py:17-18): sc[b,t,s] = b_res + w_res . tanh(src[b,s] + tgt[b,t]).
 *      src_mask [B,S] / row_mask [B*T] (optional, 1 = compute): positions the caller will mask anyway. */
int fira_copy_scores_fwd(const void* src_proj, const void* tgt_proj, const float* w_res, const float* b_res,
                         const unsigned char* src_mask, const unsigned char* row_mask, float* scores,
                         int B, int T_len, int S, int dim, int dtype, void* stream);
int fira_copy_scores_bwd(const void* src_proj, const void* tgt_proj, const float* w_res, const float* d_scores,
                         const unsigned char* row_active, void* d_src_proj, float* d_tgt_proj, float* d_w_res,
                         float* d_b_res, int B, int T_len, int S, int dim, int dtype, void* stream);

/* The same for a PACKED batch: the source rows of commit b are the two row ranges ranges[b] of src_proj (global rows);
 * scores stay [B, T, S] over the commit's own memory positions (S = mask pitch); d_src_proj rows outside the ranges
 * are not written. */
int fira_copy_scores_packed_fwd(const void* src_proj, const void* tgt_proj, const float* w_res, const float* b_res,
                                const int* ranges, const unsigned char* src_mask, const unsigned char* row_mask,
                                float* scores, int B, int T_len, int S, int dim, int dtype, void* stream);
int fira_copy_scores_packed_bwd(const void* src_proj, const void* tgt_proj, const float* w_res, const float* d_scores,
                                const unsigned char* row_active, const int* ranges, void* d_src_proj, float* d_tgt_proj,
                                float* d_w_res, float* d_b_res, int B, int T_len, int S, int dim, int dtype, void* stream);

/* ---- dual-copy mixture, loss and argmax (Model.py:54-86).  stats: 8 floats per row
 *      (vmax, vsum, cmax, csum, g0, g1, p_label, 0).  argmax_out may be NULL (training).
 *      logits / d_logits: 16-byte aligned, ld_logits a multiple of 8 (rows are read / written 8 elements at a time). */
int fira_pointer_mix_nll_fwd(const void* logits, long ld_logits, const float* copy_scores, const float* gate_logits,
                             const unsigned char* mem_mask, const int* label, float* stats, float* nll,
                             int* argmax_out, long rows, int T_len, int V, int S, int dtype, void* stream);
int fira_pointer_mix_nll_bwd(const void* logits, long ld_logits, const float* copy_scores,
                             const unsigned char* mem_mask, const int* label, const float* stats,
                             const float* upstream, void* d_logits, float* d_copy_scores, float* d_gate_logits,
                             unsigned char* row_active, long rows, int T_len, int V, int S, int dtype, void* stream);

/* ---- training on the vocabulary-label rows only (a row whose label is 0 or a copy label takes nothing from the
 *      vocabulary softmax, Model.py:64-81, so its logits are never needed):
 *   fira_vocab_rows: label [rows] -> vslot [rows] = compact slot of each row with 0 < label < V in row order, else -1;
 *                    vrows [cap] = the row of each slot, -1 in the slots past the count (count <= cap: the caller's
 *                    bound; rows beyond it get no slot, and the _rows loss gives such a row a NaN loss).
 *   fira_gather_rows: dst[i] = idx[i] >= 0 ? src[idx[i]] : 0 for i < n (rows of `width` elements, width, ld_src, ld_dst
 *                    multiples of 8, 16-byte aligned): gathers dec rows by vrows, and scatters the slots' input gradient
 *                    back to the rows by vslot.
 *   _rows twins of the loss kernels: logits / d_logits hold one row per slot (vslot NULL: one per row, as the entry points
 *                    above, which call these).  The forward cannot take argmax_out with vslot.  The backward writes the
 *                    slots of vocabulary-label rows and zero-fills the unused slots s < cap (cap <= rows); rows without
 *                    a slot write no logits gradient. */
int fira_vocab_rows(const int* label, long rows, int V, int* vslot, int* vrows, int cap, void* stream);
/* ---- the live target rows of a training batch: the rows before each commit's last non-zero shifted label (no later row
 *      carries a loss, and causal self-attention never lets an earlier row read one).  label [B,T] ->
 *      tlen [B] = 1 + the last t with label != 0 (0 without one); toff [B+1] = each commit's first slot, slots in row
 *      order; trows [cap] = b*T + t of each slot, -1 past the count.  B <= 1024.  A count above cap (the caller's bound)
 *      leaves the commits past it short of slots (toff clamps to cap): fira_decoder_fwd_rows gives those rows NaN. */
int fira_target_rows(const int* label, int B, int T, int* tlen, int* toff, int* trows, int cap, void* stream);
int fira_gather_rows(const void* src, long ld_src, const int* idx, void* dst, long ld_dst, long n, int width, int dtype,
                     void* stream);
int fira_pointer_mix_nll_fwd_rows(const void* logits, long ld_logits, const float* copy_scores, const float* gate_logits,
                                  const unsigned char* mem_mask, const int* label, const int* vslot, float* stats,
                                  float* nll, int* argmax_out, long rows, int T_len, int V, int S, int dtype,
                                  void* stream);
int fira_pointer_mix_nll_bwd_rows(const void* logits, long ld_logits, const float* copy_scores,
                                  const unsigned char* mem_mask, const int* label, const int* vslot, const int* vrows,
                                  int cap, const float* stats, const float* upstream, void* d_logits,
                                  float* d_copy_scores, float* d_gate_logits, unsigned char* row_active, long rows,
                                  int T_len, int V, int S, int dtype, void* stream);
/* Sequence-weighted backward (self-critical training, fira_icse_b200/scst.py): fira_pointer_mix_nll_bwd_rows for
 *      loss_sum = sum_row seq_weight[row / T_len] * nll[row], seq_weight [rows / T_len] fp32 (device, not NULL): row
 *      `row` takes upstream *upstream * seq_weight[row / T_len].  A row whose weight is exactly 0 is treated as a
 *      label-0 row: no gradient, row_active 0 (the copy-score backward skips it).  Weights of 1.0 give bit for bit the
 *      results of fira_pointer_mix_nll_bwd_rows. */
int fira_pointer_mix_nll_bwd_rows_weighted(const void* logits, long ld_logits, const float* copy_scores,
                                           const unsigned char* mem_mask, const int* label, const int* vslot,
                                           const int* vrows, int cap, const float* stats, const float* upstream,
                                           void* d_logits, float* d_copy_scores, float* d_gate_logits,
                                           unsigned char* row_active, long rows, int T_len, int V, int S, int dtype,
                                           void* stream, const float* seq_weight);

/* ---- one seeded sampling step from the same mixture (fira_icse_b200/sample.py).  Rows are (commit b, sample n),
 *      B*N of them: logits [B*N, ld_logits], copy_scores [B, N, S], gate_logits [B*N, 2], mem_mask / copy_src [B, S]
 *      (copy_src: the vocabulary id behind each memory position).  Candidates: vocabulary entries and unmasked copy
 *      positions whose mixture probability P_j is > 0 in fp32; s_j = log P_j / temperature, ranked by s descending then
 *      index ascending; top_k > 0 keeps the first top_k ranks; top_p < 1 then keeps the shortest rank prefix whose
 *      weight sum(exp(s_j - max s)) reaches top_p times the kept weight; the draw picks the smallest kept index whose
 *      running weight in index order exceeds u * (total kept weight).  u in [0, 1): uniforms[row] when uniforms is
 *      not NULL, else 24 bits of Philox4x32-7 keyed by *seed with counter (*first_index + b, n, stream, pos) --
 *      seed / first_index are device scalars, so one captured graph per position serves every batch.
 *      A row not yet finished writes, at column pos + 1 of seq / raw / token_logprob / tok_mask ([B*N, ld_out]):
 *      the next input token (j, or copy_src[b, j - V] for a copy), the raw index j, log(clamp(P_j, 1e-10, 1)) (=
 *      -nll of fira_pointer_mix_nll_fwd for label j), token != pad_id; also next_tok[row] = the token, length[row] += 1,
 *      logprob[row] += the log-probability, finished[row] = 1 on eos_id.  A finished row writes pad_id / 0 and keeps
 *      length and logprob.  V + S <= 32767; temperature > 0, top_k >= 0, 0 < top_p <= 1. */
int fira_pointer_mix_sample(const void* logits, long ld_logits, const float* copy_scores, const float* gate_logits,
                            const unsigned char* mem_mask, const int* copy_src, const uint64_t* seed,
                            const int* first_index, const float* uniforms, float temperature, int top_k, float top_p,
                            int eos_id, int pad_id, int* next_tok, int* seq, int* raw, float* token_logprob,
                            unsigned char* tok_mask, long ld_out, int pos, unsigned char* finished, int* length,
                            float* logprob, int B, int N, int V, int S, int dtype, void* stream);

/* ---- one n-best beam step from the same mixture (fira_icse_b200/beam.py nbest).  Rows are (commit b, slot k), B*K
 *      of them: logits [B*K, ld_logits], copy_scores [B, K, S], gate_logits [B*K, 2], mem_mask / copy_src [B, S].
 *      Slot state is double-buffered: seq / raw / token_logprob [2, B*K, T_len], length / logprob / score / status
 *      [2, B*K]; position `pos` reads half pos & 1 and writes half 1 - (pos & 1) (a slot's new history comes from
 *      another row).  status: 0 live, 1 finished, 2 inactive (slots 1..K-1 before position 0).  length counts <start>.
 *      Rule: lp_j = log(clamp(P_j, 1e-10, 1)) (= -nll of fira_pointer_mix_nll_fwd for label j) for every vocabulary
 *      entry and every unmasked copy position; a live slot i proposes (i, j) with L = logprob_i + lp_j (fp32) and
 *      n = length_i tokens generated, a finished slot proposes itself once as j = C = V + S, an inactive slot nothing;
 *      score = L / powf((5 + n) / 6, length_penalty); the K best by (score descending, then i * (C + 1) + j
 *      ascending) become slots 0..K-1 in that order.  Two launches: per live row its top K (lp, j) into workspace
 *      [B*K, K] (uint64 rank keys, caller-owned), then per commit the merge.  A grown slot writes its parent's history
 *      with column pos + 1 = (token, j, lp_j) (token = j, or copy_src[b, j - V] for a copy), length + 1, logprob L,
 *      its score, status 1 on eos_id; a carried finished slot copies its state unchanged.  Every slot writes
 *      parent[b*K + k] = b*K + i (int64, for the caller's cache reorder) and next_tok[b*K + k] = its token (pad_id
 *      when carried).  1 <= K <= 16, K <= V, V + S <= 32767, length_penalty >= 0, 0 <= pos <= T_len - 2. */
int fira_pointer_mix_beam_step(const void* logits, long ld_logits, const float* copy_scores, const float* gate_logits,
                               const unsigned char* mem_mask, const int* copy_src, float length_penalty, int eos_id,
                               int pad_id, uint64_t* workspace, int* seq, int* raw, float* token_logprob, int* length,
                               float* logprob, float* score, unsigned char* status, long* parent, int* next_tok,
                               int T_len, int pos, int B, int K, int V, int S, int dtype, void* stream);

/* ---- one diverse n-best beam step (fira_icse_b200/beam.py nbest with groups > 1).  Arguments and slot state as
 *      fira_pointer_mix_beam_step, plus `groups` G (G divides K, Kg = K / G), `diversity` lambda, chosen [B*K] int32
 *      and lp_workspace [B*K, Kg] fp32 (caller-owned, like workspace [B*K, Kg]).  Group g owns slots
 *      g*Kg .. (g+1)*Kg - 1 (the caller starts slot g*Kg of every group live, the others inactive).  Rule: the groups
 *      choose in order g = 0 .. G-1; h_g(w) = the number of slots of groups 0..g-1 that grew at this position with
 *      token w (the token of j is j, or copy_src[b, j - V] for a copy; <eos> counts like any word, a carried slot
 *      counts nothing).  Only group g's slots propose, with the candidates of fira_pointer_mix_beam_step: a live slot
 *      i proposes (i, j) with score = (logprob_i + lp_j) / powf((5 + length_i) / 6, length_penalty) and rank value
 *      score - diversity * h_g(token of j); a finished slot proposes itself once with its stored score as rank value.
 *      The Kg best by (rank value descending, then i * (C + 1) + j ascending, i the slot index within the commit)
 *      become slots g*Kg + 0 .. Kg-1 in that order, their parents inside the group; chosen[b*K + g*Kg + k] = the
 *      token the new slot grew with, -1 when carried.  The penalty is never stored: length, logprob, score,
 *      token_logprob, parent and next_tok are written as fira_pointer_mix_beam_step writes them.  2G launches on
 *      `stream` (per group its row stage, then its merge); both rank by the same fp32 value (correctly rounded
 *      operations), so the row stage's prefilter to each row's Kg best is exact.  1 <= G <= K, K % G == 0,
 *      diversity finite and >= 0, and the bounds of fira_pointer_mix_beam_step. */
int fira_pointer_mix_diverse_beam_step(const void* logits, long ld_logits, const float* copy_scores,
                                       const float* gate_logits, const unsigned char* mem_mask, const int* copy_src,
                                       float length_penalty, int eos_id, int pad_id, uint64_t* workspace, int* seq,
                                       int* raw, float* token_logprob, int* length, float* logprob, float* score,
                                       unsigned char* status, long* parent, int* next_tok, int T_len, int pos, int B,
                                       int K, int V, int S, int groups, float diversity, int* chosen,
                                       float* lp_workspace, int dtype, void* stream);

/* ---- the three steps above with forced positions (a prefix per commit; fira_icse_b200 `prefix=`, sample.score).
 *      Arguments as the step without the suffix, plus prefix [B, ld_prefix] int32 and prefix_len [B] int32 (device;
 *      prefix NULL = nothing forced, the step without the suffix).  Rule: a live row of commit b (not finished; for the
 *      beam steps status 0) is forced at position pos iff pos < prefix_len[b]; its label is then
 *      j = prefix[b * ld_prefix + pos] in the label encoding of the training loss (j < V a vocabulary id, V + s memory
 *      position s) and its lp = log(clamp(P_j, 1e-10, 1)) is formed with the same expressions, bit for bit -nll of
 *      fira_pointer_mix_nll_fwd for label j.  The sampler's forced row skips the candidate, top-k, top-p and draw
 *      passes and writes what a drawn j writes (token, raw, lp, mask, length, logprob, finished on eos_id); the Philox
 *      counter of a later free position is (first_index + b, n, pos) as without a prefix.  A forced row of a beam step
 *      emits exactly one row winner, (lp, j) (the diverse step: with its rank value and row lp), every other entry
 *      empty; the select stages are unchanged.  n-best starts with slot 0 (each group's first slot) alone live, so a
 *      forced commit grows that slot with j, its parent itself, while the other slots stay inactive; the search
 *      branches at the commit's first free position.  The caller keeps every label < V + S with its copy position
 *      unmasked, and prefix_len[b] <= ld_prefix; pos < ld_prefix. */
int fira_pointer_mix_sample_prefix(const void* logits, long ld_logits, const float* copy_scores,
                                   const float* gate_logits, const unsigned char* mem_mask, const int* copy_src,
                                   const uint64_t* seed, const int* first_index, const float* uniforms,
                                   float temperature, int top_k, float top_p, int eos_id, int pad_id, int* next_tok,
                                   int* seq, int* raw, float* token_logprob, unsigned char* tok_mask, long ld_out,
                                   int pos, unsigned char* finished, int* length, float* logprob, int B, int N, int V,
                                   int S, int dtype, void* stream, const int* prefix, int ld_prefix,
                                   const int* prefix_len);
int fira_pointer_mix_beam_step_prefix(const void* logits, long ld_logits, const float* copy_scores,
                                      const float* gate_logits, const unsigned char* mem_mask, const int* copy_src,
                                      float length_penalty, int eos_id, int pad_id, uint64_t* workspace, int* seq,
                                      int* raw, float* token_logprob, int* length, float* logprob, float* score,
                                      unsigned char* status, long* parent, int* next_tok, int T_len, int pos, int B,
                                      int K, int V, int S, int dtype, void* stream, const int* prefix, int ld_prefix,
                                      const int* prefix_len);
int fira_pointer_mix_diverse_beam_step_prefix(const void* logits, long ld_logits, const float* copy_scores,
                                              const float* gate_logits, const unsigned char* mem_mask,
                                              const int* copy_src, float length_penalty, int eos_id, int pad_id,
                                              uint64_t* workspace, int* seq, int* raw, float* token_logprob,
                                              int* length, float* logprob, float* score, unsigned char* status,
                                              long* parent, int* next_tok, int T_len, int pos, int B, int K, int V,
                                              int S, int groups, float diversity, int* chosen, float* lp_workspace,
                                              int dtype, void* stream, const int* prefix, int ld_prefix,
                                              const int* prefix_len);

/* ---- the three _prefix steps with n-gram repeat blocking and a minimum message length (fira_icse_b200
 *      `no_repeat_ngram=`, `min_length=`).  Arguments as the _prefix step (prefix may be NULL), plus no_repeat_ngram
 *      n >= 0 and min_length m >= 0 (0 = off; both 0 = the _prefix step, bit for bit).  Rule: the words of a live,
 *      non-forced row at position pos are its seq ids in columns 1..pos (a copy is its word copy_src[b, j - V]; forced
 *      prefix words count); the sampler reads its own seq row, the beam steps the read half.  Label j with word w is
 *      banned at column pos + 1 if, with n >= 1, some i >= 1 with i + n - 1 <= pos has words[i .. i+n-2] ==
 *      words[pos-n+2 .. pos] and words[i+n-1] == w (n = 1: no word twice), or if w == eos_id and pos < m (fewer than m
 *      words).  A banned label is not a candidate: the sampler drops it before the top-k / top-p cuts (nothing is
 *      renormalised, the Philox counter is unchanged), the beam row stages never offer it to their top K (a row with
 *      fewer allowed entries proposes fewer); the select stages and every emitted lp are unchanged.  Forced rows are
 *      exempt.  With a rule on: T_len <= 32 (the sampler: ld_out <= 32). */
int fira_pointer_mix_sample_rules(const void* logits, long ld_logits, const float* copy_scores,
                                  const float* gate_logits, const unsigned char* mem_mask, const int* copy_src,
                                  const uint64_t* seed, const int* first_index, const float* uniforms,
                                  float temperature, int top_k, float top_p, int eos_id, int pad_id, int* next_tok,
                                  int* seq, int* raw, float* token_logprob, unsigned char* tok_mask, long ld_out,
                                  int pos, unsigned char* finished, int* length, float* logprob, int B, int N, int V,
                                  int S, int dtype, void* stream, const int* prefix, int ld_prefix,
                                  const int* prefix_len, int no_repeat_ngram, int min_length);
int fira_pointer_mix_beam_step_rules(const void* logits, long ld_logits, const float* copy_scores,
                                     const float* gate_logits, const unsigned char* mem_mask, const int* copy_src,
                                     float length_penalty, int eos_id, int pad_id, uint64_t* workspace, int* seq,
                                     int* raw, float* token_logprob, int* length, float* logprob, float* score,
                                     unsigned char* status, long* parent, int* next_tok, int T_len, int pos, int B,
                                     int K, int V, int S, int dtype, void* stream, const int* prefix, int ld_prefix,
                                     const int* prefix_len, int no_repeat_ngram, int min_length);
int fira_pointer_mix_diverse_beam_step_rules(const void* logits, long ld_logits, const float* copy_scores,
                                             const float* gate_logits, const unsigned char* mem_mask,
                                             const int* copy_src, float length_penalty, int eos_id, int pad_id,
                                             uint64_t* workspace, int* seq, int* raw, float* token_logprob,
                                             int* length, float* logprob, float* score, unsigned char* status,
                                             long* parent, int* next_tok, int T_len, int pos, int B, int K, int V,
                                             int S, int groups, float diversity, int* chosen, float* lp_workspace,
                                             int dtype, void* stream, const int* prefix, int ld_prefix,
                                             const int* prefix_len, int no_repeat_ngram, int min_length);

/* ---- lexically constrained n-best (fira_icse_b200.beam.nbest `constraints=`; dynamic beam allocation, Post & Vilar,
 *      2018).  Arguments as the n-best _rules step, with workspace [B*K, K+4] keys (not [B*K, K]), plus constraints
 *      int32 [B, 4, 4] on the device: commit b's phrases of up to 4 vocabulary ids, 0 = padding after a phrase's last
 *      word; Tc = commit b's nonzero entries (<= 16; 0 = no constraints).  The words of a row are its seq ids in columns
 *      1..pos, as for the rules.  Progress of phrase c (length L) on words h: L if c occurs contiguously in h, else the
 *      largest m < L with h ending in c_1..c_m (0 if none); a row meets its constraints when the sum over its phrases
 *      is Tc.  Row stage per live, non-forced row: <eos> is banned while its progress is below Tc (next to the rules);
 *      it proposes (a) its K best allowed labels as the _rules step, and (b) per phrase it has not met, in phrase
 *      order, the best label by (lp, then smaller j) among j = w and the unmasked copies of w, w = the phrase's next
 *      word c_{prog+1}, unless w is banned, an earlier phrase proposed w or the label is in (a).  A forced row proposes
 *      its one label.  Each proposal's bank = the progress of the row's words with its word appended.  Select stage,
 *      L, n and score as the n-best step: with Tc = 0, the K best by (score descending, i * (C + 1) + j ascending),
 *      bit for bit the _rules step; with Tc > 0, the carried finished slots first (best score first), then the live
 *      candidates by (r ascending, bank descending), r = the candidate's rank by (score, index) within its bank.  The
 *      chosen slots become slots 0..K-1 in that order.  Bounds: K <= 16 and T_len <= 32. */
int fira_pointer_mix_beam_step_lexical(const void* logits, long ld_logits, const float* copy_scores,
                                       const float* gate_logits, const unsigned char* mem_mask, const int* copy_src,
                                       float length_penalty, int eos_id, int pad_id, uint64_t* workspace, int* seq,
                                       int* raw, float* token_logprob, int* length, float* logprob, float* score,
                                       unsigned char* status, long* parent, int* next_tok, int T_len, int pos, int B,
                                       int K, int V, int S, int dtype, void* stream, const int* prefix, int ld_prefix,
                                       const int* prefix_len, int no_repeat_ngram, int min_length,
                                       const int* constraints);

/* ---- ensemble decoding (fira_icse_b200/ensemble.py): M <= 8 models' mixtures (Model.py:54-86) averaged into one fp32
 *      triple the three step kernels above read with dtype FIRA_F32.  Member m: logits[m] (`dtype`, [B*N, ld_logits],
 *      16-byte aligned), copy_scores[m] [B, N, S] fp32, gate_logits[m] [B*N, 2] fp32 (host arrays of M device
 *      pointers, copied into the launch); log_weights [M] fp32 device (log w_m, sum w_m = 1; read at run time, so a
 *      captured launch follows new weights); mem_mask [B, S].  With P^m_j = g0^m softmax(x^m)_j (j < V) and
 *      g1^m softmax(masked c^m)_s (j = V + s), and member m's row statistics vmax, vsum, cmax, csum, g0, g1 formed as
 *      its own step kernel forms them, G0 = sum_m w_m g0^m, G1 = sum_m w_m g1^m:
 *        x'_j = LSE over m with w_m g0^m > 0 of [log(w_m g0^m / G0) + x^m_j - vmax^m - log vsum^m]
 *        c'_s = LSE over m with w_m g1^m > 0 of [log(w_m g1^m / G1) + c^m_s - cmax^m - log csum^m]  (masked s: -1e9)
 *        gl'  = (log G0, log G1)
 *      so the step kernels' mixture of (x', c', gl') is P = sum_m w_m P^m up to fp32 rounding.  G0 == 0 (G1 == 0) uses
 *      log w_m as the offsets of x' (c'), and gl'_0 = -inf (gl'_1) makes that gate exactly 0.  Output: logits_out
 *      [B*N, ld_out] fp32 (16-byte aligned, columns >= V untouched), copy_out [B, N, S], gate_out [B*N, 2].  One CTA of
 *      256 threads per row.  1 <= M <= 8, ld_logits and ld_out multiples of 8 and >= V, V + S <= 32767. */
int fira_pointer_mix_ensemble(const void* const* logits, long ld_logits, const float* const* copy_scores,
                              const float* const* gate_logits, int M, const float* log_weights,
                              const unsigned char* mem_mask, float* logits_out, long ld_out, float* copy_out,
                              float* gate_out, int B, int N, int V, int S, int dtype, void* stream);

/* ---- nearest-neighbour decoding (fira_icse_b200/knn.py, knn.cu): exact k-nearest search of a datastore of N 256-wide
 *      bf16 keys, then the mixture of a row's P with its neighbours' words.
 *   knn_search: queries [R, ld_q] (`dtype`, rounded to bf16), keys [N, 256] bf16, norms [N] fp32 (sum of key^2 over
 *      the bf16 values), all 16-byte aligned, ld_q a multiple of 8 and >= 256 -> idx [R, k] int32 and dist [R, k] fp32:
 *      the k entries with the smallest (d_i, i), ascending, d_i = fma(-2, q . key_i, |q|^2 + norm_i) with the bf16
 *      products accumulated in fp32 in a fixed order and |q|^2 in fp32.  Ties in d go to the smaller index.  A row's
 *      output depends only on its query and the datastore (not on R, the other rows or the tiling): graph replays and
 *      repeated runs agree bit for bit.  workspace: 16-byte aligned device memory of workspace_bytes >= 8 k R.  The
 *      keys are split P ways, P = min(SMs / ceil(R / 128), workspace_bytes / (8 k R), ceil(N / 64), 256) (at least
 *      1), one sorted candidate list per (split, row); so 8 k max(R, 128 SMs) bytes always give the full split
 *      (8.7 MB at k = 64 on 132 SMs, for any R up to 16,896).  1 <= k <= 64, k <= N < 2^31.  Two launches: the
 *      mma.sync distance product with the candidate lists in its epilogue, and a merge of the P lists per row.
 *   pointer_mix_knn: the model's triple (logits `dtype` [B*N, ld_logits], copy_scores [B, N, S] fp32, gate_logits
 *      [B*N, 2] fp32), mem_mask [B, S], nb_idx / nb_dist [B*N, k] from knn_search, words [N_store] int32 (the
 *      entries' vocabulary ids), params [2] fp32 device = (lam, tau) (read at run time, so a captured launch follows
 *      new values) -> the fp32 triple (logits_out [B*N, ld_out], copy_out [B, N, S], gate_out [B*N, 2]) whose step
 *      kernel mixture is P'_j = (1 - lam) P_j + lam q_j (j < V), P'_{V+s} = (1 - lam) P_{V+s}, up to fp32 rounding;
 *      q_w = sum over the neighbours with word w of exp(-(d_i - d_1) / tau) / Z.  With P's row statistics from the step
 *      kernels' own expressions, a0 = (1 - lam) g0, a1 = (1 - lam) g1, G0 = a0 + lam:
 *        gl' = (log G0, log a1),  x'_j = log a0 - log G0 + x_j - vmax - log vsum,  c'_s = c_s (masked s: -1e9),
 *        x'_w = LSE(that, log(lam q_w) - log G0) for each neighbour word w.
 *      a0 == 0 in fp32 gives x'_j = -1e9 for every word whose P' is 0 (no neighbour mass, or lam q_w underflowed
 *      to 0); a1 == 0 gives gl'_1 = -inf.  One CTA of 256 threads per row.  1 <= k <= 64, ld_logits / ld_out
 *      multiples of 8 and >= V, V + S <= 32767, 0 < lam < 1, tau > 0 (the caller checks lam and tau). */
int fira_knn_search(const void* queries, long ld_q, int dtype, const void* keys, const float* norms, long N, int R,
                    int k, void* workspace, long workspace_bytes, int* idx, float* dist, void* stream);
int fira_pointer_mix_knn(const void* logits, long ld_logits, const float* copy_scores, const float* gate_logits,
                         const unsigned char* mem_mask, const int* nb_idx, const float* nb_dist, const int* words,
                         int k, const float* params, float* logits_out, long ld_out, float* copy_out, float* gate_out,
                         int B, int N, int V, int S, int dtype, void* stream);

/* ---- knowledge distillation (fira_icse_b200/distill.py): the student's mixture P against a teacher's fp32 triple
 *      (t_logits [rows, ld_t], t_copy_scores [B, T_len, S], t_gate_logits [rows, 2]; fira_pointer_mix_ensemble's output
 *      with N = T_len), whose mixture t is formed by the same expressions.  Student operands as
 *      fira_pointer_mix_nll_fwd.  Row r with shifted label y = label[r] != 0 (a y = 0 row carries no loss and no kernel
 *      reads its logits, copy scores or teacher row):
 *        nll_r  = -log clamp(P_y, 1e-10, 1)                 (fira_pointer_mix_nll_fwd's value; a copy label beyond S: 0)
 *        kd_r   = -sum_{j < V+S} t_j log clamp(P_j, 1e-10, 1)   (a masked copy position has t_j = 0 and adds 0)
 *        loss_r = (1 - alpha) nll_r + alpha kd_r,  0 <= alpha <= 1
 *      Backward with u = *upstream (d(sum_r loss_r)), live_j = (1e-10 <= P_j <= 1), the clamp's pass-through:
 *        a_j = [(1 - alpha) [j == y] + alpha t_j] live_j,  A_V = sum_{j < V} a_j,  A_C = sum_s a_{V+s}
 *        d_logits_k = u (softmax(x)_k A_V - a_k),  d_copy_scores_s = u (softmax(masked c)_s A_C - a_{V+s}) (0 if masked)
 *        d_gate_logits = u ((g0, g1) (A_V + A_C) - (A_V, A_C)),  row_active = (A_C != 0)
 *      With alpha = 0 every output equals fira_pointer_mix_nll_fwd / _bwd's bit for bit.  stats: 16 floats per row
 *      (the student's vmax, vsum, cmax, csum, g0, g1, p_label, 0, the teacher's six, A_V, A_C) from the forward, read by
 *      the backward.  nll / kd / loss [rows]; d_logits dense [rows, ld_logits] (zeros on y = 0 rows).  One CTA of 256
 *      threads per row.  logits, d_logits, t_logits 16-byte aligned, ld_logits and ld_t multiples of 8 and >= V,
 *      V + S <= 32767, alpha in [0, 1]. */
int fira_pointer_mix_kd_fwd(const void* logits, long ld_logits, const float* copy_scores, const float* gate_logits,
                            const unsigned char* mem_mask, const int* label, const float* t_logits, long ld_t,
                            const float* t_copy_scores, const float* t_gate_logits, float alpha, float* stats,
                            float* nll, float* kd, float* loss, long rows, int T_len, int V, int S, int dtype,
                            void* stream);
int fira_pointer_mix_kd_bwd(const void* logits, long ld_logits, const float* copy_scores,
                            const unsigned char* mem_mask, const int* label, const float* t_logits, long ld_t,
                            const float* t_copy_scores, float alpha, const float* stats, const float* upstream,
                            void* d_logits, float* d_copy_scores, float* d_gate_logits, unsigned char* row_active,
                            long rows, int T_len, int V, int S, int dtype, void* stream);

/* ---- offline distillation (fira_icse_b200/distill.py KDTargets): the teacher's top-k labels, stored once, and the
 *      loss against them.
 * fira_pointer_mix_topk: the teacher's fp32 triple as fira_pointer_mix_kd_fwd reads it, mem_mask and the shifted labels.
 *      Row r with label[r] != 0: P = the triple's mixture (the step kernels' expressions); the candidates are every
 *      vocabulary entry and every unmasked copy position with P_j > 0 in fp32; the kept labels are the k candidates with
 *      the largest key (P_j descending, then j ascending; the sampler's 47-bit key taken on P), in key order, in
 *      t_label [rows, k] int32 (j < V a vocabulary id, V + s copy position s).  mass[r] = the kept P_j summed in key
 *      order in fp32, t_prob [rows, k] = P_j / mass.  A row with fewer than k candidates fills the rest with label -1
 *      and probability 0; a label-0 row reads nothing and writes labels -1, probabilities 0 and mass 0.  One CTA of 256
 *      threads per row, (V + S) * 4 bytes of dynamic shared memory; a row's result depends on that row alone.
 *      1 <= k <= 64, t_logits 16-byte aligned, ld_t a multiple of 8 and >= V, V + S <= 32767.
 * fira_pointer_mix_kd_sparse_fwd / _bwd: fira_pointer_mix_kd_fwd / _bwd with the teacher's t replaced by the dense
 *      vector that holds t_prob[r, i] at label t_label[r, i] and 0 elsewhere (entries with label -1 or probability 0
 *      add nothing); the student operands, the outputs, the rule and the argument checks are theirs, plus
 *      1 <= k <= 64.  With alpha = 0 every output equals fira_pointer_mix_nll_fwd / _bwd's bit for bit.  stats: 10
 *      floats per row (the student's vmax, vsum, cmax, csum, g0, g1, p_label, 0, A_V, A_C).  The forward reads the
 *      student row once; the backward writes it once and then rewrites the <= k + 1 columns with a_j != 0. */
int fira_pointer_mix_topk(const float* t_logits, long ld_t, const float* t_copy_scores, const float* t_gate_logits,
                          const unsigned char* mem_mask, const int* label, int k, int* t_label, float* t_prob,
                          float* mass, long rows, int T_len, int V, int S, void* stream);
int fira_pointer_mix_kd_sparse_fwd(const void* logits, long ld_logits, const float* copy_scores,
                                   const float* gate_logits, const unsigned char* mem_mask, const int* label,
                                   const int* t_label, const float* t_prob, int k, float alpha, float* stats,
                                   float* nll, float* kd, float* loss, long rows, int T_len, int V, int S, int dtype,
                                   void* stream);
int fira_pointer_mix_kd_sparse_bwd(const void* logits, long ld_logits, const float* copy_scores,
                                   const unsigned char* mem_mask, const int* label, const int* t_label,
                                   const float* t_prob, int k, float alpha, const float* stats, const float* upstream,
                                   void* d_logits, float* d_copy_scores, float* d_gate_logits,
                                   unsigned char* row_active, long rows, int T_len, int V, int S, int dtype,
                                   void* stream);

/* ---- minimum-Bayes-risk selection among each commit's N samples (fira_icse_b200/mbr.py).  seq [B, N, ld_seq] int32
 *      (row (b, n) at (b*N + n) * ld_seq, columns 0..T_len-1), length [B, N] int32 (counts <start>; clamped to
 *      [1, T_len]).  Rule:
 *        words_n   = seq[b, n, 1:length[b, n]] without every id equal to start_id, eos_id or pad_id
 *        BLEU(i,j) = bleu.sentence_bleu_method2([words_j], words_i) over the ids, in float64: clipped n-gram matches,
 *                    n = 1..4; denominator max(1, c - n + 1) (c = len(words_i)), +1 on numerator and denominator for
 *                    n >= 2; 0 for c = 0 or no unigram match; BP = 1 if c > r else exp(1 - r / c), r = len(words_j)
 *        U_i       = (sum over j != i, j ascending, of BLEU(i, j)) / (N - 1)      (fixed order, no atomics)
 *        best[b]   = the smallest i with the largest U_i
 *      utility [B, N] float64; pair_bleu [B, N, N] float64 (pair_bleu[b, i, j] = BLEU(i, j), diagonal included) or
 *      NULL.  2 <= N <= 32, 2 <= T_len <= 32, ld_seq >= T_len, B >= 0 (B = 0: nothing is launched). */
int fira_mbr_select(const int* seq, const int* length, long ld_seq, int start_id, int eos_id, int pad_id,
                    double* pair_bleu, double* utility, int* best, int B, int N, int T_len, void* stream);

/* ---- self-critical rewards (fira_icse_b200/scst.py): each of a commit's N samples scored against its reference.
 *      seq / length as fira_mbr_select; ref [B, ld_ref] int32, the commit's target ids (<start> first).  Rule:
 *        words_n   = as fira_mbr_select
 *        ref_b     = ref[b, 1:e] without start_id / pad_id ids, e = the first column >= 1 holding eos_id (T_len if none)
 *        reward    = bleu.sentence_bleu_method2([ref_b], words_n) over the ids, in float64 (the BLEU of fira_mbr_select
 *                    with r = len(ref_b))
 *        advantage = (sum over m != n, m ascending, of (reward[b, n] - reward[b, m])) / (N - 1)
 *                    (reward minus the mean of the other samples' rewards, written so that tied rewards give exactly 0)
 *      reward, advantage [B, N] float64.  One CTA per commit, one warp per sample.  2 <= N <= 32, 2 <= T_len <= 32,
 *      ld_seq >= T_len, ld_ref >= T_len, B >= 0 (B = 0: nothing is launched). */
int fira_bleu_reward(const int* seq, const int* length, long ld_seq, const int* ref, long ld_ref, int start_id,
                     int eos_id, int pad_id, double* reward, double* advantage, int B, int N, int T_len, void* stream);

/* ---- HOST-side batch preparation (CPU only: every pointer below is HOST memory, there is no stream).
 *
 * fira_host_build_adjacency: the commit graph of Dataset.py:220-294 + process_edge (Dataset.py:346-357).
 *   Relations are int32 pair lists [n,2] exactly as stored in DataSet/edge_*.json: (edit c, code j),
 *   (edit c, AST a), (AST a, code j), (AST a, AST b); code_sub = (code j, sub-token k) pairs
 *   (Dataset.py:173-192, 255-259); n_diff = diff tokens before padding (the sequential chain covers
 *   <start> t1..tn <eos>, Dataset.py:263-266); n_ast = AST nodes (edit nodes follow them).
 *   Node ids: code j -> j+1, sub-token k -> diff_len+k, AST a -> diff_len+sub_len+a, edit c -> ...+n_ast+c;
 *   pairs whose code id reaches diff_len are dropped (Dataset.py:228,243).  Output: undirected,
 *   de-duplicated, self loop on every node, in CSR order: deg[n_nodes], col[nnz], val[nnz] =
 *   1/sqrt(deg_row)/sqrt(deg_col) in float64 (Dataset.py:277-291).  *nnz_out is set even when cap is
 *   too small (FIRA_ERR_SHAPE).
 *
 * fira_host_batch_dims: segment lengths a batch needs after dropping the padding ALL its commits share:
 *   dims[3] = {c0, c1, c2} = position after the last non-zero id over commits index[0..batch) of the
 *   code / sub-token / AST+edit id tables, rounded up to mult_* (mult <= 0: keep the full length).
 *
 * fira_host_gather_batch: the loader step (Dataset.py:336-343 __getitem__ + default collate, minus the dense
 *   float64 toarray()): gathers commits index[0..batch) from the packed split arrays (int32 id tables
 *   [n, len], deg uint8 [n, n_nodes], col int16 / val float64 concatenated, edge_ptr int64 [n+1]) into
 *   caller-owned staging buffers (pinned memory): int64 id tensors [batch, c*] written with row length
 *   dims[0..2] (from fira_host_batch_dims, or any larger lengths up to the full 210/160/280), batch CSR
 *   rowptr int32 [batch*(c0+c1+c2)+1], col int32, val fp32.  The nodes cut away are isolated self loops
 *   (Dataset.py:271-275); sub-token copy labels (Dataset.py:213) shift by the removed code padding.
 *   Fails if a commit has a real id or a neighbour beyond dims. */
int fira_host_build_adjacency(const int* change_code, int n_change_code, const int* change_ast, int n_change_ast,
                              const int* ast_code, int n_ast_code, const int* ast_ast, int n_ast_ast,
                              const int* code_sub, int n_code_sub, int n_diff, int n_ast, int diff_len, int sub_len,
                              int ast_change_len, int* deg, int* col, double* val, int cap, int* nnz_out);
int fira_host_batch_dims(const int* sou, const int* sub_token, const int* ast_change, const long* index, int batch,
                         int diff_len, int sub_len, int ast_change_len, int mult_code, int mult_sub, int mult_ast,
                         int* dims);
int fira_host_gather_batch(const int* sou, const int* tar, const int* mark, const int* ast_change,
                           const int* tar_label, const int* sub_token, const unsigned char* deg, const short* col,
                           const double* val, const long* edge_ptr, const long* index, int batch, int diff_len,
                           int sub_len, int ast_change_len, int msg_len, int vocab_size, const int* dims,
                           long* o_sou, long* o_tar, long* o_mark, long* o_ast_change, long* o_tar_label,
                           long* o_sub_token, int* o_rowptr, int* o_col, float* o_val, long edge_cap, int* nnz_out);

/* fira_host_packed_dims / fira_host_gather_packed: the PER-COMMIT packed batch (SURVEY.md 8f rank 4, replaces the
 *   fixed 210/160/280 padding of Dataset.py:80-94).  Per commit and segment only the positions up to the last non-zero
 *   id are kept; node rows are segment-major and ragged: [code rows of all commits | pad][sub-token rows | pad]
 *   [AST/edit rows | pad].  packed_dims -> dims[6] = {code rows, sub rows, AST rows, max memory rows of a commit, nnz,
 *   max over commits of ceil(code rows / 128) + ceil(sub rows / 128) = the key chunks fira_attn_packed_* needs}.
 *   gather_packed: pad_dims[4] = {Rc, Rs, Ra, S} buffer sizes (>= dims, bucketed by the caller); writes int32 node ids
 *   (o_code, o_mark, o_pos = position in the commit for the positional encoding; o_sub; o_ast), o_off[3][batch+1]
 *   (row offsets of each commit inside its segment), o_ranges[batch][4] = {first code row, code rows, first sub row
 *   (global), sub rows}, o_mem_mask[batch][S], the decoder input o_tar[batch][msg_len] + o_tar_mask, the SHIFTED labels
 *   (Model.py:71-79) with copy labels renumbered to the commit's own memory rows (V + m), and the adjacency as a CSR in
 *   buffer order with global column ids (what fira_gcn_layer_fwd / fira_gcn_aggregate(B=1) consume). */
int fira_host_packed_dims(const int* sou, const int* sub_token, const int* ast_change, const unsigned char* deg,
                          const long* index, int batch, int diff_len, int sub_len, int ast_change_len, int* dims);
int fira_host_gather_packed(const int* sou, const int* tar, const int* mark, const int* ast_change,
                            const int* tar_label, const int* sub_token, const unsigned char* deg, const short* col,
                            const double* val, const long* edge_ptr, const long* index, int batch, int diff_len,
                            int sub_len, int ast_change_len, int msg_len, int vocab_size, const int* pad_dims,
                            int* o_code, int* o_mark, int* o_pos, int* o_sub, int* o_ast, int* o_off, int* o_ranges,
                            unsigned char* o_mem_mask, int* o_tar, int* o_label, unsigned char* o_tar_mask,
                            int* o_rowptr, int* o_col, float* o_val, long edge_cap, int* nnz_out);

#ifdef __cplusplus
}
#endif
#endif /* FIRA_B200_H_ */
