"""Host orchestration of the CUDA hot path: three autograd Functions (encoder, decoder, output
head) whose forward/backward are explicit sequences of libfira_b200 launches on the current
stream.  No torch compute op sits on the path (torch supplies memory, streams, autograd glue).

Precision modes (cfg["bf16"]):
  * fp32 parity mode  : fp32 activations, every Linear on fira_gemm_f32 (fp32 FFMA) -- logits within
                        1e-4 of the reference.
  * bf16 throughput   : bf16 activations, every large Linear on fira_gemm_bf16_tc (wgmma, register
                        fp32 accumulators, TMA operands); statistics, parameters, parameter gradients
                        and the handful of tiny products (4 x 256 value table, 256^3 weight merges,
                        2-wide gate) stay fp32.

Buffer conventions
  * node buffer: segment-major rows  [B*210 code | B*160 sub-token | B*280 AST/edit] x 256
    (kills the per-layer torch.cat/slice of gnn_transformer.py:58,86); `Xc` holds the code rows a
    Combination reads, `Gin` holds every row a GCN layer reads.
"""
import ctypes
import os

import torch

from . import _lib
from . import optim as _optim
from ._lib import FIRA_BF16, FIRA_F32, call

D = 256

# gradients produced on the side stream are consumed by AccumulateGrad on the main stream after Fork.join():
# the stream mismatch autograd warns about is intentional
if hasattr(torch.autograd.graph, "set_warn_on_accumulate_grad_stream_mismatch"):
    torch.autograd.graph.set_warn_on_accumulate_grad_stream_mismatch(False)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t, off=0):
    if t is None:
        return None
    return t.data_ptr() + off * t.element_size()


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.FiraLibraryError(
                "fira_icse_b200: tensors must live on a CUDA device -- this package has no CPU path "
                "(the CPU reference lives in oracle/ and is test infrastructure only)")


def _ceil(a, b):
    return (a + b - 1) // b


def _gdest(ts, shape, zero=False):
    """fp32 buffer for the gradient of parameter(s) `ts`: a view of the optimizer's flat gradient buffer when the
    parameters are re-homed by optim.FlatAdam (already zero-filled, adopted by autograd without a copy), else a new
    tensor (`zero`: the producer accumulates atomically)."""
    if not isinstance(ts, (list, tuple)):
        ts = (ts,)
    v = _optim.grad_dest(ts, shape)
    if v is not None:
        return v
    return (torch.zeros if zero else torch.empty)(shape, dtype=torch.float32, device=ts[0].device)


def _num_sms():
    """SMs of the current device, as the library sizes its own grids (fira_num_sms)"""
    return _lib.lib().fira_num_sms()


# ----------------------------------------------------------------------------- fp32 GEMM (parity mode)
def _pick_splits(M, N, K, relu):
    if relu:
        return 1
    if _ceil(M, 128) * _ceil(N, 128) >= _num_sms():
        return 1
    tiles = _ceil(M, 64) * _ceil(N, 64)
    want = _ceil(2 * _num_sms(), tiles)
    return max(1, min(want, _ceil(K, 16) // 8))


def gemm_raw(A, lda, a_k, Bp, ldb, b_k, C, ldc, M, N, K, bias=None, rs=None, rc=None, relu=False,
             accumulate=False, splits=None):
    if splits is None:
        splits = _pick_splits(M, N, K, relu)
    call("fira_gemm_f32", A, lda, int(a_k), Bp, ldb, int(b_k), C, ldc, M, N, K, _ptr(bias), _ptr(rs), _ptr(rc),
         int(relu), int(accumulate), splits, _stream())


def linear(x, W, b=None, relu=False, out=None, ld_out=None, rs=None, rc=None, M=None, x_off=0, ldx=None):
    """fp32: y[M,N] = x[M,K] W[N,K]^T + b (+ rs[m]*rc[n]).  Returns `out` ([M, ld_out] buffer)."""
    N, K = W.shape
    M = x.shape[0] if M is None else M
    ldx = K if ldx is None else ldx
    ld_out = N if ld_out is None else ld_out
    if out is None:
        out = torch.empty((M, ld_out), dtype=torch.float32, device=x.device)
    gemm_raw(_ptr(x, x_off), ldx, 1, _ptr(W), K, 1, _ptr(out), ld_out, M, N, K, bias=b, rs=rs, rc=rc, relu=relu)
    return out


def linear_dx(dy, ld_dy, W, M, out=None, accumulate=False, dy_off=0, n=None):
    """fp32: dx[M,K] (+)= dy[M,N] W[N,K]."""
    N, K = W.shape
    n = N if n is None else n
    if out is None:
        out = torch.empty((M, K), dtype=torch.float32, device=dy.device)
    gemm_raw(_ptr(dy, dy_off), ld_dy, 1, _ptr(W), K, 0, _ptr(out), K, M, K, n, accumulate=accumulate)
    return out


def linear_dw(dy, ld_dy, x, ldx, M, N, K, dy_off=0, x_off=0, out=None):
    """fp32: dW[N,K] = dy[M,N]^T x[M,K]."""
    dW = torch.empty((N, K), dtype=torch.float32, device=dy.device) if out is None else out
    gemm_raw(_ptr(dy, dy_off), ld_dy, 0, _ptr(x, x_off), ldx, 0, _ptr(dW), K, N, K, M)
    return dW


# ----------------------------------------------------------------------------- bf16 wgmma GEMM
def gemm_tc(A, lda, a_kmajor, Bm, ldb, b_kmajor, C, ldc, M, N, K, bias=None, rs=None, rc=None, relu=False,
            accumulate=False, splits=1, a_off=0, b_off=0, c_off=0):
    """C[M,N] = A(MxK) B(KxN) (+bias, +rs*rc, relu) on wgmma; A/B bf16, C fp32 or bf16 (by C.dtype)."""
    call("fira_gemm_bf16_tc", _ptr(A, a_off), lda, int(a_kmajor), _ptr(Bm, b_off), ldb, int(b_kmajor), _ptr(C, c_off),
         ldc, int(C.dtype == torch.bfloat16), M, N, K, _ptr(bias), _ptr(rs), _ptr(rc), int(relu), int(accumulate),
         splits, _stream())
    return C


# CTAs a split-K weight-gradient product may spread over.  These products run on the side streams NEXT TO the main
# chain: filling all 132 SMs shortens the product itself but takes the SMs (and, through the fp32 atomics of split-K,
# the L2 atomic throughput) away from the critical path.
_WGRAD_CTAS_ENV = os.environ.get("FIRA_WGRAD_CTAS")


def _wgrad_ctas():
    return max(1, int(_WGRAD_CTAS_ENV)) if _WGRAD_CTAS_ENV else _num_sms()


def _tc_splits(tiles, kblocks):
    """split-K factor of a small-output GEMM: at least 8 k-blocks per split, at most _wgrad_ctas() CTAs in all"""
    wgrad_ctas = _wgrad_ctas()
    if tiles >= wgrad_ctas:
        return 1
    return max(1, min(kblocks // 8 if kblocks >= 16 else 1, _ceil(wgrad_ctas, tiles)))


def colsum(x, ld, M, N, weight=None, x_off=0, dtype=None, out=None):
    """out[n] (+)= sum_m w[m] x[m, n]; `out` must be zero-filled (atomic accumulation)"""
    if dtype is None:
        dtype = FIRA_BF16 if x.dtype == torch.bfloat16 else FIRA_F32
    if out is None:
        out = torch.zeros(N, dtype=torch.float32, device=x.device)
    call("fira_colsum", _ptr(x, x_off), ld, M, N, _ptr(weight), _ptr(out), dtype, _stream())
    return out


class Prec:
    """Precision context of one forward/backward pair: dtype codes, buffers, Linear dispatch."""

    def __init__(self, bf16, wcache=None, seed_ctr=None):
        self.bf16 = bool(bf16)
        self.seed_ctr = seed_ctr          # device uint64 counter added to the dropout seed (CUDA-graph replays)
        self.code = FIRA_BF16 if self.bf16 else FIRA_F32
        self.tdt = torch.bfloat16 if self.bf16 else torch.float32
        self.wcache = {} if wcache is None else wcache

    def empty(self, shape, dev):
        return torch.empty(shape, dtype=self.tdt, device=dev)

    def w(self, W):
        """GEMM-operand form of a parameter: itself (fp32 mode) or a bf16 copy cached for fwd+bwd."""
        if not self.bf16:
            return W
        m = _optim.mirror_of(W)                 # parameters re-homed by optim.FlatAdam: a view of its bf16 mirror
        if m is not None:
            return m
        k = (W.data_ptr(), tuple(W.shape))
        if k not in self.wcache:
            self.wcache[k] = (W, W.detach().to(torch.bfloat16))     # keep W alive: the key is its address
        return self.wcache[k][1]

    # y = x W^T + b
    def linear(self, x, W, b=None, relu=False, out=None, ld_out=None, rs=None, rc=None, M=None, ldx=None, x_off=0):
        if not self.bf16:
            return linear(x, W, b, relu=relu, out=out, ld_out=ld_out, rs=rs, rc=rc, M=M, ldx=ldx, x_off=x_off)
        N, K = W.shape
        M = x.shape[0] if M is None else M
        ldx = K if ldx is None else ldx
        ld_out = N if ld_out is None else ld_out
        if out is None:
            out = torch.empty((M, ld_out), dtype=torch.bfloat16, device=x.device)
        return gemm_tc(x, ldx, 1, self.w(W), K, 1, out, ld_out, M, N, K, bias=b, rs=rs, rc=rc, relu=relu, a_off=x_off)

    # dx (+)= dy W
    def linear_dx(self, dy, ld_dy, W, M, out=None, accumulate=False, dy_off=0):
        if not self.bf16:
            return linear_dx(dy, ld_dy, W, M, out=out, accumulate=accumulate, dy_off=dy_off)
        N, K = W.shape
        if out is None:
            out = torch.empty((M, K), dtype=torch.bfloat16, device=dy.device)
        return gemm_tc(dy, ld_dy, 1, self.w(W), K, 0, out, K, M, K, N, accumulate=accumulate, a_off=dy_off)

    def linear_dx_relu(self, dy, ld_dy, W, M, h):
        """dx = relu'(h) * (dy W): the relu backward of the FeedForward block (gnn_transformer.py:172); bf16 mode: folded
        into the epilogue of the input-gradient product (fira_gemm_bf16_tc_dx_relu) unless FIRA_DX_RELU=0"""
        N, K = W.shape
        if self.bf16 and FUSE_DX_RELU:
            out = torch.empty((M, K), dtype=torch.bfloat16, device=dy.device)
            call("fira_gemm_bf16_tc_dx_relu", _ptr(dy), ld_dy, _ptr(self.w(W)), K, _ptr(out), K, _ptr(h), M, K, N, _stream())
            return out
        out = self.linear_dx(dy, ld_dy, W, M)
        call("fira_relu_bwd", _ptr(h), _ptr(out), M * K, self.code, _stream())
        return out

    # dW = dy^T x   (fp32 result in both modes)
    def linear_dw(self, dy, ld_dy, x, ldx, M, N, K, dy_off=0, x_off=0, out=None, dbias=None):
        """dW = dy^T x.  dbias: zero-filled fp32 [N] that receives the bias gradient colsum(dy) -- in bf16 mode from the
        same launch (fira_gemm_bf16_tc_dbias sums the dy tiles in shared memory), in fp32 mode from fira_colsum."""
        if not self.bf16:
            if dbias is not None:
                colsum(dy, ld_dy, M, N, x_off=dy_off, out=dbias)
            return linear_dw(dy, ld_dy, x, ldx, M, N, K, dy_off=dy_off, x_off=x_off, out=out)
        dW = torch.empty((N, K), dtype=torch.float32, device=dy.device) if out is None else out
        bn = 256 if K > 128 else (128 if K > 64 else 64)
        splits = _tc_splits(_ceil(N, 128) * _ceil(K, bn), _ceil(M, 64))
        if dbias is not None and os.environ.get("FIRA_DBIAS_FUSED", "1") != "0":
            call("fira_gemm_bf16_tc_dbias", _ptr(dy, dy_off), ld_dy, _ptr(x, x_off), ldx, 0, _ptr(dW), K, 0, N, K, M, 0, splits,
                 _ptr(dbias), _stream())
            return dW
        if dbias is not None:
            colsum(dy, ld_dy, M, N, x_off=dy_off, out=dbias)
        return gemm_tc(dy, ld_dy, 0, x, ldx, 0, dW, K, N, K, M, splits=splits, a_off=dy_off, b_off=x_off)

    def linear_ln(self, x, W, b, resid, gamma, beta, outA, outB, split, rows, p, seed, sid, rs=None, rc=None):
        """z = x W^T + b (+ rs rc^T);  out = LN(dropout(z) + resid) -> (z, stats): the GEMM, then the LayerNorm kernel
        (fira_ln_residual_fwd)"""
        z = self.linear(x, W, b, rs=rs, rc=rc, M=rows)
        return z, self.ln_fwd(z, resid, gamma, beta, outA, outB, split, rows, p, seed, sid)

    def ln_fwd(self, z, resid, gamma, beta, outA, outB, split, rows, p, seed, sid):
        stats = torch.empty((2, rows), dtype=torch.float32, device=z.device)
        call("fira_ln_residual_fwd", _ptr(z), _ptr(resid), _ptr(gamma), _ptr(beta), _ptr(outA), _ptr(outB), split,
             _ptr(stats), _ptr(stats, rows), rows, D, float(p), seed, _ptr(self.seed_ctr), sid, self.code, _stream())
        return stats

    def ln_bwd(self, dA, dB, split, z, resid, stats, gamma, rows, p, seed, sid, d_resid=None, accum=False, beta=None,
               rows_map=None):
        """beta: the LayerNorm bias parameter; with (gamma, beta) re-homed back to back by optim.FlatAdam their
        gradients are accumulated straight into its flat gradient buffer.  rows_map: the rows are slots of
        fira_target_rows (dropout mask of row rows_map[r], zeros for a pad slot)"""
        dz = torch.empty_like(z)
        if d_resid is None:
            d_resid = torch.empty_like(z)
        dgb = _gdest((gamma, beta), (2, D), zero=True) if beta is not None else \
            torch.zeros((2, D), dtype=torch.float32, device=z.device)
        call("fira_ln_residual_bwd_rows", _ptr(dA), _ptr(dB), split, _ptr(z), _ptr(resid), _ptr(stats),
             _ptr(stats, rows), _ptr(gamma), _ptr(dz), _ptr(d_resid), int(accum), _ptr(dgb), _ptr(dgb, D), _ptr(rows_map),
             rows, D, float(p), seed, _ptr(self.seed_ctr), sid, self.code, _stream())
        return dz, d_resid, dgb[0], dgb[1]


# fp32-mode free functions kept for the kernel unit tests
_F32 = Prec(False)


def ln_fwd(z, resid, gamma, beta, outA, outB, split, rows, p, seed, sid):
    return _F32.ln_fwd(z, resid, gamma, beta, outA, outB, split, rows, p, seed, sid)


def ln_bwd(dA, dB, split, z, resid, stats, gamma, rows, p, seed, sid, d_resid=None, accum=False):
    return _F32.ln_bwd(dA, dB, split, z, resid, stats, gamma, rows, p, seed, sid, d_resid=d_resid, accum=accum)


_SIDE_STREAMS = {}
# side work of a backward pass is many INDEPENDENT groups of small launches (a weight-gradient GEMM + its bias column
# sums + fp32 adjoints of the weight merges): on one side stream they serialise into a chain that is longer than the
# input-gradient chain of the main stream (timeline of GPU run F: 2.3 ms of the 4.1 ms step on that stream), so the
# groups rotate over several streams = parallel branches of the captured graph
N_SIDE = max(1, int(os.environ.get("FIRA_SIDE_STREAMS", "8")))
FUSE_DX_RELU = os.environ.get("FIRA_DX_RELU", "1") != "0" and os.environ.get("FIRA_GEMM_TMA_STORE", "1") != "0"
# the 256^3 fp32 products of the GCN weight merge (W2 W1 and its two adjoints) are 16 CTAs of the 64 x 64 tile: split-K
# spreads them over 64 CTAs; bf16 mode only -- the fp32 parity mode keeps the deterministic single-pass sum
MERGE_SPLITS = max(1, int(os.environ.get("FIRA_MERGE_SPLITS", "4")))
_TURN = [0]            # rotation shared by every Fork, so consecutive Forks do not all start on the same stream


class Fork:
    """Runs the weight-gradient / bias-gradient work of a backward pass on side streams.

    In a backward step `dZ` feeds three independent consumers: the input-gradient GEMM (critical
    path), the weight-gradient GEMM and the bias column sums.  The last two use a handful of CTAs
    each; issued on other streams they overlap with the critical path (and become parallel
    branches when the step is captured into a CUDA graph).  Every `with fork(...)` group takes the next
    side stream in rotation.  Tensors read on a side stream are kept alive until join(), tensors produced
    there are only consumed after join()."""

    def __init__(self, device, n_side=None):
        self.main = torch.cuda.current_stream(device)
        key = (device.index if device.index is not None else torch.cuda.current_device())
        if key not in _SIDE_STREAMS:
            _SIDE_STREAMS[key] = [torch.cuda.Stream(device=device) for _ in range(N_SIDE)]
        self.sides = _SIDE_STREAMS[key][:n_side] if n_side else _SIDE_STREAMS[key]
        self.side = self.sides[0]
        self.keep = []
        self.used = set()

    def __call__(self, *tensors, lane=None):
        """lane: pin the group to one side stream (groups that accumulate into the same tensor must serialise)"""
        self.keep.extend(tensors)
        if lane is None:
            lane = _TURN[0]
            _TURN[0] += 1
        self.side = self.sides[lane % len(self.sides)]
        self.side.wait_stream(self.main)
        self.used.add(self.side)
        return torch.cuda.stream(self.side)

    def join(self):
        for s in self.used:
            self.main.wait_stream(s)
        self.used.clear()
        self.keep.clear()


class Prefetch:
    """Weight-side preparation (concatenations, W2 @ W1 merges, the 4-row value table, bf16 operand copies)
    issued on the side stream so it runs while the main stream computes; `event` marks completion."""

    def __init__(self):
        self.wcache = {}
        self.items = None
        self.event = None
        self.layer_table = None            # prefetch_decoder, bf16: fira_decoder_fwd's host pointer table


def _prep_encoder_layer(pr, fork, mark_emb, Wq, bq, Wk, bk, Wv, bv, Wo, W1, b1, W2, fused=True):
    """Weight-only preparation of one encoder layer, as THREE independent groups on different side streams (each a few
    tiny launches): the 4-row value table, the merged GCN weight W2 W1 (+ its bf16 operand copies), the merged bias
    W2 b1.  Returns the tensors and one event per group; the consumer waits for a group right before it needs it."""
    f32 = dict(dtype=torch.float32, device=Wq.device)

    def done():
        ev = torch.cuda.Event()
        ev.record()
        return ev
    with fork(mark_emb, Wq, bq, Wk, bk, Wv, bv, Wo):
        Wqk = _optim.cat_rows((Wq, Wk))                              # views when optim.FlatAdam laid them out back to back
        bqk = _optim.cat_rows((bq, bk))
        Vtab = linear(mark_emb, Wv, bv)                            # fp32 [4, 256]: value has 4 distinct rows
        for w in (Wqk, Wo):
            pr.w(w)                                                # bf16 operand copies (views of the mirror / no-op in fp32)
        ev_comb = done()
    with fork(W1, W2):
        Wc = torch.empty((D, D), **f32)                            # W2 @ W1
        gemm_raw(_ptr(W2), D, 1, _ptr(W1), D, 0, _ptr(Wc), D, D, D, D, splits=MERGE_SPLITS if pr.bf16 else 1)
        pr.w(Wc)
        # the fused GCN backward multiplies by Wc itself ([out, in] read as K = out): its B operand is Wc^T stored K-major
        WcT16 = Wc.t().contiguous().to(torch.bfloat16) if (pr.bf16 and fused) else None
        ev_wc = done()
    with fork(W2, b1):
        c1 = torch.empty((D,), **f32)                              # W2 @ b1
        gemm_raw(_ptr(W2), D, 1, _ptr(b1), D, 1, _ptr(c1), 1, D, 1, D, splits=1)
        ev_c1 = done()
    return (Wqk, bqk, Vtab, Wc, c1, WcT16), (ev_comb, ev_wc, ev_c1)


def prefetch_decoder(bf16, lp, device):
    """Called by TransModel.forward BEFORE the encoder runs: the decoder's weight preparation (12-way K/V
    concatenation, per-layer QKV concatenations, ~40 bf16 casts) overlaps with the encoder."""
    pf = Prefetch()
    pr = Prec(bf16, pf.wcache)
    L = len(lp) // DEC_LAYER_PARAMS
    fork = Fork(device)
    with fork(*lp):
        Wkv = _optim.cat_rows([t for i in range(L) for t in (lp[i * 26 + 12], lp[i * 26 + 14])])     # [L*512, 256]
        bkv = _optim.cat_rows([t for i in range(L) for t in (lp[i * 26 + 13], lp[i * 26 + 15])])
        pr.w(Wkv)
        layers = []
        for i in range(L):
            q = lp[i * 26:(i + 1) * 26]
            Wqkv = _optim.cat_rows((q[0], q[2], q[4]))
            bqkv = _optim.cat_rows((q[1], q[3], q[5]))
            for w in (Wqkv, q[6], q[10], q[16], q[20], q[22]):     # Wqkv, self Wo, cross Wq, cross Wo, W1, W2
                pr.w(w)
            layers.append((Wqkv, bqkv))
        if bf16:
            # fira_decoder_fwd's [L][18] table of per-layer weight / bias / LayerNorm pointers (copied into its launch
            # parameters, so a captured graph keeps the addresses it was built with)
            ptrs = []
            for i in range(L):
                q = lp[i * 26:(i + 1) * 26]
                Wqkv, bqkv = layers[i]
                ptrs += [pr.w(Wqkv), bqkv, pr.w(q[6]), q[7], q[8], q[9], pr.w(q[10]), q[11], pr.w(q[16]), q[17], q[18],
                         q[19], pr.w(q[20]), q[21], pr.w(q[22]), q[23], q[24], q[25]]
            pf.layer_table = (ctypes.c_void_p * len(ptrs))(*[t.data_ptr() for t in ptrs])
        pf.items = (Wkv, bkv, layers)
        pf.event = torch.cuda.Event()
        pf.event.record()
    pf.fork = fork                                                 # keeps the inputs alive; joined by the consumer
    return pf


def prefetch_head(bf16, Wout, Ws, Wt):
    pf = Prefetch()
    if bf16:
        pr = Prec(True, pf.wcache)
        fork = Fork(Wout.device)
        with fork(Wout, Ws, Wt):
            for w in (Wout, Ws, Wt):
                pr.w(w)
            pf.event = torch.cuda.Event()
            pf.event.record()
        pf.fork = fork
    return pf


def make_seed():
    """64-bit dropout seed drawn from torch's CPU generator (so torch.manual_seed controls it)."""
    return int(torch.randint(0, 2 ** 62, (1,)).item())


# ============================================================================= encoder
ENC_LAYER_PARAMS = 16   # comb: Wq bq Wk bk Wv bv Wo bo lnw lnb ; gcn: W1 b1 W2 b2 lnw lnb


class EncoderFn(torch.autograd.Function):
    """gnn_transformer.py:45-62: 6 x [Combination on the code rows -> GCN on all 650 rows].

    GCN algebra (no non-linearity between fc1 and fc2, gnn_transformer.py:78-82):
        fc2(A fc1(H)) = (A H) (W2 W1)^T + rowsum(A) (W2 b1)^T + b2
    so a layer is ONE gather-reduce over H plus ONE 256x256 GEMM instead of two GEMMs and a
    650x650 dense bmm per graph.
    """

    @staticmethod
    def forward(ctx, cfg, sou, mark, ast_change, sub_token, edges, pos_table, emb, ast_emb, mark_emb, *lp):
        _require_cuda(sou, emb)
        B, n_code = sou.shape
        n_sub, n_ast = sub_token.shape[1], ast_change.shape[1]
        N = n_code + n_sub + n_ast
        assert edges.N == N and edges.B == B, "adjacency / batch mismatch"
        R, Mc = B * N, B * n_code
        L = len(lp) // ENC_LAYER_PARAMS
        training, seed = cfg["training"], cfg["seed"]
        p_comb = cfg["p_comb"] if training else 0.0
        p_gcn = cfg["p_gcn"] if training else 0.0
        heads = cfg["heads"]
        pr = Prec(cfg.get("bf16", False), seed_ctr=cfg.get("seed_ctr"))
        dev = emb.device
        f32 = dict(dtype=torch.float32, device=dev)
        st = _stream()

        Xc = pr.empty((Mc, D), dev)
        Gin = pr.empty((R, D), dev)
        # packed batches (packed.py) come as ONE ragged "graph": B = 1, the three segments hold the real rows of every
        # commit, cfg["pos"] gives each code row its position inside its commit (positional encoding)
        if cfg.get("pos") is not None:
            call("fira_embed_nodes_pos_fwd", _ptr(sou), _ptr(cfg["pos"]), _ptr(sub_token), _ptr(ast_change), _ptr(emb),
                 _ptr(ast_emb), _ptr(pos_table), _ptr(Xc), _ptr(Gin), B, n_code, n_sub, n_ast, D, pr.code, st)
        else:
            call("fira_embed_nodes_fwd", _ptr(sou), _ptr(sub_token), _ptr(ast_change), _ptr(emb), _ptr(ast_emb),
                 _ptr(pos_table), _ptr(Xc), _ptr(Gin), B, n_code, n_sub, n_ast, D, pr.code, st)
        # GCN layer: scatter (fira_gcn_aggregate) -> wgmma GEMM -> LayerNorm.  FIRA_GCN_FUSED=1 (bf16 mode) runs the whole
        # layer as ONE kernel instead (gather -> wgmma -> LayerNorm epilogue, csrc/gcn_fused.cu): validated by the tests,
        # opt-in (its speed against the three launches has not been measured on the H100)
        fused = pr.bf16 and os.environ.get("FIRA_GCN_FUSED", "0") != "0"
        rs = None if fused else edges.rowsum(n_code, n_sub, n_ast)
        erows = edges.rows_csr(n_code, n_sub, n_ast) if fused else None
        saved = []
        # weight-only work of ALL layers goes to the side stream, layer 0 first; the main stream waits for
        # layer i's event right before it needs it, so only the first layer's ~8 tiny launches are exposed
        fork = Fork(dev)
        preps, events = [], []
        for i in range(L):
            Wq, bq, Wk, bk, Wv, bv, Wo, bo, clw, clb, W1, b1, W2, b2, glw, glb = lp[i * 16:(i + 1) * 16]
            t, e = _prep_encoder_layer(pr, fork, mark_emb, Wq, bq, Wk, bk, Wv, bv, Wo, W1, b1, W2, fused=fused)
            preps.append(t)
            events.append(e)
        for i in range(L):
            Wq, bq, Wk, bk, Wv, bv, Wo, bo, clw, clb, W1, b1, W2, b2, glw, glb = lp[i * 16:(i + 1) * 16]
            sid = cfg["stream_base"] + i * 8
            cur = torch.cuda.current_stream()
            cur.wait_event(events[i][0])                               # q|k views, value table
            Wqk, bqk, Vtab, Wc, c1, WcT16 = preps[i]
            # ---- Combination (gnn_transformer.py:192-205, combination_layer.py:7-17)
            QK = pr.linear(Xc, Wqk, bqk)                               # [Mc, 512] = [q | k]
            Cd = pr.empty((Mc, D), dev)
            call("fira_comb_gate_fwd", _ptr(QK), 2 * D, _ptr(Vtab), _ptr(mark), _ptr(Cd), Mc, D, D // heads,
                 float(p_comb), seed, _ptr(pr.seed_ctr), sid + 0, pr.code, st)
            Zc, st_c = pr.linear_ln(Cd, Wo, bo, Xc, clw, clb, Gin, Gin, Mc, Mc, p_comb, seed, sid + 1)   # -> Gin[:Mc]
            # ---- GCN (gnn_transformer.py:74-86)
            Xc_n = pr.empty((Mc, D), dev)
            Gin_n = pr.empty((R, D), dev)
            cur.wait_event(events[i][1])                               # merged weight W2 W1
            cur.wait_event(events[i][2])                               # merged bias W2 b1
            if fused:
                G = None
                Z = pr.empty((R, D), dev)
                st_g = torch.empty((2, R), **f32)
                call("fira_gcn_layer_fwd", _ptr(erows[0]), _ptr(erows[1]), _ptr(erows[2]), _ptr(Gin), _ptr(pr.w(Wc)),
                     _ptr(b2), _ptr(c1), _ptr(glw), _ptr(glb), _ptr(Z), _ptr(Xc_n), _ptr(Gin_n), Mc, _ptr(st_g),
                     _ptr(st_g, R), R, D, float(p_gcn), seed, _ptr(pr.seed_ctr), sid + 2, st)
            else:
                G = pr.empty((R, D), dev)
                call("fira_gcn_aggregate", _ptr(edges.rowptr), _ptr(edges.col), _ptr(edges.val), _ptr(Gin), None,
                     _ptr(G), B, n_code, n_sub, n_ast, D, pr.code, st)
                Z, st_g = pr.linear_ln(G, Wc, b2, Gin, glw, glb, Xc_n, Gin_n, Mc, R, p_gcn, seed, sid + 2, rs=rs, rc=c1)
            saved.append((Xc, QK, Vtab, Cd, Zc, st_c, Gin, G, Z, st_g, Wqk, Wc, c1, WcT16))
            Xc, Gin = Xc_n, Gin_n
        memory = pr.empty((B, n_code + n_sub, D), dev)
        call("fira_pack_memory", _ptr(Xc), _ptr(Gin), _ptr(memory), B, n_code, n_sub, D, pr.code, st)
        fork.join()

        ctx.saved = saved
        ctx.wcache = pr.wcache
        ctx.misc = (cfg, sou, mark, ast_change, sub_token, edges, rs, B, n_code, n_sub, n_ast, p_comb, p_gcn, fused)
        ctx.save_for_backward(emb, ast_emb, mark_emb, *lp)
        return memory

    @staticmethod
    def backward(ctx, d_mem):
        cfg, sou, mark, ast_change, sub_token, edges, rs, B, n_code, n_sub, n_ast, p_comb, p_gcn, fused = ctx.misc
        emb, ast_emb, mark_emb, *lp = ctx.saved_tensors
        N = n_code + n_sub + n_ast
        R, Mc = B * N, B * n_code
        L = len(lp) // ENC_LAYER_PARAMS
        seed, heads = cfg["seed"], cfg["heads"]
        pr = Prec(cfg.get("bf16", False), ctx.wcache, seed_ctr=cfg.get("seed_ctr"))
        dev = emb.device
        f32 = dict(dtype=torch.float32, device=dev)
        st = _stream()
        et = edges.t()
        etrows = et.rows_csr(n_code, n_sub, n_ast) if fused else None
        d_mem = d_mem.contiguous().to(pr.tdt)
        dXc = pr.empty((Mc, D), dev)
        dGin = pr.empty((R, D), dev)
        call("fira_unpack_memory", _ptr(d_mem), _ptr(dXc), _ptr(dGin), B, n_code, n_sub, n_ast, D, pr.code, st)
        d_mark_emb = _gdest(mark_emb, tuple(mark_emb.shape), zero=True)
        grads = [None] * len(lp)
        fork = Fork(dev)
        for i in reversed(range(L)):
            Wq, bq, Wk, bk, Wv, bv, Wo, bo, clw, clb, W1, b1, W2, b2, glw, glb = lp[i * 16:(i + 1) * 16]
            Xc, QK, Vtab, Cd, Zc, st_c, Gin, G, Z, st_g, Wqk, Wc, c1, WcT16 = ctx.saved[i]
            sid = cfg["stream_base"] + i * 8
            # ---- GCN backward
            dZ, dRes, d_glw, d_glb = pr.ln_bwd(dXc, dGin, Mc, Z, Gin, st_g, glw, R, p_gcn, seed, sid + 2, beta=glb)
            dGin_i = pr.empty((R, D), dev)
            if fused:
                # one kernel: AdZ = A^T dZ (kept for the weight gradients), dGin_i = AdZ Wc + dRes
                AdZ = pr.empty((R, D), dev)
                call("fira_gcn_layer_bwd", _ptr(etrows[0]), _ptr(etrows[1]), _ptr(etrows[2]), _ptr(dZ), _ptr(WcT16),
                     _ptr(dRes), _ptr(AdZ), _ptr(dGin_i), R, D, st)
            with fork(dZ, G, rs, W1, W2, b1):
                d_b2 = _gdest(b2, (D,), zero=True)
                if fused:                       # dZ^T (A H) = (A^T dZ)^T H ;  sum_i rowsum(A)_i dZ_i = colsum(A^T dZ)
                    fork.keep.append(AdZ)
                    colsum(dZ, D, R, D, out=d_b2)
                    d_c1 = torch.zeros(D, dtype=torch.float32, device=dev)
                    dWc = pr.linear_dw(AdZ, D, Gin, D, R, D, D, dbias=d_c1)
                else:
                    d_c1 = colsum(dZ, D, R, D, weight=rs)
                    dWc = pr.linear_dw(dZ, D, G, D, R, D, D, dbias=d_b2)
                ev_dwc = torch.cuda.Event()
                ev_dwc.record()
                fork.keep.extend((dWc, d_c1))
            # the three fp32 adjoints of the weight merge are independent of each other: two more side streams, so the
            # last layer's chain dWc -> d_W2 -> d_W1 -> d_b1 does not trail the main stream
            with fork():
                torch.cuda.current_stream().wait_event(ev_dwc)
                d_W2 = _gdest(W2, (D, D))               # dWc W1^T + d_c1 b1^T
                gemm_raw(_ptr(dWc), D, 1, _ptr(W1), D, 1, _ptr(d_W2), D, D, D, D, rs=d_c1, rc=b1, splits=MERGE_SPLITS if pr.bf16 else 1)
            with fork():
                torch.cuda.current_stream().wait_event(ev_dwc)
                d_W1 = _gdest(W1, (D, D))               # W2^T dWc
                gemm_raw(_ptr(W2), D, 0, _ptr(dWc), D, 0, _ptr(d_W1), D, D, D, D, splits=MERGE_SPLITS if pr.bf16 else 1)
                d_b1 = _gdest(b1, (D,))                 # W2^T d_c1
                gemm_raw(_ptr(W2), D, 0, _ptr(d_c1), 1, 0, _ptr(d_b1), 1, D, 1, D, splits=1)
            if not fused:
                dG = pr.linear_dx(dZ, D, Wc, R)
                call("fira_gcn_aggregate", _ptr(et.rowptr), _ptr(et.col), _ptr(et.val), _ptr(dG), _ptr(dRes),
                     _ptr(dGin_i), B, n_code, n_sub, n_ast, D, pr.code, st)
            # ---- Combination backward (rows < Mc of dGin_i are d(comb output))
            dXc_n = pr.empty((Mc, D), dev)
            dZc, _, d_clw, d_clb = pr.ln_bwd(dGin_i, dGin_i, Mc, Zc, Xc, st_c, clw, Mc, p_comb, seed, sid + 1,
                                             d_resid=dXc_n, beta=clb)
            with fork(dZc, Cd):
                d_bo = _gdest(bo, (D,), zero=True)
                d_Wo = pr.linear_dw(dZc, D, Cd, D, Mc, D, D, out=_gdest(Wo, (D, D)), dbias=d_bo)
            dCd = pr.linear_dx(dZc, D, Wo, Mc)
            dQK = pr.empty((Mc, 2 * D), dev)
            dVtab = torch.zeros((4, D), **f32)
            call("fira_comb_gate_bwd", _ptr(QK), 2 * D, _ptr(Vtab), _ptr(mark), _ptr(dCd), _ptr(dQK), _ptr(dVtab),
                 Mc, D, D // heads, float(p_comb), seed, _ptr(pr.seed_ctr), sid + 0, pr.code, st)
            with fork(dQK, Xc):
                d_bqk = _gdest((bq, bk), (2 * D,), zero=True)
                d_Wqk = pr.linear_dw(dQK, 2 * D, Xc, D, Mc, 2 * D, D, out=_gdest((Wq, Wk), (2 * D, D)), dbias=d_bqk)
            with fork(dVtab, mark_emb, Wv):
                d_Wv = linear_dw(dVtab, D, mark_emb, D, 4, D, D, out=_gdest(Wv, (D, D)))
                d_bv = colsum(dVtab, D, 4, D, out=_gdest(bv, (D,), zero=True))
            with fork(dVtab, Wv, lane=0):                           # d_mark_emb accumulates across layers: one stream, in order
                linear_dx(dVtab, D, Wv, 4, out=d_mark_emb, accumulate=True)
            pr.linear_dx(dQK, 2 * D, Wqk, Mc, out=dXc_n, accumulate=True)
            grads[i * 16:(i + 1) * 16] = [d_Wqk[:D], d_bqk[:D], d_Wqk[D:], d_bqk[D:], d_Wv, d_bv, d_Wo, d_bo,
                                          d_clw, d_clb, d_W1, d_b1, d_W2, d_b2, d_glw, d_glb]
            dXc, dGin = dXc_n, dGin_i
            ctx.saved[i] = None
        d_emb = _gdest(emb, tuple(emb.shape), zero=True)
        d_ast = _gdest(ast_emb, tuple(ast_emb.shape), zero=True)
        call("fira_embed_nodes_bwd", _ptr(sou), _ptr(sub_token), _ptr(ast_change), _ptr(dXc), _ptr(dGin),
             _ptr(d_emb), _ptr(d_ast), B, n_code, n_sub, n_ast, D, pr.code, st)
        fork.join()
        d_mark_emb[0].zero_()     # padding_idx=0 (gnn_transformer.py:39)
        return (None, None, None, None, None, None, None, d_emb, d_ast, d_mark_emb, *grads)


# ============================================================================= decoder
DEC_LAYER_PARAMS = 26   # self: Wq bq Wk bk Wv bv Wo bo lnw lnb ; cross: same 10 ; ffn: W1 b1 W2 b2 lnw lnb


class DecoderFn(torch.autograd.Function):
    """gnn_transformer.py:108-122: embedding + PE, 6 x [self-attn, cross-attn, FFN], all post-LN.
    The 12 cross-attention K/V projections of the (layer-invariant) memory run as ONE GEMM.

    cfg["label"] (the shifted labels [B, T] of a packed bf16 training batch, else absent): the backward runs on the live
    target rows alone, the rows before each commit's last label (fira_target_rows, at most pk.Rt).  No later row carries
    a loss, and causal self-attention never lets a live row read one, so they change neither the loss nor a gradient;
    their output rows are zero.  Precondition: tar_mask[b, 0] = 1 for every commit with a label.  A row whose causal
    keys are all padding attends uniformly over all T rows (attn_mma.cuh), dead rows included, and the slot backward
    would drop the gradient those rows receive; row 0 as a valid key rules such a live row out.  The loader never breaks
    it: every target starts with the <start> token."""

    @staticmethod
    def forward(ctx, cfg, tar, memory, mem_mask, tar_mask, pos_table, dec_emb, *lp):
        _require_cuda(tar, memory, dec_emb)
        B, T = tar.shape
        pk = cfg.get("packed")                      # packed batch: memory is [1, Rc + Rs, D], keys of commit b = pk.ranges[b]
        S = pk.S if pk is not None else memory.shape[1]
        Mt, Ms = B * T, memory.shape[0] * memory.shape[1]
        L = len(lp) // DEC_LAYER_PARAMS
        H = cfg["heads"]
        training, seed = cfg["training"], cfg["seed"]
        p = cfg["p_dec"] if training else 0.0
        pr = Prec(cfg.get("bf16", False), seed_ctr=cfg.get("seed_ctr"))
        dev = dec_emb.device
        f32 = dict(dtype=torch.float32, device=dev)
        st = _stream()
        mem_dtype = memory.dtype
        memory = memory.contiguous().to(pr.tdt)

        if not pr.bf16:
            X = pr.empty((Mt, D), dev)
            call("fira_embed_rows_fwd", _ptr(tar), _ptr(dec_emb), _ptr(pos_table), _ptr(X), Mt, T, D, pr.code, st)
        pf = cfg.get("prefetch")
        if pf is None:
            pf = prefetch_decoder(pr.bf16, lp, dev)
        torch.cuda.current_stream().wait_event(pf.event)
        pf.fork.join()
        pr.wcache.update(pf.wcache)
        Wkv, bkv, qkv_layers = pf.items
        ldkv = L * 2 * D
        KV = pr.linear(memory.view(Ms, D), Wkv, bkv)                                              # [Ms, L*512]
        if pr.bf16:
            # the whole stack in ONE launch (csrc/decoder_fwd.cu): every tensor the backward reads, leading dim = layer,
            # R rows each: the live-row slots of a packed training batch (fira_target_rows), else every row
            label = cfg.get("label")
            rmap = None
            R = Mt
            if label is not None and pk is not None:
                R = pk.Rt
                rmap = torch.empty((2 * B + 1 + R,), dtype=torch.int32, device=dev)      # tlen | toff | trows
                call("fira_target_rows", _ptr(label), B, T, _ptr(rmap), _ptr(rmap, B), _ptr(rmap, 2 * B + 1), R, st)
            bf = dict(dtype=torch.bfloat16, device=dev)
            Xs = torch.empty((L, R, D), **bf)                      # each layer's input
            out = torch.empty((Mt, D), **bf)
            QKV, Hh = torch.empty((L, R, 3 * D), **bf), torch.empty((L, R, 4 * D), **bf)
            ctx1, Z1, X1, Q, ctx2, Z2, X2, Z3 = torch.empty((8, L, R, D), **bf)
            st1, st2 = torch.empty((2, L, B, H, T, 2), **f32)
            ls1, ls2, ls3 = torch.empty((3, L, 2, R), **f32)
            call("fira_decoder_fwd_rows", _ptr(tar), _ptr(dec_emb), _ptr(pos_table), _ptr(tar_mask), _ptr(KV), ldkv,
                 _ptr(mem_mask), _ptr(pk.ranges) if pk is not None else None, S, ctypes.addressof(pf.layer_table), L,
                 _ptr(Xs), _ptr(out), _ptr(QKV), _ptr(ctx1), _ptr(st1), _ptr(Z1), _ptr(ls1), _ptr(X1), _ptr(Q),
                 _ptr(ctx2), _ptr(st2), _ptr(Z2), _ptr(ls2), _ptr(X2), _ptr(Hh), _ptr(Z3), _ptr(ls3), _ptr(rmap),
                 _ptr(rmap, B), R, B, T, float(p), seed, _ptr(pr.seed_ctr), cfg["stream_base"] + 64, st)
            ctx.saved = [(Xs[i], qkv_layers[i][0], QKV[i], ctx1[i], st1[i], Z1[i], ls1[i], X1[i], Q[i], ctx2[i], st2[i],
                          Z2[i], ls2[i], X2[i], Hh[i], Z3[i], ls3[i]) for i in range(L)]
            ctx.wcache = pr.wcache
            ctx.misc = (cfg, tar, memory, mem_mask, tar_mask, KV, Wkv, B, T, S, p, mem_dtype, Ms, R, rmap)
            ctx.save_for_backward(dec_emb, *lp)
            return out.view(B, T, D)
        saved = []
        for i in range(L):
            (sWq, sbq, sWk, sbk, sWv, sbv, sWo, sbo, slw, slb,
             cWq, cbq, cWk, cbk, cWv, cbv, cWo, cbo, clw, clb,
             fW1, fb1, fW2, fb2, flw, flb) = lp[i * 26:(i + 1) * 26]
            sid = cfg["stream_base"] + 64 + i * 8
            # ---- masked self-attention (gnn_transformer.py:117-119)
            Wqkv, bqkv = qkv_layers[i]
            QKV = pr.linear(X, Wqkv, bqkv)                               # [Mt, 768]
            ctx1 = pr.empty((Mt, D), dev)
            st1 = torch.empty((B, H, T, 2), **f32)
            call("fira_attn_fwd", _ptr(QKV), 3 * D, _ptr(QKV, D), 3 * D, _ptr(QKV, 2 * D), 3 * D, _ptr(tar_mask), 1,
                 _ptr(ctx1), D, _ptr(st1), B, H, T, T, D // H, pr.code, st)
            X1 = pr.empty((Mt, D), dev)
            Z1, ls1 = pr.linear_ln(ctx1, sWo, sbo, X, slw, slb, X1, X1, Mt, Mt, p, seed, sid + 0)
            # ---- cross-attention over the encoder memory (gnn_transformer.py:120)
            Q = pr.linear(X1, cWq, cbq)
            ctx2 = pr.empty((Mt, D), dev)
            st2 = torch.empty((B, H, T, 2), **f32)
            if pk is not None:
                call("fira_attn_packed_fwd", _ptr(Q), D, _ptr(KV, i * 2 * D), ldkv, _ptr(KV, i * 2 * D + D), ldkv,
                     _ptr(pk.ranges), Ms, _ptr(mem_mask), S, pk.chunks, _ptr(ctx2), D, _ptr(st2), B, H, T, D // H, pr.code, st)
            else:
                call("fira_attn_fwd", _ptr(Q), D, _ptr(KV, i * 2 * D), ldkv, _ptr(KV, i * 2 * D + D), ldkv,
                     _ptr(mem_mask), 0, _ptr(ctx2), D, _ptr(st2), B, H, T, S, D // H, pr.code, st)
            X2 = pr.empty((Mt, D), dev)
            Z2, ls2 = pr.linear_ln(ctx2, cWo, cbo, X1, clw, clb, X2, X2, Mt, Mt, p, seed, sid + 1)
            # ---- feed-forward (gnn_transformer.py:170-174)
            Hh = pr.linear(X2, fW1, fb1, relu=True)                       # [Mt, 1024]
            X3 = pr.empty((Mt, D), dev)
            Z3, ls3 = pr.linear_ln(Hh, fW2, fb2, X2, flw, flb, X3, X3, Mt, Mt, p, seed, sid + 2)
            saved.append((X, Wqkv, QKV, ctx1, st1, Z1, ls1, X1, Q, ctx2, st2, Z2, ls2, X2, Hh, Z3, ls3))
            X = X3
        ctx.saved = saved
        ctx.wcache = pr.wcache
        ctx.misc = (cfg, tar, memory, mem_mask, tar_mask, KV, Wkv, B, T, S, p, mem_dtype, Ms, Mt, None)
        ctx.save_for_backward(dec_emb, *lp)
        return X.view(B, T, D)

    @staticmethod
    def backward(ctx, d_out):
        # R rows per saved tensor; rmap = tlen [B] | toff [B+1] | trows [R] of the live-row slots, or None (R = B*T)
        cfg, tar, memory, mem_mask, tar_mask, KV, Wkv, B, T, S, p, mem_dtype, Ms, R, rmap = ctx.misc
        dec_emb, *lp = ctx.saved_tensors
        Mt = B * T
        pk = cfg.get("packed")
        L = len(lp) // DEC_LAYER_PARAMS
        H, seed = cfg["heads"], cfg["seed"]
        pr = Prec(cfg.get("bf16", False), ctx.wcache, seed_ctr=cfg.get("seed_ctr"))
        dev = dec_emb.device
        st = _stream()
        ldkv = L * 2 * D
        dX = d_out.contiguous().to(pr.tdt).view(Mt, D)
        toff = trows = None
        if rmap is not None:
            toff, trows = rmap[B:2 * B + 1], rmap[2 * B + 1:]
            dXs = pr.empty((R, D), dev)
            call("fira_gather_rows", _ptr(dX), D, _ptr(trows), _ptr(dXs), D, R, D, pr.code, st)
            dX = dXs
        dKV = pr.empty((Ms, ldkv), dev)
        if pk is not None:          # the attention kernels write the rows of every commit; the segment padding stays
            call("fira_zero_pad_rows", _ptr(dKV), ldkv, ldkv, _ptr(pk.off), B, pk.Rc, pk.Rs, pr.code, st)
        grads = [None] * len(lp)
        F = 4 * D
        fork = Fork(dev)
        for i in reversed(range(L)):
            (sWq, sbq, sWk, sbk, sWv, sbv, sWo, sbo, slw, slb,
             cWq, cbq, cWk, cbk, cWv, cbv, cWo, cbo, clw, clb,
             fW1, fb1, fW2, fb2, flw, flb) = lp[i * 26:(i + 1) * 26]
            X, Wqkv, QKV, ctx1, st1, Z1, ls1, X1, Q, ctx2, st2, Z2, ls2, X2, Hh, Z3, ls3 = ctx.saved[i]
            sid = cfg["stream_base"] + 64 + i * 8
            # ---- FFN
            dZ3, dX2, d_flw, d_flb = pr.ln_bwd(dX, dX, R, Z3, X2, ls3, flw, R, p, seed, sid + 2, beta=flb, rows_map=trows)
            with fork(dZ3, Hh):
                d_fb2 = _gdest(fb2, (D,), zero=True)
                d_fW2 = pr.linear_dw(dZ3, D, Hh, F, R, D, F, out=_gdest(fW2, (D, F)), dbias=d_fb2)
            dHh = pr.linear_dx_relu(dZ3, D, fW2, R, Hh)                  # [R, 1024], relu backward in the epilogue
            with fork(dHh, X2):
                d_fb1 = _gdest(fb1, (F,), zero=True)
                d_fW1 = pr.linear_dw(dHh, F, X2, D, R, F, D, out=_gdest(fW1, (F, D)), dbias=d_fb1)
            pr.linear_dx(dHh, F, fW1, R, out=dX2, accumulate=True)
            # ---- cross-attention
            dZ2, dX1, d_clw, d_clb = pr.ln_bwd(dX2, dX2, R, Z2, X1, ls2, clw, R, p, seed, sid + 1, beta=clb, rows_map=trows)
            with fork(dZ2, ctx2):
                d_cbo = _gdest(cbo, (D,), zero=True)
                d_cWo = pr.linear_dw(dZ2, D, ctx2, D, R, D, D, out=_gdest(cWo, (D, D)), dbias=d_cbo)
            dctx2 = pr.linear_dx(dZ2, D, cWo, R)
            dQ = pr.empty((R, D), dev)
            if toff is not None:        # query rows = the commit's slots, keys = its memory ranges
                call("fira_attn_bwd_rows", _ptr(Q), D, _ptr(KV, i * 2 * D), ldkv, _ptr(KV, i * 2 * D + D), ldkv,
                     _ptr(pk.ranges), _ptr(mem_mask), S, 0, _ptr(toff), R, _ptr(ctx2), _ptr(dctx2), D, _ptr(st2), _ptr(dQ), D,
                     _ptr(dKV, i * 2 * D), ldkv, _ptr(dKV, i * 2 * D + D), ldkv, B, H, T, D // H, pr.code, st)
            elif pk is not None:
                call("fira_attn_packed_bwd", _ptr(Q), D, _ptr(KV, i * 2 * D), ldkv, _ptr(KV, i * 2 * D + D), ldkv,
                     _ptr(pk.ranges), Ms, _ptr(mem_mask), S, pk.chunks, _ptr(ctx2), _ptr(dctx2), D, _ptr(st2), _ptr(dQ), D,
                     _ptr(dKV, i * 2 * D), ldkv, _ptr(dKV, i * 2 * D + D), ldkv, B, H, T, D // H, pr.code, st)
            else:
                call("fira_attn_bwd", _ptr(Q), D, _ptr(KV, i * 2 * D), ldkv, _ptr(KV, i * 2 * D + D), ldkv,
                     _ptr(mem_mask), 0, _ptr(ctx2), _ptr(dctx2), D, _ptr(st2), _ptr(dQ), D, _ptr(dKV, i * 2 * D), ldkv,
                     _ptr(dKV, i * 2 * D + D), ldkv, B, H, T, S, D // H, pr.code, st)
            with fork(dQ, X1):
                d_cbq = _gdest(cbq, (D,), zero=True)
                d_cWq = pr.linear_dw(dQ, D, X1, D, R, D, D, out=_gdest(cWq, (D, D)), dbias=d_cbq)
            pr.linear_dx(dQ, D, cWq, R, out=dX1, accumulate=True)
            # ---- self-attention
            dZ1, dX0, d_slw, d_slb = pr.ln_bwd(dX1, dX1, R, Z1, X, ls1, slw, R, p, seed, sid + 0, beta=slb, rows_map=trows)
            with fork(dZ1, ctx1):
                d_sbo = _gdest(sbo, (D,), zero=True)
                d_sWo = pr.linear_dw(dZ1, D, ctx1, D, R, D, D, out=_gdest(sWo, (D, D)), dbias=d_sbo)
            dctx1 = pr.linear_dx(dZ1, D, sWo, R)
            dQKV = pr.empty((R, 3 * D), dev)
            if toff is not None:        # queries and keys = the commit's slots
                call("fira_attn_bwd_rows", _ptr(QKV), 3 * D, _ptr(QKV, D), 3 * D, _ptr(QKV, 2 * D), 3 * D, None,
                     _ptr(tar_mask), T, 1, _ptr(toff), R, _ptr(ctx1), _ptr(dctx1), D, _ptr(st1), _ptr(dQKV), 3 * D,
                     _ptr(dQKV, D), 3 * D, _ptr(dQKV, 2 * D), 3 * D, B, H, T, D // H, pr.code, st)
            else:
                call("fira_attn_bwd", _ptr(QKV), 3 * D, _ptr(QKV, D), 3 * D, _ptr(QKV, 2 * D), 3 * D, _ptr(tar_mask), 1,
                     _ptr(ctx1), _ptr(dctx1), D, _ptr(st1), _ptr(dQKV), 3 * D, _ptr(dQKV, D), 3 * D, _ptr(dQKV, 2 * D),
                     3 * D, B, H, T, T, D // H, pr.code, st)
            with fork(dQKV, X):
                d_bqkv = _gdest((sbq, sbk, sbv), (3 * D,), zero=True)
                d_Wqkv = pr.linear_dw(dQKV, 3 * D, X, D, R, 3 * D, D, out=_gdest((sWq, sWk, sWv), (3 * D, D)), dbias=d_bqkv)
            pr.linear_dx(dQKV, 3 * D, Wqkv, R, out=dX0, accumulate=True)
            grads[i * 26:(i + 1) * 26] = [
                d_Wqkv[:D], d_bqkv[:D], d_Wqkv[D:2 * D], d_bqkv[D:2 * D], d_Wqkv[2 * D:], d_bqkv[2 * D:],
                d_sWo, d_sbo, d_slw, d_slb,
                d_cWq, d_cbq, None, None, None, None, d_cWo, d_cbo, d_clw, d_clb,
                d_fW1, d_fb1, d_fW2, d_fb2, d_flw, d_flb]
            dX = dX0
            ctx.saved[i] = None
        # hoisted K/V projections of the memory: one weight-grad GEMM, one input-grad GEMM
        mem2 = memory.view(Ms, D)
        with fork(dKV, mem2):
            kv_w = [t for i in range(L) for t in (lp[i * 26 + 12], lp[i * 26 + 14])]
            kv_b = [t for i in range(L) for t in (lp[i * 26 + 13], lp[i * 26 + 15])]
            d_bkv = _gdest(kv_b, (ldkv,), zero=True)
            d_Wkv = pr.linear_dw(dKV, ldkv, mem2, D, Ms, ldkv, D, out=_gdest(kv_w, (ldkv, D)), dbias=d_bkv)
        d_mem = pr.linear_dx(dKV, ldkv, Wkv, Ms).view(memory.shape).to(mem_dtype)
        for i in range(L):
            o = i * 2 * D
            grads[i * 26 + 12], grads[i * 26 + 13] = d_Wkv[o:o + D], d_bkv[o:o + D]
            grads[i * 26 + 14], grads[i * 26 + 15] = d_Wkv[o + D:o + 2 * D], d_bkv[o + D:o + 2 * D]
        d_emb = _gdest(dec_emb, tuple(dec_emb.shape), zero=True)
        call("fira_embed_rows_bwd_rows", _ptr(tar), _ptr(trows), _ptr(dX), _ptr(d_emb), R, D, pr.code, st)
        fork.join()
        return (None, None, d_mem, None, None, None, d_emb, *grads)


# ============================================================================= output head
def _ld_logits(V):
    return (V + 63) // 64 * 64


def copy_scores_fwd(pr, memory2, dec2, Ws, Wt, wres, bres, B, T, S, src_mask=None, row_mask=None, ranges=None):
    src = pr.linear(memory2, Ws)                  # [B*S, 256] (packed batches: [Rc + Rs, 256])
    tgt = pr.linear(dec2, Wt)                     # [B*T, 256]
    sc = torch.empty((B, T, S), dtype=torch.float32, device=dec2.device)
    if ranges is not None:
        call("fira_copy_scores_packed_fwd", _ptr(src), _ptr(tgt), _ptr(wres), _ptr(bres), _ptr(ranges), _ptr(src_mask),
             _ptr(row_mask), _ptr(sc), B, T, S, D, pr.code, _stream())
    else:
        call("fira_copy_scores_fwd", _ptr(src), _ptr(tgt), _ptr(wres), _ptr(bres), _ptr(src_mask), _ptr(row_mask),
             _ptr(sc), B, T, S, D, pr.code, _stream())
    return src, tgt, sc


def head_products(pr, memory2, dec2, dec32, dec_v, cap, Wout, bout, Ws, Wt, Wres, bres, Wp, bp, B, T, S, mem_mask,
                  row_mask, ranges=None):
    """The output head's three products (Model.py:54-60): out_fc logits of the `cap` rows dec_v ([cap, _ld_logits(V)],
    pr's dtype), the pointer scores [B, T, S] with the two projections their backward reads, and the fp32 gate logits
    [B*T, 2] of dec32 -> (logits, src, tgt, sc, gl)."""
    logits = pr.empty((cap, _ld_logits(Wout.shape[0])), dec2.device)
    pr.linear(dec_v, Wout, bout, out=logits, ld_out=logits.shape[1])
    src, tgt, sc = copy_scores_fwd(pr, memory2, dec2, Ws, Wt, Wres, bres, B, T, S, src_mask=mem_mask, row_mask=row_mask,
                                   ranges=ranges)
    gl = linear(dec32, Wp, bp)                # fp32 [Mt, 2]
    return logits, src, tgt, sc, gl


class HeadFn(torch.autograd.Function):
    """Model.py:54-86 fused: out_fc, CopyNet, both softmaxes, gate mixing, log(clamp), shifted-label
    NLL -- returns (loss_sum, per-position nll, argmax ids or None).  The B x 30 x 25,020 distribution
    is never built.  seq_weight (fp32 [B] on the device, padded batches only): loss_sum = sum_b seq_weight[b] *
    sum_t nll[b, t] (self-critical training, scst.py); a target sequence of weight 0 takes no gradient.
    teacher (padded training batches only, not with seq_weight): (t_logits fp32 [B*T, >= V], t_copy_scores fp32
    [B, T, S], t_gate_logits fp32 [B*T, 2], alpha, kd fp32 [B*T]), a teacher's triple (distill.teacher_targets):
    loss_sum = sum_r (1 - alpha) nll_r + alpha kd_r with kd_r = -sum_j t_j log clamp(P_j, 1e-10, 1), written to `kd`
    (fira_pointer_mix_kd_fwd / _bwd; distill.py).
    sparse (instead of teacher, on the same path): (t_label int32 [B*T, k], t_prob fp32 [B*T, k], alpha, kd fp32
    [B*T]), a batch's stored top-k targets (distill.KDTargets.batch): the same loss with t_j = t_prob at the labels
    t_label and 0 elsewhere (fira_pointer_mix_kd_sparse_fwd / _bwd)."""

    @staticmethod
    def forward(ctx, want_argmax, bf16, pf, memory, dec, mem_mask, label, Wout, bout, Ws, Wt, Wres, bres, Wp, bp,
                pk=None, seq_weight=None, teacher=None, sparse=None):
        _require_cuda(memory, dec, Wout)
        B, T = dec.shape[0], dec.shape[1]
        S = pk.S if pk is not None else memory.shape[1]      # packed batch: memory is [1, Rc + Rs, D]
        V = Wout.shape[0]
        if seq_weight is not None:
            if pk is not None or want_argmax:
                raise ValueError("HeadFn: seq_weight applies to the padded training path only")
            if seq_weight.dtype != torch.float32 or tuple(seq_weight.shape) != (B,) or not seq_weight.is_cuda:
                raise ValueError(f"HeadFn: seq_weight must be a CUDA fp32 tensor of shape ({B},)")
            seq_weight = seq_weight.contiguous()
        Mt, Ms = B * T, memory.shape[0] * memory.shape[1]
        if teacher is not None:
            if pk is not None or want_argmax or seq_weight is not None:
                raise ValueError("HeadFn: a teacher applies to the padded training path without seq_weight")
            t_logits, t_sc, t_gl, alpha, kd = teacher
            ok = all(t is not None and t.is_cuda and t.dtype == torch.float32 for t in (t_logits, t_sc, t_gl, kd))
            if not ok or t_logits.dim() != 2 or t_logits.shape[0] != Mt or t_logits.shape[1] < V or \
                    t_logits.stride(1) != 1 or tuple(t_sc.shape) != (B, T, S) or not t_sc.is_contiguous() or \
                    tuple(t_gl.shape) != (Mt, 2) or not t_gl.is_contiguous() or kd.numel() != Mt or \
                    not kd.is_contiguous():
                raise ValueError(f"HeadFn: the teacher needs CUDA fp32 logits [{Mt}, >= {V}], copy scores "
                                 f"[{B}, {T}, {S}], gate logits [{Mt}, 2] and a kd buffer of {Mt}")
        if sparse is not None:
            if pk is not None or want_argmax or seq_weight is not None or teacher is not None:
                raise ValueError("HeadFn: sparse targets apply to the padded training path without seq_weight or a "
                                 "teacher")
            t_label, t_prob, _, kd = sparse
            ok = all(t is not None and t.is_cuda and t.is_contiguous() for t in (t_label, t_prob, kd)) and \
                t_label.dtype == torch.int32 and t_prob.dtype == torch.float32 and kd.dtype == torch.float32
            if not ok or t_label.dim() != 2 or t_label.shape[0] != Mt or not 1 <= t_label.shape[1] <= 64 or \
                    t_prob.shape != t_label.shape or kd.numel() != Mt:
                raise ValueError(f"HeadFn: sparse targets need contiguous CUDA int32 labels and fp32 probabilities "
                                 f"[{Mt}, k] with 1 <= k <= 64 and an fp32 kd buffer of {Mt}")
        pr = Prec(bf16)
        if pf is not None and pf.event is not None:
            torch.cuda.current_stream().wait_event(pf.event)
            pf.fork.join()
            pr.wcache.update(pf.wcache)
        dev = dec.device
        f32 = dict(dtype=torch.float32, device=dev)
        st = _stream()
        memory2 = memory.contiguous().to(pr.tdt).view(Ms, D)
        dec2 = dec.contiguous().to(pr.tdt).view(Mt, D)
        dec32 = dec2 if not pr.bf16 else dec2.float()            # the 2-wide gate stays on the fp32 path
        ldl = _ld_logits(V)
        kdt = teacher is not None or sparse is not None
        if want_argmax or kdt:                        # every loss row of a teacher's batch reads its logits
            cap, vslot, vrows, dec_v = Mt, None, None, dec2
        else:
            # training: out_fc runs on the vocabulary-label rows alone, compacted into `cap` slots (a packed batch
            # bounds them by pk.Rv); no other row reads the vocabulary softmax.  A padded batch has no such bound:
            # cap = B*T, and it pays the row list and the two row copies for no gain, to keep one code path
            cap = Mt if pk is None else pk.Rv
            vslot = torch.empty((Mt,), dtype=torch.int32, device=dev)
            vrows = torch.empty((cap,), dtype=torch.int32, device=dev)
            call("fira_vocab_rows", _ptr(label), Mt, V, _ptr(vslot), _ptr(vrows), cap, st)
            dec_v = pr.empty((cap, D), dev)
            call("fira_gather_rows", _ptr(dec2), D, _ptr(vrows), _ptr(dec_v), D, cap, D, pr.code, st)
        # training only needs pointer scores of real source positions at target rows whose label is a COPY
        # label (vocabulary-label rows take their loss from the vocabulary softmax alone, Model.py:64-81); with a
        # teacher every loss row spreads over the copy positions too
        row_mask = None if want_argmax else ((label != 0) if kdt else (label >= V)).to(torch.uint8)
        logits, src, tgt, sc, gl = head_products(pr, memory2, dec2, dec32, dec_v, cap, Wout, bout, Ws, Wt, Wres, bres,
                                                 Wp, bp, B, T, S, mem_mask, row_mask,
                                                 ranges=pk.ranges if pk is not None else None)
        stats = torch.empty((Mt, 16 if teacher is not None else 10 if sparse is not None else 8), **f32)
        nll = torch.empty((Mt,), **f32)
        amax = torch.empty((Mt,), dtype=torch.int32, device=dev) if want_argmax else None
        if sparse is not None:
            loss_rows = torch.empty((Mt,), **f32)
            call("fira_pointer_mix_kd_sparse_fwd", _ptr(logits), ldl, _ptr(sc), _ptr(gl), _ptr(mem_mask), _ptr(label),
                 _ptr(t_label), _ptr(t_prob), t_label.shape[1], float(sparse[2]), _ptr(stats), _ptr(nll), _ptr(kd),
                 _ptr(loss_rows), Mt, T, V, S, pr.code, st)
        elif teacher is None:
            call("fira_pointer_mix_nll_fwd_rows", _ptr(logits), ldl, _ptr(sc), _ptr(gl), _ptr(mem_mask), _ptr(label),
                 _ptr(vslot), _ptr(stats), _ptr(nll), _ptr(amax), Mt, T, V, S, pr.code, st)
        else:
            loss_rows = torch.empty((Mt,), **f32)
            call("fira_pointer_mix_kd_fwd", _ptr(logits), ldl, _ptr(sc), _ptr(gl), _ptr(mem_mask), _ptr(label),
                 _ptr(t_logits), t_logits.stride(0), _ptr(t_sc), _ptr(t_gl), float(alpha), _ptr(stats), _ptr(nll),
                 _ptr(kd), _ptr(loss_rows), Mt, T, V, S, pr.code, st)
        ctx.misc = (pr, memory2, dec2, dec32, mem_mask, label, logits, ldl, src, tgt, sc, stats, B, T, S, V,
                    memory.dtype, dec.dtype, pk, memory.shape, cap, vslot, vrows, dec_v, seq_weight, teacher, sparse)
        ctx.save_for_backward(Wout, Ws, Wt, Wres, Wp, bout, bres, bp)
        if kdt:
            loss_sum = colsum(loss_rows, 1, Mt, 1).view(())
        elif seq_weight is None:
            loss_sum = colsum(nll, 1, Mt, 1).view(())
        else:                                      # per position t: sum_b w[b] nll[b, t], then over t
            loss_sum = colsum(colsum(nll, T, B, T, weight=seq_weight), 1, T, 1).view(())
        ids = amax.view(B, T) if want_argmax else None
        nll2 = nll.view(B, T)
        ctx.mark_non_differentiable(*([nll2, ids] if ids is not None else [nll2]))
        return loss_sum, nll2, ids

    @staticmethod
    def backward(ctx, g_loss, g_nll, g_ids):
        (pr, memory2, dec2, dec32, mem_mask, label, logits, ldl, src, tgt, sc, stats, B, T, S, V,
         mem_dt, dec_dt, pk, mem_shape, cap, vslot, vrows, dec_v, seq_weight, teacher, sparse) = ctx.misc
        Wout, Ws, Wt, Wres, Wp, bout, bres, bp = ctx.saved_tensors
        Mt, Ms = B * T, memory2.shape[0]
        dev = dec2.device
        f32 = dict(dtype=torch.float32, device=dev)
        st = _stream()
        up = g_loss.contiguous().float()
        dlogits = pr.empty((cap, ldl), dev)
        dsc = torch.empty((B, T, S), **f32)
        dgl = torch.empty((Mt, 2), **f32)
        active = torch.empty((Mt,), dtype=torch.uint8, device=dev)
        args = (_ptr(logits), ldl, _ptr(sc), _ptr(mem_mask), _ptr(label), _ptr(vslot), _ptr(vrows), cap, _ptr(stats),
                _ptr(up), _ptr(dlogits), _ptr(dsc), _ptr(dgl), _ptr(active), Mt, T, V, S, pr.code, st)
        if sparse is not None:
            t_label, t_prob, alpha, _ = sparse
            call("fira_pointer_mix_kd_sparse_bwd", _ptr(logits), ldl, _ptr(sc), _ptr(mem_mask), _ptr(label),
                 _ptr(t_label), _ptr(t_prob), t_label.shape[1], float(alpha), _ptr(stats), _ptr(up), _ptr(dlogits),
                 _ptr(dsc), _ptr(dgl), _ptr(active), Mt, T, V, S, pr.code, st)
        elif teacher is not None:
            t_logits, t_sc, _, alpha, _ = teacher
            call("fira_pointer_mix_kd_bwd", _ptr(logits), ldl, _ptr(sc), _ptr(mem_mask), _ptr(label), _ptr(t_logits),
                 t_logits.stride(0), _ptr(t_sc), float(alpha), _ptr(stats), _ptr(up), _ptr(dlogits), _ptr(dsc),
                 _ptr(dgl), _ptr(active), Mt, T, V, S, pr.code, st)
        elif seq_weight is None:
            call("fira_pointer_mix_nll_bwd_rows", *args)
        else:
            call("fira_pointer_mix_nll_bwd_rows_weighted", *args, _ptr(seq_weight))
        # pointer scores
        d_src = pr.empty((Ms, D), dev)
        d_tgt = torch.zeros((Mt, D), **f32)
        d_wres = _gdest(Wres, (1, D), zero=True)
        d_bres = _gdest(bres, (1,), zero=True)
        if pk is not None:
            call("fira_zero_pad_rows", _ptr(d_src), D, D, _ptr(pk.off), B, pk.Rc, pk.Rs, pr.code, st)
            call("fira_copy_scores_packed_bwd", _ptr(src), _ptr(tgt), _ptr(Wres), _ptr(dsc), _ptr(active), _ptr(pk.ranges),
                 _ptr(d_src), _ptr(d_tgt), _ptr(d_wres), _ptr(d_bres), B, T, S, D, pr.code, st)
        else:
            call("fira_copy_scores_bwd", _ptr(src), _ptr(tgt), _ptr(Wres), _ptr(dsc), _ptr(active), _ptr(d_src),
                 _ptr(d_tgt), _ptr(d_wres), _ptr(d_bres), B, T, S, D, pr.code, st)
        fork = Fork(dev)
        with fork(d_src, memory2):                           # three independent groups, three side streams
            d_Ws = pr.linear_dw(d_src, D, memory2, D, Ms, D, D, out=_gdest(Ws, (D, D)))
        with fork(dlogits, dec_v):
            d_bout = _gdest(bout, (V,), zero=True)
            d_Wout = pr.linear_dw(dlogits, ldl, dec_v, D, cap, V, D, out=_gdest(Wout, (V, D)), dbias=d_bout)
        with fork(dgl, dec32, d_tgt):
            d_bp = colsum(dgl, 2, Mt, 2, out=_gdest(bp, (2,), zero=True))
            d_Wp = linear_dw(dgl, 2, dec32, D, Mt, 2, D, out=_gdest(Wp, (2, D)))
            d_Wt = linear_dw(d_tgt, D, dec32, D, Mt, D, D, out=_gdest(Wt, (D, D)))
        d_mem = pr.linear_dx(d_src, D, Ws, Ms)
        # vocabulary projection (the big one), gate and target projection; d_dec accumulates in fp32
        if pr.bf16:
            d_dec = torch.empty((cap, D), **f32)
            gemm_tc(dlogits, ldl, 1, pr.w(Wout), D, 0, d_dec, D, cap, D, V,
                    splits=_tc_splits(_ceil(cap, 128), _ceil(V, 64)))
        else:
            d_dec = linear_dx(dlogits, ldl, Wout, cap)
        if vslot is not None:                      # slots -> rows; rows without a slot get zeros
            d_dec_v, d_dec = d_dec, torch.empty((Mt, D), **f32)
            call("fira_gather_rows", _ptr(d_dec_v), D, _ptr(vslot), _ptr(d_dec), D, Mt, D, FIRA_F32, st)
        linear_dx(dgl, 2, Wp, Mt, out=d_dec, accumulate=True)
        linear_dx(d_tgt, D, Wt, Mt, out=d_dec, accumulate=True)
        fork.join()
        return (None, None, None, d_mem.view(mem_shape).to(mem_dt), d_dec.view(B, T, D).to(dec_dt), None, None, d_Wout,
                d_bout, d_Ws, d_Wt, d_wres, d_bres, d_Wp, d_bp, None, None, None, None)


# ============================================================================= module-surface pieces
class LinearFn(torch.autograd.Function):
    """y = x W^T + b through fira_gemm_f32 (model.out_fc(x), run_model.py:257)."""

    @staticmethod
    def forward(ctx, x, W, b):
        _require_cuda(x, W)
        N, K = W.shape
        x2 = x.contiguous().float().view(-1, K)
        M = x2.shape[0]
        ld = (N + 3) // 4 * 4
        out = torch.empty((M, ld), dtype=torch.float32, device=x.device)
        linear(x2, W, b, out=out, ld_out=ld)
        ctx.save_for_backward(x2, W)
        ctx.has_bias = b is not None
        ctx.shape = x.shape
        return out[:, :N].view(*x.shape[:-1], N)

    @staticmethod
    def backward(ctx, dy):
        x2, W = ctx.saved_tensors
        N, K = W.shape
        M = x2.shape[0]
        dy2 = dy.contiguous().float().view(M, N)
        dx = linear_dx(dy2, N, W, M).view(ctx.shape)
        dW = linear_dw(dy2, N, x2, K, M, N, K)
        db = colsum(dy2, N, M, N) if ctx.has_bias else None
        return dx, dW, db


class CopyScoresFn(torch.autograd.Function):
    """model.copy_net(memory, tar_em) -> raw pointer scores [B,T,S] (Model.py:15-18), fp32 path."""

    @staticmethod
    def forward(ctx, memory, dec, Ws, Wt, Wres, bres):
        _require_cuda(memory, dec, Ws)
        B, S, _ = memory.shape
        T = dec.shape[1]
        memory2 = memory.contiguous().float().view(B * S, D)
        dec2 = dec.contiguous().float().view(B * T, D)
        src, tgt, sc = copy_scores_fwd(_F32, memory2, dec2, Ws, Wt, Wres, bres, B, T, S)
        ctx.misc = (memory2, dec2, src, tgt, B, T, S)
        ctx.save_for_backward(Ws, Wt, Wres)
        return sc

    @staticmethod
    def backward(ctx, dsc):
        memory2, dec2, src, tgt, B, T, S = ctx.misc
        Ws, Wt, Wres = ctx.saved_tensors
        Mt, Ms = B * T, B * S
        f32 = dict(dtype=torch.float32, device=dec2.device)
        dsc = dsc.contiguous().float()
        active = torch.ones((Mt,), dtype=torch.uint8, device=dec2.device)
        d_src = torch.empty((Ms, D), **f32)
        d_tgt = torch.zeros((Mt, D), **f32)
        d_wres = torch.zeros((1, D), **f32)
        d_bres = torch.zeros((1,), **f32)
        call("fira_copy_scores_bwd", _ptr(src), _ptr(tgt), _ptr(Wres), _ptr(dsc), _ptr(active), _ptr(d_src),
             _ptr(d_tgt), _ptr(d_wres), _ptr(d_bres), B, T, S, D, FIRA_F32, _stream())
        d_Ws = linear_dw(d_src, D, memory2, D, Ms, D, D)
        d_mem = linear_dx(d_src, D, Ws, Ms).view(B, S, D)
        d_Wt = linear_dw(d_tgt, D, dec2, D, Mt, D, D)
        d_dec = linear_dx(d_tgt, D, Wt, Mt).view(B, T, D)
        return d_mem, d_dec, d_Ws, d_Wt, d_wres, d_bres
