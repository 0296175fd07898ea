"""KV-cached incremental evaluation of the Decoder for beam search (SURVEY.md section 8f rank 1).

The reference's test loop (run_model.py:187-380) re-runs the whole 30-position decoder for every beam at
every step and reads one row of the result.  The decoder is causal (gnn_transformer.py:117: pad mask AND
lower-triangular mask) and post-LN without dropout at inference, so row t of its output depends on tokens
0..t only: evaluating JUST row t against cached keys/values of rows 0..t-1 gives the same numbers.

Per batch (`start`):  cross-attention K/V of the encoder memory for all 6 layers, one GEMM
                      (the K beams of a commit share them: they are the K "query rows" of that commit).
Per step  (`step`):   embed the newest token of every beam, and per layer: QKV projection of that one row,
                      append K/V to the beam's cache, 1 x (t+1) self-attention, K x S cross-attention, FFN.
After ranking (`reorder`): caches follow their beams.

With `graphs=True` the kernel sequence of step t is captured once into a CUDA graph (one per position; all
buffers are static) and replayed for every later batch: a decoding step then costs one graph launch instead
of ~75 C-ABI calls.

The arithmetic goes through a 4-function backend (embed / linear / attention / layer-norm).  The product
backend launches the libfira_b200 kernels; there is no CPU implementation in this package (tests inject a
torch one to check the cache bookkeeping against the oracle on CPU).
"""
import torch

from . import ops
from ._lib import FIRA_BF16, FIRA_F32, call

D = ops.D


def weights_key(module, decoder=None):
    """A key that changes whenever a parameter of `module` may have changed.  `weights_epoch` of `decoder` (default:
    `module`) is bumped by engine.GraphedTrainStep after every replay: parameter updates made INSIDE a captured CUDA
    graph change neither _version nor data_ptr."""
    ps = list(module.parameters())
    return (getattr(module if decoder is None else decoder, "weights_epoch", 0),) + tuple(p._version for p in ps) + \
        tuple(p.data_ptr() for p in ps)


def replay_or_capture(graphs, key, launches):
    """Replay graphs[key]; on a miss run `launches()` (every launch on the current stream) eagerly, which gives this
    call's result and warms up the capture, then record the same launches into a CUDA graph kept as graphs[key]."""
    g = graphs.get(key)
    if g is not None:
        g.replay()
        return
    launches()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        launches()
    graphs[key] = g


class CudaBackend:
    """libfira_b200 kernels on the current stream; fp32 parity mode or bf16 throughput mode."""

    def __init__(self, bf16):
        self.bf16 = bool(bf16)
        self.tdt = torch.bfloat16 if self.bf16 else torch.float32
        self.code = FIRA_BF16 if self.bf16 else FIRA_F32
        self.pr = ops.Prec(self.bf16)

    def weight(self, W):
        """GEMM-operand form of a parameter (a bf16 copy in throughput mode)."""
        return W.detach().to(torch.bfloat16) if self.bf16 else W.detach()

    def embed(self, ids_i32, table, pos_row, out):
        rows = ids_i32.shape[0]
        call("fira_embed_rows_fwd", ops._ptr(ids_i32), ops._ptr(table), ops._ptr(pos_row), ops._ptr(out), rows, 1, D,
             self.code, ops._stream())
        return out

    def linear(self, x, Wop, b, relu=False, out=None):
        N, K = Wop.shape
        M = x.shape[0]
        if out is None:
            out = torch.empty((M, N), dtype=self.tdt, device=x.device)
        if self.bf16:
            ops.gemm_tc(x, x.stride(0), 1, Wop, K, 1, out, out.stride(0), M, N, K, bias=b, relu=relu)
        else:
            ops.gemm_raw(ops._ptr(x), x.stride(0), 1, ops._ptr(Wop), K, 1, ops._ptr(out), out.stride(0), M, N, K, bias=b,
                         relu=relu)
        return out

    def attention(self, q, k, v, key_mask, B, H, Lq, Lk):
        """q [B*Lq, D] / k, v [B*Lk, D] row-strided views; key_mask uint8 [B, Lk] -> ctx [B*Lq, D]."""
        ctx = torch.empty((B * Lq, D), dtype=self.tdt, device=q.device)
        call("fira_attn_fwd", ops._ptr(q), q.stride(0), ops._ptr(k), k.stride(0), ops._ptr(v), v.stride(0),
             ops._ptr(key_mask), 0, ops._ptr(ctx), D, None, B, H, Lq, Lk, D // H, self.code, ops._stream())
        return ctx

    def layer_norm(self, z, resid, gamma, beta):
        out = torch.empty_like(z)
        rows = z.shape[0]
        self.pr.ln_fwd(z, resid, gamma, beta, out, out, rows, rows, 0.0, 0, 0)
        return out


class IncrementalDecoder:
    """decoder = fira_icse_b200.modules.Decoder; B commits x K beams; rows are ordered (commit, beam).
    share: another IncrementalDecoder of the same B, K and tar_len whose token buffer and pad mask this one reads (the
    members of an ensemble decode the same tokens)."""

    MIN_ROWS = 128          # row count the projections run on (tensor-core tiles are 128 rows; pad rows are zeros)

    def __init__(self, decoder, B, K, tar_len, mem_len, graphs=False, backend=None, share=None):
        self.dec, self.B, self.K, self.T, self.S = decoder, B, K, tar_len, mem_len
        self.H = decoder.num_head
        self.L = len(decoder.attention_list)
        self.be = backend if backend is not None else CudaBackend(getattr(decoder, "bf16", False))
        self.use_graphs = bool(graphs) and backend is None
        dev = decoder.embedding.weight.device
        self.dev = dev
        tdt = self.be.tdt
        self.R = B * K
        self.Rp = max(self.R, self.MIN_ROWS)
        if share is None:
            self.tok = torch.zeros(self.Rp, dtype=torch.int32, device=dev)
            self.tok_mask = torch.zeros((self.R, tar_len), dtype=torch.uint8, device=dev)
        else:
            assert (share.R, share.T) == (self.R, tar_len)
            self.tok, self.tok_mask = share.tok, share.tok_mask
        self.kv_self = torch.zeros((self.L, self.R, tar_len, 2 * D), dtype=tdt, device=dev)
        self.kv_mem = torch.zeros((B * mem_len, self.L * 2 * D), dtype=tdt, device=dev)
        self.mem_mask = torch.zeros((B, mem_len), dtype=torch.uint8, device=dev)
        self.out = torch.zeros((self.Rp, D), dtype=tdt, device=dev)
        self.pos = decoder.pos_encode.to(dev)
        self.graphs = {}
        self.w = None
        self.w_version = None

    # ------------------------------------------------------------------ weights
    def _prepare_weights(self):
        """Concatenated / operand-form weights in STATIC tensors (captured graphs keep pointing at them);
        refreshed only when a parameter changed."""
        version = weights_key(self.dec)
        if version == self.w_version:
            return
        be = self.be
        layers = []
        kv_w, kv_b = [], []
        for a, c, f in zip(self.dec.attention_list, self.dec.cross_attention_list, self.dec.feed_forward_list):
            layers.append(dict(
                Wqkv=be.weight(torch.cat((a.fc_q.weight, a.fc_k.weight, a.fc_v.weight), 0)),
                bqkv=torch.cat((a.fc_q.bias, a.fc_k.bias, a.fc_v.bias), 0).detach(),
                sWo=be.weight(a.fc_o.weight), sbo=a.fc_o.bias.detach(),
                sg=a.layernorm.weight.detach(), sb=a.layernorm.bias.detach(),
                cWq=be.weight(c.fc_q.weight), cbq=c.fc_q.bias.detach(),
                cWo=be.weight(c.fc_o.weight), cbo=c.fc_o.bias.detach(),
                cg=c.layernorm.weight.detach(), cb=c.layernorm.bias.detach(),
                W1=be.weight(f.fc1.weight), b1=f.fc1.bias.detach(), W2=be.weight(f.fc2.weight), b2=f.fc2.bias.detach(),
                fg=f.layernorm.weight.detach(), fb=f.layernorm.bias.detach()))
            kv_w += [c.fc_k.weight, c.fc_v.weight]
            kv_b += [c.fc_k.bias, c.fc_v.bias]
        new = dict(layers=layers, Wkv=be.weight(torch.cat(kv_w, 0)), bkv=torch.cat(kv_b, 0).detach(),
                   emb=self.dec.embedding.weight.detach())
        if self.w is None:
            self.w = new
        else:                                   # keep the addresses the graphs captured
            for old, cur in zip(self.w["layers"], new["layers"]):
                for k in old:
                    if old[k].data_ptr() != cur[k].data_ptr():      # views of unchanged parameters need no copy
                        old[k].copy_(cur[k])
            for k in ("Wkv", "bkv"):
                self.w[k].copy_(new[k])
            if self.w["emb"].data_ptr() != new["emb"].data_ptr():
                self.w["emb"] = new["emb"]
                self.graphs.clear()
        self.w_version = version

    # ------------------------------------------------------------------ per batch
    def start(self, memory, mem_mask):
        """memory [B, S, D] (encoder output), mem_mask bool/uint8 [B, S]."""
        assert memory.shape[0] == self.B and memory.shape[1] == self.S
        self._prepare_weights()
        mem = memory.contiguous().to(self.be.tdt).view(self.B * self.S, D)
        self.be.linear(mem, self.w["Wkv"], self.w["bkv"], out=self.kv_mem)
        self.mem_mask.copy_(mem_mask.to(torch.uint8))
        self.tok_mask.zero_()
        self.kv_self.zero_()
        return self

    # ------------------------------------------------------------------ one decoding step
    def _layers(self, t):
        be, R, Rp, K, B, T, S, H = self.be, self.R, self.Rp, self.K, self.B, self.T, self.S, self.H
        X = torch.zeros((Rp, D), dtype=be.tdt, device=self.dev) if Rp > R else torch.empty((Rp, D), dtype=be.tdt,
                                                                                         device=self.dev)
        be.embed(self.tok, self.w["emb"], self.pos[t], X)
        for l, w in enumerate(self.w["layers"]):
            qkv = be.linear(X, w["Wqkv"], w["bqkv"])                                   # [Rp, 3D]
            cache = self.kv_self[l]                                                    # [R, T, 2D]
            cache[:, t].copy_(qkv[:R, D:])
            flat = cache.view(R * T, 2 * D)
            ctx = be.attention(qkv[:R, :D], flat[:, :D], flat[:, D:], self.tok_mask, R, H, 1, T)
            X1 = be.layer_norm(be.linear(self._pad(ctx), w["sWo"], w["sbo"]), X, w["sg"], w["sb"])
            q = be.linear(X1, w["cWq"], w["cbq"])
            kv = self.kv_mem[:, l * 2 * D:(l + 1) * 2 * D]
            ctx = be.attention(q[:R], kv[:, :D], kv[:, D:], self.mem_mask, B, H, K, S)
            X2 = be.layer_norm(be.linear(self._pad(ctx), w["cWo"], w["cbo"]), X1, w["cg"], w["cb"])
            hid = be.linear(X2, w["W1"], w["b1"], relu=True)
            X = be.layer_norm(be.linear(hid, w["W2"], w["b2"]), X2, w["fg"], w["fb"])
        self.out.copy_(X)

    def _pad(self, x):
        if x.shape[0] == self.Rp:
            return x
        full = torch.zeros((self.Rp, x.shape[1]), dtype=x.dtype, device=x.device)
        full[:x.shape[0]].copy_(x)
        return full

    def step(self, tokens, t, pad_id=0):
        """tokens: int64 [B*K] = token at position t of every beam -> decoder output row t, [B*K, D]
        (a view of a static buffer: consume it before the next step)."""
        self.tok[:self.R].copy_(tokens)
        self.tok_mask[:, t].copy_(tokens != pad_id)
        return self.advance(t)

    def advance(self, t):
        """Decoder output row t for the tokens already in `tok[:B*K]` and `tok_mask[:, t]` (step() fills them from the
        host side; the sampler's kernel writes them on the device)."""
        if self.use_graphs:
            replay_or_capture(self.graphs, t, lambda: self._layers(t))
        else:
            self._layers(t)
        return self.out[:self.R]

    def reorder(self, src_rows, tok_mask=True):
        """src_rows int64 [B*K]: new row r continues old row src_rows[r] (beam re-ranking).  tok_mask=False leaves the
        pad mask alone (a shared mask moved by its owner)."""
        self.kv_self.copy_(self.kv_self.index_select(1, src_rows))
        if tok_mask:
            self.tok_mask.copy_(self.tok_mask.index_select(0, src_rows))
