#!/usr/bin/env python
"""A/B timings of single kernels with CUDA events (warm L2 like inside a training step, 20 launches after 5 warm-ups),
at the shapes the bf16 bench step launches: attention forward/backward (FFMA vs tensor cores, FIRA_ATTN_TC), the GCN layer
(scatter + GEMM + LayerNorm vs the fused kernel, forward and backward) and the decoder forward (the per-layer launch
sequence vs fira_decoder_fwd).  One JSON line per measurement.

    python tools/bench_kernels.py [--batch 64] [--only attention|gcn|decoder]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
DEV = "cuda:0"
BF = torch.bfloat16


def timeit(fn, reps=10, iters=10, warm=3):
    """GPU time per call: `reps` back-to-back launches captured into ONE CUDA graph (no host launch overhead between
    them, the way the training step replays them), replayed `iters` times between CUDA events."""
    for _ in range(warm):
        fn()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    torch.cuda.synchronize()
    for a, b in ev:
        a.record()
        g.replay()
        b.record()
    torch.cuda.synchronize()
    us = sorted(1e3 * a.elapsed_time(b) / reps for a, b in ev)
    return {"avg_us": sum(us) / len(us), "min_us": us[0], "med_us": us[len(us) // 2], "timing": f"{reps} launches per graph replay"}


def st():
    return torch.cuda.current_stream().cuda_stream


def attention(B, out):
    """Padded cross / causal self-attention, the packed cross-attention of the bench's first synthetic batch and one
    incremental-decoding position (5 beams against 30 cached keys, no statistics), each on the FFMA kernels
    (FIRA_ATTN_TC=0) and on the tensor cores."""
    from fira_icse_b200 import _lib
    from fira_icse_b200.packed import PackedTables, pack_from_dataset
    from fira_icse_b200.synth import SynthDataset
    H, T, dh, D = 8, 30, 32, 256
    g = torch.Generator().manual_seed(0)
    cases = []
    for name, Lq, Lk, causal, valid, with_bwd in (("cross S=304 (127 valid)", T, 304, 0, 127, True),
                                                   ("cross S=370 (all valid)", T, 370, 0, 370, True),
                                                   ("self T=30 causal", T, 30, 1, 30, True),
                                                   ("incremental Lq=5 Lk=30 (no stats)", 5, 30, 0, 30, False)):
        mask = torch.zeros(B, Lk, dtype=torch.uint8)
        mask[:, :valid] = 1
        cases.append((name, Lq, torch.randn(B * Lk, 2 * D, generator=g).to(BF).to(DEV), 2 * D, mask.to(DEV), None,
                      Lk, causal, with_bwd))
    # the bench step's cross-attention: K / V of layer 0 of the [Ms, 6 layers x 512] projection of the packed memory
    pb = pack_from_dataset(PackedTables(SynthDataset(0, B, 24650, 71)), np.arange(B), 24650).to(DEV)
    Ms = pb.Rc + pb.Rs
    cases.append((f"packed cross, bench batch 0 (S={pb.S}, {int(pb.mem_mask.sum())} valid keys)", T,
                  torch.randn(Ms, 12 * D, generator=g).to(BF).to(DEV), 12 * D, pb.mem_mask, pb, pb.S, 0, True))
    for name, Lq, kv, ld, mask, pk, Lk, causal, with_bwd in cases:
        q = torch.randn(B * Lq, D, generator=g).to(BF).to(DEV)
        ctx = torch.empty(B * Lq, D, device=DEV, dtype=BF)
        stats = torch.empty(B, H, Lq, 2, device=DEV) if with_bwd else None
        go = torch.randn(B * Lq, D, generator=g).to(BF).to(DEV)
        dq, dkv = torch.empty_like(q), torch.zeros_like(kv)
        sp = stats.data_ptr() if stats is not None else None

        def fwd():
            if pk is None:
                _lib.call("fira_attn_fwd", q.data_ptr(), D, kv.data_ptr(), ld, kv.data_ptr() + D * 2, ld, mask.data_ptr(),
                          causal, ctx.data_ptr(), D, sp, B, H, Lq, Lk, dh, 1, st())
            else:
                _lib.call("fira_attn_packed_fwd", q.data_ptr(), D, kv.data_ptr(), ld, kv.data_ptr() + D * 2, ld,
                          pk.ranges.data_ptr(), kv.shape[0], mask.data_ptr(), Lk, pk.chunks, ctx.data_ptr(), D, sp, B, H,
                          Lq, dh, 1, st())

        def bwd():
            if pk is None:
                _lib.call("fira_attn_bwd", q.data_ptr(), D, kv.data_ptr(), ld, kv.data_ptr() + D * 2, ld, mask.data_ptr(),
                          causal, ctx.data_ptr(), go.data_ptr(), D, sp, dq.data_ptr(), D, dkv.data_ptr(), ld,
                          dkv.data_ptr() + D * 2, ld, B, H, Lq, Lk, dh, 1, st())
            else:
                _lib.call("fira_attn_packed_bwd", q.data_ptr(), D, kv.data_ptr(), ld, kv.data_ptr() + D * 2, ld,
                          pk.ranges.data_ptr(), kv.shape[0], mask.data_ptr(), Lk, pk.chunks, ctx.data_ptr(), go.data_ptr(),
                          D, sp, dq.data_ptr(), D, dkv.data_ptr(), ld, dkv.data_ptr() + D * 2, ld, B, H, Lq, dh, 1, st())
        for tc in ("0", "1"):
            os.environ["FIRA_ATTN_TC"] = tc
            fwd()
            out({"kernel": "attention fwd", "case": name, "tensor_cores": tc == "1", **timeit(fwd)})
            if with_bwd:
                out({"kernel": "attention bwd", "case": name, "tensor_cores": tc == "1", **timeit(bwd)})
    os.environ.pop("FIRA_ATTN_TC", None)


def gcn(B, out):
    from fira_icse_b200 import PackedEdges, _lib, ops
    from fira_icse_b200.data import trim_batch_host
    from fira_icse_b200.synth import N_NODES, synth_batch
    ids, coo = synth_batch(0, B, 24650, 71)
    t = {k: torch.from_numpy(v) for k, v in ids.items()}
    rowptr, col, val = PackedEdges.pack_host(coo, N_NODES, pin=False)
    lst = trim_batch_host([t["sou"], t["tar"], None, t["mark"], t["ast_change"], (rowptr, col, val), t["tar_label"],
                           t["sub_token"]], 24650)
    n = (lst[0].shape[1], lst[7].shape[1], lst[4].shape[1])
    N, R, Mc = sum(n), B * sum(n), B * n[0]
    pe = PackedEdges.from_host(*lst[5], B, N, DEV)
    er = pe.rows_csr(*n)
    pr = ops.Prec(True)
    H = torch.randn(R, 256, device=DEV).to(BF)
    Wc = torch.randn(256, 256, device=DEV) / 16
    Wc16, WcT16 = Wc.to(BF), Wc.t().contiguous().to(BF)
    b2, c1 = torch.randn(256, device=DEV) * 0.1, torch.randn(256, device=DEV) * 0.1
    gamma, beta = torch.ones(256, device=DEV), torch.zeros(256, device=DEV)
    rs = pe.rowsum(*n)
    G, Z = torch.empty_like(H), torch.empty_like(H)
    oA, oB = torch.empty(Mc, 256, device=DEV, dtype=BF), torch.empty_like(H)
    stats = torch.empty(2, R, device=DEV)
    p, seed = 0.2, 1234

    def unfused_fwd():
        _lib.call("fira_gcn_aggregate", pe.rowptr.data_ptr(), pe.col.data_ptr(), pe.val.data_ptr(), H.data_ptr(), None,
                  G.data_ptr(), B, n[0], n[1], n[2], 256, 1, st())
        z = pr.linear(G, Wc, b2, rs=rs, rc=c1, out=Z)
        pr.ln_fwd(z, H, gamma, beta, oA, oB, Mc, R, p, seed, 2)

    def fused_fwd():
        _lib.call("fira_gcn_layer_fwd", er[0].data_ptr(), er[1].data_ptr(), er[2].data_ptr(), H.data_ptr(), Wc16.data_ptr(),
                  b2.data_ptr(), c1.data_ptr(), gamma.data_ptr(), beta.data_ptr(), Z.data_ptr(), oA.data_ptr(),
                  oB.data_ptr(), Mc, stats.data_ptr(), stats.data_ptr() + 4 * R, R, 256, p, seed, None, 2, st())
    dZ, dRes = torch.randn(R, 256, device=DEV).to(BF), torch.randn(R, 256, device=DEV).to(BF)
    dG, dH, AdZ = torch.empty_like(H), torch.empty_like(H), torch.empty_like(H)

    def unfused_bwd():
        pr.linear_dx(dZ, 256, Wc, R, out=dG)
        _lib.call("fira_gcn_aggregate", pe.rowptr.data_ptr(), pe.col.data_ptr(), pe.val.data_ptr(), dG.data_ptr(),
                  dRes.data_ptr(), dH.data_ptr(), B, n[0], n[1], n[2], 256, 1, st())

    def fused_bwd():
        _lib.call("fira_gcn_layer_bwd", er[0].data_ptr(), er[1].data_ptr(), er[2].data_ptr(), dZ.data_ptr(),
                  WcT16.data_ptr(), dRes.data_ptr(), AdZ.data_ptr(), dH.data_ptr(), R, 256, st())
    info = {"rows": R, "segments": n, "nnz": pe.nnz}
    out({"kernel": "GCN layer fwd: scatter + wgmma GEMM + LayerNorm (3 launches)", **info, **timeit(unfused_fwd)})
    out({"kernel": "GCN layer fwd: fused (1 launch)", **info, **timeit(fused_fwd)})
    out({"kernel": "GCN layer bwd (dX path): GEMM + scatter (2 launches)", **info, **timeit(unfused_bwd)})
    out({"kernel": "GCN layer bwd (dX path): fused (1 launch)", **info, **timeit(fused_bwd)})
    # algorithmic bytes of the fused forward (SURVEY.md 8d with H in / out replacing X1 / X2): read H, write Z and out,
    # CSR metadata, the weight once per launch
    alg = 3 * R * 256 * 2 + (R + 1) * 4 + pe.nnz * 8 + 256 * 256 * 2
    out({"kernel": "GCN layer fwd fused: algorithmic bytes", "bytes": alg})


DEC_NAMES = ("wqkv", "bqkv", "swo", "sbo", "slw", "slb", "cwq", "cbq", "cwo", "cbo", "clw", "clb",
             "w1", "b1", "w2", "b2", "flw", "flb")


def decoder(B, out):
    """The bf16 decoder forward of a training step (six layers, T = 30, dropout 0.1): fira_decoder_fwd, one launch,
    against the 67-launch sequence it replaced (embedding, then per layer the q|k|v product, self-attention, Wo product,
    LayerNorm, q product, cross-attention, Wo product, LayerNorm, FFN1, FFN2, LayerNorm; products on the wgmma GEMM),
    on the bench's first packed batch and on a padded batch (S = 304, 127 valid keys).  The hoisted K/V product that
    precedes both is not timed."""
    import ctypes
    from fira_icse_b200 import _lib, ops
    from fira_icse_b200.packed import PackedTables, pack_from_dataset
    from fira_icse_b200.synth import SynthDataset
    T, H, L, F, D, V = 30, 8, 6, 1024, 256, 24650
    p, seed, sid = 0.1, 1234, 64
    g = torch.Generator().manual_seed(0)

    def r16(*s, scale=1.0):
        return (torch.randn(*s, generator=g) * scale).to(BF).to(DEV)

    def r32(*s, scale=1.0, shift=0.0):
        return (torch.randn(*s, generator=g) * scale + shift).to(DEV)
    shapes = {"wqkv": (3 * D, D), "swo": (D, D), "cwq": (D, D), "cwo": (D, D), "w1": (F, D), "w2": (D, F)}
    W = [{n: (r16(*shapes[n], scale=shapes[n][1] ** -0.5) if n in shapes else
              r32(D, scale=0.2, shift=1.0) if n.endswith("lw") else r32({"bqkv": 3 * D, "b1": F}.get(n, D), scale=0.1))
          for n in DEC_NAMES} for _ in range(L)]
    table = (ctypes.c_void_p * (18 * L))(*[w[n].data_ptr() for w in W for n in DEC_NAMES])
    tar = torch.randint(0, V, (B, T), generator=g, dtype=torch.int32).to(DEV)
    tar_mask = (torch.arange(T)[None] < torch.randint(5, T + 1, (B,), generator=g)[:, None]).to(torch.uint8).to(DEV)
    emb, pe = r32(V, D), r32(T, D)
    pb = pack_from_dataset(PackedTables(SynthDataset(0, B, V, 71)), np.arange(B), V).to(DEV)
    pad_mask = torch.zeros(B, 304, dtype=torch.uint8, device=DEV)
    pad_mask[:, :127] = 1
    Mt = B * T
    bf = dict(dtype=BF, device=DEV)
    f32 = dict(dtype=torch.float32, device=DEV)
    for name, Ms, mask, pk, S in ((f"packed, bench batch 0 (S={pb.S}, {int(pb.mem_mask.sum())} valid keys)",
                                   pb.Rc + pb.Rs, pb.mem_mask, pb, pb.S),
                                  ("padded S=304 (127 valid keys)", B * 304, pad_mask, None, 304)):
        KV = r16(Ms, L * 2 * D)
        ldkv = L * 2 * D
        Xs = torch.empty(L + 1, Mt, D, **bf)
        QKV, Hh = torch.empty(L, Mt, 3 * D, **bf), torch.empty(L, Mt, F, **bf)
        ctx1, Z1, X1, Q, ctx2, Z2, X2, Z3 = torch.empty(8, L, Mt, D, **bf)
        st1, st2 = torch.empty(2, L, B, H, T, 2, **f32)
        ls1, ls2, ls3 = torch.empty(3, L, 2, Mt, **f32)

        def fused():
            _lib.call("fira_decoder_fwd", tar.data_ptr(), emb.data_ptr(), pe.data_ptr(), tar_mask.data_ptr(), KV.data_ptr(),
                      ldkv, mask.data_ptr(), pk.ranges.data_ptr() if pk is not None else None, S, ctypes.addressof(table),
                      L, *[t.data_ptr() for t in (Xs, QKV, ctx1, st1, Z1, ls1, X1, Q, ctx2, st2, Z2, ls2, X2, Hh, Z3, ls3)],
                      B, T, p, seed, None, sid, st())
        pr = ops.Prec(True)

        def sequence():
            _lib.call("fira_embed_rows_fwd", tar.data_ptr(), emb.data_ptr(), pe.data_ptr(), Xs[0].data_ptr(), Mt, T, D, 1, st())
            for i, w in enumerate(W):
                X = Xs[i]
                ops.gemm_tc(X, D, 1, w["wqkv"], D, 1, QKV[i], 3 * D, Mt, 3 * D, D, bias=w["bqkv"])
                q = QKV[i].data_ptr()
                _lib.call("fira_attn_fwd", q, 3 * D, q + 2 * D, 3 * D, q + 4 * D, 3 * D, tar_mask.data_ptr(), 1,
                          ctx1[i].data_ptr(), D, st1[i].data_ptr(), B, H, T, T, 32, 1, st())
                ops.gemm_tc(ctx1[i], D, 1, w["swo"], D, 1, Z1[i], D, Mt, D, D, bias=w["sbo"])
                pr.ln_fwd(Z1[i], X, w["slw"], w["slb"], X1[i], X1[i], Mt, Mt, p, seed, sid + 8 * i)
                ops.gemm_tc(X1[i], D, 1, w["cwq"], D, 1, Q[i], D, Mt, D, D, bias=w["cbq"])
                k = KV.data_ptr() + 2 * i * 2 * D
                if pk is not None:
                    _lib.call("fira_attn_packed_fwd", Q[i].data_ptr(), D, k, ldkv, k + 2 * D, ldkv, pk.ranges.data_ptr(),
                              Ms, mask.data_ptr(), S, pk.chunks, ctx2[i].data_ptr(), D, st2[i].data_ptr(), B, H, T, 32, 1,
                              st())
                else:
                    _lib.call("fira_attn_fwd", Q[i].data_ptr(), D, k, ldkv, k + 2 * D, ldkv, mask.data_ptr(), 0,
                              ctx2[i].data_ptr(), D, st2[i].data_ptr(), B, H, T, S, 32, 1, st())
                ops.gemm_tc(ctx2[i], D, 1, w["cwo"], D, 1, Z2[i], D, Mt, D, D, bias=w["cbo"])
                pr.ln_fwd(Z2[i], X1[i], w["clw"], w["clb"], X2[i], X2[i], Mt, Mt, p, seed, sid + 8 * i + 1)
                ops.gemm_tc(X2[i], D, 1, w["w1"], D, 1, Hh[i], F, Mt, F, D, bias=w["b1"], relu=True)
                ops.gemm_tc(Hh[i], F, 1, w["w2"], F, 1, Z3[i], D, Mt, D, F, bias=w["b2"])
                pr.ln_fwd(Z3[i], X2[i], w["flw"], w["flb"], Xs[i + 1], Xs[i + 1], Mt, Mt, p, seed, sid + 8 * i + 2)
        sequence()
        ref = Xs[L].float().clone()
        fused()
        torch.cuda.synchronize()
        info = {"case": name, "commits": B,
                "max_abs_diff_output_vs_sequence": (Xs[L].float() - ref).abs().max().item()}
        out({"kernel": "decoder forward: 67-launch sequence", **info, **timeit(sequence, reps=2)})
        out({"kernel": "decoder forward: fira_decoder_fwd (1 launch)", **info, **timeit(fused, reps=2)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--only", choices=["attention", "gcn", "decoder"], default=None)
    a = ap.parse_args()
    import __graft_entry__
    __graft_entry__.build()

    def out(d):
        print(json.dumps(d), flush=True)
    for name, fn in (("attention", attention), ("gcn", gcn), ("decoder", decoder)):
        if a.only in (None, name):
            fn(a.batch, out)


if __name__ == "__main__":
    main()
