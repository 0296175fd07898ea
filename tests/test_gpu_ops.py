"""Per-kernel parity: every C-ABI entry point against a plain torch fp64/fp32 restatement of the
same op on the same seeded inputs (bit-exact for index work, fp32 round-off tolerances otherwise)."""
import math

import numpy as np
import pytest
import torch

from fira_testlib import golden_batch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def ops():
    from fira_icse_b200 import ops as o
    return o


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def close(a, b, rtol=1e-4, atol=1e-5):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    err = (a - b).abs().max().item()
    ref = b.abs().max().item()
    assert err <= atol + rtol * ref, f"max err {err:.3e} vs ref scale {ref:.3e}"


# ------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("M,N,K", [(1, 1, 1), (4, 256, 256), (130, 70, 50), (333, 257, 129), (1920, 256, 1024),
                                   (300, 2, 256), (257, 24650, 64), (2000, 512, 256)])
def test_gemm_forward_shapes(M, N, K):
    o = ops()
    x, W, b = rnd(M, K, seed=1), rnd(N, K, seed=2), rnd(N, seed=3)
    y = o.linear(x, W, b)
    close(y, x.double() @ W.double().T + b.double(), rtol=2e-5, atol=1e-5)
    y = o.linear(x, W, None, relu=True)
    close(y, torch.relu(x.double() @ W.double().T), rtol=2e-5, atol=1e-5)


def test_gemm_rank1_padded_ld_and_splits():
    o = ops()
    M, N, K = 515, 250, 300
    x, W, b, rs, rc = rnd(M, K, seed=1), rnd(N, K, seed=2), rnd(N, seed=3), rnd(M, seed=4), rnd(N, seed=5)
    out = torch.full((M, 256), 7.0, device=DEV)
    o.linear(x, W, b, out=out, ld_out=256, rs=rs, rc=rc)
    ref = x.double() @ W.double().T + b.double() + rs.double()[:, None] * rc.double()[None]
    close(out[:, :N], ref, rtol=2e-5)
    assert (out[:, N:] == 7.0).all()          # padding columns untouched
    for splits in (2, 5, 19):
        c = torch.empty((M, N), device=DEV)
        o.gemm_raw(o._ptr(x), K, 1, o._ptr(W), K, 1, o._ptr(c), N, M, N, K, bias=b, rs=rs, rc=rc, splits=splits)
        close(c, ref, rtol=2e-5)
    c0 = rnd(M, N, seed=9)
    c = c0.clone()
    o.gemm_raw(o._ptr(x), K, 1, o._ptr(W), K, 1, o._ptr(c), N, M, N, K, bias=b, accumulate=True, splits=1)
    close(c, c0.double() + x.double() @ W.double().T + b.double(), rtol=2e-5)
    c = c0.clone()
    o.gemm_raw(o._ptr(x), K, 1, o._ptr(W), K, 1, o._ptr(c), N, M, N, K, accumulate=True, splits=4)
    close(c, c0.double() + x.double() @ W.double().T, rtol=2e-5)


@pytest.mark.parametrize("M,N,K", [(5, 3, 2), (1920, 24650, 256), (777, 300, 130), (4, 256, 256), (41600, 256, 256)])
def test_gemm_backward_shapes(M, N, K):
    o = ops()
    dy, W, x = rnd(M, N, seed=1, scale=0.1), rnd(N, K, seed=2), rnd(M, K, seed=3)
    close(o.linear_dx(dy, N, W, M), dy.double() @ W.double(), rtol=3e-5, atol=1e-5)
    close(o.linear_dw(dy, N, x, K, M, N, K), dy.double().T @ x.double(), rtol=3e-5, atol=1e-5)
    close(o.colsum(dy, N, M, N), dy.double().sum(0), rtol=3e-5, atol=1e-5)
    w = rnd(M, seed=4)
    close(o.colsum(dy, N, M, N, weight=w), (dy.double() * w.double()[:, None]).sum(0), rtol=3e-5, atol=1e-5)


def test_gemm_small_weight_products():
    """the W2@W1, W2@b1 merges and their adjoints used by the fused GCN layer"""
    o = ops()
    D = 256
    W1, W2, b1, dWc, dc1 = rnd(D, D, seed=1), rnd(D, D, seed=2), rnd(D, seed=3), rnd(D, D, seed=4), rnd(D, seed=5)
    Wc = torch.empty(D, D, device=DEV)
    o.gemm_raw(o._ptr(W2), D, 1, o._ptr(W1), D, 0, o._ptr(Wc), D, D, D, D, splits=1)
    close(Wc, W2.double() @ W1.double(), rtol=2e-5)
    c1 = torch.empty(D, device=DEV)
    o.gemm_raw(o._ptr(W2), D, 1, o._ptr(b1), D, 1, o._ptr(c1), 1, D, 1, D, splits=1)
    close(c1, W2.double() @ b1.double(), rtol=2e-5)
    dW2 = torch.empty(D, D, device=DEV)
    o.gemm_raw(o._ptr(dWc), D, 1, o._ptr(W1), D, 1, o._ptr(dW2), D, D, D, D, rs=dc1, rc=b1, splits=1)
    close(dW2, dWc.double() @ W1.double().T + torch.outer(dc1.double(), b1.double()), rtol=2e-5)
    dW1 = torch.empty(D, D, device=DEV)
    o.gemm_raw(o._ptr(W2), D, 0, o._ptr(dWc), D, 0, o._ptr(dW1), D, D, D, D, splits=1)
    close(dW1, W2.double().T @ dWc.double(), rtol=2e-5)
    db1 = torch.empty(D, device=DEV)
    o.gemm_raw(o._ptr(W2), D, 0, o._ptr(dc1), 1, 0, o._ptr(db1), 1, D, 1, D, splits=1)
    close(db1, W2.double().T @ dc1.double(), rtol=2e-5)


# ------------------------------------------------------------------------------------ LN block
def _ln_ref(z, resid, gamma, beta, mask=None, scale=1.0):
    y = (z * mask * scale if mask is not None else z) + resid
    return torch.nn.functional.layer_norm(y, (256,), gamma, beta, 1e-5)


@pytest.mark.parametrize("rows", [2, 7, 1000, 41600])
def test_ln_residual_fwd_bwd(rows):
    o = ops()
    z, r = rnd(rows, 256, seed=1), rnd(rows, 256, seed=2)
    gamma, beta = rnd(256, seed=3) * 0.5 + 1.0, rnd(256, seed=4)
    split = max(1, rows // 3)
    outA, outB = torch.zeros(rows, 256, device=DEV), torch.zeros(rows, 256, device=DEV)
    stats = o.ln_fwd(z, r, gamma, beta, outA, outB, split, rows, 0.0, 0, 0)
    zz, rr, gg, bb = (t.double().requires_grad_(True) for t in (z, r, gamma, beta))
    ref = _ln_ref(zz, rr, gg, bb)
    close(outA[:split], ref[:split], rtol=1e-5, atol=1e-5)
    close(outB[split:], ref[split:], rtol=1e-5, atol=1e-5)
    assert (outB[:split] == 0).all() and (outA[split:] == 0).all()
    go = rnd(rows, 256, seed=5)
    ref.backward(go.double())
    dz, dres, dg, db = o.ln_bwd(go, go, split, z, r, stats, gamma, rows, 0.0, 0, 0)
    close(dz, zz.grad, rtol=2e-5, atol=1e-5)
    close(dres, rr.grad, rtol=2e-5, atol=1e-5)
    close(dg, gg.grad, rtol=1e-4, atol=1e-4)
    close(db, bb.grad, rtol=1e-4, atol=1e-4)
    # accumulate into an existing d_resid
    base = rnd(rows, 256, seed=6)
    acc = base.clone()
    o.ln_bwd(go, go, split, z, r, stats, gamma, rows, 0.0, 0, 0, d_resid=acc, accum=True)
    close(acc, base.double() + rr.grad, rtol=2e-5, atol=1e-5)


def test_ln_dropout_mask_is_consistent_between_fwd_and_bwd():
    o = ops()
    rows, p, seed, sid = 2048, 0.2, 1234567, 5
    ones, zero = torch.ones(rows, 256, device=DEV), torch.zeros(rows, 256, device=DEV)
    g1, b0 = torch.ones(256, device=DEV), torch.zeros(256, device=DEV)
    out = torch.empty(rows, 256, device=DEV)
    o.ln_fwd(ones, zero, g1, b0, out, out, rows, rows, p, seed, sid)
    mask = (out > 0).double()                    # kept entries sit above the row mean
    keep = mask.mean().item()
    assert abs(keep - (1 - p)) < 0.01, keep
    out2 = torch.empty_like(out)
    o.ln_fwd(ones, zero, g1, b0, out2, out2, rows, rows, p, seed, sid)
    assert torch.equal(out, out2)                # pure function of (seed, stream, index)
    o.ln_fwd(ones, zero, g1, b0, out2, out2, rows, rows, p, seed, sid + 1)
    assert not torch.equal(out, out2)
    z, r = rnd(rows, 256, seed=1), rnd(rows, 256, seed=2)
    gamma, beta = rnd(256, seed=3) * 0.5 + 1.0, rnd(256, seed=4)
    o_ = torch.empty_like(z)
    stats = o.ln_fwd(z, r, gamma, beta, o_, o_, rows, rows, p, seed, sid)
    zz, rr = z.double().requires_grad_(True), r.double().requires_grad_(True)
    ref = _ln_ref(zz, rr, gamma.double(), beta.double(), mask, 1.0 / (1 - p))
    close(o_, ref, rtol=1e-5, atol=1e-5)
    go = rnd(rows, 256, seed=5)
    ref.backward(go.double())
    dz, dres, _, _ = o.ln_bwd(go, go, rows, z, r, stats, gamma, rows, p, seed, sid)
    close(dz, zz.grad, rtol=2e-5, atol=1e-5)
    close(dres, rr.grad, rtol=2e-5, atol=1e-5)


# ------------------------------------------------------------------------------------ Combination gate
def test_comb_gate_fwd_bwd():
    from fira_icse_b200 import _lib
    o = ops()
    rows = 3001
    qk, vtab = rnd(rows, 512, seed=1), rnd(4, 256, seed=2)
    mark = torch.randint(0, 4, (rows,), generator=torch.Generator().manual_seed(3)).to(torch.int32).to(DEV)
    out = torch.empty(rows, 256, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    _lib.call("fira_comb_gate_fwd", qk.data_ptr(), 512, vtab.data_ptr(), mark.data_ptr(), out.data_ptr(), rows, 256,
              32, 0.0, 0, None, 0, 0, st)
    qkd, vd = qk.double().requires_grad_(True), vtab.double().requires_grad_(True)
    q, k, v = qkd[:, :256], qkd[:, 256:], vd[mark.long()]
    # reference formulation: softmax over the stacked pair (combination_layer.py:8-14)
    w = torch.softmax(torch.stack((q * k, q * v), -1) / math.sqrt(32), -1)
    ref = w[..., 0] * k + w[..., 1] * v
    close(out, ref, rtol=1e-5, atol=1e-5)
    go = rnd(rows, 256, seed=4)
    ref.backward(go.double())
    dqk = torch.empty(rows, 512, device=DEV)
    dv = torch.zeros(4, 256, device=DEV)
    _lib.call("fira_comb_gate_bwd", qk.data_ptr(), 512, vtab.data_ptr(), mark.data_ptr(), go.data_ptr(),
              dqk.data_ptr(), dv.data_ptr(), rows, 256, 32, 0.0, 0, None, 0, 0, st)
    close(dqk, qkd.grad, rtol=2e-5, atol=1e-5)
    close(dv, vd.grad, rtol=1e-4, atol=1e-4)
    # dropout: zeros of fwd and bwd coincide
    p = 0.1
    _lib.call("fira_comb_gate_fwd", qk.data_ptr(), 512, vtab.data_ptr(), mark.data_ptr(), out.data_ptr(), rows, 256,
              32, p, 99, None, 3, 0, st)
    dropped = out == 0
    assert abs(dropped.float().mean().item() - p) < 0.01
    close(out[~dropped], (ref.detach() / (1 - p))[~dropped], rtol=1e-5, atol=1e-5)
    _lib.call("fira_comb_gate_bwd", qk.data_ptr(), 512, vtab.data_ptr(), mark.data_ptr(), go.data_ptr(),
              dqk.data_ptr(), dv.data_ptr(), rows, 256, 32, p, 99, None, 3, 0, st)
    assert (dqk[:, :256][dropped] == 0).all() and (dqk[:, 256:][dropped] == 0).all()


# ------------------------------------------------------------------------------------ graph
def _seg_perm(B, n0, n1, n2):
    """segment-major row -> (b, node) flat index"""
    N = n0 + n1 + n2
    idx = []
    for lo, n in ((0, n0), (n0, n1), (n0 + n1, n2)):
        for b in range(B):
            idx += [b * N + lo + i for i in range(n)]
    return torch.tensor(idx)


def test_csr_from_dense_and_aggregate_match_dense_bmm():
    from fira_icse_b200 import PackedEdges, _lib
    B = 6
    edge = golden_batch(0, B)[5]                                  # float64 [B,650,650] as the reference feeds it
    pe = PackedEdges.from_dense(edge.to(DEV))
    assert torch.equal(pe.to_dense(torch.float32), edge.float())   # exact fp32 cast of the fp64 values
    assert pe.t().nnz == pe.nnz
    x = rnd(B * 650, 256, seed=1)
    add = rnd(B * 650, 256, seed=2)
    perm = _seg_perm(B, 210, 160, 280).to(DEV)
    st = torch.cuda.current_stream().cuda_stream
    for addend in (None, add):
        y = torch.empty_like(x)
        _lib.call("fira_gcn_aggregate", pe.rowptr.data_ptr(), pe.col.data_ptr(), pe.val.data_ptr(), x.data_ptr(),
                  addend.data_ptr() if addend is not None else None, y.data_ptr(), B, 210, 160, 280, 256, 0, st)
        xb = torch.empty(B * 650, 256, device=DEV, dtype=torch.float64)
        xb[perm] = x.double()                                     # to (b, node) order
        ref = torch.bmm(edge.to(DEV).float().double(), xb.view(B, 650, 256)).view(B * 650, 256)[perm]
        if addend is not None:
            ref = ref + addend.double()
        close(y, ref, rtol=1e-5, atol=1e-5)
        # bf16 activations (throughput mode): same sums on the bf16-rounded inputs,
        # fp32 accumulation, one bf16 rounding of the result
        x16 = x.to(torch.bfloat16)
        a16 = addend.to(torch.bfloat16) if addend is not None else None
        y16 = torch.empty_like(x16)
        _lib.call("fira_gcn_aggregate", pe.rowptr.data_ptr(), pe.col.data_ptr(), pe.val.data_ptr(), x16.data_ptr(),
                  a16.data_ptr() if a16 is not None else None, y16.data_ptr(), B, 210, 160, 280, 256, 1, st)
        xb[perm] = x16.double()
        ref16 = torch.bmm(edge.to(DEV).float().double(), xb.view(B, 650, 256)).view(B * 650, 256)[perm]
        if a16 is not None:
            ref16 = ref16 + a16.double()
        assert torch.equal(y16, ref16.to(torch.float32).to(torch.bfloat16)) or \
            (y16.double() - ref16).abs().max().item() <= 2 ** -7 * ref16.abs().max().item()
    rs = pe.rowsum(210, 160, 280)
    close(rs, edge.float().double().sum(-1).view(-1).to(DEV)[perm], rtol=1e-6, atol=1e-6)
    # packed-from-COO path (what the loader emits) is identical to dense->CSR
    coo = golden_batch(0, B, dense_edge=False)[5]
    pc = PackedEdges.from_coo_lists(coo, 650, DEV)
    assert torch.equal(pc.rowptr, pe.rowptr) and torch.equal(pc.col, pe.col) and torch.equal(pc.val, pe.val)


def test_csr_from_dense_nonsymmetric_strided_f32():
    from fira_icse_b200 import PackedEdges
    g = torch.Generator().manual_seed(0)
    a = torch.rand(3, 40, 40, generator=g)
    a = torch.where(a > 0.9, a, torch.zeros(()))
    big = torch.zeros(3, 40, 64)
    big[:, :, :40] = a
    pe = PackedEdges.from_dense(big.to(DEV)[:, :, :40])           # non-contiguous view
    assert torch.equal(pe.to_dense(torch.float32), a)
    assert torch.equal(pe.t().to_dense(torch.float32), a.transpose(1, 2))


def test_aggregate_single_segment_synthetic():
    """one segment (identity row map) against float64: a random 3 %-dense graph in fp32, and the config-5 stress graphs
    (N = 2048, about 64 neighbours per row) with an addend in fp32 and bf16"""
    from fira_icse_b200 import PackedEdges, _lib
    from fira_icse_b200.synth import synth_stress_graphs
    B, N = 3, 512
    g = torch.Generator().manual_seed(1)
    a = torch.rand(B, N, N, generator=g)
    a = torch.where(a > 0.97, a, torch.zeros(()))
    pe = PackedEdges.from_dense(a.to(DEV))
    x = rnd(B * N, 256, seed=3)
    y = torch.empty_like(x)
    _lib.call("fira_gcn_aggregate", pe.rowptr.data_ptr(), pe.col.data_ptr(), pe.val.data_ptr(), x.data_ptr(), None,
              y.data_ptr(), B, N, 0, 0, 256, 0, torch.cuda.current_stream().cuda_stream)
    close(y, torch.bmm(a.to(DEV).double(), x.double().view(B, N, 256)).view(B * N, 256), rtol=1e-5, atol=1e-5)
    B, N = 4, 2048
    pe = PackedEdges.from_coo_lists(synth_stress_graphs(0, B), N, DEV)
    a = pe.to_dense(torch.float64).to(DEV)
    for code, dt, rtol in ((0, torch.float32, 1e-5), (1, torch.bfloat16, 2 ** -7)):
        x, add = rnd(B * N, 256, seed=4).to(dt), rnd(B * N, 256, seed=5).to(dt)
        y = torch.empty_like(x)
        _lib.call("fira_gcn_aggregate", pe.rowptr.data_ptr(), pe.col.data_ptr(), pe.val.data_ptr(), x.data_ptr(),
                  add.data_ptr(), y.data_ptr(), B, N, 0, 0, 256, code, torch.cuda.current_stream().cuda_stream)
        close(y, torch.bmm(a, x.double().view(B, N, 256)).view(B * N, 256) + add.double(), rtol=rtol, atol=0)


# ------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("Lk,causal", [(30, 1), (370, 0), (33, 0)])
def test_attention_fwd_bwd(Lk, causal):
    from fira_icse_b200 import _lib
    B, H, Lq, dh = 5, 8, 30, 32
    Dm = H * dh
    q = rnd(B * Lq, Dm, seed=1)
    kv = rnd(B * Lk, 2 * Dm + 64, seed=2)                         # K at col 0, V at col Dm+64 (strided views)
    gm = torch.Generator().manual_seed(3)
    mask = (torch.rand(B, Lk, generator=gm) > 0.3)
    mask[:, 0] = True
    mask[1] = False if not causal else mask[1]                    # one fully masked commit (uniform softmax)
    mask_u8 = mask.to(torch.uint8).to(DEV)
    ld = kv.shape[1]
    ctx = torch.empty(B * Lq, Dm, device=DEV)
    stats = torch.empty(B, H, Lq, 2, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    voff = Dm + 64
    _lib.call("fira_attn_fwd", q.data_ptr(), Dm, kv.data_ptr(), ld, kv.data_ptr() + voff * 4, ld, mask_u8.data_ptr(),
              causal, ctx.data_ptr(), Dm, stats.data_ptr(), B, H, Lq, Lk, dh, 0, st)
    qd = q.double().requires_grad_(True)
    kvd = kv.double().requires_grad_(True)
    Q = qd.view(B, Lq, H, dh).transpose(1, 2)
    K = kvd[:, :Dm].reshape(B, Lk, H, dh).transpose(1, 2)
    V = kvd[:, voff:voff + Dm].reshape(B, Lk, H, dh).transpose(1, 2)
    m = mask.to(DEV)[:, None, None, :]
    if causal:
        m = m & torch.tril(torch.ones(Lq, Lk, dtype=torch.bool, device=DEV))[None, None]
    s = (Q @ K.transpose(-1, -2) / math.sqrt(dh)).masked_fill(~m, -1e9)
    ref = (torch.softmax(s, -1) @ V).transpose(1, 2).reshape(B * Lq, Dm)
    close(ctx, ref, rtol=2e-5, atol=1e-5)
    go = rnd(B * Lq, Dm, seed=4)
    ref.backward(go.double())
    dq = torch.empty_like(q)
    dkv = torch.zeros_like(kv)
    _lib.call("fira_attn_bwd", q.data_ptr(), Dm, kv.data_ptr(), ld, kv.data_ptr() + voff * 4, ld, mask_u8.data_ptr(),
              causal, ctx.data_ptr(), go.data_ptr(), Dm, stats.data_ptr(), dq.data_ptr(), Dm, dkv.data_ptr(), ld,
              dkv.data_ptr() + voff * 4, ld, B, H, Lq, Lk, dh, 0, st)
    close(dq, qd.grad, rtol=5e-5, atol=1e-5)
    close(dkv, kvd.grad, rtol=5e-5, atol=1e-5)


# ------------------------------------------------------------------------------------ copy scores + head
def test_copy_scores_fwd_bwd():
    from fira_icse_b200 import _lib
    B, T, S = 3, 30, 370
    src, tgt = rnd(B * S, 256, seed=1), rnd(B * T, 256, seed=2)
    w, b = rnd(1, 256, seed=3, scale=0.2), rnd(1, seed=4)
    sc = torch.empty(B, T, S, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    _lib.call("fira_copy_scores_fwd", src.data_ptr(), tgt.data_ptr(), w.data_ptr(), b.data_ptr(), None, None,
              sc.data_ptr(), B, T, S, 256, 0, st)
    sd_, td_, wd, bd = (t.double().requires_grad_(True) for t in (src, tgt, w, b))
    ref = (torch.tanh(sd_.view(B, 1, S, 256) + td_.view(B, T, 1, 256)) * wd.view(1, 1, 1, 256)).sum(-1) + bd
    close(sc, ref, rtol=1e-5, atol=1e-5)
    # optional masks: skipped positions are written as 0, the others are unchanged
    gmask = torch.Generator().manual_seed(11)
    sm = (torch.rand(B, S, generator=gmask) > 0.5).to(torch.uint8).to(DEV)
    rm = (torch.rand(B * T, generator=gmask) > 0.5).to(torch.uint8).to(DEV)
    sc2 = torch.full_like(sc, 7.0)
    _lib.call("fira_copy_scores_fwd", src.data_ptr(), tgt.data_ptr(), w.data_ptr(), b.data_ptr(), sm.data_ptr(),
              rm.data_ptr(), sc2.data_ptr(), B, T, S, 256, 0, st)
    keep = rm.view(B, T, 1).bool() & sm.view(B, 1, S).bool()
    assert torch.equal(sc2[keep], sc[keep]) and (sc2[~keep] == 0).all()
    gm = torch.Generator().manual_seed(5)
    active = (torch.rand(B * T, generator=gm) > 0.7).to(torch.uint8).to(DEV)
    dsc = rnd(B, T, S, seed=6) * active.view(B, T, 1)
    dsc[:, :, 5] = 0                                              # exact zeros inside active rows are skipped too
    ref.backward(dsc.double())
    d_src = torch.empty_like(src)
    d_tgt = torch.zeros_like(tgt)
    d_w = torch.zeros(1, 256, device=DEV)
    d_b = torch.zeros(1, device=DEV)
    _lib.call("fira_copy_scores_bwd", src.data_ptr(), tgt.data_ptr(), w.data_ptr(), dsc.data_ptr(), active.data_ptr(),
              d_src.data_ptr(), d_tgt.data_ptr(), d_w.data_ptr(), d_b.data_ptr(), B, T, S, 256, 0, st)
    close(d_src, sd_.grad, rtol=5e-5, atol=1e-5)
    close(d_tgt, td_.grad, rtol=5e-5, atol=1e-4)
    close(d_w, wd.grad, rtol=5e-5, atol=1e-4)
    close(d_b, bd.grad, rtol=5e-5, atol=1e-4)


def test_pointer_mix_nll_fwd_bwd():
    from fira_icse_b200 import _lib
    B, T, V, S = 4, 30, 1000, 370
    Mt = B * T
    ldl = 1024
    logits = rnd(Mt, ldl, seed=1, scale=3.0)
    sc = rnd(B, T, S, seed=2, scale=2.0)
    gl = rnd(Mt, 2, seed=3)
    gm = torch.Generator().manual_seed(4)
    mask = torch.rand(B, S, generator=gm) > 0.4
    mask[:, 0] = True
    label = torch.randint(0, V + S, (Mt,), generator=gm)
    label[::5] = 0                                                # padded positions
    label[3] = V + int(torch.nonzero(~mask[0])[0])                # copy label on a masked source -> p = 0 -> clamp
    lab32 = label.to(torch.int32).to(DEV)
    mu8 = mask.to(torch.uint8).to(DEV)
    stats = torch.empty(Mt, 8, device=DEV)
    nll = torch.empty(Mt, device=DEV)
    amax = torch.empty(Mt, dtype=torch.int32, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    _lib.call("fira_pointer_mix_nll_fwd", logits.data_ptr(), ldl, sc.data_ptr(), gl.data_ptr(), mu8.data_ptr(),
              lab32.data_ptr(), stats.data_ptr(), nll.data_ptr(), amax.data_ptr(), Mt, T, V, S, 0, st)
    # reference formulation, Model.py:54-86, in float64
    L, Sc, G = (t.double().requires_grad_(True) for t in (logits, sc, gl))
    gen = torch.softmax(L[:, :V], -1)
    cp = torch.softmax(Sc.view(Mt, S).masked_fill(~mask.to(DEV).repeat_interleave(T, 0), -1e9), -1)
    gate = torch.softmax(G, -1)
    dist = torch.cat((gate[:, :1] * gen, gate[:, 1:] * cp), -1)
    logp = torch.log(dist.clamp(min=1e-10, max=1))
    lab = label.to(DEV)
    ref = torch.nn.functional.nll_loss(logp, lab, reduction="none").masked_fill(lab == 0, 0)
    close(nll, ref, rtol=1e-5, atol=1e-5)
    assert torch.equal(amax.long().cpu(), logp.float().argmax(-1).cpu()) or \
        (amax.long().cpu() != logp.argmax(-1).cpu()).float().mean() < 0.02
    up = torch.tensor(0.37, device=DEV)
    (ref.sum() * up.double()).backward()
    dl = torch.full((Mt, ldl), 5.0, device=DEV)
    dsc = torch.empty(B, T, S, device=DEV)
    dgl = torch.empty(Mt, 2, device=DEV)
    act = torch.empty(Mt, dtype=torch.uint8, device=DEV)
    _lib.call("fira_pointer_mix_nll_bwd", logits.data_ptr(), ldl, sc.data_ptr(), mu8.data_ptr(), lab32.data_ptr(),
              stats.data_ptr(), up.data_ptr(), dl.data_ptr(), dsc.data_ptr(), dgl.data_ptr(), act.data_ptr(), Mt, T,
              V, S, 0, st)
    close(dl[:, :V], L.grad[:, :V], rtol=5e-5, atol=1e-6)
    close(dsc, Sc.grad, rtol=5e-5, atol=1e-6)
    close(dgl, G.grad, rtol=5e-5, atol=1e-6)
    copy_rows = (lab >= V) & (lab != 0)
    # active rows = copy labels that point at an unmasked source position (others have p = 0 -> clamp -> no grad)
    src_ok = mask.to(DEV).repeat_interleave(T, 0).gather(1, (lab - V).clamp(min=0).view(-1, 1)).view(-1)
    assert torch.equal(act.bool(), copy_rows & src_ok)


# ------------------------------------------------------------------------------------ embeddings / pack
def test_embeddings_and_memory_pack():
    from fira_icse_b200 import _lib
    B, n0, n1, n2 = 3, 210, 160, 280
    gm = torch.Generator().manual_seed(0)
    V, VA = 500, 71
    sou = torch.randint(0, V, (B, n0), generator=gm, dtype=torch.int32).to(DEV)
    sub = torch.randint(0, V, (B, n1), generator=gm, dtype=torch.int32).to(DEV)
    ast = torch.randint(0, VA, (B, n2), generator=gm, dtype=torch.int32).to(DEV)
    sou[:, 100:] = 0
    emb, aemb, pe = rnd(V, 256, seed=1), rnd(VA, 256, seed=2), rnd(n0, 256, seed=3)
    R, Mc = B * (n0 + n1 + n2), B * n0
    xc = torch.empty(Mc, 256, device=DEV)
    rest = torch.zeros(R, 256, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    _lib.call("fira_embed_nodes_fwd", sou.data_ptr(), sub.data_ptr(), ast.data_ptr(), emb.data_ptr(), aemb.data_ptr(),
              pe.data_ptr(), xc.data_ptr(), rest.data_ptr(), B, n0, n1, n2, 256, 0, st)
    assert torch.equal(xc.view(B, n0, 256), emb[sou.long()] + pe[None])
    assert torch.equal(rest[Mc:Mc + B * n1].view(B, n1, 256), emb[sub.long()])
    assert torch.equal(rest[Mc + B * n1:].view(B, n2, 256), aemb[ast.long()])
    mem = torch.empty(B, n0 + n1, 256, device=DEV)
    _lib.call("fira_pack_memory", xc.data_ptr(), rest.data_ptr(), mem.data_ptr(), B, n0, n1, 256, 0, st)
    assert torch.equal(mem, torch.cat((xc.view(B, n0, 256), rest[Mc:Mc + B * n1].view(B, n1, 256)), 1))
    dmem = rnd(B, n0 + n1, 256, seed=5)
    dxc = torch.empty_like(xc)
    drest = torch.full_like(rest, 3.0)
    _lib.call("fira_unpack_memory", dmem.data_ptr(), dxc.data_ptr(), drest.data_ptr(), B, n0, n1, n2, 256, 0, st)
    assert torch.equal(dxc.view(B, n0, 256), dmem[:, :n0])
    assert torch.equal(drest[Mc:Mc + B * n1].view(B, n1, 256), dmem[:, n0:])
    assert (drest[Mc + B * n1:] == 0).all()
    # dense embedding gradients, padding_idx = 0 skipped
    demb, daemb = torch.zeros_like(emb), torch.zeros_like(aemb)
    drest[Mc + B * n1:] = rnd(B * n2, 256, seed=6)
    _lib.call("fira_embed_nodes_bwd", sou.data_ptr(), sub.data_ptr(), ast.data_ptr(), dxc.data_ptr(), drest.data_ptr(),
              demb.data_ptr(), daemb.data_ptr(), B, n0, n1, n2, 256, 0, st)
    ref = torch.zeros(V, 256, device=DEV, dtype=torch.float64)
    ref.index_add_(0, sou.long().view(-1), dxc.double())
    ref.index_add_(0, sub.long().view(-1), drest[Mc:Mc + B * n1].double())
    ref[0] = 0
    close(demb, ref, rtol=1e-5, atol=1e-5)
    refa = torch.zeros(VA, 256, device=DEV, dtype=torch.float64)
    refa.index_add_(0, ast.long().view(-1), drest[Mc + B * n1:].double())
    refa[0] = 0
    close(daemb, refa, rtol=1e-5, atol=1e-5)
    # decoder rows
    T = 30
    tar = torch.randint(0, V, (B * T,), generator=gm, dtype=torch.int32).to(DEV)
    pe30 = rnd(T, 256, seed=7)
    x = torch.empty(B * T, 256, device=DEV)
    _lib.call("fira_embed_rows_fwd", tar.data_ptr(), emb.data_ptr(), pe30.data_ptr(), x.data_ptr(), B * T, T, 256, 0, st)
    assert torch.equal(x.view(B, T, 256), emb[tar.long()].view(B, T, 256) + pe30[None])
    g = rnd(B * T, 256, seed=8)
    d = torch.zeros_like(emb)
    _lib.call("fira_embed_rows_bwd", tar.data_ptr(), g.data_ptr(), d.data_ptr(), B * T, 256, 0, st)
    ref = torch.zeros(V, 256, device=DEV, dtype=torch.float64)
    ref.index_add_(0, tar.long(), g.double())
    close(d, ref, rtol=1e-5, atol=1e-5)
    h = rnd(B * T, 1024, seed=9)
    dd = rnd(B * T, 1024, seed=10)
    exp = torch.where(h > 0, dd, torch.zeros(()).to(DEV))
    _lib.call("fira_relu_bwd", h.data_ptr(), dd.data_ptr(), B * T * 1024, 0, st)
    assert torch.equal(dd, exp)


def test_bad_arguments_return_error_codes_not_crashes():
    from fira_icse_b200 import _lib
    x = rnd(8, 128, seed=1)
    with pytest.raises(_lib.FiraLibraryError, match="multiple of 8"):
        _lib.call("fira_relu_bwd", x.data_ptr(), x.data_ptr(), 7, 0, 0)
    with pytest.raises(_lib.FiraLibraryError):
        _lib.call("fira_ln_residual_fwd", x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(),
                  x.data_ptr(), 0, None, None, 8, 128, 0.0, 0, None, 0, 0, 0)
    with pytest.raises(_lib.FiraLibraryError, match="dtype"):
        _lib.call("fira_relu_bwd", x.data_ptr(), x.data_ptr(), 8, 9, 0)
