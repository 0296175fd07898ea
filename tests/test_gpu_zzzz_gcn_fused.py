"""The fused GCN layer kernels (csrc/gcn_fused.cu: gather -> wgmma -> LayerNorm epilogue in ONE launch per
direction) against a float64 restatement of gnn_transformer.py:74-86 on the bf16-rounded operands, and against the
three-launch CUDA sequence they replace.  Runs last (file name): a protocol bug in an mbarrier pipeline traps the context."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def seg_row(B, n, b, j):
    n0, n1, n2 = n
    j = np.asarray(j)
    return np.where(j < n0, b * n0 + j,
                    np.where(j < n0 + n1, B * n0 + b * n1 + (j - n0), B * (n0 + n1) + b * n2 + (j - n0 - n1)))


def random_graphs(B, n, seed, extra=2.0, symmetric=True):
    """per-graph COO lists with a self loop on every node + ~extra random neighbours per node"""
    rng = np.random.default_rng(seed)
    N = sum(n)
    out = []
    for b in range(B):
        m = int(extra * N / 2)
        r = rng.integers(0, N, m)
        c = rng.integers(0, N, m)
        keep = r != c
        r, c = r[keep], c[keep]
        v = rng.uniform(0.1, 1.0, r.size)
        if symmetric:
            key = np.minimum(r, c) * N + np.maximum(r, c)
            _, first = np.unique(key, return_index=True)
            r, c, v = r[first], c[first], v[first]
            r, c, v = np.concatenate((r, c)), np.concatenate((c, r)), np.concatenate((v, v))
        else:
            _, first = np.unique(r * N + c, return_index=True)
            r, c, v = r[first], c[first], v[first]
        diag = np.arange(N)
        out.append((np.concatenate((r, diag)), np.concatenate((c, diag)), np.concatenate((v, rng.uniform(0.3, 1.0, N)))))
    return out


def global_sparse(graphs, B, n):
    """float64 sparse [R, R] adjacency in buffer (segment-major) order, values rounded to fp32 like the packed CSR"""
    N = sum(n)
    rows, cols, vals = [], [], []
    for b, (r, c, v) in enumerate(graphs):
        rows.append(seg_row(B, n, b, r)); cols.append(seg_row(B, n, b, c)); vals.append(np.asarray(v, np.float32))
    idx = torch.from_numpy(np.stack((np.concatenate(rows), np.concatenate(cols)))).long()
    A = torch.sparse_coo_tensor(idx, torch.from_numpy(np.concatenate(vals)).double(), (B * N, B * N)).coalesce()
    return A.to(DEV)


def rnd(*shape, seed=0, scale=1.0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


def check(out, ref, rel, glob, what):
    out, ref = out.double(), ref.double()
    scale = ref.abs().max().item()
    bound = rel * ref.abs() + glob * scale
    over = ((out - ref).abs() - bound)
    bad = over > 0
    if bad.any():
        i = torch.nonzero(bad)[:5].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} off (worst {over.max().item():.3e} over bound, "
                             f"scale {scale:.3e}); first at {i}")


def st():
    return torch.cuda.current_stream().cuda_stream


CASES = [
    dict(B=3, n=(96, 40, 56), seed=1, extra=2.0),            # a few CTAs, one tile each, 192 rows / graph
    dict(B=4, n=(210, 160, 280), seed=2, extra=1.2),         # the reference's 650-node layout
    dict(B=48, n=(200, 104, 136), seed=3, extra=1.5),        # 21,120 rows: two tiles per CTA on 132 SMs (gather of one tile overlaps the epilogue of the other)
    dict(B=2, n=(64, 32, 32), seed=4, extra=40.0),           # dense tiles: > 1024 edges per tile (metadata read from global)
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"B{c['B']}_N{sum(c['n'])}_x{c['extra']}")
def test_gcn_layer_fwd(case):
    from fira_icse_b200 import PackedEdges, _lib, ops
    B, n = case["B"], case["n"]
    N, R = sum(n), case["B"] * sum(n)
    Mc = B * n[0]
    graphs = random_graphs(B, n, case["seed"], case["extra"])
    pe = PackedEdges.from_coo_lists(graphs, N, DEV)
    er = pe.rows_csr(*n)
    A = global_sparse(graphs, B, n)
    # the buffer-order CSR itself
    rp = er[0].long()
    assert int(rp[-1]) == pe.nnz and (rp[1:] >= rp[:-1]).all()
    H = rnd(R, 256, seed=10, dtype=BF)
    Wc = rnd(256, 256, seed=11, scale=1 / 16)
    Wc16 = Wc.to(BF)
    b2, c1 = rnd(256, seed=12, scale=0.1), rnd(256, seed=13, scale=0.1)
    gamma, beta = rnd(256, seed=14, scale=0.3) + 1.0, rnd(256, seed=15, scale=0.2)
    Z = torch.full((R, 256), 7.0, device=DEV, dtype=BF)
    outA = torch.zeros(Mc, 256, device=DEV, dtype=BF)
    outB = torch.zeros(R, 256, device=DEV, dtype=BF)
    stats = torch.zeros(2, R, device=DEV)
    _lib.call("fira_gcn_layer_fwd", er[0].data_ptr(), er[1].data_ptr(), er[2].data_ptr(), H.data_ptr(), Wc16.data_ptr(),
              b2.data_ptr(), c1.data_ptr(), gamma.data_ptr(), beta.data_ptr(), Z.data_ptr(), outA.data_ptr(),
              outB.data_ptr(), Mc, stats.data_ptr(), stats.data_ptr() + 4 * R, R, 256, 0.0, 0, None, 0, st())
    torch.cuda.synchronize()
    # float64 restatement on the rounded operands; the kernel rounds the aggregated tile to bf16 (it is the MMA operand)
    G = torch.sparse.mm(A, H.double())
    G16 = G.to(torch.float32).to(BF).double()
    rs = torch.sparse.sum(A, 1).to_dense()
    Zref = G16 @ Wc16.double().T + rs[:, None] * c1.double()[None] + b2.double()[None]
    # 2^-8 relative (one bf16 rounding) + the bf16 rounding of G entering a 256-term sum
    check(Z, Zref, 2.0 ** -8, 2.0 ** -8, "Z")
    y = Z.double() + H.double()                                   # the kernel normalises the STORED (rounded) Z
    ref = torch.nn.functional.layer_norm(y, (256,), gamma.double(), beta.double(), 1e-5)
    out = torch.cat((outA, outB[Mc:]), 0)
    check(out, ref, 2.0 ** -8, 2.0 ** -8, "LN output")
    assert (outB[:Mc] == 0).all()                                 # rows < split only go to outA
    mean, var = y.mean(1), y.var(1, unbiased=False)
    check(stats[0], mean, 1e-4, 1e-4, "mean")
    check(stats[1], (var + 1e-5).rsqrt(), 1e-3, 1e-4, "rstd")
    # against the three-launch CUDA sequence (scatter -> wgmma GEMM -> LayerNorm kernel)
    pr = ops.Prec(True)
    G3 = torch.empty(R, 256, device=DEV, dtype=BF)
    _lib.call("fira_gcn_aggregate", pe.rowptr.data_ptr(), pe.col.data_ptr(), pe.val.data_ptr(), H.data_ptr(), None,
              G3.data_ptr(), B, n[0], n[1], n[2], 256, 1, st())
    Z3 = pr.linear(G3, Wc, b2, rs=pe.rowsum(*n), rc=c1)
    check(Z, Z3.double(), 2.0 ** -7, 2.0 ** -8, "Z vs unfused")
    # dropout: the fused epilogue draws the SAME mask as fira_ln_residual_fwd for (seed, site, element)
    p, seed, sid = 0.2, 12345, 7
    _lib.call("fira_gcn_layer_fwd", er[0].data_ptr(), er[1].data_ptr(), er[2].data_ptr(), H.data_ptr(), Wc16.data_ptr(),
              b2.data_ptr(), c1.data_ptr(), gamma.data_ptr(), beta.data_ptr(), Z.data_ptr(), outA.data_ptr(),
              outB.data_ptr(), Mc, stats.data_ptr(), stats.data_ptr() + 4 * R, R, 256, p, seed, None, sid, st())
    oA, oB = torch.zeros_like(outA), torch.zeros_like(outB)
    st2 = pr.ln_fwd(Z, H, gamma, beta, oA, oB, Mc, R, p, seed, sid)
    check(torch.cat((outA, outB[Mc:]), 0), torch.cat((oA, oB[Mc:]), 0), 2.0 ** -7, 2.0 ** -7, "dropout path vs ln_fwd")
    check(stats[0], st2[0], 1e-4, 1e-4, "mean (dropout)")


@pytest.mark.parametrize("case", CASES[:3], ids=lambda c: f"B{c['B']}_N{sum(c['n'])}")
def test_gcn_layer_bwd(case):
    from fira_icse_b200 import PackedEdges, _lib
    B, n = case["B"], case["n"]
    N, R = sum(n), case["B"] * sum(n)
    graphs = random_graphs(B, n, case["seed"] + 100, case["extra"], symmetric=False)
    gt = [(c, r, v) for r, c, v in graphs]                        # the transposed adjacency, packed on its own
    pet = PackedEdges.from_coo_lists(gt, N, DEV, symmetric=False)
    ert = pet.rows_csr(*n)
    At = global_sparse(gt, B, n)
    dZ = rnd(R, 256, seed=20, dtype=BF)
    dRes = rnd(R, 256, seed=21, dtype=BF)
    Wc = rnd(256, 256, seed=22, scale=1 / 16)
    WcT16 = Wc.t().contiguous().to(BF)
    AdZ = torch.zeros(R, 256, device=DEV, dtype=BF)
    dH = torch.zeros(R, 256, device=DEV, dtype=BF)
    _lib.call("fira_gcn_layer_bwd", ert[0].data_ptr(), ert[1].data_ptr(), ert[2].data_ptr(), dZ.data_ptr(),
              WcT16.data_ptr(), dRes.data_ptr(), AdZ.data_ptr(), dH.data_ptr(), R, 256, st())
    torch.cuda.synchronize()
    ref_agg = torch.sparse.mm(At, dZ.double())
    check(AdZ, ref_agg, 2.0 ** -8, 2.0 ** -16, "A^T dZ")
    ref = AdZ.double() @ WcT16.double().T + dRes.double()         # (A^T dZ) Wc, Wc^T stored [in, out]
    check(dH, ref, 2.0 ** -8, 2.0 ** -9, "dH")
    # no addend
    _lib.call("fira_gcn_layer_bwd", ert[0].data_ptr(), ert[1].data_ptr(), ert[2].data_ptr(), dZ.data_ptr(),
              WcT16.data_ptr(), None, AdZ.data_ptr(), dH.data_ptr(), R, 256, st())
    check(dH, AdZ.double() @ WcT16.double().T, 2.0 ** -8, 2.0 ** -9, "dH (no addend)")


def test_encoder_with_fused_gcn_matches_unfused_path():
    """the whole bf16 encoder + its gradients with FIRA_GCN_FUSED=1 against FIRA_GCN_FUSED=0 on real commits"""
    import copy
    from fira_testlib import golden_batch, seeded_model
    m = copy.deepcopy(seeded_model()).to(DEV).eval().set_precision("bf16")
    batch = [b.to(DEV) for b in golden_batch(0, 8)]
    res = {}
    old = os.environ.get("FIRA_GCN_FUSED")
    try:
        for flag in ("0", "1"):
            os.environ["FIRA_GCN_FUSED"] = flag
            m.zero_grad(set_to_none=True)
            loss_sum, n_tok = m(*batch, "train")
            (loss_sum / n_tok).backward()
            res[flag] = (loss_sum.item(), {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None})
    finally:
        if old is None:
            os.environ.pop("FIRA_GCN_FUSED", None)
        else:
            os.environ["FIRA_GCN_FUSED"] = old
    l0, g0 = res["0"]
    l1, g1 = res["1"]
    assert abs(l0 - l1) <= 5e-3 * abs(l0), (l0, l1)
    worst = 1.0
    for k in g0:
        # fc_k.bias / LinearRes.bias: zero in exact arithmetic (softmax shift invariance), round-off noise here
        if g0[k].norm().item() < 1e-6 or k.endswith("fc_k.bias") or k.endswith("LinearRes.bias"):
            continue
        c = float((g0[k].double().flatten() @ g1[k].double().flatten()) / (g0[k].double().norm() * g1[k].double().norm()))
        worst = min(worst, c)
        assert c > 0.99, (k, c)
    print("fused vs unfused GCN: loss", l0, l1, "worst gradient cosine", worst)
