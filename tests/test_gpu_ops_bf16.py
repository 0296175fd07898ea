"""Per-kernel parity of the bf16 (throughput-mode) instantiations: every C-ABI entry point that takes
`dtype` is run with FIRA_BF16 on bf16-ROUNDED inputs and compared with a float64 restatement of the same op
evaluated on those rounded inputs.  The kernels accumulate in fp32 and round their outputs to bf16 once, so
the bound is one bf16 rounding of the result (2^-8 relative, element-wise) plus the fp32 round-off of the
reduction; where an op consumes a bf16-rounded intermediate of its own forward (attention / LayerNorm
backward) the bound is stated relative to the largest reference element.  The fp32 instantiations are
checked in tests/test_gpu_ops.py; the wgmma GEMM in tests/test_gpu_tc.py."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16
EPS = 2.0 ** -8            # half an ulp of bf16 is 2^-9 relative; 2^-8 leaves room for the fp32 reduction order


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def rnd16(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(BF).to(DEV)


def rnd32(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def close16(out, ref, rel=EPS, glob=0.0, what=""):
    """|out - ref| <= rel*|ref| + (glob + 2^-16)*max|ref| element-wise"""
    out, ref = out.detach().double().cpu(), ref.detach().double().cpu()
    scale = ref.abs().max().item()
    bound = rel * ref.abs() + (glob + 2.0 ** -16) * scale
    bad = (out - ref).abs() > bound
    assert not bad.any(), f"{what}: {int(bad.sum())} elements off, worst {((out - ref).abs() - bound).max().item():.3e} " \
                          f"over the bound (scale {scale:.3e})"


def st():
    return torch.cuda.current_stream().cuda_stream


def _ln_ref(z, resid, gamma, beta):
    return torch.nn.functional.layer_norm(z + resid, (256,), gamma, beta, 1e-5)


# ------------------------------------------------------------------------------------ LN block
@pytest.mark.parametrize("rows", [7, 1000, 20000])
def test_ln_residual_bf16(rows):
    from fira_icse_b200 import ops
    pr = ops.Prec(True)
    z, r = rnd16(rows, 256, seed=1), rnd16(rows, 256, seed=2)
    gamma, beta = rnd32(256, seed=3) * 0.5 + 1.0, rnd32(256, seed=4)
    split = max(1, rows // 3)
    outA, outB = torch.zeros(rows, 256, device=DEV, dtype=BF), torch.zeros(rows, 256, device=DEV, dtype=BF)
    stats = pr.ln_fwd(z, r, gamma, beta, outA, outB, split, rows, 0.0, 0, 0)
    zz, rr, gg, bb = (t.double().requires_grad_(True) for t in (z, r, gamma, beta))
    ref = _ln_ref(zz, rr, gg, bb)
    close16(outA[:split], ref[:split], what="ln fwd A")
    close16(outB[split:], ref[split:], what="ln fwd B")
    assert (outB[:split] == 0).all() and (outA[split:] == 0).all()
    go = rnd16(rows, 256, seed=5)
    ref.backward(go.double())
    dz, dres, dg, db = pr.ln_bwd(go, go, split, z, r, stats, gamma, rows, 0.0, 0, 0)
    assert dz.dtype == BF and dres.dtype == BF and dg.dtype == torch.float32
    close16(dz, zz.grad, glob=2.0 ** -9, what="ln dz")
    close16(dres, rr.grad, glob=2.0 ** -9, what="ln dres")
    close16(dg, gg.grad, rel=1e-4, glob=1e-4, what="ln dgamma")
    close16(db, bb.grad, rel=1e-4, glob=1e-4, what="ln dbeta")
    base = rnd16(rows, 256, seed=6)
    acc = base.clone()
    pr.ln_bwd(go, go, split, z, r, stats, gamma, rows, 0.0, 0, 0, d_resid=acc, accum=True)
    close16(acc, base.double() + rr.grad, glob=2.0 ** -8, what="ln dres accumulate")


def test_ln_dropout_bf16_mask_matches_fp32_mask():
    """the keep-mask is a function of (seed, site, element index) only: bf16 and fp32 kernels drop the same elements"""
    from fira_icse_b200 import ops
    rows, p, seed, sid = 1024, 0.2, 99, 3
    ones, zero = torch.ones(rows, 256, device=DEV), torch.zeros(rows, 256, device=DEV)
    g1, b0 = torch.ones(256, device=DEV), torch.zeros(256, device=DEV)
    o32 = torch.empty(rows, 256, device=DEV)
    ops.Prec(False).ln_fwd(ones, zero, g1, b0, o32, o32, rows, rows, p, seed, sid)
    o16 = torch.empty(rows, 256, device=DEV, dtype=BF)
    ops.Prec(True).ln_fwd(ones.to(BF), zero.to(BF), g1, b0, o16, o16, rows, rows, p, seed, sid)
    assert torch.equal(o32 > 0, o16 > 0)


# ------------------------------------------------------------------------------------ Combination gate
def test_comb_gate_bf16():
    from fira_icse_b200 import _lib
    rows = 3001
    qk, vtab = rnd16(rows, 512, seed=1), rnd32(4, 256, seed=2)
    mark = torch.randint(0, 4, (rows,), generator=torch.Generator().manual_seed(3)).to(torch.int32).to(DEV)
    out = torch.empty(rows, 256, device=DEV, dtype=BF)
    _lib.call("fira_comb_gate_fwd", qk.data_ptr(), 512, vtab.data_ptr(), mark.data_ptr(), out.data_ptr(), rows, 256,
              32, 0.0, 0, None, 0, 1, st())
    qkd, vd = qk.double().requires_grad_(True), vtab.double().requires_grad_(True)
    q, k, v = qkd[:, :256], qkd[:, 256:], vd[mark.long()]
    w = torch.softmax(torch.stack((q * k, q * v), -1) / math.sqrt(32), -1)     # combination_layer.py:8-14
    ref = w[..., 0] * k + w[..., 1] * v
    close16(out, ref, what="comb fwd")
    go = rnd16(rows, 256, seed=4)
    ref.backward(go.double())
    dqk = torch.empty(rows, 512, device=DEV, dtype=BF)
    dv = torch.zeros(4, 256, device=DEV)
    _lib.call("fira_comb_gate_bwd", qk.data_ptr(), 512, vtab.data_ptr(), mark.data_ptr(), go.data_ptr(),
              dqk.data_ptr(), dv.data_ptr(), rows, 256, 32, 0.0, 0, None, 0, 1, st())
    close16(dqk, qkd.grad, what="comb dqk")
    close16(dv, vd.grad, rel=1e-4, glob=1e-4, what="comb dvtab")


# ------------------------------------------------------------------------------------ graph
def test_aggregate_bf16_random_graph():
    from fira_icse_b200 import PackedEdges, _lib
    B, n0, n1, n2 = 3, 96, 40, 56
    N = n0 + n1 + n2
    g = torch.Generator().manual_seed(1)
    a = torch.rand(B, N, N, generator=g)
    a = torch.where(a > 0.97, a, torch.zeros(())) + torch.eye(N)
    pe = PackedEdges.from_dense(a.to(DEV))
    # segment-major row order
    idx = []
    for lo, n in ((0, n0), (n0, n1), (n0 + n1, n2)):
        for b in range(B):
            idx += [b * N + lo + i for i in range(n)]
    perm = torch.tensor(idx, device=DEV)
    x = rnd16(B * N, 256, seed=3)
    add = rnd16(B * N, 256, seed=4)
    y = torch.empty_like(x)
    _lib.call("fira_gcn_aggregate", pe.rowptr.data_ptr(), pe.col.data_ptr(), pe.val.data_ptr(), x.data_ptr(),
              add.data_ptr(), y.data_ptr(), B, n0, n1, n2, 256, 1, st())
    xb = torch.empty(B * N, 256, device=DEV, dtype=torch.float64)
    xb[perm] = x.double()
    ref = torch.bmm(a.to(DEV).float().double(), xb.view(B, N, 256)).view(B * N, 256)[perm] + add.double()
    close16(y, ref, what="aggregate")


# ------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("Lk,causal", [(30, 1), (370, 0), (33, 0), (136, 0)])
def test_attention_bf16(Lk, causal):
    from fira_icse_b200 import _lib
    B, H, Lq, dh = 5, 8, 30, 32
    Dm = H * dh
    q = rnd16(B * Lq, Dm, seed=1)
    kv = rnd16(B * Lk, 2 * Dm + 64, seed=2)                       # K at col 0, V at col Dm+64 (strided views)
    gm = torch.Generator().manual_seed(3)
    mask = (torch.rand(B, Lk, generator=gm) > 0.3)
    mask[:, 0] = True
    mask[1] = False if not causal else mask[1]                    # one fully masked commit (uniform softmax)
    mask_u8 = mask.to(torch.uint8).to(DEV)
    ld = kv.shape[1]
    ctx = torch.empty(B * Lq, Dm, device=DEV, dtype=BF)
    stats = torch.empty(B, H, Lq, 2, device=DEV)
    voff = Dm + 64
    _lib.call("fira_attn_fwd", q.data_ptr(), Dm, kv.data_ptr(), ld, kv.data_ptr() + voff * 2, ld, mask_u8.data_ptr(),
              causal, ctx.data_ptr(), Dm, stats.data_ptr(), B, H, Lq, Lk, dh, 1, st())
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
    # P is rounded to bf16 before the P.V product on the tensor-core path: 2^-9 per probability, i.e. at most
    # 2^-9 * max|V| on the output
    close16(ctx, ref, glob=2.0 ** -8, what="attention fwd")
    go = rnd16(B * Lq, Dm, seed=4)
    ref.backward(go.double())
    dq = torch.empty_like(q)
    dkv = torch.zeros_like(kv)
    _lib.call("fira_attn_bwd", q.data_ptr(), Dm, kv.data_ptr(), ld, kv.data_ptr() + voff * 2, ld, mask_u8.data_ptr(),
              causal, ctx.data_ptr(), go.data_ptr(), Dm, stats.data_ptr(), dq.data_ptr(), Dm, dkv.data_ptr(), ld,
              dkv.data_ptr() + voff * 2, ld, B, H, Lq, Lk, dh, 1, st())
    # backward consumes the bf16-rounded forward output (delta = dO . O) and bf16 P / dS operands
    close16(dq, qd.grad, glob=2.0 ** -6, what="attention dq")
    close16(dkv, kvd.grad, glob=2.0 ** -6, what="attention dkv")
    # masked keys get exactly zero gradient (cross-attention)
    if not causal:
        dead = ~mask.to(DEV)
        dead[1] = False
        rows = dead.view(-1)
        assert (dkv[rows][:, :Dm] == 0).all() and (dkv[rows][:, voff:voff + Dm] == 0).all()


# ------------------------------------------------------------------------------------ copy scores + head
def test_copy_scores_bf16():
    from fira_icse_b200 import _lib
    B, T, S = 3, 30, 370
    src, tgt = rnd16(B * S, 256, seed=1), rnd16(B * T, 256, seed=2)
    w, b = rnd32(1, 256, seed=3, scale=0.2), rnd32(1, seed=4)
    sc = torch.empty(B, T, S, device=DEV)
    _lib.call("fira_copy_scores_fwd", src.data_ptr(), tgt.data_ptr(), w.data_ptr(), b.data_ptr(), None, None,
              sc.data_ptr(), B, T, S, 256, 1, st())
    sd_, td_, wd, bd = (t.double().requires_grad_(True) for t in (src, tgt, w, b))
    ref = (torch.tanh(sd_.view(B, 1, S, 256) + td_.view(B, T, 1, 256)) * wd.view(1, 1, 1, 256)).sum(-1) + bd
    close16(sc, ref, rel=1e-4, glob=1e-5, what="copy scores fwd")          # fp32 output, fp32 math
    gm = torch.Generator().manual_seed(5)
    active = (torch.rand(B * T, generator=gm) > 0.7).to(torch.uint8).to(DEV)
    dsc = rnd32(B, T, S, seed=6) * active.view(B, T, 1)
    ref.backward(dsc.double())
    d_src = torch.empty_like(src)
    d_tgt = torch.zeros(B * T, 256, device=DEV)
    d_w = torch.zeros(1, 256, device=DEV)
    d_b = torch.zeros(1, device=DEV)
    _lib.call("fira_copy_scores_bwd", src.data_ptr(), tgt.data_ptr(), w.data_ptr(), dsc.data_ptr(), active.data_ptr(),
              d_src.data_ptr(), d_tgt.data_ptr(), d_w.data_ptr(), d_b.data_ptr(), B, T, S, 256, 1, st())
    close16(d_src, sd_.grad, what="copy d_src")
    close16(d_tgt, td_.grad, rel=1e-4, glob=1e-4, what="copy d_tgt")
    close16(d_w, wd.grad, rel=1e-4, glob=1e-4, what="copy d_w")
    close16(d_b, bd.grad, rel=1e-4, glob=1e-4, what="copy d_b")


def test_pointer_mix_nll_bf16():
    from fira_icse_b200 import _lib
    B, T, V, S = 4, 30, 1000, 370
    Mt = B * T
    ldl = 1024
    logits = rnd16(Mt, ldl, seed=1, scale=3.0)
    sc = rnd32(B, T, S, seed=2, scale=2.0)
    gl = rnd32(Mt, 2, seed=3)
    gm = torch.Generator().manual_seed(4)
    mask = torch.rand(B, S, generator=gm) > 0.4
    mask[:, 0] = True
    label = torch.randint(0, V + S, (Mt,), generator=gm)
    label[::5] = 0
    label[3] = V + int(torch.nonzero(~mask[0])[0])                # copy label on a masked source -> p = 0 -> clamp
    lab32 = label.to(torch.int32).to(DEV)
    mu8 = mask.to(torch.uint8).to(DEV)
    stats = torch.empty(Mt, 8, device=DEV)
    nll = torch.empty(Mt, device=DEV)
    amax = torch.empty(Mt, dtype=torch.int32, device=DEV)
    _lib.call("fira_pointer_mix_nll_fwd", logits.data_ptr(), ldl, sc.data_ptr(), gl.data_ptr(), mu8.data_ptr(),
              lab32.data_ptr(), stats.data_ptr(), nll.data_ptr(), amax.data_ptr(), Mt, T, V, S, 1, st())
    L, Sc, G = (t.double().requires_grad_(True) for t in (logits, sc, gl))
    gen = torch.softmax(L[:, :V], -1)
    cp = torch.softmax(Sc.view(Mt, S).masked_fill(~mask.to(DEV).repeat_interleave(T, 0), -1e9), -1)
    gate = torch.softmax(G, -1)
    dist = torch.cat((gate[:, :1] * gen, gate[:, 1:] * cp), -1)
    logp = torch.log(dist.clamp(min=1e-10, max=1))
    lab = label.to(DEV)
    ref = torch.nn.functional.nll_loss(logp, lab, reduction="none").masked_fill(lab == 0, 0)
    close16(nll, ref, rel=2e-5, glob=1e-6, what="nll")                      # fp32 statistics on bf16 logits
    # argmax: identical wherever the float64 top-1 / top-2 gap exceeds fp32 round-off
    top2 = logp.topk(2, -1).values
    decided = (top2[:, 0] - top2[:, 1]) > 1e-5
    assert torch.equal(amax.long()[decided], logp.argmax(-1)[decided])
    up = torch.tensor(0.37, device=DEV)
    (ref.sum() * up.double()).backward()
    dl = torch.full((Mt, ldl), 5.0, device=DEV, dtype=BF)
    dsc = torch.empty(B, T, S, device=DEV)
    dgl = torch.empty(Mt, 2, device=DEV)
    act = torch.empty(Mt, dtype=torch.uint8, device=DEV)
    _lib.call("fira_pointer_mix_nll_bwd", logits.data_ptr(), ldl, sc.data_ptr(), mu8.data_ptr(), lab32.data_ptr(),
              stats.data_ptr(), up.data_ptr(), dl.data_ptr(), dsc.data_ptr(), dgl.data_ptr(), act.data_ptr(), Mt, T,
              V, S, 1, st())
    close16(dl[:, :V], L.grad[:, :V], what="d_logits")
    close16(dsc, Sc.grad, rel=5e-5, glob=1e-6, what="d_copy_scores")
    close16(dgl, G.grad, rel=5e-5, glob=1e-6, what="d_gate")


# ------------------------------------------------------------------------------------ embeddings / pack
def test_embeddings_pack_relu_colsum_bf16():
    from fira_icse_b200 import _lib
    B, n0, n1, n2 = 3, 96, 40, 56
    gm = torch.Generator().manual_seed(0)
    V, VA = 500, 71
    sou = torch.randint(0, V, (B, n0), generator=gm, dtype=torch.int32).to(DEV)
    sub = torch.randint(0, V, (B, n1), generator=gm, dtype=torch.int32).to(DEV)
    ast = torch.randint(0, VA, (B, n2), generator=gm, dtype=torch.int32).to(DEV)
    sou[:, 50:] = 0
    emb, aemb, pe = rnd32(V, 256, seed=1), rnd32(VA, 256, seed=2), rnd32(n0, 256, seed=3)
    R, Mc = B * (n0 + n1 + n2), B * n0
    xc = torch.empty(Mc, 256, device=DEV, dtype=BF)
    rest = torch.zeros(R, 256, device=DEV, dtype=BF)
    _lib.call("fira_embed_nodes_fwd", sou.data_ptr(), sub.data_ptr(), ast.data_ptr(), emb.data_ptr(), aemb.data_ptr(),
              pe.data_ptr(), xc.data_ptr(), rest.data_ptr(), B, n0, n1, n2, 256, 1, st())
    assert torch.equal(xc.view(B, n0, 256), (emb[sou.long()] + pe[None]).to(BF))       # one rounding of the fp32 sum
    assert torch.equal(rest[Mc:Mc + B * n1].view(B, n1, 256), emb[sub.long()].to(BF))
    assert torch.equal(rest[Mc + B * n1:].view(B, n2, 256), aemb[ast.long()].to(BF))
    mem = torch.empty(B, n0 + n1, 256, device=DEV, dtype=BF)
    _lib.call("fira_pack_memory", xc.data_ptr(), rest.data_ptr(), mem.data_ptr(), B, n0, n1, 256, 1, st())
    assert torch.equal(mem, torch.cat((xc.view(B, n0, 256), rest[Mc:Mc + B * n1].view(B, n1, 256)), 1))
    dmem = rnd16(B, n0 + n1, 256, seed=5)
    dxc = torch.empty_like(xc)
    drest = torch.full_like(rest, 3.0)
    _lib.call("fira_unpack_memory", dmem.data_ptr(), dxc.data_ptr(), drest.data_ptr(), B, n0, n1, n2, 256, 1, st())
    assert torch.equal(dxc.view(B, n0, 256), dmem[:, :n0])
    assert torch.equal(drest[Mc:Mc + B * n1].view(B, n1, 256), dmem[:, n0:])
    assert (drest[Mc + B * n1:] == 0).all()
    demb, daemb = torch.zeros_like(emb), torch.zeros_like(aemb)
    drest[Mc + B * n1:] = rnd16(B * n2, 256, seed=6)
    _lib.call("fira_embed_nodes_bwd", sou.data_ptr(), sub.data_ptr(), ast.data_ptr(), dxc.data_ptr(), drest.data_ptr(),
              demb.data_ptr(), daemb.data_ptr(), B, n0, n1, n2, 256, 1, st())
    ref = torch.zeros(V, 256, device=DEV, dtype=torch.float64)
    ref.index_add_(0, sou.long().view(-1), dxc.double())
    ref.index_add_(0, sub.long().view(-1), drest[Mc:Mc + B * n1].double())
    ref[0] = 0
    close16(demb, ref, rel=1e-5, glob=1e-6, what="d_emb")                               # fp32 accumulators
    refa = torch.zeros(VA, 256, device=DEV, dtype=torch.float64)
    refa.index_add_(0, ast.long().view(-1), drest[Mc + B * n1:].double())
    refa[0] = 0
    close16(daemb, refa, rel=1e-5, glob=1e-6, what="d_ast_emb")
    T = 30
    tar = torch.randint(0, V, (B * T,), generator=gm, dtype=torch.int32).to(DEV)
    pe30 = rnd32(T, 256, seed=7)
    x = torch.empty(B * T, 256, device=DEV, dtype=BF)
    _lib.call("fira_embed_rows_fwd", tar.data_ptr(), emb.data_ptr(), pe30.data_ptr(), x.data_ptr(), B * T, T, 256, 1, st())
    assert torch.equal(x.view(B, T, 256), (emb[tar.long()].view(B, T, 256) + pe30[None]).to(BF))
    g = rnd16(B * T, 256, seed=8)
    d = torch.zeros_like(emb)
    _lib.call("fira_embed_rows_bwd", tar.data_ptr(), g.data_ptr(), d.data_ptr(), B * T, 256, 1, st())
    ref = torch.zeros(V, 256, device=DEV, dtype=torch.float64)
    ref.index_add_(0, tar.long(), g.double())
    close16(d, ref, rel=1e-5, glob=1e-6, what="d_dec_emb")
    h = rnd16(B * T, 1024, seed=9)
    dd = rnd16(B * T, 1024, seed=10)
    exp = torch.where(h > 0, dd, torch.zeros((), dtype=BF, device=DEV))
    _lib.call("fira_relu_bwd", h.data_ptr(), dd.data_ptr(), B * T * 1024, 1, st())
    assert torch.equal(dd, exp)
    y = rnd16(777, 300, seed=11)
    w = rnd32(777, seed=12)
    out = torch.zeros(296, device=DEV)
    _lib.call("fira_colsum", y.data_ptr(), 300, 777, 296, None, out.data_ptr(), 1, st())
    close16(out, y.double()[:, :296].sum(0), rel=1e-5, glob=1e-6, what="colsum")
    out.zero_()
    _lib.call("fira_colsum", y.data_ptr(), 300, 777, 296, w.data_ptr(), out.data_ptr(), 1, st())
    close16(out, (y.double()[:, :296] * w.double()[:, None]).sum(0), rel=1e-5, glob=1e-6, what="weighted colsum")
