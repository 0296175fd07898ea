"""Every dropout-masking kernel against the rule of tests/philox_rule.py, in fp32 and bf16: the forward against a
float64 restatement that applies the rule's mask (one wrong mask bit is an O(1) error at these bounds), the backward's
exact zeros against the rule's dropped set bit for bit (the upstream gradients contain no zeros), and the sampler's
Philox draws against sample_uniform.  Edge cases: seed_ctr NULL and set, seeds whose low word overflows into the high
word with the counter, 2^62 - 1 and 2^64 - 1, p in {0.1, 0.2, 0.3}, and row counts that take more than one pass of the
kernels' grid-stride loops (41,600 rows: 132 SMs x 16 CTAs x 8 rows = 16,896 rows per forward pass)."""
import ctypes
import functools
import math

import numpy as np
import pytest
import torch

import philox_rule as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16
EPS = 2.0 ** -8

# (seed, seed_ctr or None, p)
CASES = [
    (0, None, 0.1),
    (2 ** 32 - 1, 1, 0.2),                 # seed + counter carries into the high key word
    (2 ** 62 - 1, None, 0.3),              # the largest seed ops.make_seed draws
    (2 ** 64 - 1, 1, 0.1),                 # wraps to key 0
    (0x0123456789ABCDEF, 2 ** 40 + 3, 0.2),
]
ROWS = 41600


def _case_id(c):
    return f"seed{c[0]:#x}_ctr{c[1]}_p{c[2]}"


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def st():
    return torch.cuda.current_stream().cuda_stream


def rnd(*shape, seed=0, scale=1.0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(*shape, generator=g) * scale
    x = torch.where(x == 0, torch.full_like(x, 0.5), x)          # upstream gradients without zeros
    return x.to(dtype).to(DEV)


@functools.lru_cache(maxsize=64)
def keep(seed, ctr, sid, rows, p):
    """the rule's keep mask [rows, 256] on the device"""
    return torch.from_numpy(R.keep_mask(seed, ctr or 0, sid, rows, p)).to(DEV)


def ctr_tensor(ctr):
    return None if ctr is None else torch.tensor([ctr], dtype=torch.int64, device=DEV)


def ptr(t):
    return None if t is None else t.data_ptr()


def close(out, ref, bf16, rtol=1e-5, atol=1e-5, glob16=0.0, what=""):
    """fp32: |out - ref| <= atol + rtol max|ref|; bf16: element-wise 2^-8 |ref| + (glob16 + 2^-16) max|ref|"""
    out, ref = out.detach().double(), ref.detach().double()
    scale = ref.abs().max().item()
    if bf16:
        bound = EPS * ref.abs() + (glob16 + 2.0 ** -16) * scale
    else:
        bound = torch.full_like(ref, atol + rtol * scale)
    bad = (out - ref).abs() > bound
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.numel()} elements off, worst " \
                          f"{((out - ref).abs() - bound).max().item():.3e} over the bound (scale {scale:.3e})"


def apart(k, v):
    """k moved off v where they are equal: at k == v the gate's d_q is exactly zero whatever the mask (d/dq of
    v + sigmoid(s q (k - v)) (k - v) vanishes), which in bf16 happens for ~1 element in 1,000"""
    return torch.where(k == v, k + 0.25, k)


def same_zeros(t, k, what):
    """exact zeros of t [rows, 256] == the rule's dropped set"""
    z = t == 0
    if not torch.equal(z, ~k):
        extra, missing = int((z & k).sum()), int((~z & ~k).sum())
        raise AssertionError(f"{what}: {extra} zeros where the rule keeps, {missing} non-zeros where it drops")


# ------------------------------------------------------------------------------------ LayerNorm block
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_ln_residual_applies_the_rule(case, bf16):
    from fira_icse_b200 import ops
    seed, ctr, p = case
    rows, sid = ROWS, 37
    tdt = BF if bf16 else torch.float32
    pr = ops.Prec(bf16, seed_ctr=ctr_tensor(ctr))
    z, r = rnd(rows, 256, seed=1, dtype=tdt), rnd(rows, 256, seed=2, dtype=tdt)
    gamma, beta = rnd(256, seed=3) * 0.5 + 1.0, rnd(256, seed=4)
    split = rows // 3
    outA, outB = (torch.zeros(rows, 256, device=DEV, dtype=tdt) for _ in range(2))
    stats = pr.ln_fwd(z, r, gamma, beta, outA, outB, split, rows, p, seed, sid)
    k = keep(seed, ctr, sid, rows, p)
    zz, rr, gg, bb = (t.double().requires_grad_(True) for t in (z, r, gamma, beta))
    y = zz * k * R.keep_scale(p) + rr
    ref = torch.nn.functional.layer_norm(y, (256,), gg, bb, 1e-5)
    assert (outB[:split] == 0).all() and (outA[split:] == 0).all()
    close(torch.cat((outA[:split], outB[split:])), ref, bf16, what="LN output")
    close(stats[0], y.detach().mean(1), False, rtol=1e-5, atol=1e-6, what="mean")
    # backward: rows < split read the gradient of outA, the others that of outB; d_resid accumulates
    gA, gB = rnd(rows, 256, seed=5, dtype=tdt), rnd(rows, 256, seed=6, dtype=tdt)
    ref.backward(torch.cat((gA[:split], gB[split:])).double())
    base = rnd(rows, 256, seed=7, dtype=tdt)
    acc = base.clone()
    dz, _, dg, db = pr.ln_bwd(gA, gB, split, z, r, stats, gamma, rows, p, seed, sid, d_resid=acc, accum=True)
    same_zeros(dz, k, "d_z")
    close(dz, zz.grad, bf16, rtol=2e-5, atol=1e-5, glob16=2.0 ** -9, what="d_z")
    close(acc, base.double() + rr.grad, bf16, rtol=2e-5, atol=1e-5, glob16=2.0 ** -8, what="d_resid accumulate")
    close(dg, gg.grad, False, rtol=1e-4, atol=1e-4, what="d_gamma")
    close(db, bb.grad, False, rtol=1e-4, atol=1e-4, what="d_beta")


# ------------------------------------------------------------------------------------ Combination gates
def _gate(q, k, v):
    """combination_layer.py:8-14: softmax over the stacked pair"""
    w = torch.softmax(torch.stack((q * k, q * v), -1) / math.sqrt(32), -1)
    return w[..., 0] * k + w[..., 1] * v


@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_comb_gate_applies_the_rule(case, bf16):
    from fira_icse_b200 import _lib
    seed, ctr, p = case
    rows, sid = ROWS, 8
    tdt, code = (BF, 1) if bf16 else (torch.float32, 0)
    c = ctr_tensor(ctr)
    qk, vtab = rnd(rows, 512, seed=1, dtype=tdt), rnd(4, 256, seed=2)
    mark = torch.randint(0, 4, (rows,), generator=torch.Generator().manual_seed(3)).to(torch.int32).to(DEV)
    qk[:, 256:] = apart(qk[:, 256:].float(), vtab[mark.long()]).to(tdt)
    out = torch.empty(rows, 256, device=DEV, dtype=tdt)
    _lib.call("fira_comb_gate_fwd", qk.data_ptr(), 512, vtab.data_ptr(), mark.data_ptr(), out.data_ptr(), rows, 256,
              32, p, seed, ptr(c), sid, code, st())
    k = keep(seed, ctr, sid, rows, p)
    same_zeros(out, k, "gate output")
    qkd, vd = qk.double().requires_grad_(True), vtab.double().requires_grad_(True)
    ref = _gate(qkd[:, :256], qkd[:, 256:], vd[mark.long()]) * k * R.keep_scale(p)
    close(out, ref, bf16, what="gate output")
    go = rnd(rows, 256, seed=4, dtype=tdt)
    ref.backward(go.double())
    dqk = torch.empty(rows, 512, device=DEV, dtype=tdt)
    dv = torch.zeros(4, 256, device=DEV)
    _lib.call("fira_comb_gate_bwd", qk.data_ptr(), 512, vtab.data_ptr(), mark.data_ptr(), go.data_ptr(),
              dqk.data_ptr(), dv.data_ptr(), rows, 256, 32, p, seed, ptr(c), sid, code, st())
    same_zeros(dqk[:, :256], k, "d_q")
    same_zeros(dqk[:, 256:], k, "d_k")
    close(dqk, qkd.grad, bf16, rtol=2e-5, atol=1e-5, what="d_qk")
    close(dv, vd.grad, False, rtol=1e-4, atol=1e-4, what="d_vtab")


@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_comb_gate3_applies_the_rule(case, bf16):
    from fira_icse_b200 import _lib
    seed, ctr, p = case
    rows, sid = ROWS, 0
    tdt, code = (BF, 1) if bf16 else (torch.float32, 0)
    c = ctr_tensor(ctr)
    q, kk, v = (rnd(rows, 256, seed=s, dtype=tdt) for s in (1, 2, 3))
    kk = apart(kk, v)
    out = torch.empty(rows, 256, device=DEV, dtype=tdt)
    _lib.call("fira_comb_gate3_fwd", q.data_ptr(), kk.data_ptr(), v.data_ptr(), out.data_ptr(), rows, 256, 32, p, seed,
              ptr(c), sid, code, st())
    k = keep(seed, ctr, sid, rows, p)
    same_zeros(out, k, "gate3 output")
    qd, kd, vd = (t.double().requires_grad_(True) for t in (q, kk, v))
    ref = _gate(qd, kd, vd) * k * R.keep_scale(p)
    close(out, ref, bf16, what="gate3 output")
    go = rnd(rows, 256, seed=4, dtype=tdt)
    ref.backward(go.double())
    dq, dk, dv = (torch.empty(rows, 256, device=DEV, dtype=tdt) for _ in range(3))
    _lib.call("fira_comb_gate3_bwd", q.data_ptr(), kk.data_ptr(), v.data_ptr(), go.data_ptr(), dq.data_ptr(),
              dk.data_ptr(), dv.data_ptr(), rows, 256, 32, p, seed, ptr(c), sid, code, st())
    for name, got, want in (("d_q", dq, qd.grad), ("d_k", dk, kd.grad), ("d_v", dv, vd.grad)):
        same_zeros(got, k, name)
        close(got, want, bf16, rtol=2e-5, atol=1e-5, what=name)


# ------------------------------------------------------------------------------------ fused GCN layer (bf16)
@pytest.mark.parametrize("ci", range(4), ids=lambda i: f"gcn_case{i}")
def test_gcn_layer_fwd_applies_the_rule(ci):
    from fira_icse_b200 import PackedEdges, _lib
    from test_gpu_zzzz_gcn_fused import CASES as GCN_CASES, check, global_sparse, random_graphs
    case = GCN_CASES[ci]
    seed, ctr, p = CASES[ci + 1]
    sid = 5 * 8 + 2
    B, n = case["B"], case["n"]
    N, Rn = sum(n), case["B"] * sum(n)
    Mc = B * n[0]
    graphs = random_graphs(B, n, case["seed"], case["extra"])
    er = PackedEdges.from_coo_lists(graphs, N, DEV).rows_csr(*n)
    H = rnd(Rn, 256, seed=10, dtype=BF)
    Wc16 = rnd(256, 256, seed=11, scale=1 / 16).to(BF)
    b2, c1 = rnd(256, seed=12, scale=0.1), rnd(256, seed=13, scale=0.1)
    gamma, beta = rnd(256, seed=14, scale=0.3) + 1.0, rnd(256, seed=15, scale=0.2)
    Z = torch.full((Rn, 256), 7.0, device=DEV, dtype=BF)
    outA = torch.zeros(Mc, 256, device=DEV, dtype=BF)
    outB = torch.zeros(Rn, 256, device=DEV, dtype=BF)
    stats = torch.zeros(2, Rn, device=DEV)
    c = ctr_tensor(ctr)
    _lib.call("fira_gcn_layer_fwd", er[0].data_ptr(), er[1].data_ptr(), er[2].data_ptr(), H.data_ptr(), Wc16.data_ptr(),
              b2.data_ptr(), c1.data_ptr(), gamma.data_ptr(), beta.data_ptr(), Z.data_ptr(), outA.data_ptr(),
              outB.data_ptr(), Mc, stats.data_ptr(), stats.data_ptr() + 4 * Rn, Rn, 256, p, seed, ptr(c), sid, st())
    torch.cuda.synchronize()
    # Z itself is undropped (the backward recomputes the mask from it): one bf16 rounding of the float64 product
    A = global_sparse(graphs, B, n)
    G16 = torch.sparse.mm(A, H.double()).to(torch.float32).to(BF).double()
    rs = torch.sparse.sum(A, 1).to_dense()
    check(Z, G16 @ Wc16.double().T + rs[:, None] * c1.double()[None] + b2.double()[None], 2.0 ** -8, 2.0 ** -8, "Z")
    k = keep(seed, ctr, sid, Rn, p)
    y = Z.double() * k * R.keep_scale(p) + H.double()                # the epilogue drops the stored (rounded) Z
    ref = torch.nn.functional.layer_norm(y, (256,), gamma.double(), beta.double(), 1e-5)
    check(torch.cat((outA, outB[Mc:]), 0), ref, 2.0 ** -8, 2.0 ** -8, "LN output")
    assert (outB[:Mc] == 0).all()
    check(stats[0], y.mean(1), 1e-4, 1e-4, "mean")


# ------------------------------------------------------------------------------------ persistent decoder forward
DEC_CASES = ["padded T=30", "padded T=32", "packed hand T=30", "packed golden T=30"]


@pytest.mark.parametrize("ci", range(4), ids=lambda i: DEC_CASES[i])
def test_decoder_fwd_applies_the_rule(ci):
    """all 18 LayerNorm sites of fira_decoder_fwd (6 layers x self-attention, cross-attention, FFN) against the float64
    LayerNorm of the kernel's own z and residual under the rule's mask, with a non-zero base stream id"""
    from fira_icse_b200 import _lib
    from test_gpu_decoder_fwd import CASES as D_CASES, L, ln
    bt = D_CASES[DEC_CASES[ci]]()
    seed, ctr, p = CASES[ci]
    base = 16
    sid0 = base + R.DEC_OFFSET                          # what DecoderFn passes: stream_base + 64
    B, T = bt.B, bt.T
    Mt, D, F, H = B * T, 256, 1024, 8
    nan = float("nan")

    def e(*shape, dtype=BF):
        return torch.full(shape, nan, dtype=dtype, device=DEV)
    o = {"X": e(L + 1, Mt, D), "qkv": e(L, Mt, 3 * D), "hh": e(L, Mt, F)}
    for nm in ("ctx1", "z1", "x1", "q", "ctx2", "z2", "x2", "z3"):
        o[nm] = e(L, Mt, D)
    for nm in ("st1", "st2"):
        o[nm] = e(L, B, H, T, 2, dtype=torch.float32)
    for nm in ("ls1", "ls2", "ls3"):
        o[nm] = e(L, 2, Mt, dtype=torch.float32)
    q = {k: v.data_ptr() for k, v in o.items()}
    c = ctr_tensor(ctr)
    _lib.call("fira_decoder_fwd", bt.tar.data_ptr(), bt.emb.data_ptr(), bt.pe.data_ptr(), bt.tar_mask.data_ptr(),
              bt.kv.data_ptr(), bt.kv.shape[1], bt.mem_mask.data_ptr(),
              bt.ranges.data_ptr() if bt.ranges is not None else None, bt.S, ctypes.addressof(bt.table), L,
              q["X"], q["qkv"], q["ctx1"], q["st1"], q["z1"], q["ls1"], q["x1"], q["q"], q["ctx2"],
              q["st2"], q["z2"], q["ls2"], q["x2"], q["hh"], q["z3"], q["ls3"], B, T, float(p), seed, ptr(c), sid0, st())
    torch.cuda.synchronize()
    sites = ("self_attn", "cross_attn", "ffn")
    for i, w in enumerate(bt.w):
        for s, (z, res, out, ls, g, be) in enumerate(((o["z1"][i], o["X"][i], o["x1"][i], o["ls1"][i], w["slw"], w["slb"]),
                                                      (o["z2"][i], o["x1"][i], o["x2"][i], o["ls2"][i], w["clw"], w["clb"]),
                                                      (o["z3"][i], o["x2"][i], o["X"][i + 1], o["ls3"][i], w["flw"], w["flb"]))):
            sid = R.decoder_sid(base, i, sites[s])
            assert sid == sid0 + 8 * i + s
            zd = z.double() * keep(seed, ctr, sid, Mt, p) * R.keep_scale(p)
            ref, mean, rstd = ln(zd, res, g, be)
            close(out, ref, True, what=f"L{i} {sites[s]} LayerNorm")
            close(ls[0], mean, False, rtol=1e-5, atol=1e-6, what=f"L{i} {sites[s]} mean")
    assert not any(bool(t.isnan().any()) for t in o.values())


# ------------------------------------------------------------------------------------ sampler
def _sample(logits, sc, gl, mem_mask, copy_src, N, V, k, top_p, seed, first, pos, temp=1.0):
    """one fira_pointer_mix_sample step at position `pos` with the Philox draw (uniforms = NULL) -> (raw, log-prob)"""
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import FIRA_BF16, FIRA_F32, call
    Rr, S = logits.shape[0], sc.shape[-1]
    i32 = dict(dtype=torch.int32, device=DEV)
    ld = pos + 2
    nxt = torch.zeros(Rr, **i32)
    seq, raw = torch.zeros((Rr, ld), **i32), torch.zeros((Rr, ld), **i32)
    tlp = torch.zeros((Rr, ld), dtype=torch.float32, device=DEV)
    msk = torch.zeros((Rr, ld), dtype=torch.uint8, device=DEV)
    fin = torch.zeros(Rr, dtype=torch.uint8, device=DEV)
    length = torch.full((Rr,), pos + 1, **i32)
    lp = torch.zeros(Rr, dtype=torch.float32, device=DEV)
    seed_t = torch.tensor([seed - 2 ** 64 if seed >= 2 ** 63 else seed], dtype=torch.int64, device=DEV)
    first_t = torch.tensor([first], **i32)
    P = ops._ptr
    call("fira_pointer_mix_sample", P(logits), logits.stride(0), P(sc), P(gl), P(mem_mask), P(copy_src), P(seed_t),
         P(first_t), None, float(temp), int(k), float(top_p), -1, 0, P(nxt), P(seq), P(raw), P(tlp), P(msk), ld, pos,
         P(fin), P(length), P(lp), Rr // N, N, V, S, FIRA_BF16 if logits.dtype == torch.bfloat16 else FIRA_F32,
         ops._stream())
    torch.cuda.synchronize()
    return raw[:, pos + 1].cpu().numpy(), tlp[:, pos + 1].cpu().numpy()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_sampler_philox_draws_follow_the_rule(dtype):
    from sample_rule import draw, mixture
    from test_gpu_sample import _inputs
    V, S, B, N = 61, 13, 3, 4
    Rr = B * N
    gen = torch.Generator().manual_seed(21 + (dtype == torch.bfloat16))
    logits, sc, gl, mem_mask, copy_src = _inputs(gen, B, N, V, S, dtype)
    x = logits.float().cpu().numpy()[:, :V].astype(np.float64)
    scn, gln, mk = sc.cpu().numpy().reshape(Rr, S), gl.cpu().numpy(), mem_mask.cpu().numpy()
    rows = [mixture(x[r], scn[r], gln[r], mk[r // N]) for r in range(Rr)]
    checked = skipped = 0
    for seed, first, pos in [(0xC0FFEE0012345678, 5, 7), (2 ** 64 - 1, 0, 1), (2 ** 32 + 9, 1000, 28)]:
        for k, top_p in [(0, 1.0), (5, 1.0), (0, 0.9)]:
            raw, _ = _sample(logits, sc, gl, mem_mask, copy_src, N, V, k, top_p, seed, first, pos)
            for r in range(Rr):
                u = float(R.sample_uniform(seed, first, r // N, r % N, pos))
                ref, near = draw(rows[r], mk[r // N], V, 1.0, k, top_p, u)
                if near:
                    skipped += 1
                    continue
                checked += 1
                assert int(raw[r]) == ref, (seed, first, pos, k, top_p, r, int(raw[r]), ref)
    assert skipped <= 0.05 * (checked + skipped), (checked, skipped)


def test_sampler_draw_depends_only_on_the_commit_index():
    """a commit at position b of a B = 3 call with first_index f draws exactly what it draws alone with f + b"""
    from test_gpu_sample import _inputs
    V, S, B, N = 24650, 370, 3, 4
    gen = torch.Generator().manual_seed(5)
    logits, sc, gl, mem_mask, copy_src = _inputs(gen, B, N, V, S, torch.float32)
    seed, f, pos = 0xABCDEF0123456789, 40, 3
    raw, tlp = _sample(logits, sc, gl, mem_mask, copy_src, N, V, 0, 1.0, seed, f, pos)
    for b in range(B):
        rs = slice(b * N, (b + 1) * N)
        raw1, tlp1 = _sample(logits[rs].contiguous(), sc[b:b + 1].contiguous(), gl[rs].contiguous(),
                             mem_mask[b:b + 1].contiguous(), copy_src[b:b + 1].contiguous(), N, V, 0, 1.0, seed, f + b,
                             pos)
        assert np.array_equal(raw1, raw[rs]) and np.array_equal(tlp1.view(np.uint32), tlp[rs].view(np.uint32)), b
    other, _ = _sample(logits, sc, gl, mem_mask, copy_src, N, V, 0, 1.0, seed, f + 1, pos)
    assert not np.array_equal(other, raw)                # the commit index does enter the draw
