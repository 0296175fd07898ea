"""Offline distillation on the GPU: fira_pointer_mix_topk against the float64 rule (tests/kd_topk_rule.py), the sparse
loss kernels against the rule and, at alpha = 0, against the NLL kernels bit for bit, against the dense kd kernels on an
exactly k-sparse teacher, HeadFn with sparse targets and the whole loss against float64 autograd of the oracle, and
`run_model.py kd-targets` -> `distill` -> `test`."""
import numpy as np
import pytest
import torch

from bf16_bound import close
from fira_testlib import golden_batch, seeded_model
from kd_topk_rule import dense, row as rule_row, topk as rule_topk
from sample_rule import mixture
from test_gpu_cli import _run_model, trained  # noqa: F401  (the trained-model fixture)
from test_gpu_distill import (_ensemble_teacher, _head_reference, _head_teacher, _kd, _oracle_loss, _random_teacher,
                              _student)
from test_gpu_scst import EPS_HEAD, HEAD_PARAMS, _head_inputs, _plain

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
V0 = 24650
# sparse vs dense kd kernels on an exactly k-sparse teacher: the worst relative difference measured on an H100 80GB
# HBM3 was 3.5e-7 (fp32 summation order and t~ = P / mass against the dense kernel's t); the bound is the smallest
# power of two at least twice that
EPS_DENSE = 2.0 ** -20


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _topk(teacher, mm, lab, T, V, S, k):
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import call
    tx, tsc, tgl = teacher
    R = lab.numel()
    tl = torch.full((R, k), 7, dtype=torch.int32, device=DEV)
    tp = torch.full((R, k), float("nan"), device=DEV)
    mass = torch.full((R,), float("nan"), device=DEV)
    call("fira_pointer_mix_topk", ops._ptr(tx), tx.stride(0), ops._ptr(tsc), ops._ptr(tgl), ops._ptr(mm), ops._ptr(lab),
         k, ops._ptr(tl), ops._ptr(tp), ops._ptr(mass), R, T, V, S, ops._stream())
    torch.cuda.synchronize()
    return tl, tp, mass


def _sparse(student, tl, tp, alpha, T, V, S, up=1.0):
    """both sparse kernels -> (nll, kd, loss, stats, d_logits, d_copy_scores, d_gate_logits, row_active)"""
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import call
    logits, sc, gl, mm, lab = student
    R, ld, k = lab.numel(), logits.shape[1], tl.shape[1]
    B = R // T
    code = 1 if logits.dtype == torch.bfloat16 else 0
    p, st = ops._ptr, ops._stream()
    f = dict(device=DEV, dtype=torch.float32)
    stats = torch.full((R, 10), float("nan"), **f)
    nll, kd, loss = (torch.full((R,), float("nan"), **f) for _ in range(3))
    call("fira_pointer_mix_kd_sparse_fwd", p(logits), ld, p(sc), p(gl), p(mm), p(lab), p(tl), p(tp), k, float(alpha),
         p(stats), p(nll), p(kd), p(loss), R, T, V, S, code, st)
    dl = torch.full_like(logits, 7.0)
    dsc = torch.full((B, T, S), 7.0, **f)
    dgl = torch.full((R, 2), 7.0, **f)
    act = torch.full((R,), 7, dtype=torch.uint8, device=DEV)
    u = torch.tensor([up], **f)
    call("fira_pointer_mix_kd_sparse_bwd", p(logits), ld, p(sc), p(mm), p(lab), p(tl), p(tp), k, float(alpha),
         p(stats), p(u), p(dl), p(dsc), p(dgl), p(act), R, T, V, S, code, st)
    torch.cuda.synchronize()
    return nll, kd, loss, stats, dl, dsc, dgl, act


# ============================================================================= top-k
def _check_topk(teacher, mm, lab, T, V, S, k):
    tl, tp, mass = _topk(teacher, mm, lab, T, V, S, k)
    tx, tsc, tgl = (a.cpu().numpy().astype(np.float64) for a in teacher)
    R = lab.numel()
    tsc = tsc.reshape(R, S)
    mk = mm.cpu().numpy()
    tl_, tp_, mass_ = tl.cpu().numpy(), tp.cpu().numpy(), mass.cpu().numpy()
    near = 0
    for r in range(R):
        if int(lab[r]) == 0:
            assert (tl_[r] == -1).all() and (tp_[r] == 0).all() and mass_[r] == 0
            continue
        m = mk[r // T]
        P = mixture(tx[r, :V], tsc[r], tgl[r], m)
        labels, probs, ms = rule_topk(P, m, V, k)
        if not np.array_equal(labels, tl_[r]):
            # only a swap across fp32 rounding: the float64 probabilities of the differing slots agree to it
            diff = labels != tl_[r]
            assert (labels[diff] >= 0).all() and (tl_[r][diff] >= 0).all(), (r, labels, tl_[r])
            np.testing.assert_allclose(P[tl_[r][diff]], P[labels[diff]], rtol=2e-6, err_msg=str(r))
            near += 1
        got_p = P[np.maximum(tl_[r], 0)] * (tl_[r] >= 0)
        np.testing.assert_allclose(tp_[r], got_p / got_p.sum() if got_p.sum() else got_p, rtol=1e-5, atol=1e-30)
        assert abs(mass_[r] - got_p.sum()) <= 1e-5 * got_p.sum(), (r, mass_[r], got_p.sum())
        assert abs(mass_[r] - ms) <= 1e-5 * ms
    return tl, tp, mass, near


@pytest.mark.parametrize("V,S", [(V0, 370), (61, 13)])
@pytest.mark.parametrize("k", [1, 8, 64])
def test_topk_matches_float64_rule(V, S, k):
    B, T = 3, 8
    logits, sc, gl, mm, lab = _student(V + k, B, T, V, S, torch.float32)
    teacher = _random_teacher(V + k, B, T, V, S)
    tx = teacher[0]
    tx[5, 3:9] = tx[5, :V].max()                           # an exact tie at the top: the smaller labels first
    tx[4, :V] = -1e30                                     # one vocabulary candidate: fewer than 64 when S is small
    tx[4, 2] = 0.0
    teacher[2][4] = torch.tensor([0.0, 0.0], device=DEV)
    tl, tp, mass, near = _check_topk(teacher, mm, lab, T, V, S, k)
    if k == 64 and S < 64:
        assert int((tl[4] >= 0).sum()) == 1 + int(mm[0].sum()) and int(tl[4, -1]) == -1
    tied = [j for j in tl[5].tolist() if 3 <= j <= 8]
    assert tied == sorted(tied)
    print(f"[kd-targets] V={V} S={S} k={k}: {near} rows differ from float64 across an fp32 near-tie")
    # a row's result depends on that row alone: twice, and with the first commit removed from the batch
    again = _topk(teacher, mm, lab, T, V, S, k)
    assert all(torch.equal(a, b) for a, b in zip((tl, tp, mass), again))
    sub = _topk(tuple(a[T:] if a.dim() == 2 and a.shape[0] == B * T else a[1:] for a in teacher), mm[1:], lab[T:], T, V,
                S, k)
    assert torch.equal(sub[0], tl[T:]) and torch.equal(sub[1], tp[T:]) and torch.equal(sub[2], mass[T:])


# ============================================================================= the sparse loss
def _check_rule(student, tl, tp, alpha, T, V, S):
    nll, kd, loss, stats, dl, dsc, dgl, act = _sparse(student, tl, tp, alpha, T, V, S)
    logits, sc, gl, mm, lab = student
    R = lab.numel()
    bf16 = logits.dtype == torch.bfloat16
    x64 = logits.float().cpu().numpy()[:, :V].astype(np.float64)
    c64 = sc.cpu().numpy().reshape(R, S).astype(np.float64)
    g64, mk = gl.cpu().numpy().astype(np.float64), mm.cpu().numpy()
    tl_, tp_ = tl.cpu().numpy(), tp.cpu().numpy().astype(np.float64)
    out = [a.float().cpu().numpy() for a in (nll, kd, loss, dl[:, :V], dsc.reshape(R, S), dgl)]
    A_C = stats[:, 9].cpu().numpy()
    for r in range(R):
        y = int(lab[r])
        want = rule_row(x64[r], c64[r], g64[r], mk[r // T], tl_[r], tp_[r], y, alpha)
        for i, (g, w) in enumerate(zip(out[:3], want[:3])):
            assert abs(g[r] - w) <= 2e-5 * max(1.0, abs(w)), (r, y, i, g[r], w)
        for i, (g, w) in enumerate(zip(out[3:], want[3:])):
            scale = max(float(np.abs(w).max()), 1e-30)
            tol = 1e-5 * scale + (2.0 ** -8 * np.abs(w) if (bf16 and i == 0) else 0.0)
            if i == 2:
                tol = 2e-6
            assert (np.abs(g[r] - w) <= tol).all(), (r, y, i, float(np.abs(g[r] - w).max()), scale)
        assert int(act[r]) == int(A_C[r] != 0)
        if y == 0:
            assert not out[3][r].any() and int(act[r]) == 0


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("V,S", [(V0, 370), (61, 13)])
@pytest.mark.parametrize("alpha", [0.3, 1.0])
def test_sparse_kernels_match_float64_rule(dtype, V, S, alpha):
    B, T, k = 3, 8, 8
    student = _student(V + S + 5, B, T, V, S, dtype)
    lab, mm = student[4], student[3]
    tl, tp, _ = _topk(_random_teacher(V + 1, B, T, V, S), mm, lab, T, V, S, k)
    tl[3, 5:] = -1                                        # missing slots
    tp[3, 5:] = 0.0
    tp[4, 2] = 0.0                                        # a kept label with probability 0
    y7 = int(lab[7])                                      # the row's own label kept, and not kept
    if y7 != 0 and y7 < V + S:
        tl[7, 1] = y7
    _check_rule(student, tl, tp, alpha, T, V, S)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("V,S", [(V0, 370), (61, 13)])
def test_alpha_zero_equals_the_nll_kernels(dtype, V, S):
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import call
    B, T, k = 3, 8, 8
    student = _student(V + 11, B, T, V, S, dtype)
    logits, sc, gl, mm, lab = student
    R, ld = lab.numel(), logits.shape[1]
    code = 1 if dtype == torch.bfloat16 else 0
    p, st = ops._ptr, ops._stream()
    stats = torch.empty((R, 8), device=DEV)
    nll = torch.empty(R, device=DEV)
    call("fira_pointer_mix_nll_fwd", p(logits), ld, p(sc), p(gl), p(mm), p(lab), p(stats), p(nll), None, R, T, V, S,
         code, st)
    dl = torch.full_like(logits, 7.0)
    dsc = torch.full((B, T, S), 7.0, device=DEV)
    dgl = torch.full((R, 2), 7.0, device=DEV)
    act = torch.full((R,), 7, dtype=torch.uint8, device=DEV)
    up = 0.37
    u = torch.tensor([up], device=DEV)
    call("fira_pointer_mix_nll_bwd", p(logits), ld, p(sc), p(mm), p(lab), p(stats), p(u), p(dl), p(dsc), p(dgl),
         p(act), R, T, V, S, code, st)
    torch.cuda.synchronize()
    tl, tp, _ = _topk(_random_teacher(V, B, T, V, S), mm, lab, T, V, S, k)
    snll, _, sloss, _, sdl, sdsc, sdgl, sact = _sparse(student, tl, tp, 0.0, T, V, S, up=up)
    assert torch.equal(snll, nll) and torch.equal(sloss, nll)
    assert torch.equal(sdl[:, :V], dl[:, :V])
    assert torch.equal(sdsc, dsc) and torch.equal(sdgl, dgl) and torch.equal(sact, act)
    assert int(act.sum()) > 0 and int((lab == 0).sum()) > 0


def _k_sparse_teacher(seed, mm, B, T, V, S, k):
    """a triple with k entries above -1e30 per row (k - 3 vocabulary entries, 3 unmasked copy positions): its fp32
    mixture is exactly k-sparse"""
    from fira_icse_b200 import ops
    g = torch.Generator().manual_seed(seed)
    R = B * T
    tx = torch.full((R, ops._ld_logits(V)), -1e30)
    tsc = torch.full((R, S), -1e30)
    tgl = torch.randn((R, 2), generator=g)
    mk = mm.cpu()
    for r in range(R):
        tx[r, torch.randperm(V, generator=g)[:k - 3]] = torch.randn(k - 3, generator=g) * 2
        ok = torch.nonzero(mk[r // T]).view(-1)
        tsc[r, ok[torch.randperm(len(ok), generator=g)[:3]]] = torch.randn(3, generator=g) * 2
    return tx.to(DEV), tsc.view(B, T, S).to(DEV), tgl.to(DEV)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("V,S", [(V0, 370), (61, 13)])
def test_sparse_kernels_agree_with_the_dense_ones_on_a_k_sparse_teacher(dtype, V, S):
    B, T, k = 3, 8, 8
    student = _student(V + 2, B, T, V, S, dtype)
    lab, mm = student[4], student[3]
    teacher = _k_sparse_teacher(V, mm, B, T, V, S, k)
    tl, tp, _ = _topk(teacher, mm, lab, T, V, S, k)
    assert bool((tl[lab != 0] >= 0).all())
    dn = _kd(student, teacher, 0.6, T, V, S, up=0.5)
    sp = _sparse(student, tl, tp, 0.6, T, V, S, up=0.5)
    worst = 0.0
    for i in (0, 1, 2, 4, 5, 6):
        a, b = sp[i].double(), dn[i].double()
        a, b = a.reshape(lab.numel(), -1), b.reshape(lab.numel(), -1)
        if i == 4:
            a, b = a[:, :V], b[:, :V]
        scale = b.abs().amax(1, keepdim=True).clamp_min(1e-30)
        worst = max(worst, float(((a - b).abs() / scale).max()))
    assert torch.equal(sp[7], dn[7])
    print(f"[kd-targets] sparse vs dense kd kernels ({dtype}, V={V}): worst relative difference {worst:.3e}")
    assert worst <= EPS_DENSE


def test_kernels_refuse_invalid_arguments():
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import lib
    V, S, B, T, k = 61, 13, 2, 8, 4
    logits, sc, gl, mm, lab = _student(1, B, T, V, S, torch.float32)
    tx, tsc, tgl = _random_teacher(1, B, T, V, S)
    R, ld = lab.numel(), logits.shape[1]
    f = dict(device=DEV, dtype=torch.float32)
    tl, tp = torch.zeros((R, k), dtype=torch.int32, device=DEV), torch.zeros((R, k), **f)
    stats, nll, kd, loss, mass = (torch.empty((R, 10), **f), *(torch.empty(R, **f) for _ in range(4)))
    dl, dsc, dgl = torch.empty_like(logits), torch.empty((B, T, S), **f), torch.empty((R, 2), **f)
    act, u = torch.empty(R, dtype=torch.uint8, device=DEV), torch.ones(1, **f)
    p, st = ops._ptr, ops._stream()
    codes = dict(shape=1, align=2, dtype=4, arg=5)

    def topk(**o):
        a = dict(tx=p(tx), ldt=tx.stride(0), tsc=p(tsc), tgl=p(tgl), mm=p(mm), lab=p(lab), k=k, tl=p(tl), tp=p(tp),
                 mass=p(mass), R=R, T=T, V=V, S=S)
        a.update(o)
        return lib().fira_pointer_mix_topk(*a.values(), st)

    def fwd(**o):
        a = dict(logits=p(logits), ld=ld, sc=p(sc), gl=p(gl), mm=p(mm), lab=p(lab), tl=p(tl), tp=p(tp), k=k, alpha=0.5,
                 stats=p(stats), nll=p(nll), kd=p(kd), loss=p(loss), R=R, T=T, V=V, S=S, dtype=0)
        a.update(o)
        return lib().fira_pointer_mix_kd_sparse_fwd(*a.values(), st)

    def bwd(**o):
        a = dict(logits=p(logits), ld=ld, sc=p(sc), mm=p(mm), lab=p(lab), tl=p(tl), tp=p(tp), k=k, alpha=0.5,
                 stats=p(stats), u=p(u), dl=p(dl), dsc=p(dsc), dgl=p(dgl), act=p(act), R=R, T=T, V=V, S=S, dtype=0)
        a.update(o)
        return lib().fira_pointer_mix_kd_sparse_bwd(*a.values(), st)

    assert topk() == 0 and fwd() == 0 and bwd() == 0
    assert topk(R=0) == 0 and fwd(R=0) == 0 and bwd(R=0) == 0
    for o, code in [(dict(k=0), "arg"), (dict(k=65), "arg"), (dict(tx=None), "arg"), (dict(tl=None), "arg"),
                    (dict(mass=None), "arg"), (dict(ldt=ld + 4), "align"), (dict(tx=p(tx) + 8), "align"),
                    (dict(V=32767 - S + 1, ldt=32768), "shape"), (dict(S=0), "shape"), (dict(R=-1), "shape"),
                    (dict(ldt=56), "shape")]:
        assert topk(**o) == codes[code], o
    common = [(dict(alpha=-0.1), "arg"), (dict(alpha=1.01), "arg"), (dict(alpha=float("nan")), "arg"),
              (dict(k=0), "arg"), (dict(k=65), "arg"), (dict(logits=None), "arg"), (dict(tl=None), "arg"),
              (dict(tp=None), "arg"), (dict(stats=None), "arg"), (dict(ld=ld + 4), "align"),
              (dict(logits=p(logits) + 4), "align"), (dict(V=32767 - S + 1, ld=32768), "shape"), (dict(S=0), "shape"),
              (dict(T=0), "shape"), (dict(R=-1), "shape"), (dict(ld=56), "shape"), (dict(dtype=7), "dtype")]
    for o, code in common + [(dict(gl=None), "arg"), (dict(kd=None), "arg"), (dict(loss=None), "arg")]:
        assert fwd(**o) == codes[code], o
    for o, code in common + [(dict(u=None), "arg"), (dict(dl=None), "arg"), (dict(act=None), "arg"),
                             (dict(dl=p(dl) + 4), "align")]:
        assert bwd(**o) == codes[code], o
    torch.cuda.synchronize()


# ============================================================================= HeadFn and the whole loss
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_head_with_sparse_targets_matches_float64(bf16):
    from fira_icse_b200 import ops
    alpha, k = 0.4, 8
    memory, dec, mem_valid, label = _head_inputs(bf16)
    B, T = label.shape
    S = mem_valid.shape[1]
    teacher, _ = _head_teacher(B, T, S, mem_valid)
    mm = mem_valid.to(torch.uint8).to(DEV)
    lab = label.to(torch.int32).reshape(-1).to(DEV)
    tl, tp, _ = _topk(teacher, mm, lab, T, V0, S, k)
    t = torch.from_numpy(np.stack([dense(a, b, V0 + S) for a, b in zip(tl.cpu().numpy(), tp.cpu().double().numpy())]))
    model = seeded_model()
    params = [dict(model.named_parameters())[n].detach().to(DEV).clone().requires_grad_(True) for n in HEAD_PARAMS]
    m = memory.to(DEV).requires_grad_(True)
    d = dec.to(DEV).requires_grad_(True)
    kd = torch.empty(lab.numel(), device=DEV)
    loss, nll, _ = ops.HeadFn.apply(False, bf16, None, m, d, mm, lab, *params, None, None, None, (tl, tp, alpha, kd))
    loss.backward()
    torch.cuda.synchronize()
    ref = _head_reference(alpha, t.view(B, T, -1), memory, dec, mem_valid, label, rounded=bf16)
    names = ["loss", "nll", "kd", "d_memory", "d_dec"] + list(HEAD_PARAMS)
    got = [loss, nll.view(B, T), kd.view(B, T), m.grad, d.grad] + [q.grad for q in params]
    for n, g, r in zip(names, got, [ref[0], ref[1], ref[2], ref[3], ref[4]] + ref[5]):
        g, r = g.detach().cpu().double(), r.detach().double()
        if n == "copy_net.LinearRes.bias":
            continue
        if not bf16:
            err = float((g - r).abs().max())
            assert err <= 1e-4 * float(r.abs().max()), (n, err, float(r.abs().max()))
        elif n == "loss":
            assert abs(float(g) - float(r)) <= EPS_HEAD * abs(float(r))
        else:
            close(f"sparse kd head {n}", g, r, EPS_HEAD, rows=n in ("nll", "kd", "d_memory", "d_dec"))
    with pytest.raises(ValueError, match="sparse targets need"):
        ops.HeadFn.apply(False, bf16, None, m, d, mm, lab, *params, None, None, None, (tl[:, :0], tp, alpha, kd))


def _sparse_of(b, ens, m, k):
    from fira_icse_b200 import distill
    bd = [t.to(DEV) for t in b]
    label = m.shifted_label(bd[6])
    targets = distill.teacher_targets(ens, bd, label)
    mm = torch.cat((bd[0] != 0, bd[7] != 0), dim=1).to(torch.uint8)
    tl, tp, _ = distill.topk_targets(targets, mm, label, m.vocab_size, k)
    B, T = label.shape
    t = np.stack([dense(a, c, m.vocab_size + mm.shape[1]) for a, c in zip(tl.cpu().numpy(), tp.cpu().double().numpy())])
    return distill.SparseTargets(tl, tp), torch.from_numpy(t).view(B, T, -1)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_whole_loss_with_stored_targets_matches_float64(precision, monkeypatch):
    from fira_icse_b200 import distill
    m = _plain(precision)
    b = golden_batch(0, 3)
    ens, _, _ = _ensemble_teacher()
    sparse, t = _sparse_of(b, ens, m, 8)
    m.zero_grad(set_to_none=True)
    bd = [x.to(DEV) for x in b]
    label = m.shifted_label(bd[6])
    loss, _, _ = distill.distill_loss(m, bd, sparse, label, 0.5)
    n = int((label != 0).sum())
    (loss / n).backward()
    torch.cuda.synchronize()
    loss = loss.item() / n
    grads = {k: q.grad for k, q in m.named_parameters() if q.grad is not None}
    if precision == "fp32":
        ref_loss, ref = _oracle_loss(m, b, t, 0.5)
        assert abs(loss - ref_loss) <= 1e-4 * abs(ref_loss)
        for k, g in grads.items():
            r = ref[k].numpy()
            if k.endswith("fc_k.bias") or k == "copy_net.LinearRes.bias":
                continue
            np.testing.assert_allclose(g.cpu().numpy(), r, rtol=5e-3, atol=1e-7 + 5e-4 * float(np.abs(r).max()),
                                       err_msg=k)
    else:
        from test_gpu_bf16_step import check_step, record_gates
        gates = {}
        record_gates(monkeypatch, gates)
        ref_loss, ref = _oracle_loss(m, b, t, 0.5)
        check_step("distill/stored targets", loss, grads, ref_loss, ref, gates)


def test_step_with_stored_targets_runs_no_teacher():
    from fira_icse_b200 import distill, optim
    m = _plain("fp32")
    b = golden_batch(0, 4)
    ens, _, _ = _ensemble_teacher()
    sparse, _ = _sparse_of(b, ens, m, 8)
    calls = []
    orig = distill.teacher_targets
    distill.teacher_targets = lambda *a, **kw: calls.append(1) or orig(*a, **kw)
    try:
        opt = optim.FlatAdam(m.live_parameters(), lr=1e-4, groups=m.flat_groups())
        optim.attach(m, [opt])
        step = distill.distill_step(m, opt, [x.to(DEV) for x in b], sparse, alpha=0.5)
    finally:
        distill.teacher_targets = orig
    assert not calls and np.isfinite(step.loss) and step.tokens > 0 and step.kd > 0.0
    with pytest.raises(ValueError, match="sparse targets must be"):
        distill.distill_step(m, opt, [x.to(DEV) for x in b], distill.SparseTargets(sparse.t_label[1:], sparse.t_prob[1:]),
                             alpha=0.5)


# ============================================================================= CLI
def test_run_model_kd_targets_then_distill_then_test(trained):  # noqa: F811
    from fira_icse_b200.distill import KDTargets
    d, env, _ = trained
    base = open(d / "best_model.pt", "rb").read()
    r = _run_model("kd-targets", d, dict(env, FIRA_ENSEMBLE="best_model.pt", FIRA_KD_TOPK="8"))
    assert "kd-targets:" in r.stdout and "mean kept mass" in r.stdout, r.stdout
    t = KDTargets.load(d / "kd_targets.pt", k=8)
    assert t.rows > 0 and t.provenance["commits"] == t.n and len(t.provenance["fingerprints"]) == 1
    assert bool((t.mass > 0).all() and (t.mass <= 1.0001).all())
    r = _run_model("distill", d, dict(env, FIRA_MAX_BATCHES="2", FIRA_KD_TARGETS="kd_targets.pt"))
    assert "kd epoch: 0 batch: 0/" in r.stdout and "best dev bleu" in r.stdout
    assert open(d / "best_model.pt", "rb").read() == base
    kd = torch.load(d / "best_model_kd.pt", map_location="cpu")
    assert len(kd) == 338
    r = _run_model("test", d, dict(env, FIRA_CHECKPOINT="best_model_kd.pt"))
    assert "mean sentence bleu" in r.stdout
