"""Knowledge distillation on the GPU: fira_pointer_mix_kd_fwd / _bwd against the float64 rule (tests/kd_rule.py) and
against the NLL kernels at alpha = 0, a one-hot teacher, HeadFn with a teacher and the whole distillation loss against
float64 autograd of the oracle, a self-teacher, decoding after a step, and `run_model.py distill`."""
import copy
import os

import numpy as np
import pytest
import torch

from bf16_bound import close
from fira_testlib import golden_batch, seeded_model
from kd_rule import row as rule_row
from sample_rule import mixture
from test_gpu_cli import _run_model, trained  # noqa: F401  (the trained-model fixture)
from test_gpu_ensemble import _combine, _members, _two_members
from test_gpu_scst import EPS_HEAD, HEAD_PARAMS, HEAD_ROUNDED, _head_inputs, _plain, _vocab_ids

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
V0 = 24650


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


# ============================================================================= the kernels
def _student(seed, B, T, V, S, dtype, mem_mask=None):
    """wide logits (many entries below the clamp), a saturated gate each way, and labels of every kind: vocabulary,
    copy, a copy label at a masked position, one beyond S, and 0"""
    from fira_icse_b200 import ops
    g = torch.Generator().manual_seed(seed)
    R, ld = B * T, ops._ld_logits(V)
    logits = (torch.randn((R, ld), generator=g) * 6).to(dtype)
    sc = torch.randn((B, T, S), generator=g) * 3
    gl = torch.randn((R, 2), generator=g)
    gl[1], gl[2] = torch.tensor([-200.0, 0.0]), torch.tensor([0.0, -200.0])
    if mem_mask is None:
        mem_mask = (torch.rand((B, S), generator=g) < 0.7).to(torch.uint8)
        mem_mask[:, 0] = 1
        mem_mask[:, 1] = 0
    mem_mask = mem_mask.cpu()
    lab = torch.randint(1, V, (B, T), generator=g)
    for b in range(B):
        ok = torch.nonzero(mem_mask[b]).view(-1)
        for t in range(0, T, 3):
            lab[b, t] = V + int(ok[torch.randint(0, len(ok), (1,), generator=g)])
        lab[b, T - 2:] = 0
    lab[0, 1] = V + 1                            # masked position
    lab[1 % B, 4] = V + S + 2                    # beyond S
    lab[0, 2] = 0
    return (logits.to(DEV), sc.to(DEV), gl.to(DEV), mem_mask.to(DEV), lab.reshape(-1).to(torch.int32).to(DEV))


def _random_teacher(seed, B, T, V, S):
    from fira_icse_b200 import ops
    g = torch.Generator().manual_seed(seed + 99)
    R, ld = B * T, ops._ld_logits(V)
    tx = torch.randn((R, ld), generator=g) * 2
    tsc = torch.randn((B, T, S), generator=g) * 2
    tgl = torch.randn((R, 2), generator=g)
    tgl[3] = torch.tensor([-200.0, 0.0])
    return tx.to(DEV), tsc.to(DEV), tgl.to(DEV)


def _kd(student, teacher, alpha, T, V, S, up=1.0):
    """both kernels -> (nll, kd, loss, stats, d_logits, d_copy_scores, d_gate_logits, row_active)"""
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import call
    logits, sc, gl, mm, lab = student
    tx, tsc, tgl = teacher
    R, ld = lab.numel(), logits.shape[1]
    B = R // T
    code = 1 if logits.dtype == torch.bfloat16 else 0
    p, st = ops._ptr, ops._stream()
    nan = dict(device=DEV, dtype=torch.float32)
    stats = torch.full((R, 16), float("nan"), **nan)
    nll, kd, loss = (torch.full((R,), float("nan"), **nan) for _ in range(3))
    call("fira_pointer_mix_kd_fwd", p(logits), ld, p(sc), p(gl), p(mm), p(lab), p(tx), tx.stride(0), p(tsc), p(tgl),
         float(alpha), p(stats), p(nll), p(kd), p(loss), R, T, V, S, code, st)
    dl = torch.full_like(logits, 7.0)
    dsc = torch.full((B, T, S), 7.0, **nan)
    dgl = torch.full((R, 2), 7.0, **nan)
    act = torch.full((R,), 7, dtype=torch.uint8, device=DEV)
    u = torch.tensor([up], **nan)
    call("fira_pointer_mix_kd_bwd", p(logits), ld, p(sc), p(mm), p(lab), p(tx), tx.stride(0), p(tsc), float(alpha),
         p(stats), p(u), p(dl), p(dsc), p(dgl), p(act), R, T, V, S, code, st)
    torch.cuda.synchronize()
    return nll, kd, loss, stats, dl, dsc, dgl, act


def _check_rule(student, teacher, alpha, T, V, S):
    nll, kd, loss, stats, dl, dsc, dgl, act = _kd(student, teacher, alpha, T, V, S)
    logits, sc, gl, mm, lab = student
    tx, tsc, tgl = teacher
    R = lab.numel()
    bf16 = logits.dtype == torch.bfloat16
    x64 = logits.float().cpu().numpy()[:, :V].astype(np.float64)
    c64 = sc.cpu().numpy().reshape(R, S).astype(np.float64)
    g64, mk = gl.cpu().numpy().astype(np.float64), mm.cpu().numpy()
    tx64, tc64, tg64 = (a.cpu().numpy().astype(np.float64) for a in (tx[:, :V], tsc.reshape(R, S), tgl))
    out = [a.float().cpu().numpy() for a in (nll, kd, loss, dl[:, :V], dsc.reshape(R, S), dgl)]
    A_C = stats[:, 15].cpu().numpy()
    below = 0
    for r in range(R):
        m = mk[r // T]
        t = mixture(tx64[r], tc64[r], tg64[r], m)
        t[V:][m == 0] = 0.0
        y = int(lab[r])
        want = rule_row(x64[r], c64[r], g64[r], m, t, y, alpha)
        for k, (g, w) in enumerate(zip(out[:3], want[:3])):
            assert abs(g[r] - w) <= 2e-5 * max(1.0, abs(w)), (r, y, k, g[r], w)
        for k, (g, w) in enumerate(zip(out[3:], want[3:])):
            scale = max(float(np.abs(w).max()), 1e-30)
            tol = 1e-5 * scale + (2.0 ** -8 * np.abs(w) if (bf16 and k == 0) else 0.0)
            if k == 2:                           # g (A_V + A_C) - A: a difference of terms up to 1
                tol = 2e-6
            assert (np.abs(g[r] - w) <= tol).all(), (r, y, k, float(np.abs(g[r] - w).max()), scale)
        assert int(act[r]) == int(A_C[r] != 0)
        if y == 0:
            assert not out[3][r].any() and int(act[r]) == 0
        below += int((mixture(x64[r], c64[r], g64[r], m) < 1e-10).sum())
    assert below > 0
    return nll, kd


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("V,S", [(V0, 370), (61, 13)])
@pytest.mark.parametrize("alpha", [0.0, 0.3, 1.0])
def test_kernels_match_float64_rule_random_teacher(dtype, V, S, alpha):
    B, T = 3, 8
    student = _student(V + S + int(alpha * 10), B, T, V, S, dtype)
    _check_rule(student, _random_teacher(V, B, T, V, S), alpha, T, V, S)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("V,S", [(V0, 370), (61, 13)])
def test_kernels_match_float64_rule_ensemble_teacher(dtype, V, S):
    """the teacher triple of a real fira_pointer_mix_ensemble launch (three members, one saturated gate)"""
    B, T, M = 3, 8, 3
    members, mem_mask = _members(V + 7, M, B, T, V, S, dtype)
    w = np.array([0.2, 0.5, 0.3])
    teacher = _combine(members, np.log(w), mem_mask, T, V, S)
    student = _student(V + 3, B, T, V, S, dtype, mem_mask=mem_mask)
    _check_rule(student, teacher, 0.6, T, V, S)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("V,S", [(V0, 370), (61, 13)])
def test_alpha_zero_equals_the_nll_kernels(dtype, V, S):
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import call
    B, T = 3, 8
    student = _student(V + 11, B, T, V, S, dtype)
    logits, sc, gl, mm, lab = student
    R, ld = lab.numel(), logits.shape[1]
    code = 1 if dtype == torch.bfloat16 else 0
    p, st = ops._ptr, ops._stream()
    stats = torch.empty((R, 8), device=DEV)
    nll = torch.empty(R, device=DEV)
    call("fira_pointer_mix_nll_fwd_rows", p(logits), ld, p(sc), p(gl), p(mm), p(lab), None, p(stats), p(nll), None, R,
         T, V, S, code, st)
    dl = torch.full_like(logits, 7.0)
    dsc = torch.full((B, T, S), 7.0, device=DEV)
    dgl = torch.full((R, 2), 7.0, device=DEV)
    act = torch.full((R,), 7, dtype=torch.uint8, device=DEV)
    up = 0.37
    u = torch.tensor([up], device=DEV)
    call("fira_pointer_mix_nll_bwd_rows", p(logits), ld, p(sc), p(mm), p(lab), None, None, 0, p(stats), p(u), p(dl),
         p(dsc), p(dgl), p(act), R, T, V, S, code, st)
    torch.cuda.synchronize()
    knll, _, kloss, _, kdl, kdsc, kdgl, kact = _kd(student, _random_teacher(V, B, T, V, S), 0.0, T, V, S, up=up)
    assert torch.equal(knll, nll) and torch.equal(kloss, nll)
    assert torch.equal(kdl[:, :V], dl[:, :V])
    assert torch.equal(kdsc, dsc) and torch.equal(kdgl, dgl) and torch.equal(kact, act)
    assert int(act.sum()) > 0 and int((lab == 0).sum()) > 0


def _one_hot_teacher(lab, mm, T, V, S):
    """a finite triple (fills of -1e30) whose mixture is one-hot at each row's label (rows with label 0: at 1)"""
    from fira_icse_b200 import ops
    R = lab.numel()
    tx = torch.full((R, ops._ld_logits(V)), -1e30, device=DEV)
    tsc = torch.full((R, S), -1e30, device=DEV)
    tgl = torch.zeros((R, 2), device=DEV)
    for r in range(R):
        y = int(lab[r])
        if V <= y < V + S and mm[r // T, y - V]:
            tsc[r, y - V] = 0.0
            tgl[r, 0] = -1e30
        else:
            tx[r, y if 0 < y < V else 1] = 0.0
            tgl[r, 1] = -1e30
    return tx, tsc.view(R // T, T, S), tgl


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_one_hot_teacher_at_alpha_one_is_the_nll(dtype):
    V, S, B, T = V0, 370, 3, 8
    student = _student(5, B, T, V, S, dtype)
    lab, mm = student[4], student[3]
    teacher = _one_hot_teacher(lab, mm, T, V, S)
    hard = _kd(student, teacher, 0.0, T, V, S, up=0.5)
    soft = _kd(student, teacher, 1.0, T, V, S, up=0.5)
    # a copy label at a masked position or beyond S has no one-hot teacher entry: those rows differ by design
    y = lab.long()
    s = (y - V).clamp(0, S - 1)
    real = (y < V) | ((y < V + S) & (mm[torch.arange(lab.numel(), device=DEV) // T, s] != 0))
    torch.testing.assert_close(soft[2][real], hard[0][real], rtol=1e-6, atol=0)
    torch.testing.assert_close(soft[0], hard[0], rtol=0, atol=0)
    for a, b in zip(soft[4:7], hard[4:7]):
        a, b = a.reshape(lab.numel(), -1)[real], b.reshape(lab.numel(), -1)[real]
        torch.testing.assert_close(a.float(), b.float(), rtol=1e-6, atol=1e-7)


def test_kernels_refuse_invalid_arguments():
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import lib
    V, S, B, T = 61, 13, 2, 8
    logits, sc, gl, mm, lab = _student(1, B, T, V, S, torch.float32)
    tx, tsc, tgl = _random_teacher(1, B, T, V, S)
    R, ld = lab.numel(), logits.shape[1]
    f = dict(device=DEV, dtype=torch.float32)
    stats, nll, kd, loss = torch.empty((R, 16), **f), torch.empty(R, **f), torch.empty(R, **f), torch.empty(R, **f)
    dl, dsc, dgl = torch.empty_like(logits), torch.empty((B, T, S), **f), torch.empty((R, 2), **f)
    act, u = torch.empty(R, dtype=torch.uint8, device=DEV), torch.ones(1, **f)
    p, st = ops._ptr, ops._stream()
    codes = dict(shape=1, align=2, dtype=4, arg=5)

    def fwd(**o):
        a = dict(logits=p(logits), ld=ld, sc=p(sc), gl=p(gl), mm=p(mm), lab=p(lab), tx=p(tx), ldt=tx.stride(0),
                 tsc=p(tsc), tgl=p(tgl), alpha=0.5, stats=p(stats), nll=p(nll), kd=p(kd), loss=p(loss), R=R, T=T, V=V,
                 S=S, dtype=0)
        a.update(o)
        return lib().fira_pointer_mix_kd_fwd(*a.values(), st)

    def bwd(**o):
        a = dict(logits=p(logits), ld=ld, sc=p(sc), mm=p(mm), lab=p(lab), tx=p(tx), ldt=tx.stride(0), tsc=p(tsc),
                 alpha=0.5, stats=p(stats), u=p(u), dl=p(dl), dsc=p(dsc), dgl=p(dgl), act=p(act), R=R, T=T, V=V, S=S,
                 dtype=0)
        a.update(o)
        return lib().fira_pointer_mix_kd_bwd(*a.values(), st)

    assert fwd() == 0 and bwd() == 0
    assert fwd(R=0) == 0 and bwd(R=0) == 0
    common = [(dict(alpha=-0.1), "arg"), (dict(alpha=1.01), "arg"), (dict(alpha=float("nan")), "arg"),
              (dict(alpha=float("inf")), "arg"), (dict(logits=None), "arg"), (dict(tx=None), "arg"),
              (dict(mm=None), "arg"), (dict(lab=None), "arg"), (dict(stats=None), "arg"), (dict(ld=ld + 4), "align"),
              (dict(ldt=ld + 4), "align"), (dict(logits=p(logits) + 4), "align"), (dict(tx=p(tx) + 8), "align"),
              (dict(V=32767 - S + 1, ld=32768, ldt=32768), "shape"), (dict(S=0), "shape"), (dict(T=0), "shape"),
              (dict(R=-1), "shape"), (dict(ld=56), "shape"), (dict(dtype=7), "dtype")]
    for o, code in common + [(dict(gl=None), "arg"), (dict(tgl=None), "arg"), (dict(kd=None), "arg"),
                             (dict(loss=None), "arg")]:
        assert fwd(**o) == codes[code], o
    for o, code in common + [(dict(u=None), "arg"), (dict(dl=None), "arg"), (dict(act=None), "arg"),
                             (dict(dl=p(dl) + 4), "align")]:
        assert bwd(**o) == codes[code], o
    torch.cuda.synchronize()


# ============================================================================= HeadFn with a teacher
def _head_teacher(B, T, S, mem_valid):
    from fira_icse_b200 import ops
    g = torch.Generator().manual_seed(21)
    tx = torch.randn((B * T, ops._ld_logits(V0)), generator=g) * 2
    tsc = torch.randn((B, T, S), generator=g) * 2
    tgl = torch.randn((B * T, 2), generator=g)
    t = np.stack([mixture(tx[r, :V0].double().numpy(), tsc.view(-1, S)[r].double().numpy(), tgl[r].double().numpy(),
                          mem_valid[r // T].numpy()) for r in range(B * T)])
    t[:, V0:][np.repeat(mem_valid.numpy(), T, 0) == 0] = 0.0
    return (tx.to(DEV), tsc.to(DEV), tgl.to(DEV)), torch.from_numpy(t).view(B, T, -1)


def _run_head(bf16, alpha, teacher, memory, dec, mem_valid, label):
    from fira_icse_b200 import ops
    model = seeded_model()
    params = [dict(model.named_parameters())[k].detach().to(DEV).clone().requires_grad_(True) for k in HEAD_PARAMS]
    m = memory.to(DEV).requires_grad_(True)
    d = dec.to(DEV).requires_grad_(True)
    kd = torch.empty(label.numel(), device=DEV)
    loss, nll, _ = ops.HeadFn.apply(False, bf16, None, m, d, mem_valid.to(torch.uint8).to(DEV),
                                    label.to(torch.int32).reshape(-1).to(DEV), *params, None, None,
                                    (*teacher, alpha, kd))
    loss.backward()
    torch.cuda.synchronize()
    return loss, nll, kd, m.grad, d.grad, [p.grad for p in params]


def _head_reference(alpha, t, memory, dec, mem_valid, label, rounded):
    import fira_oracle as O
    named = dict(seeded_model().named_parameters())
    sd = {k: (named[k].detach().to(torch.bfloat16).double() if rounded and k in HEAD_ROUNDED else
              named[k].detach().double()).requires_grad_(True) for k in HEAD_PARAMS}
    m64 = memory.double().requires_grad_(True)
    d64 = dec.double().requires_grad_(True)
    logp, _ = O.output_distribution(sd, m64, mem_valid, d64)
    keep = label != 0
    nll = -logp.gather(-1, label.unsqueeze(-1)).squeeze(-1) * keep
    kd = -(t * logp).sum(-1) * keep
    loss = ((1 - alpha) * nll + alpha * kd).sum()
    loss.backward()
    return loss, nll, kd, m64.grad, d64.grad, [sd[k].grad for k in HEAD_PARAMS]


@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_head_with_a_teacher_matches_float64(bf16):
    alpha = 0.4
    inputs = _head_inputs(bf16)
    memory, dec, mem_valid, label = inputs
    B, T = label.shape
    teacher, t = _head_teacher(B, T, mem_valid.shape[1], mem_valid)
    got = _run_head(bf16, alpha, teacher, *inputs)
    ref = _head_reference(alpha, t, *inputs, rounded=bf16)
    names = ["loss", "nll", "kd", "d_memory", "d_dec"] + list(HEAD_PARAMS)
    pairs = list(zip(names, [got[0], got[1].view(B, T), got[2].view(B, T), got[3], got[4]] + got[5],
                     [ref[0], ref[1], ref[2], ref[3], ref[4]] + ref[5]))
    for k, g, r in pairs:
        g, r = g.detach().cpu().double(), r.detach().double()
        if k == "copy_net.LinearRes.bias":                # zero in exact arithmetic (softmax shift invariance)
            if not bf16:
                assert float(g.abs().max()) <= 1e-4 * float(ref[5][HEAD_PARAMS.index("copy_net.LinearRes.weight")].abs().max())
            continue
        if not bf16:
            err = float((g - r).abs().max())
            assert err <= 1e-4 * float(r.abs().max()), (k, err, float(r.abs().max()))
        elif k == "loss":
            assert abs(float(g) - float(r)) <= EPS_HEAD * abs(float(r))
        else:
            close(f"kd head {k}", g, r, EPS_HEAD, rows=k in ("nll", "kd", "d_memory", "d_dec"))


# ============================================================================= the whole loss
def _loss_grads(m, b, teacher, alpha):
    from fira_icse_b200 import distill
    m.zero_grad(set_to_none=True)
    bd = [t.to(DEV) for t in b]
    label = m.shifted_label(bd[6])
    targets = distill.teacher_targets(teacher, bd, label)
    loss, _, _ = distill.distill_loss(m, bd, targets, label, alpha)
    n = int((label != 0).sum())
    (loss / n).backward()
    torch.cuda.synchronize()
    return loss.item() / n, {k: p.grad for k, p in m.named_parameters() if p.grad is not None}


def _oracle_teacher(b, members, weights):
    """sum_m w_m of the members' float64 distributions [B, T, V + S]"""
    import fira_oracle as O
    t = 0
    with torch.no_grad():
        for w, mm in zip(weights, members):
            sd = {k: v.detach().cpu().double() for k, v in mm.state_dict().items()}
            det = {}
            O.forward(sd, *b, stage="train", detail=det)
            t = t + w * O.output_distribution(sd, det["memory"], det["mem_mask"], det["decoder"])[1]
    return t


def _oracle_loss(m, b, t, alpha):
    import fira_oracle as O
    sd = {k: v.detach().cpu().double().requires_grad_(v.is_floating_point()) for k, v in m.state_dict().items()}
    det = {}
    O.forward(sd, *b, stage="train", detail=det)
    keep = O.shifted_labels(b[6]) != 0
    kd = -(t * det["logp"]).sum(-1) * keep
    loss = ((1 - alpha) * det["nll"] + alpha * kd).sum() / keep.sum()
    loss.backward()
    return loss.item(), {k: v.grad for k, v in sd.items() if v.requires_grad}


def _ensemble_teacher():
    from fira_icse_b200.ensemble import Ensemble
    m1, m2 = _two_members()
    return Ensemble([m1, m2], [0.3, 0.7]), (m1, m2), (0.3, 0.7)


def test_whole_loss_gradients_fp32_match_float64():
    m = _plain("fp32")
    b = golden_batch(0, 3)
    ens, members, w = _ensemble_teacher()
    loss, grads = _loss_grads(m, b, ens, 0.5)
    ref_loss, ref = _oracle_loss(m, b, _oracle_teacher(b, members, w), 0.5)
    assert abs(loss - ref_loss) <= 1e-4 * abs(ref_loss)
    assert sorted(grads) == sorted(k for k, g in ref.items() if g is not None)
    for k, g in grads.items():
        r = ref[k].numpy()
        scale = float(np.abs(r).max())
        if k.endswith("fc_k.bias") or k == "copy_net.LinearRes.bias":
            assert float(g.abs().max()) < 1e-6, k
            continue
        np.testing.assert_allclose(g.cpu().numpy(), r, rtol=5e-3, atol=1e-7 + 5e-4 * scale, err_msg=k)


def test_whole_loss_gradients_bf16_match_float64(monkeypatch):
    """bf16 student, fp32 teacher: the teacher's triple carries fp32 rounding only, far inside the bf16 bound, so the
    shared bound of tests/test_gpu_bf16_step.py applies unchanged"""
    from test_gpu_bf16_step import check_step, record_gates
    m = _plain("bf16")
    b = golden_batch(0, 3)
    ens, members, w = _ensemble_teacher()
    loss, grads = _loss_grads(m, b, ens, 0.5)
    t = _oracle_teacher(b, members, w)
    gates = {}
    record_gates(monkeypatch, gates)                      # the student's gates only
    ref_loss, ref = _oracle_loss(m, b, t, 0.5)
    check_step("distill/padded", loss, grads, ref_loss, ref, gates)


def test_a_self_teacher_gives_no_gradient():
    """t = P is the minimum of the cross-entropy over P: alpha = 1 against an ensemble of the model's own copy"""
    from fira_icse_b200.ensemble import Ensemble
    m = _plain("fp32")
    b = golden_batch(0, 4)
    _, hard = _loss_grads(m, b, Ensemble([copy.deepcopy(m)]), 0.0)
    hard = {k: g.clone() for k, g in hard.items()}
    _, soft = _loss_grads(m, b, Ensemble([copy.deepcopy(m)]), 1.0)
    scale = max(float(g.abs().max()) for g in hard.values())
    worst = max(float(g.abs().max()) for g in soft.values())
    print(f"[distill] self-teacher: largest gradient {worst:.2e}, alpha = 0 scale {scale:.2e}")
    assert worst <= 1e-4 * scale


# ============================================================================= decoding after a step
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_sampling_after_a_step_uses_the_new_weights_without_recapture(precision):
    from fira_icse_b200 import TransModel, distill, optim
    from fira_icse_b200.decode_loop import _LOOPS
    from fira_icse_b200.sample import sample
    from fira_testlib import reference_args
    from test_gpu_sample import _model
    m = _model(precision)
    teacher = _two_members()[1].set_precision(precision)
    b = [t.to(DEV) for t in golden_batch(0, 8)]
    kw = dict(num_samples=4, top_p=0.95, seed=3, **_vocab_ids())
    opt = optim.FlatAdam(m.live_parameters(), lr=1e-3, groups=m.flat_groups())
    optim.attach(m, [opt])
    before = sample(m, b[0], b[3], b[4], b[5], b[7], **kw)
    (key, (_, _, loop)), = _LOOPS[m].items()
    graphs = dict(loop.graphs)
    assert graphs
    step = distill.distill_step(m, opt, b, teacher, alpha=0.5)
    assert np.isfinite(step.loss) and step.tokens > 0 and step.kd > 0.0
    assert abs(step.loss - (0.5 * step.nll + 0.5 * step.kd)) <= 1e-4 * step.loss
    m.eval()
    after = sample(m, b[0], b[3], b[4], b[5], b[7], **kw)
    assert _LOOPS[m][key][2] is loop and loop.graphs.keys() == graphs.keys()
    assert all(loop.graphs[k] is g for k, g in graphs.items())
    fresh = TransModel(reference_args())
    fresh.load_state_dict({k: v.cpu() for k, v in m.state_dict().items()})
    fresh = fresh.to(DEV).eval().set_precision(precision)
    ref = sample(fresh, b[0], b[3], b[4], b[5], b[7], **kw)
    # as tests/test_gpu_scst.py: compare each row up to its first differing draw (bf16 near-ties may flip)
    T = after.seq.shape[-1]
    differ = (after.seq != ref.seq) | (after.raw != ref.raw)
    first = torch.where(differ.any(-1), differ.float().argmax(-1), torch.full_like(differ[..., 0], T, dtype=torch.long))
    if precision == "fp32":
        assert bool((first == T).all())
    agree = torch.arange(T, device=DEV) < first.unsqueeze(-1)
    assert float(agree.float().mean()) >= 0.5
    tol = 1e-4 if precision == "fp32" else 0.5
    np.testing.assert_allclose(after.token_logprob[agree].cpu().numpy(), ref.token_logprob[agree].cpu().numpy(), rtol=0,
                               atol=tol)
    assert not torch.equal(after.token_logprob, before.token_logprob)


# ============================================================================= CLI
def test_run_model_distill_then_test(trained):  # noqa: F811
    d, env, _ = trained
    base = open(d / "best_model.pt", "rb").read()
    sd = torch.load(d / "best_model.pt", map_location="cpu")
    g = torch.Generator().manual_seed(4)
    second = {k: (v + torch.randn(v.shape, generator=g) * 0.05 * v.std() if v.is_floating_point() and v.numel() > 1
                  else v) for k, v in sd.items()}
    torch.save(second, d / "second.pt")
    other = open(d / "second.pt", "rb").read()
    r = _run_model("distill", d, dict(env, FIRA_MAX_BATCHES="2", FIRA_ENSEMBLE="best_model.pt,second.pt",
                                      FIRA_ENSEMBLE_WEIGHTS="2,1"))
    assert "kd epoch: 0 batch: 0/" in r.stdout and "best dev bleu" in r.stdout
    assert open(d / "best_model.pt", "rb").read() == base and open(d / "second.pt", "rb").read() == other
    kd = torch.load(d / "best_model_kd.pt", map_location="cpu")
    assert len(kd) == 338 and sorted(kd) == sorted(sd)
    assert os.path.getsize(d / "OUTPUT" / "dev_output_kd") > 0
    r = _run_model("test", d, dict(env, FIRA_CHECKPOINT="best_model_kd.pt"))
    assert "mean sentence bleu" in r.stdout
    assert os.path.getsize(d / "OUTPUT" / "output_fira") > 0
