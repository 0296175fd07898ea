"""Global-norm gradient clipping on the device: fira_grad_sumsq against float64, fira_grad_clip_finalize against the rule,
fira_adam_flat_clip against fira_adam_flat (the same bits at coef = 1) and against the rule, optim.FlatAdam(max_grad_norm)
and optim.ClipGroup against torch's clip_grad_norm_ + Adam, every GraphedTrainStep mode replay by replay against
clip_rule (tests/clip_rule.py), a non-finite step in the engine, and `run_model.py train` / `finetune` with
FIRA_CLIP_NORM."""
import copy
import gc
import os

import numpy as np
import pytest
import torch

import clip_rule
import ema_rule
from fira_testlib import ROOT, load_raw_golden, seeded_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LR, B1, B2, EPS = 1e-3, 0.9, 0.999, 1e-8
F32 = dict(dtype=torch.float32, device=DEV)
F64 = dict(dtype=torch.float64, device=DEV)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    yield
    # hand the engines' graph pools back to the device before the next module: later modules start training
    # subprocesses of their own on this GPU
    gc.collect()
    torch.cuda.empty_cache()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _blocks(n):
    from fira_icse_b200 import _lib
    return _lib.lib().fira_grad_sumsq_blocks(n)


def _sumsq(g, partials=None):
    from fira_icse_b200 import _lib
    if partials is None:
        partials = torch.full((_blocks(g.numel()),), -1.0, **F64)
    _lib.call("fira_grad_sumsq", g.data_ptr(), g.numel(), partials.data_ptr(), _stream())
    return partials


def _finalize(partials, state, c, steps=(), scale=None):
    from fira_icse_b200 import _lib
    ptrs = torch.tensor([t.data_ptr() for t in steps] or [0], dtype=torch.int64, device=DEV)
    _lib.call("fira_grad_clip_finalize", partials.data_ptr(), partials.numel(),
              scale.data_ptr() if scale is not None else None, c, state.data_ptr(), ptrs.data_ptr(), len(steps),
              _stream())
    torch.cuda.synchronize()                                   # ptrs must outlive the launch


def _state(coef=1.0, taken=1.0):
    return torch.tensor([0.0, coef, taken, 0.0, 0.0], **F64)


# ============================================================================= fira_grad_sumsq
@pytest.mark.parametrize("case", ["partial_block", "two_passes", "zeros", "fp32_overflow"])
def test_sumsq_against_float64(case):
    n = {"partial_block": 8 * 1001, "two_passes": 8 * (2 * 1024 * 256 + 77), "zeros": 8 * 5000,
         "fp32_overflow": 8 * 3001}[case]
    gen = torch.Generator(device=DEV).manual_seed(n)
    g = torch.randn(n, generator=gen, **F32)
    if case == "zeros":
        g.zero_()
    if case == "fp32_overflow":
        g *= 3e19                                              # g^2 ~ 1e39 > fp32 max; the norm (~1e22) is finite
    assert _blocks(n) == min(1024, (n // 8 + 255) // 256)
    partials = _sumsq(g)
    torch.cuda.synchronize()
    got = float(partials.sum())                                # float64 partials: their order barely matters here
    ref = float(np.sum(np.square(g.cpu().double().numpy())))
    if case == "zeros":
        assert got == 0.0 and torch.equal(partials, torch.zeros_like(partials))
    else:
        assert np.isfinite(got) and got == pytest.approx(ref, rel=1e-12)
    # the finalize's norm is the same sum
    state = _state()
    _finalize(partials, state, float("inf"))
    assert state[0].item() == pytest.approx(np.sqrt(ref), rel=1e-12, abs=0.0)


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")])
def test_sumsq_of_a_non_finite_gradient_is_not_finite(bad):
    g = torch.randn(8 * 4096, **F32)
    g[12345] = bad
    partials = _sumsq(g)
    torch.cuda.synchronize()
    assert not np.isfinite(float(partials.sum()))


def test_sumsq_is_bitwise_repeatable_and_stream_independent():
    n = 8 * (1024 * 256 + 999)
    g = torch.randn(n, **F32) * 1e3
    a = _sumsq(g)
    b = _sumsq(g)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        c = _sumsq(g)
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int64), b.view(torch.int64)) and torch.equal(a.view(torch.int64), c.view(torch.int64))
    states = []
    for p in (a, c):
        st = _state()
        _finalize(p, st, 1.0)
        states.append(st)
    assert torch.equal(states[0].view(torch.int64), states[1].view(torch.int64))


# ============================================================================= fira_grad_clip_finalize
@pytest.mark.parametrize("scaled", [False, True])
def test_finalize_follows_the_rule(scaled):
    parts = [torch.rand(_blocks(8 * k), **F64) * 10 for k in (1001, 64, 300_001)]   # three members, back to back
    partials = torch.cat(parts)
    S = float(partials.sum())
    scale = torch.tensor(37.0, **F32) if scaled else None
    s = 37.0 if scaled else 1.0
    steps = [torch.tensor(float(k), **F32) for k in (3, 5, 9)]
    state = _state()
    for c, clipped in ((1e6, 0), (1.0, 1), (float("inf"), 1)):
        _finalize(partials, state, c, steps, scale)
        nrm = np.sqrt(S) / s
        assert state[0].item() == pytest.approx(nrm, rel=1e-13)
        assert state[1].item() == clip_rule.coefficient(nrm, c)
        assert state[2].item() == 1.0 and state[3].item() == clipped and state[4].item() == 0
    assert [t.item() for t in steps] == [6.0, 8.0, 12.0]
    partials[7] = float("inf")                                 # a non-finite step: flag 0, skipped + 1, no step counted
    _finalize(partials, state, 1.0, steps, scale)
    assert state[0].item() == float("inf") and state[2].item() == 0.0
    assert state[3].item() == 1 and state[4].item() == 1 and state[1].item() == 1.0     # the last taken step's coef
    assert [t.item() for t in steps] == [6.0, 8.0, 12.0]


def test_finalize_argument_checks():
    from fira_icse_b200._lib import FiraLibraryError
    partials = torch.ones(4, **F64)
    state = _state()
    for c in (0.0, -1.0, float("nan"), float("-inf")):
        with pytest.raises(FiraLibraryError, match="max_norm"):
            _finalize(partials, state, c)
    from fira_icse_b200 import _lib
    with pytest.raises(FiraLibraryError, match="null"):
        _lib.call("fira_grad_clip_finalize", partials.data_ptr(), 4, None, 1.0, None, None, 0, _stream())
    with pytest.raises(FiraLibraryError, match="null"):
        _lib.call("fira_grad_clip_finalize", partials.data_ptr(), 4, None, 1.0, state.data_ptr(), None, 1, _stream())
    torch.cuda.synchronize()
    assert torch.equal(state, _state())                        # nothing was launched


# ============================================================================= fira_adam_flat_clip
def _adam(p, g, m, v, p16, t, scale, ema=None, d=0.0, clip=None):
    from fira_icse_b200 import _lib
    args = [p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p16.data_ptr(), p.numel(), LR, B1, B2, EPS,
            t.data_ptr(), scale.data_ptr() if scale is not None else None,
            ema.data_ptr() if ema is not None else None, d]
    if clip is None:
        _lib.call("fira_adam_flat", *args, _stream())
    else:
        _lib.call("fira_adam_flat_clip", *args, clip.data_ptr(), _stream())


def _bufs(n, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return dict(p=torch.randn(n, generator=gen, **F32), m=torch.randn(n, generator=gen, **F32) * 0.1,
                v=torch.rand(n, generator=gen, **F32) * 0.01, e=torch.randn(n, generator=gen, **F32),
                p16=torch.zeros(n, dtype=torch.bfloat16, device=DEV)), torch.randn(n, generator=gen, **F32) * 3.0


def _clone(b):
    return {k: t.clone() for k, t in b.items()}


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


KEYS = ("p", "m", "v", "e", "p16")


@pytest.mark.parametrize("n", [8 * 1001, 8 * 300_001])
@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("with_ema", [False, True])
def test_adam_clip_at_coef_one_is_fira_adam_flat(n, scaled, with_ema):
    b0, g = _bufs(n, n + 2 * scaled + with_ema)
    t = torch.tensor(7.0, **F32)
    scale = torch.tensor(37.0, **F32) if scaled else None
    d = 0.999 if with_ema else 0.0
    ref, got = _clone(b0), _clone(b0)
    _adam(ref["p"], g, ref["m"], ref["v"], ref["p16"], t, scale, ref["e"] if with_ema else None, d)
    _adam(got["p"], g, got["m"], got["v"], got["p16"], t, scale, got["e"] if with_ema else None, d, clip=_state(1.0))
    torch.cuda.synchronize()
    for k in KEYS:
        assert torch.equal(_bits(ref[k]), _bits(got[k])), k


@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("with_ema", [False, True])
def test_adam_clip_below_one_follows_the_rule(scaled, with_ema):
    n = 8 * 300_001
    b0, g = _bufs(n, 7 + scaled)
    t = torch.tensor(4.0, **F32)
    scale = torch.tensor(37.0, **F32) if scaled else None
    coef = clip_rule.coefficient(9.0, 2.0)                     # fl32(2 / (9 + 1e-6))
    d = 0.99 if with_ema else 0.0
    got = _clone(b0)
    _adam(got["p"], g, got["m"], got["v"], got["p16"], t, scale, got["e"] if with_ema else None, d,
          clip=_state(coef))
    # the same bits as fira_adam_flat fed g' = fl(fl(g * fl(1 / s)) * coef) with no scale: the clip is that product
    gp = torch.from_numpy(clip_rule.scaled_grad(g.cpu().numpy(), coef, 37.0 if scaled else None).astype(np.float32))
    gp = gp.to(DEV)
    ref = _clone(b0)
    _adam(ref["p"], gp, ref["m"], ref["v"], ref["p16"], t, None, ref["e"] if with_ema else None, d)
    torch.cuda.synchronize()
    for k in KEYS:
        assert torch.equal(_bits(ref[k]), _bits(got[k])), k
    # and against the float64 rule
    h = {k: b0[k].cpu().double().numpy() for k in ("p", "m", "v", "e")}
    gp64 = clip_rule.scaled_grad(g.cpu().numpy(), coef, 37.0 if scaled else None)
    p64, m64, v64 = ema_rule.adam(h["p"], gp64, h["m"], h["v"], 4.0, LR, B1, B2, EPS)
    # m cancels to near zero in places: its error is an fp32 rounding of the terms b1 m and (1 - b1) g' (|.| < 1)
    np.testing.assert_allclose(got["m"].cpu().double().numpy(), m64, rtol=1e-5, atol=2.0 ** -23)
    np.testing.assert_allclose(got["v"].cpu().double().numpy(), v64, rtol=1e-5, atol=1e-12)
    np.testing.assert_allclose(got["p"].cpu().double().numpy(), p64, rtol=1e-6, atol=1e-6)


def test_adam_clip_skipped_step_writes_nothing():
    n = 8 * 300_001
    b0, g = _bufs(n, 11)
    t = torch.tensor(4.0, **F32)
    got = _clone(b0)
    _adam(got["p"], g, got["m"], got["v"], got["p16"], t, None, got["e"], 0.9, clip=_state(0.5, taken=0.0))
    torch.cuda.synchronize()
    for k in KEYS:
        assert torch.equal(_bits(b0[k]), _bits(got[k])), k
    assert t.item() == 4.0


def test_adam_clip_argument_checks():
    from fira_icse_b200 import _lib
    from fira_icse_b200._lib import FiraLibraryError
    n = 64
    p, g, m, v, e = (torch.zeros(n + 8, **F32) for _ in range(5))
    p16 = torch.zeros(n, dtype=torch.bfloat16, device=DEV)
    t = torch.tensor(1.0, **F32)
    clip = _state(0.5)

    def call(clip_ptr=clip.data_ptr(), nn=n, p_ptr=p.data_ptr(), e_ptr=None, d=0.0):
        _lib.call("fira_adam_flat_clip", p_ptr, g.data_ptr(), m.data_ptr(), v.data_ptr(), p16.data_ptr(), nn, LR, B1, B2,
                  EPS, t.data_ptr(), None, e_ptr, d, clip_ptr, _stream())

    with pytest.raises(FiraLibraryError, match="null"):
        call(clip_ptr=None)
    with pytest.raises(FiraLibraryError, match="multiple of 8"):
        call(nn=60)
    with pytest.raises(FiraLibraryError, match="alignment"):
        call(p_ptr=p.data_ptr() + 4)
    with pytest.raises(FiraLibraryError, match="alignment"):
        call(clip_ptr=clip.data_ptr() + 4)
    for d in (0.0, 1.0, float("nan")):
        with pytest.raises(FiraLibraryError, match="ema_decay"):
            call(e_ptr=e.data_ptr(), d=d)
    with pytest.raises(FiraLibraryError, match="multiple of 8"):
        _lib.call("fira_grad_sumsq", g.data_ptr(), 60, clip.data_ptr(), _stream())
    with pytest.raises(FiraLibraryError, match="alignment"):
        _lib.call("fira_grad_sumsq", g.data_ptr() + 4, 64, clip.data_ptr(), _stream())
    torch.cuda.synchronize()
    for x in (p, m, v, e):
        assert torch.equal(x, torch.zeros_like(x))             # nothing was launched
    assert torch.equal(clip, _state(0.5))


# ============================================================================= FlatAdam / ClipGroup
def _params(seed):
    g = torch.Generator().manual_seed(seed)
    shapes = [(256, 256), (256,), (256, 256), (256,), (1024, 256), (1024,), (2,), (1,), (1, 256), (333, 256), (24650,)]
    return [torch.nn.Parameter(torch.randn(s, generator=g).to(DEV)) for s in shapes]


def _grads(step, params):
    g = torch.Generator().manual_seed(100 + step)
    return [torch.randn(p.shape, generator=g).to(DEV) * 10.0 ** (step % 3 - 1) for p in params]


def _set_grads(params, grads):
    for q, gr in zip(params, grads):
        q.grad = gr.clone()


def _groups(ps):
    return [[ps[0], ps[2]], [ps[1], ps[3]]]


def test_flat_adam_clip_matches_torch_clip_and_adam():
    """c between the small and the large steps' norms (about 71, 710 and 7100): some steps clip, some do not"""
    from fira_icse_b200.optim import FlatAdam
    c = 200.0
    ref, mine = _params(0), _params(0)
    opt_ref = torch.optim.Adam(ref, lr=LR)
    opt = FlatAdam(mine, lr=LR, groups=_groups(mine), max_grad_norm=c)
    norms = []
    for step in range(20):
        grads = _grads(step, ref)
        _set_grads(ref, grads)
        _set_grads(mine, grads)
        norms.append(float(torch.nn.utils.clip_grad_norm_(ref, c)))
        opt_ref.step()
        opt.step()
        assert opt.grad_norm.item() == pytest.approx(norms[-1], rel=1e-6)
    torch.cuda.synchronize()
    n_clipped = sum(x > c for x in norms)
    assert 0 < n_clipped < 20 and opt.clipped.item() == n_clipped and opt.skipped.item() == 0
    assert opt.step_t.item() == 20.0
    sd = opt.state_dict()
    for p, q, m in zip(ref, mine, sd["exp_avg"]):
        torch.testing.assert_close(q.data, p.data, rtol=2e-6, atol=2e-7)
        torch.testing.assert_close(m, opt_ref.state[p]["exp_avg"], rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("with_ema", [False, True])
def test_flat_adam_clip_at_inf_is_bitwise_flat_adam(with_ema):
    from fira_icse_b200.optim import FlatAdam
    a, b = _params(1), _params(1)
    d = 0.9 if with_ema else None
    opt_a = FlatAdam(a, lr=LR, groups=_groups(a), ema_decay=d)
    opt_b = FlatAdam(b, lr=LR, groups=_groups(b), ema_decay=d, max_grad_norm=float("inf"))
    for step in range(6):
        grads = _grads(step, a)
        _set_grads(a, grads)
        _set_grads(b, grads)
        opt_a.step()
        opt_b.step()
    torch.cuda.synchronize()
    for k in ("p", "m", "v", "p16", "step_t") + (("ema",) if with_ema else ()):
        assert torch.equal(getattr(opt_a, k), getattr(opt_b, k)), k
    assert opt_b.clipped.item() == 0 and opt_b.skipped.item() == 0 and np.isfinite(opt_b.grad_norm.item())
    assert list(opt_b.state_dict()) == list(opt_a.state_dict())


def test_flat_adam_skips_a_non_finite_step():
    from fira_icse_b200.optim import FlatAdam
    a = _params(2)
    opt = FlatAdam(a, lr=LR, groups=_groups(a), ema_decay=0.9, max_grad_norm=1.0)
    for step in range(3):
        _set_grads(a, _grads(step, a))
        opt.step()
    before = {k: getattr(opt, k).clone() for k in ("p", "m", "v", "p16", "ema", "step_t")}
    grads = _grads(3, a)
    grads[4][7, 9] = float("nan")
    _set_grads(a, grads)
    opt.step()
    torch.cuda.synchronize()
    for k, x in before.items():
        assert torch.equal(_bits(x) if x.dim() else x, _bits(getattr(opt, k)) if x.dim() else getattr(opt, k)), k
    assert opt.skipped.item() == 1 and not np.isfinite(opt.grad_norm.item())
    _set_grads(a, _grads(4, a))
    opt.step()
    torch.cuda.synchronize()
    assert opt.step_t.item() == 4.0 and np.isfinite(opt.grad_norm.item()) and not torch.equal(opt.p, before["p"])


def test_clip_group_matches_one_flat_adam():
    """two FlatAdam instances over halves of the parameters in one ClipGroup against one FlatAdam over all of them: the
    same norm (up to the grouping of the float64 partials), so the same trajectory within fp32 roundings"""
    from fira_icse_b200.optim import ClipGroup, FlatAdam
    one, two = _params(3), _params(3)
    opt = FlatAdam(one, lr=LR, max_grad_norm=30.0)
    o1, o2 = FlatAdam(two[:5], lr=LR, max_grad_norm=30.0), FlatAdam(two[5:], lr=LR, max_grad_norm=30.0)
    grp = ClipGroup([o1, o2])
    assert o1.clip is grp and o2.clip is grp
    with pytest.raises(RuntimeError, match="ClipGroup"):
        o1.step()
    for step in range(12):
        grads = _grads(step, one)
        _set_grads(one, grads)
        _set_grads(two, grads)
        opt.step()
        grp.step()
        assert grp.grad_norm.item() == pytest.approx(opt.grad_norm.item(), rel=1e-12)
    torch.cuda.synchronize()
    assert grp.clipped.item() == opt.clipped.item() > 0
    assert o1.step_t.item() == o2.step_t.item() == opt.step_t.item() == 12.0
    for p, q in zip(one, two):
        torch.testing.assert_close(q.data, p.data, rtol=1e-6, atol=1e-7)
    with pytest.raises(ValueError, match="same max_grad_norm"):
        ClipGroup([FlatAdam(_params(4), lr=LR, max_grad_norm=1.0), FlatAdam(_params(5), lr=LR, max_grad_norm=2.0)])
    with pytest.raises(ValueError, match="same max_grad_norm"):
        ClipGroup([FlatAdam(_params(4), lr=LR, max_grad_norm=1.0), FlatAdam(_params(5), lr=LR)])
    with pytest.raises(ValueError, match="max_grad_norm"):
        FlatAdam(_params(6), lr=LR, max_grad_norm=0.0)


def test_flat_adam_clip_state_dict_roundtrip_is_bit_exact():
    from fira_icse_b200.optim import FlatAdam
    a = _params(7)
    opt_a = FlatAdam(a, lr=LR, groups=_groups(a), max_grad_norm=5.0)
    for step in range(6):
        _set_grads(a, _grads(step, a))
        opt_a.step()
    sd = opt_a.state_dict()
    assert list(sd) == ["step", "lr", "betas", "eps", "exp_avg", "exp_avg_sq"] and sd["step"] == 6.0
    b = [torch.nn.Parameter(q.detach().clone()) for q in a]
    opt_b = FlatAdam(b, lr=LR, groups=_groups(b), max_grad_norm=5.0)
    opt_b.load_state_dict(sd)
    for step in range(6, 12):
        grads = _grads(step, a)
        _set_grads(a, grads)
        _set_grads(b, grads)
        opt_a.step()
        opt_b.step()
    torch.cuda.synchronize()
    for k in ("p", "m", "v", "p16", "step_t"):
        assert torch.equal(getattr(opt_a, k), getattr(opt_b, k)), k


# ============================================================================= the engine
def _hosts():
    from fira_icse_b200.packed import PackedTables, pack_from_dataset
    from test_packed import GoldenSplit, V
    tables = PackedTables(GoldenSplit())
    eight = [pack_from_dataset(tables, np.arange(lo, lo + 8), V) for lo in (0, 16)]
    six = [pack_from_dataset(tables, np.arange(lo, lo + 6), V) for lo in (40, 64)]
    return [eight[0], six[0], eight[1], six[1]]


def _engine(mode, monkeypatch, c, d=None):
    from fira_icse_b200.engine import GraphedTrainStep
    from fira_icse_b200.optim import FlatAdam
    if mode == "single_opt":
        monkeypatch.setenv("FIRA_OPT_OVERLAP", "0")
    else:
        monkeypatch.delenv("FIRA_OPT_OVERLAP", raising=False)
    m = copy.deepcopy(seeded_model()).to(DEV)
    m.train()
    m.set_precision("bf16")
    eng = GraphedTrainStep(m, 8, lambda ps: FlatAdam(ps, lr=LR, groups=m.flat_groups(), ema_decay=d, max_grad_norm=c),
                           edge_capacity=65536, split=True if mode == "split" else None)
    return m, eng


def _snap(eng):
    out = []
    for o in eng.flat_optims:
        s = {k: getattr(o, k).cpu().double().numpy() for k in ("p", "m", "v")}
        s["t"] = o.step_t.item()
        s["e"] = o.ema.cpu().double().numpy() if o.ema is not None else None
        out.append(s)
    return out


def _check_replay(eng, before, c, d):
    """the replay that just ran against clip_rule from the snapshot `before` and the gradients it left in g;
    -> coef"""
    grads = [o.g.cpu().double().numpy() for o in eng.flat_optims]
    after = _snap(eng)
    S, nrm = clip_rule.norm(grads)
    assert np.isfinite(S)
    assert eng.grad_norm.item() == pytest.approx(nrm, rel=1e-10)
    coef = clip_rule.coefficient(eng.grad_norm.item(), c)
    for b, a, g in zip(before, after, grads):
        assert a["t"] == b["t"] + 1
        gp = clip_rule.scaled_grad(g, coef)
        p64, m64, v64 = ema_rule.adam(b["p"], gp, b["m"], b["v"], a["t"], LR, B1, B2, EPS)
        for got, ref, key in ((a["m"], m64, "m"), (a["v"], v64, "v"), (a["p"], p64, "p")):
            tol = 2e-6 * np.abs(ref) + 1e-6 * float(np.abs(ref).max()) * (key != "p") + 1e-6 * (key == "p")
            err = np.abs(got - ref)
            assert np.all(err <= tol), (key, float(np.max(err / tol)))
        if d is not None:
            e64 = ema_rule.ema(b["e"], a["p"], d)
            ulp = np.spacing(np.abs(e64).astype(np.float32)).astype(np.float64)
            assert np.all(np.abs(a["e"] - e64) <= 2 * ulp)
    return coef


@pytest.mark.parametrize("c,d", [(1e-3, 0.9), (float("inf"), None)])
@pytest.mark.parametrize("mode", ["overlap", "single_opt", "split"])
def test_engine_clips_every_replay_by_the_rule(mode, c, d, monkeypatch):
    """c = 1e-3 is far below the model's gradient norm: every step clips (with the EMA on, it follows the clipped
    parameters); c = inf never clips.  Each replay is checked from a snapshot of p, m, v, t taken before it and g read
    after it (g lives until the next step's zero-fill)."""
    m, eng = _engine(mode, monkeypatch, c, d)
    hosts = [pb.to(DEV) for pb in _hosts()]
    eng.step(hosts[0])                                          # the eager first step: the optimizers exist now
    assert eng.clip is not None and len(eng.flat_optims) == (1 if mode == "single_opt" else 2)
    assert all(o.clip is eng.clip for o in eng.flat_optims)    # one norm over both halves
    steps = 6
    for k in range(1, steps + 1):
        before = _snap(eng)
        eng.step(hosts[k % len(hosts)])
        torch.cuda.synchronize()
        coef = _check_replay(eng, before, c, d)
        assert (coef < 1.0) == (c != float("inf"))
    assert len(eng.captured) >= 2
    assert eng.clipped.item() == (steps + 1 if c != float("inf") else 0) and eng.skipped.item() == 0


@pytest.mark.parametrize("mode", ["overlap", "single_opt", "split"])
def test_engine_skips_a_non_finite_step_and_goes_on(mode, monkeypatch):
    m, eng = _engine(mode, monkeypatch, 1.0, 0.9)
    hosts = [pb.to(DEV) for pb in _hosts()]
    for k in range(3):                                          # the eager step, then both shapes captured
        eng.step(hosts[k % 2])
    graphs = {key: (c.graph, getattr(c, "graph_b", None)) for key, c in eng.captured.items()}
    opt_graphs = eng.graph_opt if isinstance(eng.graph_opt, list) else [eng.graph_opt]
    w = m.out_fc.weight
    keep = w[3, 5].item()
    with torch.no_grad():
        w[3, 5] = float("inf")                                  # a used weight: every logit row sees it
    for o in eng.flat_optims:
        o.sync_mirror()
    torch.cuda.synchronize()
    before = {(i, k): getattr(o, k).clone() for i, o in enumerate(eng.flat_optims)
              for k in ("p", "m", "v", "p16", "ema", "step_t")}
    eng.step(hosts[1])
    torch.cuda.synchronize()
    assert eng.skipped.item() == 1 and not np.isfinite(eng.grad_norm.item())
    for (i, k), x in before.items():
        y = getattr(eng.flat_optims[i], k)
        assert torch.equal(_bits(x), _bits(y)) if x.dim() else torch.equal(x, y), (i, k)
    with torch.no_grad():
        w[3, 5] = keep
    for o in eng.flat_optims:
        o.sync_mirror()
    for k in range(2):                                          # training goes on by the rule, on the same graphs
        before = _snap(eng)
        eng.step(hosts[k % 2])
        torch.cuda.synchronize()
        _check_replay(eng, before, 1.0, 0.9)
    assert eng.skipped.item() == 1
    assert {key: (c.graph, getattr(c, "graph_b", None)) for key, c in eng.captured.items()} == graphs
    assert (eng.graph_opt if isinstance(eng.graph_opt, list) else [eng.graph_opt]) == opt_graphs


# ============================================================================= run_model.py
def _train_dir(tmp_path_factory, name, **extra):
    from test_data import _write_dataset
    from test_gpu_cli import _run_model
    d = tmp_path_factory.mktemp(name)
    _write_dataset(str(d), load_raw_golden())
    env = dict(os.environ, PYTHONPATH=ROOT, FIRA_EPOCHS="16", FIRA_BATCH="16", FIRA_MAX_BATCHES="1",
               FIRA_WORKERS="0", FIRA_TEST_BATCH="4")
    env.pop("FIRA_CLIP_NORM", None)
    env.update(extra)
    return d, env, _run_model("train", d, env)


def test_run_model_train_and_finetune_with_clip_norm(tmp_path_factory):
    from test_gpu_cli import _run_model
    d, env, r = _train_dir(tmp_path_factory, "cli_clip", FIRA_CLIP_NORM="1e-3")
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("epoch: ") and " batch: " in ln]
    assert len(lines) == 16, r.stdout[-2000:]
    for k, ln in enumerate(lines):
        assert " grad_norm: " in ln and f" clipped: {k + 1} skipped: 0" in ln, ln       # 1 batch per epoch, all clip
        assert float(ln.split(" grad_norm: ")[1].split()[0]) > 1e-3
    assert os.path.exists(d / "best_model.pt")
    r = _run_model("finetune", d, dict(env, FIRA_MAX_BATCHES="2", FIRA_SAMPLES="4", FIRA_CLIP_NORM="inf"))
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("scst epoch: 0 batch: 0/")]
    assert lines and " grad_norm: " in lines[0] and " clipped: 0 skipped: 0" in lines[0], r.stdout[-2000:]
    assert os.path.exists(d / "best_model_scst.pt")


def test_run_model_train_without_clip_norm_prints_no_gradient_fields(tmp_path_factory):
    d, _, r = _train_dir(tmp_path_factory, "cli_no_clip")
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("epoch: ") and " batch: " in ln]
    assert len(lines) == 16 and not any("grad_norm" in ln or "clipped" in ln for ln in lines)
    assert os.path.exists(d / "best_model.pt")
