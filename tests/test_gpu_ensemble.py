"""Ensemble decoding on the GPU: fira_pointer_mix_ensemble against the float64 rewrite (tests/ensemble_rule.py), an
ensemble of one model with itself against the model, two distinct members against their own scores, graph reuse
across batches, Ensemble objects and weights, and `run_model.py test` with FIRA_ENSEMBLE."""
import copy
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from ensemble_rule import average
from fira_testlib import ROOT, golden_batch
from sample_rule import mixture
from test_gpu_cli import _test_lines, trained  # noqa: F401  (the trained-model fixture)
from test_gpu_constraints import _check_rules, _self_score
from test_gpu_nbest import _check, _nbest
from test_gpu_prefix import _eos_prefix, _score
from test_gpu_sample import _check_bookkeeping, _head_nll, _inputs, _model, _sample, _vocab

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _combine(members, log_w, mem_mask, N, V, S, ld_out=None, rc_only=False, over=None):
    """fira_pointer_mix_ensemble on members [(logits, sc, gl)] -> (x' [R, V], c' [B, N, S], gl' [R, 2]) or its code"""
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import FIRA_BF16, FIRA_F32, lib
    R = members[0][0].shape[0]
    B = R // N
    ld_out = ops._ld_logits(V) if ld_out is None else ld_out
    out = torch.full((R, ld_out), float("nan"), dtype=torch.float32, device=DEV)
    sc = torch.empty((B, N, S), dtype=torch.float32, device=DEV)
    gl = torch.empty((R, 2), dtype=torch.float32, device=DEV)
    M = len(members)
    arr = [(ctypes.c_void_p * max(M, 1))(*[ops._ptr(t[k]) for t in members]) for k in range(3)]
    lw = torch.tensor(log_w, dtype=torch.float32, device=DEV)
    a = dict(logits=ctypes.addressof(arr[0]), ld=members[0][0].stride(0), sc=ctypes.addressof(arr[1]),
             gl=ctypes.addressof(arr[2]), M=M, lw=ops._ptr(lw), mask=ops._ptr(mem_mask), out=ops._ptr(out), ld_out=ld_out,
             sc_out=ops._ptr(sc), gl_out=ops._ptr(gl), B=B, N=N, V=V, S=S,
             dtype=FIRA_BF16 if members[0][0].dtype == torch.bfloat16 else FIRA_F32)
    a.update(over or {})
    rc = lib().fira_pointer_mix_ensemble(*a.values(), ops._stream())
    if rc_only:
        return rc
    assert rc == 0
    torch.cuda.synchronize()
    return out, sc, gl


def _members(seed, M, B, N, V, S, dtype):
    """M members' rows planted as test_gpu_sample._inputs, one shared mem_mask; the last member's gate is saturated to
    the copy side (g0 = 0 in fp32) on half the rows, and every member's on row 0 (G0 = 0)"""
    gen = torch.Generator().manual_seed(seed)
    out = [_inputs(gen, B, N, V, S, dtype) for _ in range(M)]
    mem_mask = out[0][3]
    members = []
    for m, (logits, sc, gl, _, _) in enumerate(out):
        sc = sc.masked_fill(mem_mask.unsqueeze(1) == 0, 40.0)      # masked positions would dominate if they counted
        if m == M - 1:
            gl[: gl.shape[0] // 2] = torch.tensor([-200.0, 0.0], device=DEV)
        gl[0] = torch.tensor([-200.0, 0.0], device=DEV)
        members.append((logits, sc.contiguous(), gl))
    return members, mem_mask


# relative to max(1, |log P|): x' is rounded once to fp32 and the step kernels' softmax of it adds its own fp32 rounding.
# Measured on an H100 over every case below: at most 1.3e-6 (6e-8 for M = 1); the bound keeps a 4x margin.
LOG_TOL = 5e-6


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("V,S", [(24650, 370), (61, 13)])
@pytest.mark.parametrize("M", [1, 2, 3, 8])
def test_kernel_matches_float64_rule(dtype, V, S, M):
    B, N = 3, 4
    R = B * N
    members, mem_mask = _members(V + S + 31 * M + (dtype == torch.bfloat16), M, B, N, V, S, dtype)
    w = np.linspace(1.0, 2.0, M)
    w = w / w.sum()
    x, c, gl = _combine(members, np.log(w), mem_mask, N, V, S)
    mk = mem_mask.cpu().numpy()
    xn, cn, gn = x.cpu().numpy()[:, :V].astype(np.float64), c.cpu().numpy().reshape(R, S), gl.cpu().numpy()
    assert np.isfinite(xn).all() and np.isfinite(cn).all()
    host = [(lg.float().cpu().numpy()[:, :V].astype(np.float64), sc.cpu().numpy().reshape(R, S), g.cpu().numpy())
            for lg, sc, g in members]
    worst = 0.0
    refs = []
    for r in range(R):
        rows = [(h[0][r], h[1][r], h[2][r]) for h in host]
        ref = average(rows, w, mk[r // N], mixture)
        got = mixture(xn[r], cn[r], gn[r], mk[r // N])
        refs.append(ref)
        ok = ref >= 1e-30
        lr, lg_ = np.log(ref[ok]), np.log(np.maximum(got[ok], 1e-300))
        err = np.abs(lg_ - lr) / np.maximum(1.0, np.abs(lr))
        worst = max(worst, float(err.max()))
        assert (got[V:][mk[r // N] == 0] == 0).all()
    print(f"[ensemble] {dtype} V={V} S={S} M={M}: largest relative error of log P {worst:.2e}")
    assert worst <= LOG_TOL, worst
    assert np.all(gn[0, 0] == -np.inf)                    # row 0: every member saturated, G0 = 0
    # the loss kernel on the output (FIRA_F32) returns -log P
    gen = np.random.default_rng(V + M)
    label = np.zeros(R, np.int64)
    for r in range(R):
        ok = np.nonzero(refs[r] >= 1e-10)[0]
        ok = ok[ok != 0]
        label[r] = gen.choice(ok)
    nll = _head_nll(x, c, gl, mem_mask, label, N, V)
    ref = np.array([-np.log(refs[r][label[r]]) for r in range(R)])
    np.testing.assert_array_less(np.abs(nll - ref), LOG_TOL * np.maximum(1.0, ref) + 1e-12)


def test_kernel_refuses_invalid_arguments():
    V, S, B, N = 61, 13, 2, 2
    members, mem_mask = _members(1, 2, B, N, V, S, torch.float32)
    assert _combine(members, [np.log(0.5)] * 2, mem_mask, N, V, S, rc_only=True) == 0
    codes = dict(shape=1, align=2, dtype=4, arg=5)
    for over, code in [(dict(M=0), "arg"), (dict(M=9), "arg"), (dict(lw=None), "arg"), (dict(mask=None), "arg"),
                       (dict(out=None), "arg"), (dict(logits=None), "arg"), (dict(ld=62), "align"),
                       (dict(ld_out=60), "align"), (dict(V=32767 - S + 1), "shape"), (dict(N=0), "shape"),
                       (dict(S=0), "shape"), (dict(dtype=7), "dtype")]:
        assert _combine(members, [np.log(0.5)] * 2, mem_mask, N, V, S, rc_only=True, over=over) == codes[code], over
    lg = members[0][0]
    buf = torch.zeros(lg.numel() + 8, dtype=lg.dtype, device=DEV)
    bad = [(buf[1:1 + lg.numel()].view(lg.shape),) + members[0][1:], members[1]]               # 4 bytes off
    assert _combine(bad, [np.log(0.5)] * 2, mem_mask, N, V, S, rc_only=True) == codes["align"]
    null = [members[0], (members[1][0], members[1][1], None)]                                # a member's null pointer
    assert _combine(null, [np.log(0.5)] * 2, mem_mask, N, V, S, rc_only=True) == codes["arg"]


# ------------------------------------------------------------------ end to end
def _ens(models, weights=None):
    from fira_icse_b200.ensemble import Ensemble
    return Ensemble(models, weights)


# bf16: the decoder's split-K products add fp32 partials atomically in no fixed order, so two runs of the same bf16
# model differ (measured on an H100: up to 0.03-0.12 in a token's log-probability on the sharpened model, varying from
# run to run).  The ensemble runs its members' decoders separately from the runs it is compared with, so in bf16 the
# comparison uses the bound of the other bf16 decoding tests (test_gpu_sample.py): median <= 5e-2, max <= 0.5.
BF16_MEDIAN, BF16_MAX = 5e-2, 0.5


def _close(got, want, precision, tol=1e-5):
    d = (got - want).abs()
    if precision == "fp32":
        assert (d <= tol * want.abs().clamp(min=1.0)).all(), d.max()
    else:
        assert d.median().item() <= BF16_MEDIAN and d.max().item() <= BF16_MAX, d.max()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_an_ensemble_of_a_model_with_itself_is_the_model(precision):
    m = _model(precision)
    ens = _ens([m, m], [0.3, 0.7])
    b = golden_batch(0, 8)
    v = _vocab()
    got, want = _score(ens, b).token_logprob.cpu(), _score(m, b).token_logprob.cpu()
    live = want != 0
    _close(got[live], want[live], precision)
    # greedy samples and n-best lists: identical, except where the model's own top candidates are within 1e-5 (bf16:
    # within the run-to-run bound)
    tie = 1e-5 if precision == "fp32" else BF16_MAX
    a, e = _sample(m, b, num_samples=1, top_k=1, seed=3), _sample(ens, b, num_samples=1, top_k=1, seed=3)
    ties = 0
    for r in range(8):
        if torch.equal(a.raw[r], e.raw[r]):
            continue
        t = int((a.raw[r, 0] != e.raw[r, 0]).nonzero()[0])            # first differing column
        if t == 29:                                                    # no column left for the <eos> score needs
            continue
        lab = torch.zeros((2, 30), dtype=torch.int64)
        for i, src in enumerate((a, e)):                               # score both continuations with the model
            lab[i, :t + 1] = src.raw[r, 0, :t + 1].cpu()
            lab[i, t + 1] = v["<eos>"]
        bb = [x[r:r + 1].repeat_interleave(2, 0) if torch.is_tensor(x) else x for x in b]
        bb[6] = lab
        lp = _score(m, bb).token_logprob[:, t].cpu()
        assert abs(float(lp[0] - lp[1])) <= tie, (r, t, lp)
        ties += 1
    assert precision == "bf16" or ties <= 2          # bf16: the run-to-run spread widens what counts as a near-tie
    a, e = _nbest(m, b, beam_size=4), _nbest(ens, b, beam_size=4)
    _check(e, v)
    ties = 0
    for c in range(8):
        if not torch.equal(a.raw[c], e.raw[c]):
            torch.testing.assert_close(e.score[c], a.score[c], rtol=0, atol=tie * 30)   # a near-tie swapped two slots
            ties += 1
    assert precision == "bf16" or ties <= 2
    if precision == "fp32":
        torch.testing.assert_close(e.score, a.score, rtol=0, atol=tie * 30)


def _two_members():
    m1 = _model("fp32")
    m2 = copy.deepcopy(m1)
    g = torch.Generator(device=DEV).manual_seed(1)
    with torch.no_grad():
        for p in (m2.out_fc.weight, m2.copy_net.LinearRes.weight, m2.copy_net.LinearProb.weight):
            p.add_(torch.randn(p.shape, generator=g, device=DEV) * p.std() * 0.5)
    return m1, m2


def _mix(scores, w):
    """log sum_m w_m exp(score_m) per token"""
    s = torch.stack(scores).double()
    return torch.logsumexp(s + torch.tensor(np.log(w), dtype=torch.float64).view(-1, 1, 1), 0)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_two_members_score_is_the_average_of_their_probabilities(precision):
    m1, m2 = (m.set_precision(precision) for m in _two_members())
    b = golden_batch(0, 16)
    rep = [x.to(DEV) if torch.is_tensor(x) else x for x in b]
    with torch.no_grad():                                              # the members really disagree
        assert not torch.equal(m1(*rep, "dev"), m2(*rep, "dev"))
    w = [0.3, 0.7]
    got = _score(_ens([m1, m2], w), b).token_logprob.cpu()
    members = [_score(m, b).token_logprob.cpu() for m in (m1, m2)]
    live = (b[6][:, 1:30] != 0).cpu()
    live = torch.cat((torch.zeros((16, 1), dtype=torch.bool), live), 1)
    live &= (members[0] > -23.0) & (members[1] > -23.0)               # no member clamped at 1e-10
    want = _mix(members, w).float()
    # bf16: the members' scores come from other runs of the bf16 decoder than the ensemble's (BF16_MEDIAN); log sum w
    # exp is 1-Lipschitz in the members' log-probabilities, so the run-to-run bound carries over
    assert live.sum() > 20
    _close(got[live], want[live], precision)


def test_two_members_decoders():
    m1, m2 = _two_members()
    ens = _ens([m1, m2], [0.6, 0.4])
    b = golden_batch(0, 16)
    v = _vocab()
    eos = v["<eos>"]
    s = _sample(ens, b, num_samples=3, seed=9, temperature=0.8)
    _check_bookkeeping(s, v)
    _self_score(ens, b, s, "fp32", eos)                            # token_logprob = the ensemble's rescoring
    n = _nbest(ens, b, beam_size=3, length_penalty=0.6)
    _check(n, v)
    _self_score(ens, b, n, "fp32", eos)
    pre = _eos_prefix(b[6], 2, eos)
    r = _nbest(ens, b, beam_size=3, prefix=pre, no_repeat_ngram=2, min_length=3)
    _check(r, v)
    k = (pre != 0).sum(1)
    for c in range(16):
        assert torch.equal(r.raw[c, :, 1:1 + int(k[c])].cpu(), pre[c, :int(k[c])].unsqueeze(0).expand(3, -1))
    _check_rules(r, 2, 3, eos, start=int(k.max()))
    _self_score(ens, b, r, "fp32", eos)
    dv = _nbest(ens, b, beam_size=4, groups=2, diversity=0.5)
    _check(dv, v)
    from fira_icse_b200.mbr import mbr
    out = mbr(ens, b[0], b[3], b[4], b[5].to(DEV), b[7], num_samples=4, seed=5, start_id=v["<start>"], eos_id=eos,
              pad_id=v["<pad>"])
    assert torch.equal(out.index.cpu(), torch.argmax(out.utility, 1).cpu())
    _self_score(ens, b, out.samples, "fp32", eos)


def test_graphs_are_reused_across_batches_ensembles_and_weights():
    from fira_icse_b200.decode_loop import loop_for
    from fira_icse_b200.sample import _Sampler, sample
    m1, m2 = _two_members()
    v = _vocab()
    T = 8                                      # every batch runs all T - 1 positions (the first poll is at 8)

    def run(ens, lo):
        b = golden_batch(lo, lo + 8)
        return sample(ens, b[0], b[3], b[4], b[5].to(DEV), b[7], num_samples=2, seed=1, tar_len=T,
                      start_id=v["<start>"], eos_id=v["<eos>"], pad_id=v["<pad>"])

    ens = _ens([m1, m2])
    run(ens, 0)
    S = golden_batch(0, 8)[0].shape[1] + golden_batch(0, 8)[7].shape[1]
    loop = loop_for(_Sampler, ens, 8, 2, T, S)
    keys = set(loop.graphs)
    assert len(keys) == T - 1
    run(ens, 8)                                                        # a second batch of the same shape
    again = _ens([m1, m2])                                             # a new Ensemble of the same models
    run(again, 8)
    assert loop_for(_Sampler, again, 8, 2, T, S) is loop and set(loop.graphs) == keys
    # new weights replay the same graphs, and the scores follow the formula
    b = golden_batch(0, 8)
    w = [0.9, 0.1]
    got = _score(_ens([m1, m2], w), b).token_logprob.cpu()
    assert loop_for(_Sampler, again, 8, 1, 30, S).graphs                # score's own loop (N = 1) was captured
    n_score = len(loop_for(_Sampler, again, 8, 1, 30, S).graphs)
    uniform = _score(_ens([m1, m2]), b).token_logprob.cpu()
    assert len(loop_for(_Sampler, again, 8, 1, 30, S).graphs) == n_score
    members = [_score(m, b).token_logprob.cpu() for m in (m1, m2)]
    live = torch.cat((torch.zeros((8, 1), dtype=torch.bool), (b[6][:, 1:30] != 0)), 1)
    live &= (members[0] > -23.0) & (members[1] > -23.0)
    for w_, s_ in ((w, got), ([0.5, 0.5], uniform)):
        want = _mix(members, w_).float()
        assert ((s_ - want).abs()[live] <= 1e-5 * want.abs()[live].clamp(min=1.0)).all()
    assert not torch.equal(got[live], uniform[live])


def test_run_model_ensemble(trained):  # noqa: F811
    d, base, _ = trained
    n_test, lines = _test_lines(trained, "output_fira_nbest_ens2", FIRA_DECODE="nbest", FIRA_BEAM="3",
                                FIRA_ENSEMBLE="best_model.pt,best_model.pt")
    assert len(lines) == 3 * n_test + 1 and lines[-1] == ""
    for c in range(n_test):
        fields = [ln.split("\t", 2) for ln in lines[3 * c:3 * c + 3]]
        assert all(len(f) == 3 and float(f[1]) <= 0.0 for f in fields)
        scores = [float(f[0]) for f in fields]
        assert all(x >= y for x, y in zip(scores, scores[1:])), scores
    env = dict(base, FIRA_DECODE="beam", FIRA_ENSEMBLE="best_model.pt,best_model.pt")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "run_model.py"), "test"], cwd=d, env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "FIRA_ENSEMBLE applies to FIRA_DECODE=sample, nbest and mbr" in r.stderr
