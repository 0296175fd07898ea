"""n-gram repeat blocking and minimum length on the GPU: the three `_rules` step entry points against their `_prefix`
twins (rules off) and against the float64 rules with the banned labels removed (tests/constraint_rule.py), forced rows,
and `no_repeat_ngram=` / `min_length=` end to end on the sharpened golden model, plus `run_model.py test` with
FIRA_NO_REPEAT_NGRAM / FIRA_MIN_LENGTH."""
import json

import numpy as np
import pytest
import torch

from constraint_rule import allowed, banned, candidates, repeats_ngram, sample_draw, select
from fira_testlib import golden_batch
from sample_rule import mixture
from test_gpu_cli import _run_model, trained  # noqa: F401  (the trained-model fixture)
from test_gpu_nbest import _check, _nbest, _state
from test_gpu_prefix import _code, _decode, _eos_prefix, _prefix, _rows_equal, _score
from test_gpu_sample import _check_bookkeeping, _head_nll, _inputs, _model, _teacher_forced, _vocab

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [torch.float32, torch.bfloat16]


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _histories(R, V, n, pos, salt=0):
    """seq columns 0..pos [R, pos + 1] whose last n - 1 words follow earlier occurrences of the planted top words
    V // 2 and V - 1 (even rows) or V - 1 and word 40 (odd rows), so those words are banned for n >= 1; 1 = <start>"""
    out = np.full((R, pos + 1), 1, np.int32)
    for r in range(R):
        a, b = (V // 2, V - 1) if r % 2 == 0 else (V - 1, 40)
        ctx = [10 + salt + k for k in range(n - 1)]
        words = ctx + [a] + ctx + [b] + ctx
        words = ([20 + salt + r % 3] * pos + words)[-pos:]             # filler before when pos is longer
        out[r, 1:] = words
    return out


def _plant_copies(inputs, V, eos):
    """per commit, two unmasked copy positions with high scores: one spelling the planted top word V // 2, one <eos>"""
    logits, sc, gl, mem_mask, copy_src = inputs
    for b in range(mem_mask.shape[0]):
        s = mem_mask[b].nonzero().view(-1)
        copy_src[b, s[0]], copy_src[b, s[1]] = V // 2, eos
        sc[b, :, s[0]], sc[b, :, s[1]] = 9.0, 8.5
    return inputs


# ------------------------------------------------------------------ sampler step
def _sample_call(inputs, N, V, pos, T, hist, name, extra=(), prefix=None, uniforms=None, seed=77, eos=-1, k=0, p=1.0):
    """one sampler step at `pos` with the rows' histories `hist` [R, pos + 1] -> every written buffer"""
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import call
    logits, sc, gl, mem_mask, copy_src = inputs
    R, S = logits.shape[0], sc.shape[-1]
    gen = torch.Generator().manual_seed(pos)
    i32 = dict(dtype=torch.int32, device=DEV)
    seq = torch.full((R, T), -7, dtype=torch.int32)
    seq[:, :pos + 1] = torch.from_numpy(hist)
    o = dict(nxt=torch.full((R,), -7, **i32), seq=seq.to(DEV), raw=torch.full((R, T), -7, **i32),
             tlp=torch.full((R, T), 9.0, device=DEV), msk=torch.full((R, T), 7, dtype=torch.uint8, device=DEV),
             fin=torch.zeros(R, dtype=torch.uint8, device=DEV), length=torch.full((R,), pos + 1, **i32),
             lp=(-torch.rand(R, generator=gen) * 5).to(DEV))
    o["fin"][1] = 1
    o["lp0"] = o["lp"].clone()
    seed_t = torch.tensor([seed], dtype=torch.int64, device=DEV)
    first_t = torch.tensor([3], **i32)
    P = ops._ptr
    pre = [P(prefix[0]), T, P(prefix[1])] if prefix is not None else [None, 0, None]
    call(name, P(logits), logits.stride(0), P(sc), P(gl), P(mem_mask), P(copy_src), P(seed_t), P(first_t),
         P(uniforms), 1.0, int(k), float(p), eos, 0, P(o["nxt"]), P(o["seq"]), P(o["raw"]), P(o["tlp"]), P(o["msk"]),
         T, pos, P(o["fin"]), P(o["length"]), P(o["lp"]), R // N, N, V, S, _code(logits), ops._stream(), *pre, *extra)
    torch.cuda.synchronize()
    return {key: v.cpu() for key, v in o.items()}


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("philox", [False, True])
def test_sample_rules_off_is_the_prefix_twin(dtype, philox):
    gen = torch.Generator().manual_seed(41 + philox)
    B, N, V, S, T, pos = 4, 4, 24650, 370, 12, 5
    inputs = _inputs(gen, B, N, V, S, dtype)
    hist = _histories(B * N, V, 2, pos)
    for k, p in ((0, 1.0), (5, 0.9), (50, 1.0), (0, 0.5)):
        u = None if philox else torch.rand(B * N, generator=gen).to(DEV)
        for pre in (None, _prefix(B, T, [5, None, V, None], pos)):
            kw = dict(prefix=pre, uniforms=u, k=k, p=p, eos=3)
            twin = _sample_call(inputs, N, V, pos, T, hist, "fira_pointer_mix_sample_prefix", **kw)
            got = _sample_call(inputs, N, V, pos, T, hist, "fira_pointer_mix_sample_rules", (0, 0), **kw)
            _rows_equal(got, twin, slice(None))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", [1, 2, 3])
def test_sample_draw_skips_banned_labels(dtype, n):
    gen = torch.Generator().manual_seed(53 + n + 7 * (dtype == torch.bfloat16))
    B, N, V, S, T, eos = 3, 4, 24650, 370, 12, 3                      # <eos>: a planted top word
    pos = 3 * (n - 1) + 2
    R = B * N
    inputs = _plant_copies(_inputs(gen, B, N, V, S, dtype), V, eos)
    logits, sc, gl, mem_mask, copy_src = inputs
    x = logits.float().cpu().numpy()[:, :V].astype(np.float64)
    scn, gln, mk, src = sc.cpu().numpy().reshape(R, S), gl.cpu().numpy(), mem_mask.cpu().numpy(), copy_src.cpu().numpy()
    rows = [mixture(x[r], scn[r], gln[r], mk[r // N]) for r in range(R)]
    hist = _histories(R, V, n, pos)
    checked = skipped = 0
    for m in (0, pos + 1):                                            # pos + 1: <eos> banned as well
        bans = [banned(hist[r, 1:], n, m, eos, pos + 1) for r in range(R)]
        assert all({V // 2, V - 1} & ban for ban in bans) and (m == 0 or all(eos in ban for ban in bans))
        for k, p in ((0, 1.0), (1, 1.0), (5, 1.0), (0, 0.9), (50, 0.3)):
            u = torch.rand(R, generator=gen)
            got = _sample_call(inputs, N, V, pos, T, hist, "fira_pointer_mix_sample_rules", (n, m), uniforms=u.to(DEV),
                               eos=eos, k=k, p=p)
            for r in range(R):
                if r == 1:                                            # finished row: padding
                    assert got["raw"][r, pos + 1] == 0
                    continue
                j = int(got["raw"][r, pos + 1])
                tok = j if j < V else int(src[r // N, j - V])
                assert tok not in bans[r], (n, m, k, p, r, j, tok)
                ref, near = sample_draw(rows[r], mk[r // N], src[r // N], bans[r], V, 1.0, k, p, float(u[r]))
                if near:
                    skipped += 1
                    continue
                checked += 1
                assert j == ref, (n, m, k, p, r, j, ref)
            raw = got["raw"][:, pos + 1].numpy().copy()
            nll = _head_nll(logits, sc, gl, mem_mask, raw, N, V)
            live = raw != 0
            assert (got["tlp"][:, pos + 1].numpy()[live] == -nll[live].astype(np.float32)).all()   # bit for bit
    # ~110 draws per case (test_gpu_sample.py's 5% bound is over ~430): one more near row must not fail the case
    assert skipped <= 0.1 * (checked + skipped), (checked, skipped)


@pytest.mark.parametrize("dtype", DTYPES)
def test_forced_sample_rows_take_banned_labels(dtype):
    gen = torch.Generator().manual_seed(61)
    B, N, V, S, T, pos, eos = 3, 4, 24650, 370, 12, 5, 3
    inputs = _inputs(gen, B, N, V, S, dtype)
    logits, sc, gl, mem_mask, copy_src = inputs
    hist = _histories(B * N, V, 2, pos)                               # V // 2 banned on even rows, V - 1 on every row
    labels = [V - 1, eos, None]                                       # banned by the n-gram rule, banned <eos>
    got = _sample_call(inputs, N, V, pos, T, hist, "fira_pointer_mix_sample_rules", (2, pos + 1),
                       prefix=_prefix(B, T, labels, pos), uniforms=torch.zeros(B * N, device=DEV), eos=eos)
    nll = _head_nll(logits, sc, gl, mem_mask, np.repeat(np.array([V - 1, eos, 0]), N), N, V)
    c = pos + 1
    for r in range(2 * N):
        if r == 1:
            continue
        j = labels[r // N]
        assert got["raw"][r, c] == j and got["seq"][r, c] == j and got["nxt"][r] == j
        assert got["tlp"][r, c].item() == np.float32(-nll[r])
        assert got["lp"][r] == got["lp0"][r] + got["tlp"][r, c]
        assert got["length"][r] == pos + 2 and got["fin"][r] == int(j == eos)
    for r in range(2 * N, 3 * N):                                     # the free commit obeys the rules
        assert int(got["seq"][r, c]) not in banned(hist[r, 1:], 2, pos + 1, eos, pos + 1)


# ------------------------------------------------------------------ n-best and diverse steps
def _beam_call(inputs, K, V, state, pos, T, G, name, extra=(), prefix=None, alpha=0.6, diversity=0.5, eos=3):
    """one (diverse, G given) beam step from `state` -> the written half and the outputs"""
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import call
    logits, sc, gl, mem_mask, copy_src = inputs
    R, S = logits.shape[0], sc.shape[-1]
    L, n, status, seq, raw, tlp = state
    h = pos & 1
    i32 = dict(dtype=torch.int32, device=DEV)
    bufs = dict(seq=torch.full((2, R, T), -7, **i32), raw=torch.full((2, R, T), -7, **i32),
                tlp=torch.full((2, R, T), 9.0, device=DEV), length=torch.full((2, R), -7, **i32),
                lp=torch.full((2, R), 9.0, device=DEV), score=torch.full((2, R), 9.0, device=DEV),
                status=torch.full((2, R), 7, dtype=torch.uint8, device=DEV))
    bufs["seq"][h], bufs["raw"][h], bufs["tlp"][h] = seq.to(DEV), raw.to(DEV), tlp.to(DEV)
    bufs["length"][h], bufs["lp"][h], bufs["status"][h] = n.to(DEV), L.to(DEV), status.to(DEV)
    bufs["score"][h] = (L / torch.pow((5.0 + (n - 1).float()) / 6.0, alpha)).to(DEV)
    parent = torch.full((R,), -1, dtype=torch.int64, device=DEV)
    nxt = torch.full((R,), -1, **i32)
    chosen = torch.full((R,), -7, **i32)
    work = torch.zeros(R * K, dtype=torch.int64, device=DEV)
    work_lp = torch.zeros(R * K, dtype=torch.float32, device=DEV)
    P = ops._ptr
    args = [P(logits), logits.stride(0), P(sc), P(gl), P(mem_mask), P(copy_src), float(alpha), eos, 0, P(work),
            P(bufs["seq"]), P(bufs["raw"]), P(bufs["tlp"]), P(bufs["length"]), P(bufs["lp"]), P(bufs["score"]),
            P(bufs["status"]), P(parent), P(nxt), T, pos, R // K, K, V, S]
    if G is not None:
        args += [G, float(diversity), P(chosen), P(work_lp)]
    pre = [P(prefix[0]), T, P(prefix[1])] if prefix is not None else [None, 0, None]
    call(name, *args, _code(logits), ops._stream(), *pre, *extra)
    torch.cuda.synchronize()
    out = {k: v[1 - h].cpu() for k, v in bufs.items()}
    out.update(parent=parent.cpu(), nxt=nxt.cpu())
    if G is not None:
        out["chosen"] = chosen.cpu()
    return out


def _names(G):
    base = "fira_pointer_mix_beam_step" if G is None else "fira_pointer_mix_diverse_beam_step"
    return base + "_prefix", base + "_rules"


def _beam_state(gen, B, K, T, pos, V, n_gram, Kg):
    """test_gpu_nbest's state (commit 0 at its first position with every group's first slot live, commit 1 with
    finished slots) with every slot `pos` words long and the histories of `_histories`"""
    state = _state(gen, B, K, T, pos, V, 0)
    L, n, status, seq, raw, tlp = state
    status[:K] = 2
    status[:K:Kg] = 0
    n[:] = pos + 1
    seq[:, :pos + 1] = torch.from_numpy(_histories(B * K, V, n_gram, pos, salt=7))
    return state


CONFIGS = [(1, None), (3, None), (5, None), (16, None), (4, 1), (4, 2), (4, 4), (6, 3), (16, 16)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("K,G", CONFIGS)
def test_beam_rules_off_is_the_prefix_twin(dtype, K, G):
    gen = torch.Generator().manual_seed(K * 43 + (G or 0) + (dtype == torch.bfloat16))
    B, V, S, T, pos = 3, 24650, 370, 12, 5
    inputs = _inputs(gen, B, K, V, S, dtype)
    state = _beam_state(gen, B, K, T, pos, V, 2, K // (G or 1))
    twin_name, name = _names(G)
    for pre in (None, _prefix(B, T, [9, None, None], pos)):
        twin = _beam_call(inputs, K, V, state, pos, T, G, twin_name, prefix=pre)
        _rows_equal(_beam_call(inputs, K, V, state, pos, T, G, name, (0, 0), prefix=pre), twin, slice(None))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("K,G", CONFIGS)
def test_beam_step_skips_banned_labels(dtype, K, G):
    gen = torch.Generator().manual_seed(K * 47 + (G or 0) + 3 * (dtype == torch.bfloat16))
    B, V, S, T, eos, alpha, diversity = 3, 24650, 370, 12, 3, 0.6, 0.5
    Gr = G or 1
    Kg, R, C = K // Gr, B * K, V + S
    near = compared = 0
    for n_gram in (1, 2, 3):
        pos = 3 * (n_gram - 1) + 2
        inputs = _plant_copies(_inputs(gen, B, K, V, S, dtype), V, eos)
        logits, sc, gl, mem_mask, copy_src = inputs
        x = logits.float().cpu().numpy()[:, :V].astype(np.float64)
        scn, gln, mk = sc.cpu().numpy().reshape(R, S), gl.cpu().numpy(), mem_mask.cpu().numpy()
        src = copy_src.cpu().numpy()
        Pm = np.stack([mixture(x[r], scn[r], gln[r], mk[r // K]) for r in range(R)])
        state = _beam_state(gen, B, K, T, pos, V, n_gram, Kg)
        L, n, status, seq, raw, tlp = state
        for m in (0, pos + 1):
            out = _beam_call(inputs, K, V, state, pos, T, G, _names(G)[1], (n_gram, m), alpha=alpha,
                             diversity=diversity if G else 0.0, eos=eos)
            Ld, nd = L.double().numpy(), (n - 1).double().numpy()
            bans = [banned(seq[r, 1:pos + 1].numpy(), n_gram, m, eos, pos + 1) for r in range(R)]
            for b in range(B):
                rows = slice(b * K, (b + 1) * K)
                st = status[rows].numpy()
                ok = np.stack([allowed(bans[r], V, src[b], mk[b]) for r in range(b * K, (b + 1) * K)])
                prev = []
                for g in range(Gr):
                    args = (Ld[rows], nd[rows], st, Pm[rows], ok, src[b], V, Gr, g, alpha, diversity if G else 0.0,
                            prev)
                    ref, _ = select(candidates(*args), Kg)
                    table = {(c[2], c[3]): c[0] for c in candidates(*args, keep=Kg + 8)}
                    for k in range(Kg):
                        r = b * K + g * Kg + k
                        i = int(out["parent"][r]) - b * K
                        assert g * Kg <= i < (g + 1) * Kg
                        carried = st[i] == 1
                        j = C if carried else int(out["raw"][r, pos + 1])
                        if k >= len(ref):                                 # no candidate filled the slot
                            continue
                        assert (i, j) in table, (n_gram, m, b, g, k, i, j)
                        if not carried:
                            tok = j if j < V else int(src[b, j - V])
                            assert tok not in bans[b * K + i] and (j < V or mk[b, j - V]), (n_gram, m, b, k, j)
                            assert out["seq"][r, pos + 1] == tok and out["nxt"][r] == tok
                        if (i, j) != ref[k][:2]:                          # only across a float64 near-tie
                            near += 1
                            d = abs(table[(i, j)] - ref[k][5]) / max(1e-30, abs(ref[k][5]))
                            assert d <= 1e-6, (dtype, K, G, n_gram, m, b, g, k, (i, j), ref[k][:2], d)
                        compared += 1
                    if G is not None:
                        prev += [int(out["chosen"][b * K + g * Kg + k]) for k in range(Kg)]
            grown = out["seq"][:, pos + 1] != 0
            par = out["parent"].to(DEV)
            lab = torch.where(grown, out["raw"][:, pos + 1], torch.zeros_like(out["raw"][:, pos + 1]))
            nll = _head_nll(logits[par].contiguous(), sc.view(R, S)[par].view(B, K, S).contiguous(), gl[par].contiguous(),
                            mem_mask, lab.numpy(), K, V)
            live = lab.numpy() != 0
            np.testing.assert_allclose(out["tlp"][:, pos + 1].numpy()[live], -nll[live], rtol=1e-6, atol=0)
    assert near <= 0.02 * compared, (near, compared)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("K,G", [(3, None), (4, 2), (4, 4)])
def test_forced_beam_rows_take_banned_labels(dtype, K, G):
    gen = torch.Generator().manual_seed(K * 59 + (G or 0))
    B, V, S, T, pos, eos = 3, 24650, 370, 12, 5, 3
    Kg = K // (G or 1)
    inputs = _inputs(gen, B, K, V, S, dtype)
    logits, sc, gl, mem_mask, copy_src = inputs
    state = _beam_state(gen, B, K, T, pos, V, 2, Kg)                 # V - 1 banned on every row
    L, n, status, seq, raw, tlp = state
    for j in (V - 1, eos):
        got = _beam_call(inputs, K, V, state, pos, T, G, _names(G)[1], (2, pos + 1),
                         prefix=_prefix(B, T, [j, None, None], pos), eos=eos)
        nll = _head_nll(logits, sc, gl, mem_mask, np.full(B * K, j), K, V)
        for k in range(0, K, Kg):                                     # commit 0: every group's live slot grows with j
            assert got["parent"][k] == k and got["raw"][k, pos + 1] == j and got["nxt"][k] == j
            assert got["tlp"][k, pos + 1].item() == np.float32(-nll[k])
            assert got["length"][k] == pos + 2 and got["status"][k] == int(j == eos)


# ------------------------------------------------------------------ end to end
END_TO_END = ["sample", "nbest3", "nbest5", "diverse", "mbr"]        # nbest3: alpha 0, nbest5: alpha 0.6
MIN_LENGTH = 3


def _hyps(name, out):
    return out.samples if name == "mbr" else out


def _check_rules(hyp, n, m, eos, start=0):
    """every finished hypothesis: no word at index >= start repeats an n-gram, <eos> after at least m words"""
    seq, length = hyp.seq.cpu(), hyp.length.cpu()
    checked = 0
    for r in range(seq.shape[0] * seq.shape[1]):
        s, ln = seq.view(-1, seq.shape[2])[r], int(length.view(-1)[r])
        words = s[1:ln].tolist()
        if ln <= 1:                                                    # an n-best slot never filled
            continue
        assert not repeats_ngram(words, n, start), (r, words)
        if words[-1] == eos:
            assert len(words) - 1 >= m, (r, words)
        checked += 1
    assert checked > 0


def _self_score(m, b, hyp, precision, eos):
    """sample.score of every hypothesis returns its own token_logprob.  score needs <eos> within tar_len, so an
    unfinished hypothesis is scored with <eos> at column min(length, T - 1) (after its last label, or in place of it)
    and only the columns before that one are compared (the decoder is causal: they do not depend on it)."""
    rep = _teacher_forced(m, b, hyp)
    lab = rep[6].clone()
    T = lab.shape[1]
    fin = (lab[:, 1:] == eos).any(1)
    end = torch.where(fin, T - 1, hyp.length.reshape(-1).clamp(max=T - 1))
    rows = (~fin).nonzero().view(-1)
    lab[rows, end[rows]] = eos
    rep[6] = lab
    sc = _score(m, rep)
    keep = (torch.arange(T, device=lab.device).unsqueeze(0) < end.unsqueeze(1)).cpu()
    got = sc.token_logprob.cpu()[keep]
    want = hyp.token_logprob.reshape(-1, T).cpu()[keep]
    if precision == "fp32":
        torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)
    else:                                                              # two bf16 incremental decoders of other shapes
        d = (got - want).abs()
        assert d.median().item() <= 5e-2 and d.max().item() <= 0.5


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", END_TO_END)
def test_decoders_obey_the_rules(precision, name):
    m = _model(precision)
    b = golden_batch(0, 16)
    v = _vocab()
    for n in (1, 2, 3):
        out = _decode(name, m, b, no_repeat_ngram=n, min_length=MIN_LENGTH)
        hyp = _hyps(name, out)
        if name in ("sample", "mbr"):
            _check_bookkeeping(hyp, v)
        else:
            _check(hyp, v)
        _check_rules(hyp, n, MIN_LENGTH, v["<eos>"])
        _self_score(m, b, hyp, precision, v["<eos>"])
        if name == "mbr":
            assert out.seq.shape[0] == 16 and not repeats_ngram(out.seq[0, 1:int(out.length[0])].tolist(), n)


@pytest.mark.parametrize("name", END_TO_END)
def test_rules_off_is_no_rules(name):
    m = _model("fp32")
    b = golden_batch(0, 8)
    none = _decode(name, m, b)
    off = _decode(name, m, b, no_repeat_ngram=0, min_length=0)
    assert torch.equal(none.seq, off.seq)
    if name != "mbr":
        assert torch.equal(none.raw, off.raw)


def test_the_rules_change_the_hypotheses_that_break_them():
    m = _model("fp32")
    b = golden_batch(0, 16)
    v = _vocab()
    free = _decode("nbest3", m, b)
    ruled = _decode("nbest3", m, b, no_repeat_ngram=1, min_length=MIN_LENGTH)
    _check_rules(ruled, 1, MIN_LENGTH, v["<eos>"])
    for c in range(16):
        broken = any(repeats_ngram(free.seq[c, k, 1:int(free.length[c, k])].tolist(), 1) or
                     (bool(free.finished[c, k]) and int(free.length[c, k]) - 2 < MIN_LENGTH) for k in range(3))
        if broken:
            assert not torch.equal(free.seq[c], ruled.seq[c]), c


@pytest.mark.parametrize("name", ["sample", "nbest3", "diverse", "mbr"])
def test_rules_apply_after_the_prefix(name):
    m = _model("fp32")
    b = golden_batch(0, 16)
    v = _vocab()
    first = _eos_prefix(b[6], 1, v["<eos>"])
    pre = torch.cat((first, first), 1)                                # the prefix repeats its word: exempt
    out = _decode(name, m, b, prefix=pre, no_repeat_ngram=1, min_length=MIN_LENGTH)
    hyp = _hyps(name, out)
    raw = hyp.raw[:, :, 1:3].cpu()
    assert (raw == pre.unsqueeze(1)).all()
    _check_rules(hyp, 1, MIN_LENGTH, v["<eos>"], start=2)


# ------------------------------------------------------------------ run_model.py test
@pytest.mark.parametrize("mode,name,per", [("nbest", "output_fira_nbest", 3), ("sample", "output_fira_samples", 2)])
def test_run_model_rules(trained, mode, name, per):  # noqa: F811
    d, base, _ = trained
    untagged = d / "OUTPUT" / name
    before = untagged.read_bytes() if untagged.exists() else None
    env = dict(base, FIRA_DECODE=mode, FIRA_BEAM="3", FIRA_SAMPLES="2", FIRA_NO_REPEAT_NGRAM="2", FIRA_MIN_LENGTH="3")
    r = _run_model("test", d, env)
    assert "mean sentence bleu" in r.stdout
    lines = open(d / "OUTPUT" / (name + "_norepeat2_minlen3")).read().split("\n")
    n_test = len(json.load(open(d / "all_index"))["test"])
    assert len(lines) == per * n_test + 1 and lines[-1] == ""
    assert (untagged.read_bytes() if untagged.exists() else None) == before
