"""Lexically constrained n-best on the GPU: fira_pointer_mix_beam_step_lexical against its `_rules` twin (no
constraints) and against the float64 rule (tests/lexical_rule.py), `nbest(constraints=)` end to end on the sharpened
golden model (alone, with a prefix and the rules, with a two-member ensemble), and `run_model.py test` with
FIRA_CONSTRAINT_WORDS."""
import gc
import json

import numpy as np
import pytest
import torch

from constraint_rule import banned
from fira_testlib import golden_batch
from lexical_rule import candidates, meets, phrases_of, select
from sample_rule import mixture
from test_gpu_cli import _run_model, trained  # noqa: F401  (the trained-model fixture)
from test_gpu_constraints import _beam_call, _beam_state, _check_rules, _plant_copies, _self_score
from test_gpu_ensemble import _ens, _two_members
from test_gpu_nbest import _nbest
from test_gpu_prefix import _code, _eos_prefix, _prefix, _rows_equal
from test_gpu_sample import _check_bookkeeping, _head_nll, _inputs, _model, _vocab

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [torch.float32, torch.bfloat16]
KS = [1, 3, 5, 16]


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


@pytest.fixture(autouse=True)
def _release_decoding_loops():
    """decode_loop keeps every model's decoding loops, with their captured position graphs, for the whole process (a
    loop holds its model, so the weak-keyed cache never drops one).  The GPU modules share one process, so the loops of
    the models each test here creates are dropped when it ends: the modules after this one find the device memory they
    would find without it."""
    from fira_icse_b200 import decode_loop
    before = {id(m) for m in decode_loop._LOOPS.keys()}
    yield
    for m in [m for m in decode_loop._LOOPS.keys() if id(m) not in before]:
        del decode_loop._LOOPS[m]
    gc.collect()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------ one step of the kernel
def _lex_call(inputs, K, V, state, pos, T, con, extra=(0, 0), prefix=None, alpha=0.6, eos=3):
    """one fira_pointer_mix_beam_step_lexical from `state` (test_gpu_constraints._beam_call's layout) -> the written half
    and the outputs"""
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
    work = torch.zeros(R * (K + 4), dtype=torch.int64, device=DEV)
    c = torch.zeros((R // K, 4, 4), **i32)
    c[:, :con.shape[1], :con.shape[2]] = con.to(DEV, torch.int32)
    P = ops._ptr
    pre = [P(prefix[0]), T, P(prefix[1])] if prefix is not None else [None, 0, None]
    call("fira_pointer_mix_beam_step_lexical", P(logits), logits.stride(0), P(sc), P(gl), P(mem_mask), P(copy_src),
         float(alpha), eos, 0, P(work), P(bufs["seq"]), P(bufs["raw"]), P(bufs["tlp"]), P(bufs["length"]),
         P(bufs["lp"]), P(bufs["score"]), P(bufs["status"]), P(parent), P(nxt), T, pos, R // K, K, V, S, _code(logits),
         ops._stream(), *pre, *extra, P(c))
    torch.cuda.synchronize()
    out = {k: v[1 - h].cpu() for k, v in bufs.items()}
    out.update(parent=parent.cpu(), nxt=nxt.cpu())
    return out


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("K", KS)
def test_no_constraints_is_the_rules_twin(dtype, K):
    gen = torch.Generator().manual_seed(K * 71 + (dtype == torch.bfloat16))
    B, V, S, T, pos = 3, 24650, 370, 12, 5
    inputs = _inputs(gen, B, K, V, S, dtype)
    state = _beam_state(gen, B, K, T, pos, V, 2, K)
    zero = torch.zeros((B, 4, 4), dtype=torch.int32)
    for pre in (None, _prefix(B, T, [9, None, None], pos)):
        for rules in ((0, 0), (2, pos + 1)):
            twin = _beam_call(inputs, K, V, state, pos, T, None, "fira_pointer_mix_beam_step_rules", rules, prefix=pre)
            got = _lex_call(inputs, K, V, state, pos, T, zero, rules, prefix=pre)
            _rows_equal(got, twin, slice(None))


def _constraints(seq, K, V, pos):
    """per commit: a planted top word and a plain word; a phrase the history has started (its last word) and a banned
    word (V - 1, repeated by the planted histories); the planted copy word V // 2 and a three-word phrase"""
    last = [int(seq[b * K, pos]) for b in range(3)]
    return torch.tensor([[[V // 2, 40, 0], [5, 0, 0]],
                         [[last[1], 9, 0], [V - 1, 0, 0]],
                         [[V // 2, 0, 0], [last[2], 11, 12]]], dtype=torch.int32)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("K", KS)
def test_step_matches_the_float64_rule(dtype, K):
    gen = torch.Generator().manual_seed(K * 73 + 5 * (dtype == torch.bfloat16))
    B, V, S, T, eos, alpha = 3, 24650, 370, 12, 3, 0.6
    R, C = B * K, V + S
    near = compared = 0
    for n_gram in (0, 1, 2):
        pos = 3 * max(n_gram - 1, 0) + 2
        inputs = _plant_copies(_inputs(gen, B, K, V, S, dtype), V, eos)
        logits, sc, gl, mem_mask, copy_src = inputs
        x = logits.float().cpu().numpy()[:, :V].astype(np.float64)
        scn, gln, mk = sc.cpu().numpy().reshape(R, S), gl.cpu().numpy(), mem_mask.cpu().numpy()
        src = copy_src.cpu().numpy()
        Pm = np.stack([mixture(x[r], scn[r], gln[r], mk[r // K]) for r in range(R)])
        state = _beam_state(gen, B, K, T, pos, V, max(n_gram, 1), K)
        L, n, status, seq, raw, tlp = state
        con = _constraints(seq, K, V, pos)
        for m in (0, pos + 1):
            out = _lex_call(inputs, K, V, state, pos, T, con, (n_gram, m), alpha=alpha, eos=eos)
            Ld, nd = L.double().numpy(), (n - 1).double().numpy()
            for b in range(B):
                rows = range(b * K, (b + 1) * K)
                st = status[b * K:(b + 1) * K].numpy()
                words = [seq[r, 1:pos + 1].tolist() for r in rows]
                bans = [banned(w, n_gram, m, eos, pos + 1) for w in words]
                ph = phrases_of(con[b].numpy())
                tc = sum(len(c) for c in ph)
                cand = candidates(Ld[b * K:(b + 1) * K], nd[b * K:(b + 1) * K], st, Pm[b * K:(b + 1) * K], mk[b],
                                  src[b], words, bans, ph, V, K, alpha, eos)
                ref = select(cand, K, tc)
                table = {(c[2], c[3]): c[0] for c in cand}
                for k in range(min(K, len(ref))):
                    r = b * K + k
                    i = int(out["parent"][r]) - b * K
                    carried = st[i] == 1
                    j = C if carried else int(out["raw"][r, pos + 1])
                    assert (i, j) in table, (n_gram, m, b, k, i, j)
                    if not carried:
                        tok = j if j < V else int(src[b, j - V])
                        assert out["seq"][r, pos + 1] == tok and out["nxt"][r] == tok
                        assert tok not in bans[i] and (j < V or mk[b, j - V])
                        if tok == eos:
                            assert meets(words[i], ph), (b, k, i)
                    if (i, j) != ref[k][:2]:                          # only across a float64 near-tie
                        near += 1
                        d = abs(table[(i, j)] - ref[k][4]) / max(1e-30, abs(ref[k][4]))
                        assert d <= 1e-6, (dtype, K, n_gram, m, b, k, (i, j), ref[k][:2], d)
                    compared += 1
            grown = out["seq"][:, pos + 1] != 0
            par = out["parent"].to(DEV)
            lab = torch.where(grown, out["raw"][:, pos + 1], torch.zeros_like(out["raw"][:, pos + 1]))
            nll = _head_nll(logits[par].contiguous(), sc.view(R, S)[par].view(B, K, S).contiguous(), gl[par].contiguous(),
                            mem_mask, lab.numpy(), K, V)
            live = lab.numpy() != 0
            np.testing.assert_allclose(out["tlp"][:, pos + 1].numpy()[live], -nll[live], rtol=1e-6, atol=0)
    assert near <= 0.02 * compared, (near, compared)


# ------------------------------------------------------------------ end to end
def _oracle(b, k):
    import run_model
    return run_model.oracle_constraints(b, k, _vocab())


def _phrase_constraints(b):
    """per commit: its first two reference words as one phrase, and one more diff word that the reference holds"""
    one = _oracle(b, 3)
    tar = b[1]
    con = torch.zeros((tar.shape[0], 2, 2), dtype=torch.long)
    con[:, 0] = tar[:, 1:3]
    con[:, 1, 0] = one[:, 2, 0]
    eos = _vocab()["<eos>"]
    con[(con == eos).any(-1).any(-1)] = 0                             # a message shorter than two words: none
    return con


def _host_met(out, con):
    B, K = out.seq.shape[:2]
    met = torch.zeros((B, K), dtype=torch.bool)
    for c in range(B):
        ph = phrases_of(con[c].numpy())
        for k in range(K):
            met[c, k] = meets(out.seq[c, k, 1:int(out.length[c, k])].tolist(), ph)
    return met


def _check_lexical(out, con, v):
    from fira_icse_b200.beam import constraints_met
    _check_bookkeeping(out, v)
    last = out.seq.gather(2, (out.length - 1).unsqueeze(-1)).squeeze(-1)
    assert torch.equal(out.finished, last == v["<eos>"])
    met = constraints_met(out.seq, out.length, con)
    assert met.device == out.seq.device
    host = _host_met(out, con)
    assert torch.equal(met.cpu(), host)
    assert host[out.finished.cpu()].all()                             # every finished hypothesis meets them
    key = host.float() * 1e6 + out.score.cpu().double()               # sorted by (met, score)
    assert (key[:, 1:] <= key[:, :-1]).all()
    return host


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("K", [3, 5])
def test_nbest_with_constraints(precision, K):
    m = _model(precision)
    b = golden_batch(0, 16)
    v = _vocab()
    for con in (_oracle(b, 2), _phrase_constraints(b)):
        out = _nbest(m, b, beam_size=K, length_penalty=0.6, constraints=con)
        met = _check_lexical(out, con, v)
        assert met[:, 0].float().mean() >= 0.75
        _self_score(m, b, out, precision, v["<eos>"])


def test_zero_constraints_is_nbest():
    # two loops, two decoder runs: the split-K fp32 atomics leave the log-probabilities up to a few 1e-5 apart, so the
    # ids and flags are compared exactly and the log-probabilities within 1e-4, the bound of test_gpu_nbest's
    # static-buffer test; the step itself is the _rules step bit for bit (above)
    m = _model("fp32")
    b = golden_batch(0, 16)
    for kw in (dict(beam_size=3), dict(beam_size=5, length_penalty=0.6, no_repeat_ngram=2, min_length=3)):
        a = _nbest(m, b, **kw)
        z = _nbest(m, b, constraints=torch.zeros((16, 4, 4), dtype=torch.long), **kw)
        for f in ("seq", "raw", "length", "finished"):
            assert torch.equal(getattr(a, f), getattr(z, f)), f
        for f in ("logprob", "score", "token_logprob"):
            torch.testing.assert_close(getattr(z, f), getattr(a, f), rtol=0, atol=1e-4)


def test_constraints_with_a_prefix_and_the_rules():
    m = _model("fp32")
    b = golden_batch(0, 16)
    v = _vocab()
    eos = v["<eos>"]
    pre = _eos_prefix(b[6], 1, eos)
    con = _oracle(b, 2)
    out = _nbest(m, b, beam_size=4, prefix=pre, no_repeat_ngram=2, min_length=3, constraints=con)
    _check_lexical(out, con, v)
    k = (pre != 0).sum(1)
    for c in range(16):
        assert torch.equal(out.raw[c, :, 1:1 + int(k[c])].cpu(), pre[c, :int(k[c])].unsqueeze(0).expand(4, -1))
    _check_rules(out, 2, 3, eos, start=int(k.max()))


def test_constraints_with_an_ensemble():
    m1, m2 = _two_members()
    ens = _ens([m1, m2], [0.6, 0.4])
    b = golden_batch(0, 16)
    v = _vocab()
    con = _oracle(b, 2)
    out = _nbest(ens, b, beam_size=3, constraints=con)
    _check_lexical(out, con, v)
    _self_score(ens, b, out, "fp32", v["<eos>"])


def test_a_constraint_changes_the_top_hypothesis():
    m = _model("fp32")
    b = golden_batch(0, 16)
    v = _vocab()
    free = _nbest(m, b, beam_size=3)
    con = torch.zeros((16, 1, 1), dtype=torch.long)
    special = {v[w] for w in ("<start>", "<eos>", "<pad>", "<unkm>")}
    for c in range(16):                               # a diff word the free top hypothesis does not contain
        top = set(free.seq[c, 0, :int(free.length[c, 0])].tolist())
        cands = [w for w in b[0][c].tolist() if w not in special and w not in top]
        con[c, 0, 0] = cands[0]
    out = _nbest(m, b, beam_size=3, constraints=con)
    met = _check_lexical(out, con, v)
    # the sharpened model runs most messages to tar_len unfinished, so the top hypothesis is the best one that holds
    # the word, whenever one does (sorted by (met, score))
    changed = 0
    for c in range(16):
        if met[c, 0]:
            assert int(con[c, 0, 0]) in out.seq[c, 0].tolist()
            assert not torch.equal(out.seq[c, 0], free.seq[c, 0])
            changed += 1
    assert changed >= 12, changed


# ------------------------------------------------------------------ run_model.py test
def test_run_model_constraint_words(trained):  # noqa: F811
    import run_model
    from fira_icse_b200.data import build_commit
    from fira_testlib import load_raw_golden
    d, base, _ = trained
    env = dict(base, FIRA_DECODE="nbest", FIRA_BEAM="3", FIRA_CONSTRAINT_WORDS="1")
    r = _run_model("test", d, env)
    assert "mean sentence bleu" in r.stdout and "constraints met by the top hypothesis" in r.stdout
    lines = open(d / "OUTPUT" / "output_fira_nbest_lex1").read().split("\n")
    idx = json.load(open(d / "all_index"))["test"]
    assert len(lines) == 3 * len(idx) + 1 and lines[-1] == ""
    raw = load_raw_golden()
    vocab = raw["word_vocab"]
    r_vocab = {i: w for w, i in vocab.items()}
    upper = set(raw["VOCAB_UPPER_CASE"])
    checked = held = 0
    for c, i in enumerate(idx):
        cm = build_commit(raw["raw"], i, vocab, raw["ast_change_vocab"], upper)
        sou, tar, sub = (torch.tensor(cm[k]).unsqueeze(0) for k in ("sou", "tar", "sub_token"))
        con = run_model.oracle_constraints([sou, tar, None, None, None, None, None, sub], 1, vocab)
        if not con.any():
            continue
        word = run_model.deanonymise(run_model.ids_to_text([int(con[0, 0, 0])], r_vocab), raw["raw"]["variable"][i])
        score, lp, msg = lines[3 * c].split("\t", 2)
        if float(score) == 0.0:                       # an unfilled slot
            continue
        words = msg.split()
        if len(words) < 29:                           # finished (an unfinished top line may miss its word)
            assert word[0] in words, (c, word, msg)
        held += word[0] in words
        checked += 1
    assert checked > 0 and held >= 0.5 * checked, (held, checked)
