"""Lexically constrained n-best without a device: the restated rule (tests/lexical_rule.py) on hand-worked cases, Tc = 0
against beam_rule.step, every decode_loop.check_constraints error (raised before any device work),
data.constraint_words, and run_model.py's FIRA_CONSTRAINT_WORDS refusals."""
import numpy as np
import pytest
import torch

import beam_rule
from lexical_rule import candidates, meets, phrases_of, progress, row_progress, select

EOS = 2
V, S = 12, 4
C = V + S


def _probs(rows):
    """[K, C] mixtures from {j: p} per slot, the rest spread evenly and tiny"""
    P = np.full((len(rows), C), 1e-6)
    for i, r in enumerate(rows):
        for j, p in r.items():
            P[i, j] = p
    return P


@pytest.mark.parametrize("words,c,want", [
    ([5, 6, 7], [6, 7], 2),                  # occurs at the end
    ([6, 7, 5], [6, 7], 2),                  # occurred earlier: stays met
    ([5, 6], [6, 7, 8], 1),                  # partial
    ([5, 6, 7], [6, 7, 8], 2),
    ([6, 7, 5], [6, 7, 8], 0),               # the partial match fell back
    ([6, 6], [6, 6, 7], 2),                  # the longest start the words end with
    ([6], [6, 6, 7], 1),
    ([], [6], 0),
])
def test_progress(words, c, want):
    assert progress(words, c) == want


def test_overlapping_phrases_both_count():
    ph = [[5, 6], [6, 7]]
    assert row_progress([5, 6, 7], ph) == 4 and meets([5, 6, 7], ph)
    assert row_progress([5, 6], ph) == 3 and not meets([5, 6], ph)
    assert phrases_of(np.array([[5, 6, 0, 0], [0, 0, 0, 0], [7, 0, 0, 0]])) == [[5, 6], [7]]


def _cands(words, phrases, P, K=2, status=(0,), L=(0.0,), n=(2,), copy_src=(3, 9, 9, 4), copy_ok=(1, 1, 0, 1),
           bans=None, forced=None):
    k = len(status)
    return candidates(np.array(L, float), np.array(n, float), np.array(status), P, np.array(copy_ok, bool),
                      np.array(copy_src), words, bans or [set()] * k, phrases, V, K, 0.0, EOS, forced)


def test_phrase_proposals_and_banks():
    # slot 0 has written 5; phrase [5, 6] wants 6 next, phrase [8] wants 8: neither is in the row's top 2 (3, 4)
    P = _probs([{3: 0.5, 4: 0.3, 6: 0.01, 8: 0.02, EOS: 0.1}])
    got = {c[3]: c[6] for c in _cands([[5]], [[5, 6], [8]], P)}
    assert got == {3: 0, 4: 0, 6: 2, 8: 1}             # banks: progress with the word appended (3, 4 leave [5, 6])
    assert EOS not in got                                # <eos> banned below Tc


def test_a_partial_match_falls_back():
    # slot 0 wrote 5 6 of phrase [5, 6, 7]: 7 keeps its progress (bank 3), anything else drops it to 0 (or 1 for 5)
    P = _probs([{3: 0.5, 5: 0.3, 7: 0.01}])
    got = {c[3]: c[6] for c in _cands([[5, 6]], [[5, 6, 7]], P)}
    assert got == {3: 0, 5: 1, 7: 3}


def test_a_copy_spells_the_next_word():
    # copy position 1 spells 9 with more probability than the vocabulary entry 9; copy position 2 (masked) more still
    P = _probs([{3: 0.5, 4: 0.3, 9: 0.001, V + 1: 0.01, V + 2: 0.1}])
    got = {c[3]: c[6] for c in _cands([[5]], [[9]], P)}
    assert got == {3: 0, 4: 0, V + 1: 1}


def test_a_proposal_already_in_the_top_k_is_not_repeated():
    P = _probs([{3: 0.5, 9: 0.3}])
    got = [c[3] for c in _cands([[5]], [[9], [9, 4]], P)]
    assert sorted(got) == [3, 9]


def test_a_banned_next_word_is_not_proposed():
    P = _probs([{3: 0.5, 4: 0.3, 8: 0.01}])
    got = [c[3] for c in _cands([[8, 5]], [[5, 8]], P, bans=[{8}])]    # 8 banned by the rules (e.g. n = 1)
    assert sorted(got) == [3, 4]


def test_a_forced_row_proposes_its_label_with_its_bank():
    P = _probs([{3: 0.5}])
    got = _cands([[5]], [[5, 6]], P, forced=6)
    assert [(c[3], c[6]) for c in got] == [(6, 2)]


def test_finished_slots_are_pinned_then_the_banks_are_striped():
    # slot 0 finished with a poor score; slots 1 and 2 live.  Tc = 2 (phrases [7] and [8])
    P = _probs([{}, {3: 0.6, 4: 0.2, 7: 0.01, 8: 0.005}, {3: 0.5, 7: 0.3, 8: 0.01}])
    cand = _cands([[7], [5], [7]], [[7], [8]], P, K=2, status=(1, 0, 0), L=(-30.0, -1.0, -1.5), n=(3, 3, 3))
    sel = select(cand, 3, 2)
    assert sel[0][:2] == (0, C)                          # the finished slot first, whatever its score
    # bank 2: (2, 8); bank 1: (2, 3), (2, 7), (1, 7), (1, 8); bank 0: (1, 3), (1, 4): the best of each bank, higher
    # banks first, ahead of (1, 3), the best score of all
    assert [s[:2] for s in sel[1:]] == [(2, 8), (2, 3)]
    assert [s[5] for s in sel[1:]] == [2, 1]
    # with Tc = 0 the plain order: best scores first, the finished slot last
    plain = select(_cands([[7], [5], [7]], [], P, K=2, status=(1, 0, 0), L=(-30.0, -1.0, -1.5), n=(3, 3, 3)), 3, 0)
    assert [s[:2] for s in plain] == [(1, 3), (2, 3), (1, 4)]


@pytest.mark.parametrize("seed", range(4))
def test_no_constraints_is_the_n_best_rule(seed):
    rng = np.random.default_rng(seed)
    K = 3
    P = rng.dirichlet(np.ones(C), size=K)
    status = np.array([0, 1, 0])
    L, n = -rng.random(K) * 4, np.array([2.0, 3.0, 2.0])
    copy_ok = np.array([1, 0, 1, 1], bool)
    for alpha in (0.0, 0.6):
        got = select(candidates(L, n, status, P, copy_ok, np.array([3, 4, 5, 6]), [[5, 6]] * K, [set()] * K, [], V, K,
                                alpha, EOS), K, 0)
        want, _ = beam_rule.step(L, n, status, P, copy_ok, V, K, alpha)
        assert [g[:5] for g in got] == [w[:5] for w in want]


# ------------------------------------------------------------------ check_constraints
def _check(con, B=2, tar_len=30, groups=1, pad_id=0):
    from fira_icse_b200.decode_loop import check_constraints
    return check_constraints(con, B, V=V, tar_len=tar_len, start_id=1, eos_id=EOS, pad_id=pad_id, groups=groups)


def test_valid_constraints_are_padded_to_four_by_four():
    out = _check(torch.tensor([[[5, 6], [7, 0]], [[0, 0], [0, 0]]]))
    assert out.dtype == torch.int32 and out.shape == (2, 4, 4)
    assert out[0, 0, :2].tolist() == [5, 6] and out[0, 1, 0] == 7 and int((out != 0).sum()) == 3
    assert _check(None) is None


@pytest.mark.parametrize("con,kw,match", [
    (torch.tensor([[[5.0]], [[6.0]]]), {}, "integer tensor"),
    (torch.tensor([[[True]], [[False]]]), {}, "integer tensor"),
    ([[[5]], [[6]]], {}, "integer tensor"),
    (torch.tensor([[5, 6], [7, 8]]), {}, "shape"),
    (torch.ones((3, 1, 1), dtype=torch.long) * 5, {}, "shape"),
    (torch.ones((2, 5, 1), dtype=torch.long) * 5, {}, "shape"),
    (torch.ones((2, 1, 5), dtype=torch.long) * 5, {}, "shape"),
    (torch.tensor([[[5, 0, 6]], [[5, 0, 0]]]), {}, "follows a 0"),
    (torch.tensor([[[V]], [[5]]]), {}, r"\[0, V"),
    (torch.tensor([[[-1]], [[5]]]), {}, r"\[0, V"),
    (torch.tensor([[[1]], [[5]]]), {}, "<start>"),
    (torch.tensor([[[EOS]], [[5]]]), {}, "<eos>"),
    (torch.tensor([[[9]], [[5]]]), dict(pad_id=9), "pad_id"),
    (torch.tensor([[[5, 6, 7]], [[5, 0, 0]]]), dict(tar_len=4), "at most tar_len - 2 = 2 words"),
    (torch.tensor([[[5]], [[6]]]), dict(tar_len=33), "tar_len <= 32"),
    (torch.tensor([[[5]], [[6]]]), dict(groups=2), "groups"),
])
def test_constraint_errors(con, kw, match):
    with pytest.raises(ValueError, match=match):
        _check(con, **kw)


# ------------------------------------------------------------------ data.constraint_words
def test_constraint_words_normalise_like_build_commit():
    from fira_icse_b200.data import constraint_words
    raw = {"variable": [{"myVar": "VAR1"}]}
    vocab = {"<unkm>": 3, "fix": 5, "VAR1": 6, "null": 7, "check": 8, "add": 9}
    upper = {"VAR1"}
    assert constraint_words(raw, 0, ["Fix", "null check", ["myVar"]], vocab, upper) == [[5], [7, 8], [6]]
    with pytest.raises(ValueError, match="'frobnicate' of commit 0 is not in the vocabulary"):
        constraint_words(raw, 0, ["fix frobnicate"], vocab, upper)


# ------------------------------------------------------------------ run_model.py
VOCAB = {"<start>": 1, "<eos>": 2, "<pad>": 0, "<unkm>": 3}


@pytest.mark.parametrize("mode,env", [("beam", {}), ("sample", {}), ("mbr", {}), ("nbest", {"FIRA_BEAM_GROUPS": "3"})])
def test_run_model_refuses_constraints_outside_plain_nbest(monkeypatch, mode, env):
    import run_model
    monkeypatch.setenv("FIRA_CONSTRAINT_WORDS", "1")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    with pytest.raises(SystemExit, match="FIRA_CONSTRAINT_WORDS applies to FIRA_DECODE=nbest"):
        run_model.decoder(mode, VOCAB)


def test_run_model_tags_the_constrained_output(monkeypatch):
    import run_model
    monkeypatch.setenv("FIRA_CONSTRAINT_WORDS", "2")
    monkeypatch.setenv("FIRA_NO_REPEAT_NGRAM", "2")
    assert run_model.decoder("nbest", VOCAB)[0] == "output_fira_nbest_norepeat2_lex2"
    monkeypatch.setenv("FIRA_CONSTRAINT_WORDS", "5")
    with pytest.raises(SystemExit, match=r"FIRA_CONSTRAINT_WORDS must be in \[0, 4\]"):
        run_model.decoder("nbest", VOCAB)


def test_run_model_oracle_constraints():
    import run_model
    tar = torch.tensor([[1, 7, 5, 7, 3, 8, 9, 2, 0], [1, 2, 0, 0, 0, 0, 0, 0, 0]])
    sou = torch.tensor([[1, 5, 7, 3, 9, 2], [1, 5, 2, 0, 0, 0]])
    sub = torch.tensor([[8, 0], [0, 0]])
    b = [sou, tar, None, None, None, None, None, sub]
    got = run_model.oracle_constraints(b, 3, VOCAB)
    assert got.shape == (2, 3, 1)
    assert got[0, :, 0].tolist() == [7, 5, 8] and got[1].abs().sum() == 0     # <unkm> (3) is never required
