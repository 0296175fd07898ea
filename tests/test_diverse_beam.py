"""The diverse n-best rule (float64 restatement, tests/diverse_rule.py) against the n-best rule and brute force, and the
argument checks of fira_icse_b200.beam.nbest(groups=, diversity=), on CPU.  The kernel is compared with the restatement
in tests/test_gpu_diverse_beam.py."""
import numpy as np
import pytest

import beam_rule
from diverse_rule import group_candidates, step
from sample_rule import mixture

V, S = 40, 7
C = V + S


def _rows(rng, K, ties=False):
    P = np.stack([mixture(rng.normal(0, 2, V), rng.normal(0, 2, S), rng.normal(0, 1, 2), np.ones(S, bool))
                  for _ in range(K)])
    if ties:                                          # exact ties inside a row and across rows
        P[:, [3, 9, 21]] = P[:, [3]].copy()
        P[1 % K, :] = P[0, :]
    return P


def _state(rng, K, G, finished=0):
    L = -rng.random(K) * 5
    n = rng.integers(1, 6, K).astype(float)
    status = np.zeros(K, int)
    status[rng.permutation(K)[:finished]] = 1
    return L, n, status


def _copy_src(rng):
    src = rng.integers(3, V, S)
    src[:3] = [3, 9, 21]                              # copies spelling the planted top words
    return src


@pytest.mark.parametrize("K", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("alpha", [0.0, 0.6])
def test_one_group_is_the_nbest_rule(K, alpha):
    rng = np.random.default_rng(K * 7 + int(alpha * 10))
    for trial in range(20):
        P = _rows(rng, K, ties=trial % 2 == 0)
        L, n, status = _state(rng, K, 1, finished=trial % K)
        ok = rng.random(S) > 0.3
        for prefilter in (True, False):
            [(sel, gap)], _ = step(L, n, status, P, ok, _copy_src(rng), V, 1, alpha, 2.5, prefilter)
            ref, ref_gap = beam_rule.step(L, n, status, P, ok, V, K, alpha, prefilter)
            assert [s[:5] for s in sel] == ref and gap == ref_gap


@pytest.mark.parametrize("K,G", [(2, 2), (4, 2), (6, 3), (8, 4), (16, 4)])
def test_zero_diversity_makes_every_group_an_independent_nbest(K, G):
    rng = np.random.default_rng(K + G)
    Kg = K // G
    for trial in range(10):
        P = _rows(rng, K, ties=trial % 2 == 0)
        L, n, status = _state(rng, K, G, finished=trial % K)
        ok = rng.random(S) > 0.3
        groups, _ = step(L, n, status, P, ok, _copy_src(rng), V, G, 0.6, 0.0)
        for g, (sel, _) in enumerate(groups):
            own = slice(g * Kg, (g + 1) * Kg)
            ref, _ = beam_rule.step(L[own], n[own], status[own], P[own], ok, V, Kg, 0.6)
            assert [(s[0] - g * Kg,) + s[1:5] for s in sel] == ref


@pytest.mark.parametrize("K,G", [(2, 2), (4, 2), (6, 3), (8, 4), (8, 8)])
@pytest.mark.parametrize("diversity", [0.5, 3.0])
def test_row_prefilter_by_penalised_value_then_merge_equals_brute_force(K, G, diversity):
    rng = np.random.default_rng(K * 100 + G * 10 + int(diversity))
    for trial in range(25):
        P = _rows(rng, K, ties=trial % 2 == 0)
        if trial % 3 == 0:
            P[:, 5] = P[:, 6]                         # a tie at the top of every row
            P[:, 5:7] = 0.9
        L, n, status = _state(rng, K, G, finished=trial % K)
        if trial % 4 == 0:                            # position 0: the first slot of every group alone
            status[:] = 2
            status[::K // G] = 0
            L[::K // G], n[::K // G] = 0.0, 0
        if trial % 5 == 1:                            # exact ties across the rows of a group
            P[1:K:2] = P[0:K:2][:len(P[1:K:2])]
            L[1:K:2], n[1:K:2] = L[0:K:2][:len(L[1:K:2])], n[0:K:2][:len(n[1:K:2])]
        ok = rng.random(S) > 0.3
        src = _copy_src(rng)
        fast, fast_chosen = step(L, n, status, P, ok, src, V, G, 0.6 * (trial % 2), diversity)
        brute, brute_chosen = step(L, n, status, P, ok, src, V, G, 0.6 * (trial % 2), diversity, prefilter=False)
        assert [sel for sel, _ in fast] == [sel for sel, _ in brute] and fast_chosen == brute_chosen


def test_a_copy_of_an_earlier_groups_word_is_penalised_like_the_vocabulary_entry():
    rng = np.random.default_rng(11)
    K, G = 2, 2
    P = _rows(rng, K)
    src = np.full(S, 30)
    src[2] = 3                                        # copy position 2 spells word 3
    L, n, status = np.zeros(K), np.zeros(K), np.zeros(K, int)
    ok = np.ones(S, bool)
    for diversity in (0.0, 1.5):
        cand = {c[3]: c for c in group_candidates(L, n, status, P, ok, src, V, G, 1, 0.0, diversity, [3],
                                                  prefilter=False)}
        for j in (3, V + 2):                          # the vocabulary entry and the copy of the earlier group's word
            assert cand[j][0] == cand[j][6] - diversity
        for j in (4, V + 0):                          # other words: no penalty
            assert cand[j][0] == cand[j][6]
    # a group-0 pick of word 3 through either route penalises both routes in group 1
    P[:, :] = 1e-6
    P[0, 3] = 0.9
    _, chosen = step(L, n, np.array([0, 0]), P, ok, src, V, G, 0.0, 100.0)
    assert chosen[0] == 3 and chosen[1] != 3


def test_finished_slots_are_carried_with_their_stored_score_and_no_penalty():
    rng = np.random.default_rng(4)
    K, G = 4, 2
    P = _rows(rng, K)
    L = np.array([-0.01, -9.0, -0.02, -30.0])
    n = np.array([3.0, 4.0, 2.0, 5.0])
    status = np.array([1, 0, 1, 0])
    src = _copy_src(rng)
    for alpha in (0.0, 1.0):
        groups, chosen = step(L, n, status, P, np.ones(S, bool), src, V, G, alpha, 1e3)
        for g, (sel, _) in enumerate(groups):
            carried = [s for s in sel if s[1] == C]
            assert [s[0] for s in carried] == [2 * g]               # each group keeps its finished slot
            i, j, Lk, nk, score, value = carried[0]
            assert Lk == L[i] and nk == n[i] and score == value == L[i] / ((5 + n[i]) / 6) ** alpha
            assert all(s[0] in (2 * g, 2 * g + 1) for s in sel)     # parents inside the group
        assert chosen[0] == -1 and chosen[2] == -1                # the carried slots rank first and count nothing


@pytest.mark.parametrize("kw", [dict(groups=0), dict(groups=2, beam_size=3), dict(groups=4, beam_size=2),
                                dict(groups=2.0), dict(groups=True), dict(groups="2"),
                                dict(groups=2, diversity=-0.5), dict(groups=2, diversity=float("inf")),
                                dict(groups=2, diversity=float("nan")), dict(groups=2, diversity=1e60),
                                dict(groups=2, diversity=True), dict(groups=2, diversity="0.5")])
def test_invalid_groups_or_diversity_raise_before_any_device_work(kw):
    from fira_icse_b200.beam import nbest
    args = dict(beam_size=4, length_penalty=0.0, tar_len=30)
    args.update(kw)
    with pytest.raises(ValueError):
        nbest(None, None, None, None, None, None, start_id=1, eos_id=2, **args)       # no model, no tensors needed
