"""The n-best rule (float64 restatement, tests/beam_rule.py) and the argument checks of fira_icse_b200.beam.nbest, on
CPU.  The kernel is compared with the restatement in tests/test_gpu_nbest.py."""
import numpy as np
import pytest

from beam_rule import candidates, step, token_logprob
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


def _state(rng, K, finished=0):
    L = -rng.random(K) * 5
    n = rng.integers(1, 6, K).astype(float)
    status = np.zeros(K, int)
    status[:finished] = 1
    return L, n, status


def test_k1_alpha0_is_greedy():
    rng = np.random.default_rng(0)
    for _ in range(50):
        P = _rows(rng, 1)
        ok = rng.random(S) > 0.3
        sel, _ = step([0.0], [0], [0], P, ok, V, 1, 0.0)
        masked = P[0].copy()
        masked[V:][~ok] = -1
        assert sel[0][:2] == (0, int(np.argmax(masked)))


@pytest.mark.parametrize("K", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("alpha", [0.0, 0.6, 1.5])
def test_row_top_k_prefilter_then_merge_equals_brute_force(K, alpha):
    rng = np.random.default_rng(K * 10 + int(alpha * 10))
    for trial in range(30):
        P = _rows(rng, K, ties=trial % 2 == 0)
        if trial % 3 == 0:
            P[:, 5] = P[:, 6]                         # a tie at the top of every row
            P[:, 5:7] = 0.9
        L, n, status = _state(rng, K, finished=trial % K)
        if trial % 5 == 0:
            status[1:] = 2                            # position 0: slot 0 alone
            L[0], n[0] = 0.0, 0
        ok = rng.random(S) > 0.3
        fast, _ = step(L, n, status, P, ok, V, K, alpha)
        brute, _ = step(L, n, status, P, ok, V, K, alpha, prefilter=False)
        assert fast == brute


def test_masked_copies_are_never_candidates_and_inactive_slots_propose_nothing():
    rng = np.random.default_rng(3)
    P = _rows(rng, 3)
    ok = np.zeros(S, bool)
    P[:, V:] = 0.99                                   # masked copies would win every slot
    cand = candidates([0.0, 0.0, 0.0], [0, 0, 0], [0, 2, 2], P, ok, V, 3, 0.0, prefilter=False)
    assert all(c[2] == 0 and c[3] < V for c in cand) and len(cand) == V


def test_finished_slots_are_carried_unchanged():
    rng = np.random.default_rng(4)
    K = 4
    for alpha in (0.0, 1.0):
        P = _rows(rng, K)
        L = np.array([-0.01, -9.0, -30.0, -0.02])
        n = np.array([3.0, 4.0, 5.0, 2.0])
        status = np.array([1, 0, 0, 1])
        sel, _ = step(L, n, status, P, np.ones(S, bool), V, K, alpha)
        carried = [s for s in sel if s[1] == C]
        assert sorted(s[0] for s in carried) == [0, 3]                 # both stay (nothing else scores near 0)
        for i, j, Lk, nk, score in carried:
            assert Lk == L[i] and nk == n[i] and score == L[i] / ((5 + n[i]) / 6) ** alpha


def test_alpha0_ranking_equals_fp32_product_ranking_without_underflow():
    rng = np.random.default_rng(5)
    K = 3
    checked = 0
    for _ in range(40):
        P = _rows(rng, K)
        L, n, status = _state(rng, K)
        prob = np.exp(L).astype(np.float32)
        ok = np.ones(S, bool)
        sel, _ = step(L, n, status, P, ok, V, K, 0.0)
        prod = (prob[:, None] * P.astype(np.float32)).reshape(-1)        # the reference's candidate layout
        assert (prod[prod > 0] > 1e-30).all()
        order = np.argsort(-prod, kind="stable")
        if prod[order[K - 1]] - prod[order[K]] <= 1e-5 * prod[order[K - 1]]:
            continue                                                       # fp32 near-tie: either answer is right
        assert [(s[0], s[1]) for s in sel] == [(int(o) // C, int(o) % C) for o in order[:K]]
        checked += 1
    assert checked >= 30


def test_log_rule_separates_hypotheses_whose_fp32_products_are_all_zero():
    rng = np.random.default_rng(6)
    K = 5
    P = _rows(rng, K)
    L = np.array([-120.0, -121.0, -122.5, -130.0, -131.0])             # exp(L) underflows in fp32
    n = np.full(K, 12.0)
    status = np.zeros(K, int)
    assert (np.exp(L).astype(np.float32)[:, None] * P.astype(np.float32) == 0).all()
    sel, gap = step(L, n, status, P, np.ones(S, bool), V, K, 0.0)
    scores = [s[4] for s in sel]
    assert all(a > b for a, b in zip(scores, scores[1:])) and gap > 0
    best = max((L[i] + token_logprob(P[i, j]), i, j) for i in range(K) for j in range(C))
    assert (sel[0][0], sel[0][1]) == (best[1], best[2])


def test_length_penalty_prefers_longer_hypotheses():
    # equal per-token log-probability: alpha = 0 ranks the short hypothesis first, alpha = 1 the long one
    L = np.array([-2.0, -4.0])
    n = np.array([2.0, 4.0])
    P = np.zeros((2, C))
    sel0, _ = step(L, n, [1, 1], P, np.ones(S, bool), V, 2, 0.0)
    sel1, _ = step(L, n, [1, 1], P, np.ones(S, bool), V, 2, 1.0)
    assert [s[0] for s in sel0] == [0, 1] and [s[0] for s in sel1] == [0, 1]      # -2/1.17 > -4/1.5
    sel2, _ = step(L, n, [1, 1], P, np.ones(S, bool), V, 2, 3.0)
    assert [s[0] for s in sel2] == [1, 0]                                        # -2/1.6 < -4/3.375


@pytest.mark.parametrize("kw", [dict(beam_size=0), dict(beam_size=17), dict(beam_size=2.0), dict(beam_size=True),
                                dict(length_penalty=-0.1), dict(length_penalty=float("inf")),
                                dict(length_penalty=float("nan")), dict(length_penalty=1e60),
                                dict(length_penalty="1"), dict(tar_len=1), dict(tar_len=2.5)])
def test_invalid_arguments_raise_before_any_device_work(kw):
    from fira_icse_b200.beam import nbest
    args = dict(beam_size=3, length_penalty=0.0, tar_len=30)
    args.update(kw)
    with pytest.raises(ValueError):
        nbest(None, None, None, None, None, None, start_id=1, eos_id=2, **args)       # no model, no tensors needed
