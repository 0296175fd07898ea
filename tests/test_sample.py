"""The sampling rule (float64 restatement, tests/sample_rule.py) and the argument checks of fira_icse_b200.sample, on CPU.
The kernel is compared with the restatement in tests/test_gpu_sample.py."""
import numpy as np
import pytest

from sample_rule import draw, mixture


def _row(rng, V=40, S=7):
    P = mixture(rng.normal(0, 2, V), rng.normal(0, 2, S), rng.normal(0, 1, 2), rng.random(S) > 0.3)
    return P, np.ones(S, bool)


def test_top_k_1_and_tiny_top_p_give_the_argmax():
    rng = np.random.default_rng(0)
    for _ in range(50):
        P, ok = _row(rng)
        best = int(np.argmax(P))
        for u in (0.0, 0.5, 0.999999):
            assert draw(P, ok, 40, 1.0, 1, 1.0, u)[0] == best
            assert draw(P, ok, 40, 0.7, 0, 1e-6, u)[0] == best
            assert draw(P, ok, 40, 3.0, 50, 1e-6, u)[0] == best


def test_ties_go_to_the_smaller_index():
    P = np.array([0.1, 0.3, 0.2, 0.3, 0.1])
    ok = np.ones(0, bool)
    assert draw(P, ok, 5, 1.0, 1, 1.0, 0.9)[0] == 1                   # two maxima: index 1 ranks first
    # k = 2 keeps ranks {1, 3}; u below half of their equal weights picks the smaller index
    assert draw(P, ok, 5, 1.0, 2, 1.0, 0.49)[0] == 1
    assert draw(P, ok, 5, 1.0, 2, 1.0, 0.51)[0] == 3
    # k = 3: the third rank is index 2 (0.2), not one of the two 0.1 entries
    assert sorted({draw(P, ok, 5, 1.0, 3, 1.0, u)[0] for u in np.linspace(0, 0.999, 200)}) == [1, 2, 3]
    # three-way tie at the k cut: the two smaller indices stay
    Q = np.array([0.25, 0.25, 0.25, 0.25])
    assert sorted({draw(Q, ok, 4, 1.0, 2, 1.0, u)[0] for u in np.linspace(0, 0.999, 200)}) == [0, 1]


def test_masked_and_zero_entries_are_never_kept():
    rng = np.random.default_rng(1)
    V, S = 30, 9
    for _ in range(30):
        mask = rng.random(S) > 0.5
        mask[0] = False
        P = mixture(rng.normal(0, 1, V), rng.normal(0, 1, S) + 5.0, rng.normal(0, 1, 2), mask)
        ok = mask.copy()
        P[3] = 0.0
        for u in np.linspace(0, 0.999, 64):
            for k, p, T in ((0, 1.0, 1.0), (5, 1.0, 0.5), (0, 0.9, 2.0)):
                j = draw(P, ok, V, T, k, p, u)[0]
                assert j != 3 and (j < V or mask[j - V])


def test_draw_frequencies_follow_the_tempered_weights():
    P = np.array([0.5, 0.3, 0.15, 0.05])
    us = (np.arange(100000) + 0.5) / 100000
    for T, k, p in ((1.0, 0, 1.0), (0.5, 0, 1.0), (2.0, 3, 1.0), (1.0, 0, 0.7)):
        counts = np.bincount([draw(P, np.ones(0, bool), 4, T, k, p, u)[0] for u in us], minlength=4) / len(us)
        w = P ** (1.0 / T)
        if k:
            w[k:] = 0
        if p < 1:
            keep = np.cumsum(w) / w.sum() < p
            keep[np.argmin(keep)] = True                 # the entry that reaches p stays
            w = np.where(keep, w, 0)
        np.testing.assert_allclose(counts, w / w.sum(), atol=1e-4)


@pytest.mark.parametrize("kw", [dict(num_samples=0), dict(num_samples=33), dict(num_samples=2.0),
                                dict(temperature=0.0), dict(temperature=-1.0), dict(temperature=float("inf")),
                                dict(temperature=float("nan")), dict(temperature=1e-60), dict(top_k=-1),
                                dict(top_k=1.5), dict(top_p=0.0), dict(top_p=1.5), dict(top_p=float("nan")),
                                dict(seed=-1), dict(seed=2 ** 64), dict(first_index=-1), dict(tar_len=1)])
def test_invalid_arguments_raise_before_any_device_work(kw):
    from fira_icse_b200.sample import sample
    args = dict(num_samples=2, temperature=1.0, top_k=0, top_p=1.0, seed=0, first_index=0, tar_len=30)
    args.update(kw)
    with pytest.raises(ValueError):
        sample(None, None, None, None, None, None, start_id=1, eos_id=2, **args)       # no model, no tensors needed
