"""Offline distillation on the host: the float64 top-k rule (tests/kd_topk_rule.py) on hand-made rows, KDTargets
save / load and batch(), its refusals, and the settings errors of `run_model.py kd-targets` and `distill`."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from fira_testlib import ROOT
from kd_rule import row as kd_row
from kd_topk_rule import dense, row, topk


# ============================================================================= the rule
def test_ties_go_to_the_smaller_label():
    V = 6
    P = np.array([0.1, 0.2, 0.1, 0.2, 0.05, 0.05, 0.2, 0.1])     # copy positions 0, 1 (labels 6, 7)
    labels, probs, mass = topk(P, [1, 1], V, 4)
    assert labels.tolist() == [1, 3, 6, 0]
    assert mass == pytest.approx(0.7)
    np.testing.assert_allclose(probs, P[[1, 3, 6, 0]] / 0.7)


def test_masked_copies_and_zero_probabilities_are_not_candidates():
    V = 4
    P = np.array([0.0, 0.3, 0.1, 0.0, 0.4, 0.2])                 # copy position 0 is masked
    labels, probs, mass = topk(P, [0, 1], V, 3)
    assert labels.tolist() == [1, 5, 2]
    assert mass == pytest.approx(0.6)


def test_fewer_candidates_than_k_fill_with_minus_one():
    V = 3
    P = np.array([0.0, 0.7, 0.0, 0.3, 0.0])
    labels, probs, mass = topk(P, [1, 0], V, 5)
    assert labels.tolist() == [1, 3, -1, -1, -1]
    np.testing.assert_allclose(probs, [0.7, 0.3, 0, 0, 0])
    assert mass == pytest.approx(1.0)
    assert topk(np.zeros(5), [1, 1], V, 2)[0].tolist() == [-1, -1]


def test_the_loss_is_kd_rule_on_the_renormalised_vector():
    rng = np.random.default_rng(3)
    V, S, k = 9, 4, 3
    x, c, gl = rng.normal(size=V), rng.normal(size=S), rng.normal(size=2)
    mk = np.array([1, 0, 1, 1])
    P = rng.random(V + S)
    labels, probs, _ = topk(P, mk, V, k)
    t = dense(labels, probs, V + S)
    assert t.sum() == pytest.approx(1.0) and np.count_nonzero(t) == k
    for y in (0, 2, V + 2):
        got, want = row(x, c, gl, mk, labels, probs, y, 0.4), kd_row(x, c, gl, mk, t, y, 0.4)
        for g, w in zip(got, want):
            np.testing.assert_array_equal(g, w)


# ============================================================================= KDTargets
def _targets(k=3, first=0):
    """four commits with 2, 0, 3 and 1 loss rows"""
    from fira_icse_b200.distill import KDTargets
    pos = torch.tensor([0, 2, 0, 1, 4, 1], dtype=torch.int16)
    y = torch.tensor([5, 7, 1, 9, 2, 3], dtype=torch.int32)
    R = pos.numel()
    t_label = torch.arange(R * k, dtype=torch.int32).view(R, k)
    t_prob = torch.rand((R, k), generator=torch.Generator().manual_seed(1))
    return KDTargets(torch.tensor([0, 2, 2, 5, 6]), pos, y, t_label, t_prob, torch.rand(R), vocab_size=11, k=k,
                     first=first, provenance=dict(fingerprints=["ab"], weights=[1.0], precision="fp32", commits=4))


def _labels(store, indices, T=6):
    """the shifted labels of a batch of the stored commits at `indices`"""
    lab = torch.zeros((len(indices), T), dtype=torch.int64)
    for b, i in enumerate(indices):
        i -= store.first
        for r in range(int(store.row_off[i]), int(store.row_off[i + 1])):
            lab[b, int(store.pos[r])] = int(store.y[r])
    return lab


def test_save_load_round_trip(tmp_path):
    from fira_icse_b200.distill import KDTargets
    a = _targets(first=7)
    a.save(tmp_path / "t.pt")
    b = KDTargets.load(tmp_path / "t.pt", vocab_size=11, k=3, commits=4)
    for f in ("row_off", "pos", "y", "t_label", "t_prob", "mass"):
        assert torch.equal(getattr(a, f), getattr(b, f)), f
    assert (b.vocab_size, b.k, b.first, b.n, b.rows) == (11, 3, 7, 4, 6)
    assert b.provenance == a.provenance and b.nbytes == a.nbytes
    for kw, match in ((dict(vocab_size=12), "vocab_size 11"), (dict(k=8), "k 3"), (dict(commits=5), "commits 4")):
        with pytest.raises(ValueError, match=match):
            KDTargets.load(tmp_path / "t.pt", **kw)
    torch.save({"format": "other"}, tmp_path / "o.pt")
    with pytest.raises(ValueError, match="not a distillation target file"):
        KDTargets.load(tmp_path / "o.pt")


def test_batch_returns_the_rows_of_shuffled_commits():
    s = _targets(first=10)
    order = [13, 10, 11, 12]
    T = 6
    got = s.batch(order, _labels(s, order, T))
    assert got.t_label.shape == (4 * T, 3) and got.t_label.dtype == torch.int32
    want_l = torch.full((4 * T, 3), -1, dtype=torch.int32)
    want_p = torch.zeros((4 * T, 3))
    for b, i in enumerate(order):
        i -= s.first
        for r in range(int(s.row_off[i]), int(s.row_off[i + 1])):
            want_l[b * T + int(s.pos[r])] = s.t_label[r]
            want_p[b * T + int(s.pos[r])] = s.t_prob[r]
    assert torch.equal(got.t_label, want_l) and torch.equal(got.t_prob, want_p)
    assert int((got.t_label[:, 0] >= 0).sum()) == s.rows


def test_batch_refuses_another_split_or_order():
    s = _targets()
    lab = _labels(s, [0, 1, 2])
    with pytest.raises(ValueError, match="row counts"):
        s.batch([1, 0, 2], lab)                               # commits 0 and 1 swapped
    bad = lab.clone()
    bad[0, 2] = 6                                             # the same rows, another label
    with pytest.raises(ValueError, match="positions or labels"):
        s.batch([0, 1, 2], bad)
    moved = lab.clone()
    moved[0, 2], moved[0, 3] = 0, 7                           # the same count, another position
    with pytest.raises(ValueError, match="positions or labels"):
        s.batch([0, 1, 2], moved)
    with pytest.raises(ValueError, match="outside the stored commits"):
        s.batch([0, 1, 4], _labels(s, [0, 1, 2]))
    with pytest.raises(ValueError, match="positions for a batch"):
        s.batch([0, 1], lab)


def test_constructor_and_step_refusals():
    from fira_icse_b200.distill import KDTargets, check_topk
    s = _targets()
    for k in (0, 65, 2.5, True):
        with pytest.raises(ValueError, match="k must be an integer"):
            check_topk(k)
    with pytest.raises(ValueError, match="rise from 0"):
        KDTargets(torch.tensor([0, 2, 1, 6]), s.pos, s.y, s.t_label, s.t_prob, s.mass, vocab_size=11, k=3, first=0,
                  provenance={})
    with pytest.raises(ValueError, match="t_label"):
        KDTargets(s.row_off, s.pos, s.y, s.t_label.long(), s.t_prob, s.mass, vocab_size=11, k=3, first=0,
                  provenance={})


# ============================================================================= CLI settings
def _run(stage, tmp_path, **env):
    e = dict(os.environ, PYTHONPATH=ROOT, **env)
    for k in ("FIRA_ENSEMBLE", "FIRA_ENSEMBLE_WEIGHTS", "FIRA_CHECKPOINT", "FIRA_KD_TARGETS", "FIRA_KD_TOPK"):
        if k not in env:
            e.pop(k, None)
    return subprocess.run([sys.executable, os.path.join(ROOT, "run_model.py"), stage], cwd=tmp_path, env=e,
                          capture_output=True, text=True, timeout=300)


@pytest.mark.parametrize("stage,env,match", [
    ("kd-targets", dict(FIRA_KD_TOPK="0", FIRA_ENSEMBLE="teacher.pt"), "FIRA_KD_TOPK must be in [1, 64]"),
    ("kd-targets", dict(FIRA_KD_TOPK="65", FIRA_ENSEMBLE="teacher.pt"), "FIRA_KD_TOPK must be in [1, 64]"),
    ("kd-targets", dict(FIRA_KD_TOPK="eight", FIRA_ENSEMBLE="teacher.pt"), "FIRA_KD_TOPK"),
    ("kd-targets", dict(), "needs the teacher"),
    ("kd-targets", dict(FIRA_ENSEMBLE="missing.pt"), "missing.pt not found"),
    ("kd-targets", dict(WORLD_SIZE="2"), "one GPU"),
    ("distill", dict(FIRA_KD_TARGETS="targets.pt", FIRA_ENSEMBLE="teacher.pt"), "unset FIRA_ENSEMBLE"),
    ("distill", dict(FIRA_KD_TARGETS="missing.pt"), "FIRA_KD_TARGETS: missing.pt not found"),
    ("distill", dict(FIRA_KD_TARGETS="targets.pt", FIRA_CHECKPOINT="student.pt"), "student.pt not found"),
])
def test_settings_errors(tmp_path, stage, env, match):
    for name in ("teacher.pt", "targets.pt"):
        (tmp_path / name).write_bytes(b"")
    r = _run(stage, tmp_path, **env)
    assert r.returncode != 0
    assert match in r.stderr, r.stderr[-2000:]
    assert not os.path.exists(tmp_path / "kd_targets.pt") and not os.path.exists(tmp_path / "best_model_kd.pt")
