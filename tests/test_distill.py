"""Knowledge distillation without a device: the float64 rule (tests/kd_rule.py) against float64 autograd of
-sum_j w_j log clamp(P_j, 1e-10, 1), every error distill_step and teacher_targets raise before any device work, and
the argument errors of `run_model.py distill`."""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from fira_testlib import ROOT, golden_batch, reference_args, seeded_model
from kd_rule import row
from sample_rule import mixture


def _autograd(x, c, gl, mk, t, y, alpha):
    """loss and gradients of (1 - alpha) nll + alpha kd by torch autograd in float64"""
    x, c, gl = (torch.tensor(a, dtype=torch.float64, requires_grad=True) for a in (x, c, gl))
    V = x.shape[0]
    cm = c.masked_fill(torch.from_numpy(mk == 0), -1e9)
    g = torch.softmax(gl, 0)
    P = torch.cat((g[0] * torch.softmax(x, 0), g[1] * torch.softmax(cm, 0)))
    lp = torch.log(torch.clamp(P, 1e-10, 1.0))
    w = alpha * torch.from_numpy(t)
    nll = torch.tensor(-np.log(1e-10), dtype=torch.float64)           # a copy label beyond S: the clamp floor
    if y < V + c.shape[0]:
        w[y] += 1.0 - alpha
        nll = -lp[y]
    loss = -(w * lp).sum()
    if y >= V + c.shape[0]:
        loss = loss + (1.0 - alpha) * nll
    loss.backward()
    kd = -(torch.from_numpy(t) * lp).sum()
    return nll.item(), kd.item(), loss.item(), x.grad.numpy(), c.grad.numpy(), gl.grad.numpy()


def _case(rng, V, S, y, gate=None, teacher_gate=None):
    x = rng.normal(0, 8, V)                     # wide: many entries below the clamp
    c = rng.normal(0, 3, S)
    mk = (rng.random(S) < 0.7).astype(np.uint8)
    mk[0] = 1
    gl = rng.normal(0, 1, 2) if gate is None else np.array(gate, np.float64)
    tx, tc = rng.normal(0, 2, V), rng.normal(0, 2, S)
    tg = rng.normal(0, 1, 2) if teacher_gate is None else np.array(teacher_gate, np.float64)
    t = mixture(tx, tc, tg, mk)
    t[V:][mk == 0] = 0.0
    return x, c, gl, mk, t


@pytest.mark.parametrize("alpha", [0.0, 0.3, 1.0])
def test_rule_matches_float64_autograd(alpha):
    rng = np.random.default_rng(int(alpha * 10) + 5)
    V, S = 61, 13
    cases = []
    for y in (3, 40, V + 2):                    # vocabulary labels and a copy label
        cases.append(_case(rng, V, S, y) + (y,))
    x, c, gl, mk, t = _case(rng, V, S, 0)
    masked = int(np.flatnonzero(mk == 0)[0]) if (mk == 0).any() else None
    if masked is not None:                      # a copy label at a masked position
        cases.append((x, c, gl, mk, t, V + masked))
    cases.append(_case(rng, V, S, 5, gate=[-1e4, 0.0]) + (5,))         # g0 = 0: every vocabulary entry clamped
    cases.append(_case(rng, V, S, V + 1, gate=[0.0, -1e4]) + (V + 1,))  # g1 = 0
    cases.append(_case(rng, V, S, 7, teacher_gate=[-1e4, 0.0]) + (7,))  # the teacher's G0 = 0
    cases.append(_case(rng, V, S, V + S + 4) + (V + S + 4,))           # a copy label beyond S
    below = 0
    for x, c, gl, mk, t, y in cases:
        got = row(x, c, gl, mk, t, y, alpha)
        want = _autograd(x, c, gl, mk, t, y, alpha)
        for g, w in zip(got[:3], want[:3]):
            assert abs(g - w) <= 1e-12 * max(1.0, abs(w))
        for g, w in zip(got[3:], want[3:]):
            np.testing.assert_allclose(g, w, rtol=0, atol=1e-13)
        below += int((mixture(x, c, gl, mk) < 1e-10).sum())
    assert below > 0


def test_zero_label_rows_carry_nothing():
    rng = np.random.default_rng(1)
    x, c, gl, mk, t = _case(rng, 61, 13, 0)
    nll, kd, loss, dx, dc, dgl = row(x, c, gl, mk, t, 0, 0.5)
    assert nll == kd == loss == 0.0
    assert not dx.any() and not dc.any() and not dgl.any()


def test_alpha_zero_is_the_nll_and_one_hot_teacher_is_alpha_zero():
    rng = np.random.default_rng(2)
    V, S = 61, 13
    x, c, gl, mk, _ = _case(rng, V, S, 9)
    onehot = np.zeros(V + S)
    onehot[9] = 1.0
    hard = row(x, c, gl, mk, np.full(V + S, 0.5), 9, 0.0)
    soft = row(x, c, gl, mk, onehot, 9, 1.0)
    assert hard[2] == hard[0] and abs(soft[2] - hard[0]) <= 1e-15
    for a, b in zip(hard[3:], soft[3:]):
        np.testing.assert_array_equal(a, b)


# ------------------------------------------------------------------ validation before any device work
def _step(teacher="copy", alpha=0.5, student=None):
    from fira_icse_b200.distill import distill_step
    student = seeded_model() if student is None else student
    if teacher == "copy":
        teacher = copy.deepcopy(student)
    distill_step(student, None, golden_batch(0, 2), teacher, alpha=alpha)


@pytest.mark.parametrize("alpha,exc", [(-0.1, ValueError), (1.5, ValueError), (float("nan"), ValueError),
                                       (float("inf"), ValueError), (True, TypeError), ("0.5", TypeError),
                                       (None, TypeError)])
def test_bad_alpha_raises_before_device_work(alpha, exc):
    with pytest.raises(exc, match="alpha"):
        _step(alpha=alpha)


def test_bad_teachers_raise_before_device_work():
    from fira_icse_b200 import TransModel
    from fira_icse_b200.distill import teacher_targets
    m = seeded_model()
    with pytest.raises(TypeError, match="TransModel or an Ensemble"):
        _step(teacher="best_model.pt")
    with pytest.raises(TypeError, match="TransModel or an Ensemble"):
        _step(teacher=[copy.deepcopy(m)])
    with pytest.raises(ValueError, match="the student itself"):
        _step(teacher=m)
    torch.manual_seed(0)
    small = TransModel(reference_args(vocab_size=61))
    with pytest.raises(ValueError, match="vocab_size"):
        _step(teacher=small)
    with pytest.raises(ValueError, match="meta"):
        _step(teacher=copy.deepcopy(m).to("meta"))
    with pytest.raises(TypeError, match="TransModel or an Ensemble"):
        teacher_targets("best_model.pt", golden_batch(0, 2), torch.zeros((2, 30), dtype=torch.long))


def test_ensemble_teacher_with_the_student_as_member_raises():
    """an Ensemble needs CUDA members; the identity check runs on its member tuple, so a stand-in shows it"""
    from fira_icse_b200 import distill
    from fira_icse_b200.ensemble import Ensemble
    m = seeded_model()
    ens = Ensemble.__new__(Ensemble)
    ens.models, ens.log_weights = (copy.deepcopy(m), m), (np.log(0.5),) * 2
    with pytest.raises(ValueError, match="teacher member 1 is the student"):
        distill.teacher_members(ens, m)


# ------------------------------------------------------------------ run_model.py distill
def _distill(tmp_path, **env):
    e = dict(os.environ, PYTHONPATH=ROOT, **env)
    for k in ("FIRA_ENSEMBLE", "FIRA_ENSEMBLE_WEIGHTS", "FIRA_CHECKPOINT"):
        if k not in env:
            e.pop(k, None)
    return subprocess.run([sys.executable, os.path.join(ROOT, "run_model.py"), "distill"], cwd=tmp_path, env=e,
                          capture_output=True, text=True, timeout=300)


@pytest.mark.parametrize("env,match", [
    (dict(WORLD_SIZE="2"), "one GPU"),
    (dict(FIRA_KD_ALPHA="1.5"), "FIRA_KD_ALPHA"),
    (dict(FIRA_KD_ALPHA="-0.5"), "FIRA_KD_ALPHA"),
    (dict(FIRA_KD_ALPHA="nan"), "FIRA_KD_ALPHA"),
    (dict(FIRA_KD_ALPHA="half"), "could not convert"),
    (dict(FIRA_KD_EPOCHS="0"), "FIRA_KD_EPOCHS"),
    (dict(FIRA_KD_EPOCHS="two"), "invalid literal"),
    (dict(FIRA_KD_LR="0"), "FIRA_KD_LR"),
    (dict(FIRA_KD_LR="inf"), "FIRA_KD_LR"),
    (dict(), "needs the teacher"),
    (dict(FIRA_ENSEMBLE_WEIGHTS="1,2"), "FIRA_ENSEMBLE_WEIGHTS needs FIRA_ENSEMBLE"),
    (dict(FIRA_ENSEMBLE="a.pt,b.pt", FIRA_ENSEMBLE_WEIGHTS="1"), "1 weights for 2 checkpoints"),
    (dict(FIRA_ENSEMBLE="a.pt,b.pt", FIRA_ENSEMBLE_WEIGHTS="1,-1"), "positive finite"),
    (dict(FIRA_ENSEMBLE="a.pt,,b.pt"), "1 to 8 checkpoints"),
    (dict(FIRA_ENSEMBLE="missing.pt"), "missing.pt not found"),
    (dict(FIRA_ENSEMBLE="teacher.pt"), "student checkpoint best_model.pt not found"),
    (dict(FIRA_ENSEMBLE="teacher.pt", FIRA_CHECKPOINT="student.pt"), "student.pt not found"),
    (dict(FIRA_ENSEMBLE="teacher.pt,best_model_kd.pt", FIRA_CHECKPOINT="teacher.pt"), "which distill writes"),
])
def test_distill_argument_errors(tmp_path, env, match):
    for name in ("teacher.pt", "best_model_kd.pt"):
        (tmp_path / name).write_bytes(b"")
    kd = (tmp_path / "best_model_kd.pt").read_bytes()
    r = _distill(tmp_path, **env)
    assert r.returncode != 0
    assert match in r.stderr, r.stderr[-2000:]
    assert (tmp_path / "best_model_kd.pt").read_bytes() == kd
    assert not os.path.exists(tmp_path / "OUTPUT" / "dev_output_kd")


def test_test_still_refuses_a_checkpoint_with_an_ensemble(tmp_path):
    (tmp_path / "teacher.pt").write_bytes(b"")
    e = dict(os.environ, PYTHONPATH=ROOT, FIRA_DECODE="sample", FIRA_ENSEMBLE="teacher.pt", FIRA_CHECKPOINT="x.pt")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "run_model.py"), "test"], cwd=tmp_path, env=e,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "unset FIRA_CHECKPOINT" in r.stderr
