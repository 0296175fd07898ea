"""Global-norm gradient clipping without a GPU: the float64 rule (clip_rule.py) against torch.nn.utils.clip_grad_norm_
followed by torch.optim.Adam in float64, the C prototypes, optim.check_max_grad_norm, and FIRA_CLIP_NORM in
`run_model.py train`, `finetune` and `distill`: accepted values, and refusals before any device work."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import clip_rule
from fira_testlib import ROOT

LR, B1, B2, EPS = 2.0 ** -10, 0.875, 0.9990234375, 2.0 ** -27          # exact in fp32: the rule rounds none of them


def _tensors(seed, shapes=((64, 32), (32,), (7,), (1,))):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(s, generator=g, dtype=torch.float64) for s in shapes]


@pytest.mark.parametrize("c", [1.0, float("inf")])
@pytest.mark.parametrize("grad_scale", [None, 37.0])
def test_rule_matches_torch_clip_and_adam_in_float64(c, grad_scale):
    """20 steps whose gradient norms range over four decades, so that c = 1 clips some steps and not others; step 7
    has an inf gradient and step 13 a NaN one: the rule skips them (the torch reference does not step) and the state
    is unchanged"""
    ps = [torch.nn.Parameter(t) for t in _tensors(0)]
    opt = torch.optim.Adam(ps, lr=LR, betas=(B1, B2), eps=EPS)
    state = clip_rule.new_state([p.detach().numpy() for p in ps])
    gen = torch.Generator().manual_seed(1)
    taken_clipped = taken_unclipped = 0
    for k in range(20):
        grads = [torch.randn(p.shape, generator=gen, dtype=torch.float64) * 10.0 ** (k % 4 - 2) for p in ps]
        if k in (7, 13):
            grads[k % 2][0] = float("inf") if k == 7 else float("nan")
        s = grad_scale or 1.0
        before = [dict(mb) for mb in state["members"]], state["t"]
        taken, nrm, coef = clip_rule.step(state, [g.numpy() * s for g in grads], c, LR, B1, B2, EPS, grad_scale)
        if k in (7, 13):
            assert not taken and not np.isfinite(nrm)
            for mb, mb0 in zip(state["members"], before[0]):
                for key in ("p", "m", "v"):
                    assert mb[key] is mb0[key]
            assert state["t"] == before[1]
            continue
        for p, g in zip(ps, grads):
            p.grad = g.clone()
        total = torch.nn.utils.clip_grad_norm_(ps, c)
        np.testing.assert_allclose(nrm, float(total), rtol=1e-12)
        opt.step()
        taken_clipped += coef < 1.0
        taken_unclipped += coef == 1.0
        for p, mb in zip(ps, state["members"]):
            # coef is rounded to fp32 once (and g' twice): a relative 2^-24 of the step, which Adam's m / sqrt(v) damps
            np.testing.assert_allclose(mb["p"], p.detach().numpy(), rtol=1e-6, atol=LR * 1e-5)
    assert state["skipped"] == 2 and state["t"] == 18
    assert state["clipped"] == taken_clipped
    if c == 1.0:
        assert taken_clipped >= 4 and taken_unclipped >= 4
    else:
        assert taken_clipped == 0


def test_rule_coefficient_and_fp32_order():
    assert clip_rule.coefficient(0.5, 1.0) == 1.0
    assert clip_rule.coefficient(3.0, float("inf")) == 1.0
    assert clip_rule.coefficient(4.0, 1.0) == np.float64(np.float32(1.0 / (4.0 + 1e-6)))
    g = np.array([3.0, -1e-30, 2.0 ** 100], np.float32)
    assert np.array_equal(clip_rule.scaled_grad(g, 1.0), g.astype(np.float64))      # coef 1 is the identity
    S, nrm = clip_rule.norm([np.array([3e19, 4e19], np.float32)])                     # squares overflow fp32, not float64
    assert np.isfinite(S) and nrm == pytest.approx(5e19, rel=1e-7)


def test_prototypes():
    from fira_icse_b200 import _lib
    h = _lib.parse_header()
    assert h["fira_adam_flat"][2][-3:] == ["ema", "ema_decay", "stream"]            # the existing entry point is as it was
    names = h["fira_adam_flat_clip"][2]
    assert names[:-2] == h["fira_adam_flat"][2][:-1] and names[-2:] == ["clip", "stream"]
    restype, types, names = h["fira_grad_clip_finalize"]
    assert names == ["partials", "n_partials", "grad_scale", "max_norm", "clip", "steps", "n_steps", "stream"]
    assert types[3].__name__ == "c_double"
    assert h["fira_grad_sumsq"][2] == ["g", "n", "partials", "stream"]
    assert h["fira_grad_sumsq_blocks"][2] == ["n"]


@pytest.mark.parametrize("bad", [0, -1.0, float("nan"), float("-inf"), "x", None])
def test_check_max_grad_norm_refuses(bad):
    from fira_icse_b200.optim import check_max_grad_norm
    with pytest.raises(ValueError, match="max_grad_norm"):
        check_max_grad_norm(bad)


def test_check_max_grad_norm_accepts():
    from fira_icse_b200.optim import check_max_grad_norm
    assert check_max_grad_norm("1.5") == 1.5 and check_max_grad_norm(float("inf")) == float("inf")
    assert check_max_grad_norm("inf") == float("inf") and check_max_grad_norm(1e-30) == 1e-30


# ------------------------------------------------------------------ run_model.py
def _run(tmp_path, stage, **env):
    e = dict(os.environ, PYTHONPATH=ROOT, **env)
    return subprocess.run([sys.executable, os.path.join(ROOT, "run_model.py"), stage], cwd=tmp_path, env=e,
                          capture_output=True, text=True, timeout=300)


@pytest.mark.parametrize("stage,value", [("train", "0"), ("train", "-1"), ("train", "nan"), ("train", "-inf"),
                                         ("train", "big"), ("finetune", "0"), ("distill", "nan")])
def test_clip_norm_argument_errors(tmp_path, stage, value):
    """refused before the device, the data or the model are touched: no CUDA-device message, no missing-DataSet error,
    no file written (every stage reads the setting through clip_settings, test_clip_settings covers the values)"""
    r = _run(tmp_path, stage, FIRA_CLIP_NORM=value)
    assert r.returncode != 0
    assert "FIRA_CLIP_NORM must be a positive number or inf" in r.stderr, r.stderr[-2000:]
    assert "no CUDA device" not in r.stderr and "DataSet" not in r.stderr
    assert not [f for f in os.listdir(tmp_path) if f.endswith(".pt")]


def test_clip_norm_with_the_eager_engine_is_refused(tmp_path):
    r = _run(tmp_path, "train", FIRA_CLIP_NORM="1.0", FIRA_ENGINE="eager")
    assert r.returncode != 0 and "FIRA_ENGINE=eager" in r.stderr, r.stderr[-2000:]
    assert "no CUDA device" not in r.stderr and "DataSet" not in r.stderr


def test_clip_settings(monkeypatch):
    import run_model
    monkeypatch.delenv("FIRA_CLIP_NORM", raising=False)
    monkeypatch.delenv("FIRA_ENGINE", raising=False)
    assert run_model.clip_settings() is None and run_model.clip_settings(engine_checked=True) is None
    monkeypatch.setenv("FIRA_CLIP_NORM", "0.5")
    assert run_model.clip_settings(engine_checked=True) == 0.5
    monkeypatch.setenv("FIRA_CLIP_NORM", "inf")
    assert run_model.clip_settings() == float("inf")
    for bad in ("0", "-2", "nan", "-inf", "1e", "none"):
        monkeypatch.setenv("FIRA_CLIP_NORM", bad)
        with pytest.raises(SystemExit, match="FIRA_CLIP_NORM must be a positive number or inf"):
            run_model.clip_settings()
    monkeypatch.setenv("FIRA_CLIP_NORM", "inf")
    monkeypatch.setenv("FIRA_ENGINE", "eager")
    assert run_model.clip_settings() == float("inf")                  # finetune / distill do not use the engine
    with pytest.raises(SystemExit, match="FIRA_ENGINE=eager"):
        run_model.clip_settings(engine_checked=True)


def test_clip_log_fields():
    """the progress line's fields: the window's mean norm and the group's counters, then a fresh window"""
    import run_model

    class Group:
        state = torch.tensor([0.0, 1.0, 1.0, 3.0, 1.0], dtype=torch.float64)
        grad_norm, clipped, skipped = state[0], state[3], state[4]

    grp = Group()
    log = run_model.ClipLog(lambda: None)
    log.add()
    assert log.text() == ""                                           # no group yet: no fields
    log = run_model.ClipLog(lambda: grp)
    for x in (1.0, 2.0, 6.0):
        grp.state[0] = x
        log.add()
    assert log.text() == " grad_norm: 3.0000 clipped: 3 skipped: 1"
    grp.state[0] = 5.0
    log.add()
    assert log.text() == " grad_norm: 5.0000 clipped: 3 skipped: 1"
