"""The exponential moving average of the weights without a GPU: the float64 rule of fira_adam_flat + EMA (ema_rule.py)
against torch.optim.Adam in float64 with a hand-rolled EMA, the C prototype, optim.check_ema_decay, TransModel's
constructor arguments, and the FIRA_EMA errors of `run_model.py train`, raised before any device work."""
import copy
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

import ema_rule
from fira_testlib import ROOT, reference_args


def _tensors(seed, shapes=((64, 32), (32,), (7,), (1,))):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(s, generator=g, dtype=torch.float64) for s in shapes]


@pytest.mark.parametrize("grad_scale", [None, 37.0])
@pytest.mark.parametrize("d", [0.9, 0.999])
def test_rule_matches_torch_adam_and_ema_in_float64(d, grad_scale):
    """torch.optim.Adam on float64 parameters, then e = d e + (1 - d) p by hand, against ema_rule.adam_ema fed the
    same fp32-representable constants"""
    lr, b1, b2, eps = 2.0 ** -10, 0.875, 0.9990234375, 2.0 ** -27       # exact in fp32: the rule rounds nothing
    ps = [torch.nn.Parameter(t) for t in _tensors(0)]
    opt = torch.optim.Adam(ps, lr=lr, betas=(b1, b2), eps=eps)
    dd, c = ema_rule.ema_coefficients(d)
    ema = [p.detach().clone() for p in ps]
    mine = [dict(p=p.detach().numpy().copy(), m=np.zeros(p.shape), v=np.zeros(p.shape), e=p.detach().numpy().copy())
            for p in ps]
    gen = torch.Generator().manual_seed(1)
    for t in range(1, 13):
        grads = [torch.randn(p.shape, generator=gen, dtype=torch.float64) * 10.0 ** (t % 4 - 2) for p in ps]
        for p, gr in zip(ps, grads):
            p.grad = gr / grad_scale if grad_scale else gr.clone()
        opt.step()
        with torch.no_grad():
            for e, p in zip(ema, ps):
                e.mul_(dd).add_(p.detach() * c)
        for s, gr in zip(mine, grads):
            s["p"], s["m"], s["v"], s["e"] = ema_rule.adam_ema(s["p"], gr.numpy(), s["m"], s["v"], s["e"], t, lr, b1,
                                                              b2, eps, d, grad_scale)
    for p, e, s in zip(ps, ema, mine):
        np.testing.assert_allclose(s["p"], p.detach().numpy(), rtol=1e-12, atol=1e-14)
        # the rule rounds c p to fp32 as the kernel does: a relative 2^-24 of c p per step
        np.testing.assert_allclose(s["e"], e.numpy(), rtol=0, atol=12 * 2.0 ** -24 * c * (np.abs(s["p"]).max() + 1))


def test_rule_ema_is_the_kernel_order():
    """e = d e + fl32(c p) with c = fl32(1 - d): a fixed point stays put, and the coefficients are the fp32 ones"""
    d, c = ema_rule.ema_coefficients(0.999)
    assert d == np.float64(np.float32(0.999)) and c == np.float64(np.float32(1.0) - np.float32(0.999))
    p = np.array([0.0, 1.0, -3.5, 2.0 ** -20])
    np.testing.assert_allclose(ema_rule.ema(p, p, 0.999), p, rtol=2.0 ** -23)
    assert np.all(ema_rule.ema(np.zeros(4), p, 0.5) == 0.5 * p)


def test_adam_flat_prototype_takes_the_ema_buffer():
    from fira_icse_b200 import _lib
    _, types, names = _lib.parse_header()["fira_adam_flat"]
    assert names[-3:] == ["ema", "ema_decay", "stream"]
    assert types[-3] is not None and types[-2].__name__ == "c_float"


@pytest.mark.parametrize("bad", [0, 1, 1.5, -0.1, float("nan"), float("inf"), "x", None])
def test_check_ema_decay_refuses(bad):
    from fira_icse_b200.optim import check_ema_decay
    with pytest.raises(ValueError, match="ema_decay"):
        check_ema_decay(bad)


def test_check_ema_decay_accepts():
    from fira_icse_b200.optim import check_ema_decay
    assert check_ema_decay("0.999") == 0.999 and check_ema_decay(0.5) == 0.5


def test_transmodel_keeps_its_arguments_outside_the_state_dict():
    from fira_icse_b200 import TransModel
    from fira_icse_b200.optim import ema_model
    m = TransModel(reference_args(vocab_size=50))
    assert m.args.vocab_size == 50 and m.args.embedding_dim == 256
    assert len(m.state_dict()) == 338 and not any("args" in k for k in m.state_dict())
    assert copy.deepcopy(m).args == m.args and pickle.loads(pickle.dumps(m.args)) == m.args
    with pytest.raises(ValueError, match="no optimizer with an EMA"):
        ema_model(m, [])                                      # a CPU model's parameters belong to no FlatAdam


def test_transmodel_arguments_set_as_attributes_win():
    """run_model.py's DotDict: load_globals sets vocab_size by attribute assignment, which leaves the key at 0"""
    import run_model
    from fira_icse_b200 import TransModel
    args = run_model.DotDict(reference_args(vocab_size=0))
    args.vocab_size = 50
    m = TransModel(args)
    assert m.args.vocab_size == 50 and m.args.ast_change_vocab_size == 71
    assert TransModel(m.args).out_fc.weight.shape == (50, 256)


# ------------------------------------------------------------------ run_model.py train
def _train(tmp_path, **env):
    e = dict(os.environ, PYTHONPATH=ROOT, **env)
    return subprocess.run([sys.executable, os.path.join(ROOT, "run_model.py"), "train"], cwd=tmp_path, env=e,
                          capture_output=True, text=True, timeout=300)


@pytest.mark.parametrize("env,match", [
    (dict(FIRA_EMA="0"), "FIRA_EMA must be a number in (0, 1)"),
    (dict(FIRA_EMA="1"), "FIRA_EMA must be a number in (0, 1)"),
    (dict(FIRA_EMA="-0.5"), "FIRA_EMA must be a number in (0, 1)"),
    (dict(FIRA_EMA="nan"), "FIRA_EMA must be a number in (0, 1)"),
    (dict(FIRA_EMA="inf"), "FIRA_EMA must be a number in (0, 1)"),
    (dict(FIRA_EMA="fast"), "FIRA_EMA must be a number in (0, 1)"),
    (dict(FIRA_EMA="0.999", FIRA_ENGINE="eager"), "FIRA_ENGINE=eager"),
])
def test_train_ema_argument_errors(tmp_path, env, match):
    """the setting is refused before the device, the data or the model are touched: no CUDA-device message, no
    missing-DataSet error, no file written"""
    r = _train(tmp_path, **env)
    assert r.returncode != 0
    assert match in r.stderr, r.stderr[-2000:]
    assert "no CUDA device" not in r.stderr and "DataSet" not in r.stderr
    assert not os.path.exists(tmp_path / "best_model.pt") and not os.path.exists(tmp_path / "best_model_ema.pt")


def test_ema_settings(monkeypatch):
    import run_model
    monkeypatch.delenv("FIRA_EMA", raising=False)
    monkeypatch.delenv("FIRA_ENGINE", raising=False)
    assert run_model.ema_settings() is None
    monkeypatch.setenv("FIRA_EMA", "0.995")
    assert run_model.ema_settings() == 0.995
    monkeypatch.setenv("FIRA_ENGINE", "graph")
    assert run_model.ema_settings() == 0.995
