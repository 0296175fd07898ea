"""Ensemble decoding on the host: the float64 rewrite of fira_pointer_mix_ensemble (tests/ensemble_rule.py) reproduces
the weighted average of the members' mixtures, every Ensemble argument error (raised before any device work), and
run_model.py's FIRA_ENSEMBLE settings."""
import copy

import numpy as np
import pytest
import torch

from ensemble_rule import average, rewrite
from fira_testlib import reference_args
from sample_rule import mixture


def _rows(rng, M, V, S, saturated=()):
    rows = []
    for m in range(M):
        x = rng.normal(0, 3, V)
        c = rng.normal(0, 2, S)
        gl = rng.normal(0, 1, 2)
        if m in saturated:                     # g0 = 0 exactly in float64: every word of this member has P = 0
            gl = np.array([-1e4, 0.0])
        rows.append((x, c, gl))
    return rows


def _mask(rng, S):
    mk = (rng.random(S) > 0.3).astype(np.uint8)
    mk[0] = 1
    return mk


@pytest.mark.parametrize("M,weights,saturated", [
    (1, [1.0], ()),
    (2, [0.5, 0.5], ()),
    (3, [0.2, 0.3, 0.5], ()),
    (4, [0.1, 0.2, 0.3, 0.4], (1,)),            # one member's gate saturated to the copy side
    (3, [0.6, 0.3, 0.1], (0, 1, 2)),            # every member saturated: G0 = 0
    (8, [1 / 8] * 8, (2, 5)),
])
@pytest.mark.parametrize("V,S", [(61, 13), (24650, 370)])
def test_rewrite_reproduces_the_weighted_average(M, weights, saturated, V, S):
    rng = np.random.default_rng(V + S + 17 * M + len(saturated))
    for _ in range(3):
        rows = _rows(rng, M, V, S, saturated)
        mk = _mask(rng, S)
        x, c, gl = rewrite(rows, weights, mk)
        assert np.isfinite(x).all() and np.isfinite(c).all()
        assert (c[mk == 0] == -1e9).all()
        got = mixture(x, c, gl, mk)
        ref = average(rows, weights, mk, mixture)
        np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-300)
        assert abs(got.sum() - 1.0) < 1e-12
        if len(saturated) == M:
            assert gl[0] == -np.inf and (got[:V] == 0).all()


def test_rewrite_of_one_member_is_its_own_mixture():
    rng = np.random.default_rng(3)
    (row,) = _rows(rng, 1, 61, 13)
    mk = _mask(rng, 13)
    np.testing.assert_allclose(mixture(*rewrite([row], [1.0], mk), mk), mixture(*row, mk), rtol=1e-12, atol=1e-300)


def test_rewrite_stays_finite_where_every_member_underflows():
    rng = np.random.default_rng(5)
    rows = _rows(rng, 2, 61, 13)
    for x, _, _ in rows:
        x[7] = x.max() - 900.0                  # exp underflows to 0 in float64 for both members
    mk = _mask(rng, 13)
    x, _, _ = rewrite(rows, [0.5, 0.5], mk)
    assert np.isfinite(x[7]) and x[7] < -800


# ------------------------------------------------------------------ Ensemble arguments
_SMALL = {}


def _small(vocab_size=61, precision="fp32"):
    """a CPU TransModel with a small vocabulary"""
    key = (vocab_size, precision)
    if key not in _SMALL:
        from fira_icse_b200 import TransModel
        torch.manual_seed(0)
        _SMALL[key] = TransModel(reference_args(vocab_size=vocab_size)).set_precision(precision)
    return _SMALL[key]


@pytest.mark.parametrize("models,weights,exc,match", [
    (lambda: [], None, ValueError, "1 to 8 models"),
    (lambda: [_small()] * 9, None, ValueError, "1 to 8 models"),
    (lambda: _small(), None, TypeError, "list or tuple"),
    (lambda: [_small(), "model"], None, TypeError, "member 1 is a str"),
    (lambda: [_small(), _small()], [1.0], ValueError, "2 models need 2 weights"),
    (lambda: [_small(), _small()], [1.0, 0.0], ValueError, "positive and finite"),
    (lambda: [_small(), _small()], [1.0, -2.0], ValueError, "positive and finite"),
    (lambda: [_small(), _small()], [1.0, float("inf")], ValueError, "positive and finite"),
    (lambda: [_small(), _small()], [1.0, float("nan")], ValueError, "positive and finite"),
    (lambda: [_small(), _small()], [1.0, "2"], TypeError, "numbers"),
    (lambda: [_small(), _small()], [True, 1.0], TypeError, "numbers"),
    (lambda: [_small(), _small()], "12", TypeError, "sequence"),
    (lambda: [_small(), _small(precision="bf16")], None, ValueError, "precision"),
    (lambda: [_small(), _small(vocab_size=69)], None, ValueError, "vocab_size"),
    (lambda: [_small(), _small()], None, ValueError, "CUDA device"),
])
def test_ensemble_arguments_are_checked_on_the_host(models, weights, exc, match):
    from fira_icse_b200.ensemble import Ensemble
    with pytest.raises(exc, match=match):
        Ensemble(models(), weights)


def test_ensemble_refuses_members_on_different_devices():
    from fira_icse_b200.ensemble import Ensemble
    meta = copy.deepcopy(_small()).to("meta")
    with pytest.raises(ValueError, match="member 1 is on meta"):
        Ensemble([_small(), meta])


def test_beam_search_and_scst_refuse_an_ensemble():
    from fira_icse_b200.beam import beam_search
    from fira_icse_b200.ensemble import Ensemble
    from fira_icse_b200.scst import scst_step
    ens = Ensemble.__new__(Ensemble)             # the refusal comes before anything reads the members
    with pytest.raises(TypeError, match="beam_search takes a single model"):
        beam_search(ens, None, None, None, None, None, start_id=1, eos_id=2)
    with pytest.raises(TypeError, match="scst_step takes a single model"):
        scst_step(ens, None, None, num_samples=2, start_id=1, eos_id=2)


# ------------------------------------------------------------------ run_model.py test
VOCAB = {"<start>": 1, "<eos>": 2, "<pad>": 0}


@pytest.fixture
def ckpts(tmp_path, monkeypatch):
    for n in ("a.pt", "b.pt", "c.pt"):
        (tmp_path / n).write_bytes(b"")
    monkeypatch.chdir(tmp_path)
    for v in ("FIRA_CHECKPOINT", "FIRA_ENSEMBLE", "FIRA_ENSEMBLE_WEIGHTS", "FIRA_NO_REPEAT_NGRAM", "FIRA_MIN_LENGTH",
              "FIRA_PREFIX_WORDS"):
        monkeypatch.delenv(v, raising=False)
    return monkeypatch


@pytest.mark.parametrize("env,mode,match", [
    (dict(FIRA_ENSEMBLE="a.pt,b.pt"), "beam", "FIRA_ENSEMBLE applies to FIRA_DECODE=sample, nbest and mbr"),
    (dict(FIRA_ENSEMBLE="a.pt,b.pt", FIRA_CHECKPOINT="a.pt"), "nbest", "unset FIRA_CHECKPOINT"),
    (dict(FIRA_ENSEMBLE="a.pt,b.pt", FIRA_ENSEMBLE_WEIGHTS="1"), "sample", "1 weights for 2 checkpoints"),
    (dict(FIRA_ENSEMBLE="a.pt,b.pt", FIRA_ENSEMBLE_WEIGHTS="1,0"), "mbr", "positive finite"),
    (dict(FIRA_ENSEMBLE="a.pt,b.pt", FIRA_ENSEMBLE_WEIGHTS="1,-3"), "nbest", "positive finite"),
    (dict(FIRA_ENSEMBLE="a.pt,b.pt", FIRA_ENSEMBLE_WEIGHTS="1,x"), "nbest", "numbers separated by commas"),
    (dict(FIRA_ENSEMBLE="a.pt,missing.pt"), "nbest", "checkpoint missing.pt not found"),
    (dict(FIRA_ENSEMBLE="a.pt,,b.pt"), "nbest", "1 to 8 checkpoints"),
    (dict(FIRA_ENSEMBLE=",".join(["a.pt"] * 9)), "nbest", "1 to 8 checkpoints"),
    (dict(FIRA_ENSEMBLE_WEIGHTS="1,2"), "nbest", "FIRA_ENSEMBLE_WEIGHTS needs FIRA_ENSEMBLE"),
])
def test_run_model_ensemble_settings_refuse(ckpts, env, mode, match):
    import run_model
    for k, v in env.items():
        ckpts.setenv(k, v)
    with pytest.raises(SystemExit, match=match):
        run_model.ensemble_settings(mode)


def test_run_model_ensemble_settings_and_output_tag(ckpts):
    import run_model
    assert run_model.ensemble_settings("nbest") is None
    assert run_model.decoder("nbest", VOCAB)[0] == "output_fira_nbest"
    ckpts.setenv("FIRA_ENSEMBLE", "a.pt, b.pt")
    assert run_model.ensemble_settings("sample") == (["a.pt", "b.pt"], None)
    assert run_model.decoder("nbest", VOCAB)[0] == "output_fira_nbest_ens2"
    ckpts.setenv("FIRA_NO_REPEAT_NGRAM", "2")
    assert run_model.decoder("nbest", VOCAB)[0] == "output_fira_nbest_norepeat2_ens2"
    ckpts.delenv("FIRA_NO_REPEAT_NGRAM")
    ckpts.setenv("FIRA_ENSEMBLE", "a.pt,b.pt,c.pt")
    ckpts.setenv("FIRA_ENSEMBLE_WEIGHTS", "1,2,0.5")
    assert run_model.ensemble_settings("mbr") == (["a.pt", "b.pt", "c.pt"], [1.0, 2.0, 0.5])
    assert run_model.decoder("mbr", VOCAB)[0] == "output_fira_mbr_ens3"
    assert run_model.decoder("sample", VOCAB)[0] == "output_fira_samples_ens3"
    with pytest.raises(SystemExit, match="FIRA_ENSEMBLE applies"):
        run_model.decoder("beam", VOCAB)
