"""Nearest-neighbour decoding without a GPU: the float64 rule's own properties (tests/knn_rule.py), the host-side
validation of Datastore, KNNModel and the settings, the save / load round trip with the fingerprint, and the
`run_model.py test` FIRA_KNN errors, raised before any device work."""
import numpy as np
import pytest
import torch

from fira_testlib import reference_args
from knn_rule import distances, mix, neighbour_q, search


def _store(N=10, V=50, **kw):
    from fira_icse_b200.knn import Datastore
    keys = torch.randn((N, 256)).to(torch.bfloat16)
    a = dict(keys=keys, norms=keys.float().square().sum(1), words=torch.arange(N, dtype=torch.int32) % V,
             source=torch.zeros((N, 2), dtype=torch.int32))
    a.update(kw)
    return Datastore(a["keys"], a["norms"], a["words"], a["source"], vocab_size=V, precision="fp32", fingerprint="f")


def test_rule_q_sums_to_one_and_aggregates_repeated_words():
    q = neighbour_q([4, 2, 4, 9], [1.0, 1.5, 3.0, 7.0], 2.0, 12)
    assert q.sum() == pytest.approx(1.0)
    e = np.exp(-np.array([0.0, 0.5, 2.0, 6.0]) / 2.0)
    assert q[4] == pytest.approx((e[0] + e[2]) / e.sum())
    assert q[2] == pytest.approx(e[1] / e.sum()) and q[0] == 0.0
    one = neighbour_q([3, 3, 3], [0.0, 5.0, 9.0], 1e-3, 5)
    assert one[3] == pytest.approx(1.0)


def test_rule_mixture_keeps_copy_labels_without_neighbour_mass():
    P = np.array([0.2, 0.3, 0.1, 0.4])            # V = 2 vocabulary labels, 2 copy labels
    q = np.array([0.0, 1.0])
    out = mix(P, q, 0.25, 2)
    assert out.sum() == pytest.approx(1.0)
    assert np.allclose(out, [0.15, 0.475, 0.075, 0.3])


def test_rule_search_breaks_ties_by_index():
    keys = np.random.default_rng(0).standard_normal((20, 256)).astype(np.float32)
    keys[11] = keys[4]
    keys[17] = keys[4]
    q = keys[4:5] + 1e-3
    idx, d = search(q, keys, 3)
    assert idx[0].tolist() == [4, 11, 17] and d[0, 0] == d[0, 1] == d[0, 2]
    assert np.all(np.diff(distances(q, keys)[0][idx[0]]) >= 0)


@pytest.mark.parametrize("change,match", [
    (dict(keys=torch.zeros((10, 128), dtype=torch.bfloat16)), "shape"),
    (dict(keys=torch.zeros((10, 256))), "bfloat16"),
    (dict(norms=torch.zeros(10, dtype=torch.float64)), "float32"),
    (dict(words=torch.zeros(10, dtype=torch.int64)), "int32"),
    (dict(words=torch.full((10,), 50, dtype=torch.int32)), "vocabulary ids"),
    (dict(source=torch.zeros((10, 3), dtype=torch.int32)), "source"),
    (dict(norms=torch.zeros(9)), r"\[N = 10\]"),
])
def test_datastore_validation(change, match):
    with pytest.raises(ValueError, match=match):
        _store(**change)


def test_datastore_save_load_round_trip(tmp_path):
    from fira_icse_b200.knn import Datastore
    st = _store()
    p = tmp_path / "ds.pt"
    st.save(p)
    back = Datastore.load(p, "cpu")
    for k in ("keys", "norms", "words", "source"):
        assert torch.equal(getattr(back, k), getattr(st, k))
    assert (back.vocab_size, back.precision, back.fingerprint) == (50, "fp32", "f")
    with pytest.raises(ValueError, match="vocab_size"):
        Datastore.load(p, "cpu", vocab_size=51)
    with pytest.raises(ValueError, match="built in fp32"):
        Datastore.load(p, "cpu", precision="bf16")
    torch.save({"format": "other"}, tmp_path / "x.pt")
    with pytest.raises(ValueError, match="not a kNN datastore"):
        Datastore.load(tmp_path / "x.pt", "cpu")


@pytest.mark.parametrize("k,tau,lam,match", [
    (0, 10.0, 0.25, "k must be"), (65, 10.0, 0.25, "k must be"), (True, 10.0, 0.25, "k must be"),
    (8, 0.0, 0.25, "temperature"), (8, float("inf"), 0.25, "temperature"), (8, float("nan"), 0.25, "temperature"),
    (8, 10.0, 0.0, "lam"), (8, 10.0, 1.0, "lam"), (8, 10.0, -0.1, "lam"),
])
def test_settings_refused(k, tau, lam, match):
    from fira_icse_b200.knn import check_settings
    with pytest.raises(ValueError, match=match):
        check_settings(k, tau, lam)


def test_knn_model_host_checks():
    import fira_icse_b200 as F
    from fira_icse_b200.ensemble import Ensemble
    from fira_icse_b200.knn import KNNModel, fingerprint, state_fingerprint
    torch.manual_seed(0)
    m = F.TransModel(reference_args(vocab_size=50))
    assert fingerprint(m) == state_fingerprint(m.state_dict()) == fingerprint(m)
    with pytest.raises(TypeError, match="Datastore"):
        KNNModel(m, object())
    with pytest.raises(TypeError, match="TransModel"):
        KNNModel("model", _store())
    with pytest.raises(ValueError, match="exceeds the datastore"):
        KNNModel(m, _store(N=4), k=8)
    with pytest.raises(ValueError, match="CUDA device"):           # a CPU model: checked before any device work
        KNNModel(m, _store())
    # an Ensemble is refused before its own device check
    with pytest.raises((TypeError, ValueError)):
        KNNModel(Ensemble([m]), _store())


def test_fingerprint_follows_the_weights():
    import fira_icse_b200 as F
    from fira_icse_b200.knn import state_fingerprint
    torch.manual_seed(0)
    m = F.TransModel(reference_args(vocab_size=50))
    a = state_fingerprint(m.state_dict())
    with torch.no_grad():
        m.out_fc.bias[0] += 1.0
    assert state_fingerprint(m.state_dict()) != a


def test_single_model_entry_points_refuse_a_knn_model():
    from fira_icse_b200.ensemble import refuse
    from fira_icse_b200.knn import KNNModel
    km = KNNModel.__new__(KNNModel)
    for what in ("beam_search", "scst_step", "distill_step"):
        with pytest.raises(TypeError, match=f"{what} takes a single model; a KNNModel"):
            refuse(km, what)


@pytest.fixture
def knn_env(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    for v in ("FIRA_CHECKPOINT", "FIRA_ENSEMBLE", "FIRA_ENSEMBLE_WEIGHTS", "FIRA_KNN", "FIRA_KNN_K",
              "FIRA_KNN_TEMPERATURE", "FIRA_KNN_LAMBDA", "FIRA_PRECISION"):
        monkeypatch.delenv(v, raising=False)
    import fira_icse_b200 as F
    from fira_icse_b200.knn import state_fingerprint
    torch.manual_seed(0)
    m = F.TransModel(reference_args(vocab_size=50))
    torch.save(m.state_dict(), tmp_path / "best_model.pt")
    st = _store()
    st.fingerprint = state_fingerprint(m.state_dict())
    st.save(tmp_path / "datastore.pt")
    _store().save(tmp_path / "other.pt")
    return monkeypatch


@pytest.mark.parametrize("env,mode,match", [
    (dict(FIRA_KNN="datastore.pt"), "beam", "FIRA_KNN applies to FIRA_DECODE=sample, nbest and mbr"),
    (dict(FIRA_KNN="datastore.pt", FIRA_ENSEMBLE="best_model.pt"), "sample", "unset FIRA_ENSEMBLE"),
    (dict(FIRA_KNN="datastore.pt", FIRA_KNN_K="0"), "nbest", "k must be"),
    (dict(FIRA_KNN="datastore.pt", FIRA_KNN_K="11"), "nbest", "exceeds the datastore"),
    (dict(FIRA_KNN="datastore.pt", FIRA_KNN_LAMBDA="1"), "mbr", "lam must be"),
    (dict(FIRA_KNN="datastore.pt", FIRA_KNN_TEMPERATURE="-1"), "sample", "temperature"),
    (dict(FIRA_KNN="missing.pt"), "sample", "missing.pt not found"),
    (dict(FIRA_KNN="datastore.pt", FIRA_PRECISION="bf16"), "sample", "built in fp32"),
    (dict(FIRA_KNN="other.pt"), "sample", "fingerprint mismatch"),
])
def test_run_model_knn_settings_refuse(knn_env, env, mode, match):
    import run_model
    for k, v in env.items():
        knn_env.setenv(k, v)
    with pytest.raises(SystemExit, match=match):
        run_model.knn_settings(mode, None if "FIRA_ENSEMBLE" not in env else (["best_model.pt"], None))


def test_run_model_knn_settings_and_output_tag(knn_env):
    import run_model
    vocab = {"<start>": 1, "<eos>": 2, "<pad>": 0}
    assert run_model.knn_settings("sample", None) is None
    knn_env.setenv("FIRA_KNN", "datastore.pt")
    knn_env.setenv("FIRA_KNN_K", "4")
    s = run_model.knn_settings("sample", None)
    assert s.pop("store").N == 10 and s == dict(path="datastore.pt", k=4, temperature=10.0, lam=0.25)
    assert run_model.decoder("sample", vocab)[0] == "output_fira_samples_knn4"
    knn_env.setenv("FIRA_NO_REPEAT_NGRAM", "2")
    assert run_model.decoder("nbest", vocab)[0] == "output_fira_nbest_norepeat2_knn4"
