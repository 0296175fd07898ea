"""`python run_model.py train|test` end to end on a 128-commit DataSet directory (trained once, then decoded with
FIRA_DECODE=beam, sample and nbest), and beam-search id parity against the reference's own test() loop
(tests/golden/beam_first16.npz, beam5_first16.npz)."""
import copy
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from fira_testlib import GOLDEN, ROOT, golden_batch, load_raw_golden, seeded_model
from test_data import _write_dataset

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


@pytest.mark.parametrize("golden", ["beam_first16.npz", "beam5_first16.npz"])      # beam 3 (run_model.py:43), beam 5
@pytest.mark.parametrize("mode", ["full", "graph"])
def test_beam_search_ids_match_reference_test_loop(mode, golden):
    """mode: full decoder re-run per step / KV-cached newest row replayed as CUDA graphs (the first batch runs it
    eagerly and captures it, later batches replay); goldens = outputs of the unmodified reference's test() loop
    (tests/golden/make_golden_beam.py) with beam 3 (the reference default) and beam 5 (BASELINE.json configs[3])"""
    from fira_icse_b200.beam import beam_search, best_sequences
    gold = np.load(os.path.join(GOLDEN, golden))
    raw = load_raw_golden()
    vocab = raw["word_vocab"]
    model = copy.deepcopy(seeded_model()).to(DEV).eval()
    with torch.no_grad():                      # same sharpening as tests/golden/make_golden_beam.py
        k = float(gold["sharpen"])
        model.out_fc.weight *= k; model.out_fc.bias *= k; model.copy_net.LinearRes.weight *= k
    bs = int(gold["batch"])
    for lo in range(0, gold["beam_ids"].shape[0], bs):
        b = golden_batch(lo, lo + bs)
        seq, length, prob = beam_search(model, b[0], b[3], b[4], b[5].to(DEV), b[7], beam_size=int(gold["beam"]),
                                        tar_len=30, start_id=vocab["<start>"], eos_id=vocab["<eos>"],
                                        pad_id=vocab["<pad>"], mode=mode)
        best, blen = best_sequences(seq, length, prob)
        for i in range(bs):
            ref = gold["beam_ids"][lo + i]
            ref = ref[ref >= 0]
            mine = best[i, :blen[i]].cpu().numpy()
            assert np.array_equal(mine, ref), (lo + i, mine, ref)


def _run_model(stage, cwd, env):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "run_model.py"), stage], cwd=cwd, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    return r


@pytest.fixture(scope="module")
def trained(tmp_path_factory):
    """`run_model.py train` once -> (its directory, the environment, the training run)."""
    d = tmp_path_factory.mktemp("cli")
    _write_dataset(str(d), load_raw_golden())
    env = dict(os.environ, PYTHONPATH=ROOT, FIRA_EPOCHS="1", FIRA_BATCH="16", FIRA_MAX_BATCHES="3",
               FIRA_WORKERS="0", FIRA_TEST_BATCH="4")
    return d, env, _run_model("train", d, env)


def _test_lines(trained, name, **env):
    d, base, _ = trained
    r = _run_model("test", d, dict(base, **env))
    assert "mean sentence bleu" in r.stdout
    n_test = len(json.load(open(d / "all_index"))["test"])
    return n_test, open(d / "OUTPUT" / name).read().split("\n")


def test_run_model_train_then_test(trained):
    d, _, r = trained
    assert "loss:" in r.stdout
    sd = torch.load(d / "best_model.pt", map_location="cpu")
    assert len(sd) == 338 and not any(k.startswith("module.") for k in sd)
    n_test, lines = _test_lines(trained, "output_fira")
    assert len(lines) == n_test + 1 and lines[-1] == ""


def test_run_model_test_writes_samples(trained):
    n_test, lines = _test_lines(trained, "output_fira_samples", FIRA_DECODE="sample", FIRA_SAMPLES="3",
                                FIRA_TOP_P="0.95", FIRA_SEED="3")
    assert len(lines) == 3 * n_test + 1 and lines[-1] == ""
    for ln in lines[:-1]:
        lp, _ = ln.split("\t", 1)
        assert float(lp) <= 0.0


def test_run_model_test_writes_nbest(trained):
    n_test, lines = _test_lines(trained, "output_fira_nbest", FIRA_DECODE="nbest", FIRA_BEAM="4",
                                FIRA_LENGTH_PENALTY="0.6")
    assert len(lines) == 4 * n_test + 1 and lines[-1] == ""
    for c in range(n_test):
        fields = [ln.split("\t", 2) for ln in lines[4 * c:4 * c + 4]]
        scores = [float(f[0]) for f in fields]
        assert all(float(f[1]) <= 0.0 for f in fields)
        assert all(x >= y for x, y in zip(scores, scores[1:])), scores
