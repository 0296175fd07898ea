"""Minimum-Bayes-risk selection on the GPU: fira_mbr_select against the float64 restatement (tests/mbr_rule.py),
fira_icse_b200.mbr end to end on the sharpened golden model, and `run_model.py test` with FIRA_DECODE=mbr."""
import json
import os

import numpy as np
import pytest
import torch

from fira_testlib import golden_batch, load_raw_golden
from mbr_rule import select

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
START, EOS, PAD = 2, 1, 0
TOL = 1e-12


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _kernel(seq, length, T, pairs=True):
    """fira_mbr_select on seq [B, N, ld] / length [B, N] with T_len = T -> (pair BLEU or None, utility, best)"""
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import call
    B, N, ld = seq.shape
    s = seq.to(DEV, torch.int32).contiguous()
    n = length.to(DEV, torch.int32).contiguous()
    pb = torch.full((B, N, N), -1.0, dtype=torch.float64, device=DEV) if pairs else None
    u = torch.full((B, N), -1.0, dtype=torch.float64, device=DEV)
    best = torch.full((B,), -1, dtype=torch.int32, device=DEV)
    call("fira_mbr_select", ops._ptr(s), ops._ptr(n), ld, START, EOS, PAD, ops._ptr(pb), ops._ptr(u), ops._ptr(best),
         B, N, T, ops._stream())
    torch.cuda.synchronize()
    return (pb.cpu().numpy() if pairs else None), u.cpu().numpy(), best.cpu().numpy()


def _candidates(rng, B, N, T, ld):
    """ids over a 5-id vocabulary plus the three markers at random positions; lengths 1 (only <start>) .. T, rows with
    and without <eos>; commits with duplicated and all-identical candidates; columns T..ld-1 hold ids the rule never
    reads."""
    seq = np.full((B, N, ld), PAD, np.int64)
    length = np.zeros((B, N), np.int64)
    pool = np.array([3, 4, 5, 6, 7, 3, 4, 5, 6, 7, 3, 4, PAD, START, EOS])
    for b in range(B):
        for n in range(N):
            L = int(rng.integers(1, T + 1))
            seq[b, n, 0] = START
            seq[b, n, 1:L] = rng.choice(pool, L - 1)
            if L >= 2 and rng.random() < 0.7:
                seq[b, n, L - 1] = EOS
            length[b, n] = L
        if b % 4 == 1:                                  # duplicates
            seq[b, 1::2], length[b, 1::2] = seq[b, 0], length[b, 0]
        if b % 8 == 2:                                  # every candidate the same: all utilities tie
            seq[b], length[b] = seq[b, :1], length[b, :1]
    seq[:, :, T:] = rng.integers(3, 8, (B, N, ld - T))
    return torch.from_numpy(seq), torch.from_numpy(length)


@pytest.mark.parametrize("B", [0, 1, 64])
@pytest.mark.parametrize("N", [2, 5, 32])
def test_kernel_matches_float64_rule(B, N):
    rng = np.random.default_rng(100 * N + B)
    for T, ld in ((32, 32), (30, 33)):
        seq, length = _candidates(rng, B, N, T, ld)
        pb, u, best = _kernel(seq, length, T)
        _, u2, best2 = _kernel(seq, length, T, pairs=False)
        assert np.array_equal(u, u2) and np.array_equal(best, best2)
        for b in range(B):
            ref_pairs, ref_u, _ = select(seq[b, :, :T].tolist(), length[b].tolist(), START, EOS, PAD)
            np.testing.assert_allclose(pb[b], np.array(ref_pairs), rtol=0, atol=TOL)
            np.testing.assert_allclose(u[b], np.array(ref_u), rtol=0, atol=TOL)
            assert ref_u[best[b]] >= max(ref_u) - TOL
            assert best[b] == int(np.flatnonzero(u[b] == u[b].max())[0])
            if b % 8 == 2:
                assert best[b] == 0 and (u[b] == u[b, 0]).all()


# ------------------------------------------------------------------ end to end
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_mbr_picks_the_restated_choice_among_its_samples(precision):
    from fira_icse_b200.mbr import mbr
    from test_gpu_sample import _model
    v = load_raw_golden()["word_vocab"]
    ids = dict(start_id=v["<start>"], eos_id=v["<eos>"], pad_id=v["<pad>"])
    m = _model(precision)
    b = golden_batch(0, 8)
    out = mbr(m, b[0], b[3], b[4], b[5].to(DEV), b[7], num_samples=6, top_p=0.95, seed=4, **ids)
    s = out.samples
    B, N, T = s.seq.shape
    assert out.seq.shape == (B, T) and out.utility.shape == (B, N) and out.utility.dtype == torch.float64
    rows = torch.arange(B, device=out.index.device)
    assert torch.equal(out.seq, s.seq[rows, out.index]) and torch.equal(out.length, s.length[rows, out.index])
    assert torch.equal(out.logprob, s.logprob[rows, out.index])
    seq, length, u, index = s.seq.cpu(), s.length.cpu(), out.utility.cpu().numpy(), out.index.cpu().numpy()
    for c in range(B):
        _, ref_u, _ = select(seq[c].tolist(), length[c].tolist(), ids["start_id"], ids["eos_id"], ids["pad_id"])
        np.testing.assert_allclose(u[c], np.array(ref_u), rtol=0, atol=TOL)
        assert index[c] == int(np.flatnonzero(u[c] == u[c].max())[0])


# ------------------------------------------------------------------ CLI
@pytest.fixture(scope="module")
def trained(tmp_path_factory):
    """`run_model.py train` once -> (its directory, the environment)."""
    from fira_testlib import ROOT
    from test_data import _write_dataset
    from test_gpu_cli import _run_model
    d = tmp_path_factory.mktemp("cli_mbr")
    _write_dataset(str(d), load_raw_golden())
    env = dict(os.environ, PYTHONPATH=ROOT, FIRA_EPOCHS="1", FIRA_BATCH="16", FIRA_MAX_BATCHES="3",
               FIRA_WORKERS="0", FIRA_TEST_BATCH="4")
    _run_model("train", d, env)
    return d, env


def test_run_model_test_writes_mbr_choices(trained):
    from test_gpu_cli import _run_model
    d, env = trained
    r = _run_model("test", d, dict(env, FIRA_DECODE="mbr", FIRA_SAMPLES="4"))
    assert "mean sentence bleu" in r.stdout
    n_test = len(json.load(open(d / "all_index"))["test"])
    lines = open(d / "OUTPUT" / "output_fira_mbr").read().split("\n")
    assert len(lines) == n_test + 1 and lines[-1] == ""
    for ln in lines[:-1]:
        u, lp, _ = ln.split("\t", 2)
        assert 0.0 <= float(u) <= 1.0 and float(lp) <= 0.0
