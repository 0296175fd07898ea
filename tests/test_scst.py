"""Self-critical fine-tuning without a device: the float64 reward rule (tests/scst_rule.py) on hand-made cases, every
ValueError scst_step raises before any device work, and the argument errors of `run_model.py finetune`."""
import os
import subprocess
import sys

import pytest
import torch

from fira_testlib import ROOT, golden_batch, seeded_model
from scst_rule import reference, rewards

START, EOS, PAD = 2, 1, 0


def _row(words, T=8):
    ids = [START] + list(words) + [EOS]
    return ids + [PAD] * (T - len(ids)), len(ids)


def test_sample_equal_to_the_reference_scores_one():
    tar, _ = _row([5, 6, 7, 8, 9])
    a, la = _row([5, 6, 7, 8, 9])
    b, lb = _row([9, 8])
    r, adv = rewards([a, b], [la, lb], tar, START, EOS, PAD)
    assert r[0] == 1.0
    assert adv == [r[0] - r[1], r[1] - r[0]]


def test_empty_sample_scores_zero():
    tar, _ = _row([5, 6, 7])
    empty, le = _row([])                         # <start> <eos>
    only_start = [START] + [PAD] * 7             # no word and no <eos> (length 1)
    r, _ = rewards([empty, only_start], [le, 1], tar, START, EOS, PAD)
    assert r == [0.0, 0.0]


def test_equal_rewards_give_zero_advantages():
    tar, _ = _row([5, 6, 7, 8])
    s, n = _row([5, 6, 3])
    for N in (2, 3, 4, 7, 32):
        r, adv = rewards([s] * N, [n] * N, tar, START, EOS, PAD)
        assert len(set(r)) == 1 and 0.0 < r[0] < 1.0
        assert adv == [0.0] * N


def test_reference_stops_at_its_first_eos_and_drops_markers():
    assert reference([START, 5, PAD, 6, START, EOS, 7, EOS], 8, START, EOS, PAD) == [5, 6]
    assert reference([START, 5, 6, 7], 4, START, EOS, PAD) == [5, 6, 7]          # no <eos> before T
    assert reference([START, 5, 6, 7, 8, EOS], 4, START, EOS, PAD) == [5, 6, 7]   # columns past T are not read


def test_leave_one_out_baseline_sums_in_ascending_order():
    tar, _ = _row([5, 6, 7, 8, 9, 10])
    rows = [_row(w) for w in ([5, 6, 7], [5, 6, 7, 8, 9, 10], [10, 11], [5, 7, 9, 11, 6])]
    r, adv = rewards([x for x, _ in rows], [n for _, n in rows], tar, START, EOS, PAD)
    for n in range(4):
        total = 0.0
        for m in range(4):
            if m != n:
                total += r[n] - r[m]
        assert adv[n] == total / 3
        assert abs(adv[n] - (r[n] - (sum(r) - r[n]) / 3)) <= 1e-15        # r_n minus the mean of the others


# ------------------------------------------------------------------ validation before any device work
def _step(**kw):
    from fira_icse_b200.scst import scst_step
    batch = kw.pop("batch", None) or golden_batch(0, 4)
    args = dict(num_samples=4, temperature=1.0, top_k=0, top_p=1.0, seed=0, first_index=0, no_repeat_ngram=0,
                min_length=0, tar_len=30, start_id=START, eos_id=EOS, pad_id=PAD)
    args.update(kw)
    scst_step(seeded_model(), None, batch, **args)


@pytest.mark.parametrize("kw,match", [
    (dict(num_samples=1), "num_samples"),
    (dict(num_samples=33), "num_samples"),
    (dict(num_samples=4.0), "num_samples"),
    (dict(tar_len=33), "tar_len"),
    (dict(tar_len=1), "tar_len"),
    (dict(temperature=0.0), "temperature"),
    (dict(top_k=-1), "top_k"),
    (dict(top_p=1.5), "top_p"),
    (dict(seed=-1), "seed"),
    (dict(first_index=-1), "first_index"),
    (dict(no_repeat_ngram=-1), "no_repeat_ngram"),
    (dict(min_length=29), "min_length"),
])
def test_bad_settings_raise_before_device_work(kw, match):
    with pytest.raises(ValueError, match=match):
        _step(**kw)


def test_reference_without_eos_raises():
    batch = golden_batch(0, 4)
    tar = batch[1].clone()
    tar[2] = torch.where(tar[2] == EOS, torch.full_like(tar[2], 7), tar[2])
    batch[1] = tar
    with pytest.raises(ValueError, match="<eos>"):
        _step(batch=batch)
    batch = golden_batch(0, 4)
    n = int((batch[1][0] == EOS).nonzero()[0])                 # <eos> just past a shorter tar_len
    with pytest.raises(ValueError, match="<eos>"):
        _step(batch=batch, tar_len=n)


# ------------------------------------------------------------------ run_model.py finetune
def _finetune(tmp_path, **env):
    e = dict(os.environ, PYTHONPATH=ROOT, **env)
    return subprocess.run([sys.executable, os.path.join(ROOT, "run_model.py"), "finetune"], cwd=tmp_path, env=e,
                          capture_output=True, text=True, timeout=300)


@pytest.mark.parametrize("env,match", [
    (dict(WORLD_SIZE="2"), "one GPU"),
    (dict(FIRA_SAMPLES="1"), "num_samples"),
    (dict(FIRA_SAMPLES="33"), "num_samples"),
    (dict(FIRA_SCST_LR="0"), "FIRA_SCST_LR"),
    (dict(FIRA_SCST_EPOCHS="0"), "FIRA_SCST_EPOCHS"),
    (dict(FIRA_TOP_P="1.5"), "top_p"),
    (dict(FIRA_MIN_LENGTH="29"), "min_length"),
    (dict(FIRA_SAMPLES="four"), "invalid literal"),
])
def test_finetune_argument_errors(tmp_path, env, match):
    r = _finetune(tmp_path, **env)
    assert r.returncode != 0
    assert match in r.stderr, r.stderr[-2000:]
    assert not os.path.exists(tmp_path / "best_model_scst.pt")
