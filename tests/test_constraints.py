"""n-gram repeat blocking and minimum length without a device: the restated rule (tests/constraint_rule.py) on
hand-worked histories, every decode_loop.check_rules error (raised before any device work), and run_model.py's
refusal of the rules for the reference beam search."""
import numpy as np
import pytest

from constraint_rule import allowed, banned, repeats_ngram

EOS = 2


@pytest.mark.parametrize("words,n,want", [
    ([5, 6, 5], 2, {6}),
    ([5, 6, 7, 5, 6], 3, {7}),
    ([5, 6, 7, 5, 6], 2, {7}),            # "6 7" is the only bigram starting with the last word
    ([5, 6, 7, 5, 6], 1, {5, 6, 7}),      # n = 1: every earlier word
    ([5, 6, 5], 1, {5, 6}),
    ([5, 6, 5], 4, set()),                # n longer than the history
    ([5, 6, 5], 3, set()),                # "6 5" never occurred before
    ([], 1, set()),
    ([5, 5, 5], 2, {5}),
])
def test_ngram_rule(words, n, want):
    assert banned(words, n, 0, EOS, len(words) + 1) == want


def test_min_length_rule():
    words = [5, 6, 7]                                       # length - 1 = 3 words
    assert banned(words, 0, 4, EOS, len(words) + 1) == {EOS}    # length - 1 = m - 1: <eos> banned
    assert banned(words, 0, 3, EOS, len(words) + 1) == set()    # length - 1 = m: allowed
    assert banned(words, 0, 0, EOS, len(words) + 1) == set()
    assert banned([5, 6, 5], 2, 4, EOS, 4) == {6, EOS}


def test_a_copy_and_its_word_are_banned_together():
    V = 10
    copy_src = np.array([6, 3, 6, EOS])
    ok = allowed({6, EOS}, V, copy_src, np.array([1, 1, 0, 1]))
    assert ok.tolist() == [True] * 2 + [False] + [True] * 3 + [False] + [True] * 3 + [False, True, False, False]


def test_repeated_ngram_detector():
    assert repeats_ngram([5, 6, 5, 6], 2) and not repeats_ngram([5, 6, 5, 7], 2)
    assert repeats_ngram([5, 5], 1) and not repeats_ngram([5, 5], 1, start=2)
    assert not repeats_ngram([5, 6, 5, 6, 7], 2, start=4) and repeats_ngram([5, 6, 7, 5, 6], 2, start=4)


def _check(n, m, tar_len=30):
    from fira_icse_b200.decode_loop import check_rules
    check_rules(n, m, tar_len)


def test_valid_rules():
    for n, m in ((0, 0), (1, 0), (0, 1), (29, 28), (3, 5)):
        _check(n, m)
    _check(0, 0, tar_len=64)                                # off: any tar_len


@pytest.mark.parametrize("n,m", [(True, 0), (0, False), (2.0, 0), (0, 1.5), ("2", 0), (None, 0), (np.int64(2), 0)])
def test_non_integer_rules(n, m):
    with pytest.raises(ValueError, match="must be an integer >= 0"):
        _check(n, m)


@pytest.mark.parametrize("n,m,name", [(-1, 0, "no_repeat_ngram"), (0, -1, "min_length")])
def test_negative_rules(n, m, name):
    with pytest.raises(ValueError, match=name):
        _check(n, m)


def test_rules_longer_than_the_message():
    with pytest.raises(ValueError, match="no_repeat_ngram must be <= tar_len - 1 = 29"):
        _check(30, 0)
    with pytest.raises(ValueError, match="min_length must be <= tar_len - 2 = 28"):
        _check(0, 29)


def test_rules_need_a_short_history():
    with pytest.raises(ValueError, match="tar_len <= 32"):
        _check(2, 0, tar_len=33)
    with pytest.raises(ValueError, match="tar_len <= 32"):
        _check(0, 3, tar_len=33)


@pytest.mark.parametrize("var", ["FIRA_NO_REPEAT_NGRAM", "FIRA_MIN_LENGTH"])
def test_run_model_beam_rejects_the_rules(monkeypatch, var):
    import run_model
    monkeypatch.setenv(var, "2")
    with pytest.raises(SystemExit, match="FIRA_NO_REPEAT_NGRAM and FIRA_MIN_LENGTH apply to FIRA_DECODE=sample"):
        run_model.decoder("beam", {"<start>": 1, "<eos>": 2, "<pad>": 0})


def test_run_model_tags_the_output_name(monkeypatch):
    import run_model
    vocab = {"<start>": 1, "<eos>": 2, "<pad>": 0}
    monkeypatch.setenv("FIRA_NO_REPEAT_NGRAM", "2")
    monkeypatch.setenv("FIRA_MIN_LENGTH", "3")
    monkeypatch.setenv("FIRA_PREFIX_WORDS", "1")
    assert run_model.decoder("nbest", vocab)[0] == "output_fira_nbest_prefix1_norepeat2_minlen3"
    monkeypatch.setenv("FIRA_PREFIX_WORDS", "0")
    monkeypatch.setenv("FIRA_MIN_LENGTH", "0")
    assert run_model.decoder("sample", vocab)[0] == "output_fira_samples_norepeat2"
    monkeypatch.delenv("FIRA_NO_REPEAT_NGRAM")
    assert run_model.decoder("mbr", vocab)[0] == "output_fira_mbr"
