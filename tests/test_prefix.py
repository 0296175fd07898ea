"""Prefix-constrained decoding without a device: the prefix validation of decode_loop.check_prefix and
sample.score_prefix (every error raised before any device work, on CPU tensors), and data.prefix_labels against
build_commit's tar_label on the golden raw commits."""
import numpy as np
import pytest
import torch

from fira_testlib import load_raw_golden

V, T, EOS, PAD = 50, 8, 2, 0


def _mem(B=2, n_sou=6, n_sub=4):
    """sou [B, 6] with positions 0..3 real, sub_token [B, 4] with positions 0..1 real (memory S = 10)"""
    sou = torch.zeros((B, n_sou), dtype=torch.int64)
    sou[:, :4] = torch.tensor([1, 7, 8, 9])
    sub = torch.zeros((B, n_sub), dtype=torch.int64)
    sub[:, :2] = torch.tensor([11, 12])
    return sou, sub


def _check(prefix, eos_last=True, pad_id=PAD, B=2):
    from fira_icse_b200.decode_loop import check_prefix
    sou, sub = _mem(B)
    return check_prefix(prefix, sou, sub, V=V, tar_len=T, eos_id=EOS, pad_id=pad_id, eos_last=eos_last)


def test_none_is_no_prefix():
    assert _check(None) is None


@pytest.mark.parametrize("eos_last", [True, False])
def test_valid_prefix_is_padded_to_tar_len(eos_last):
    pre = torch.tensor([[5, V + 1, V + 6, 0], [0, 0, 0, 0]], dtype=torch.int64)   # vocabulary, diff copy, sub copy
    out, n = _check(pre, eos_last)
    assert out.dtype == torch.int32 and out.shape == (2, T) and out.device.type == "cpu"
    assert out[0, :3].tolist() == [5, V + 1, V + 6] and (out[0, 3:] == 0).all() and (out[1] == 0).all()
    assert n.tolist() == [3, 0] and n.dtype == torch.int32
    out, n = _check(torch.tensor([[4, EOS], [3, 0]], dtype=torch.int32))                # <eos> last: sample / mbr
    assert n.tolist() == [2, 1]
    out, n = _check(torch.zeros((2, 0), dtype=torch.int64))                               # P = 0
    assert n.tolist() == [0, 0]


@pytest.mark.parametrize("bad", [torch.ones((2, 2)), torch.ones((2, 2), dtype=torch.bool), [[1, 2], [3, 4]],
                                 np.ones((2, 2), dtype=np.int64)])
def test_non_integer_prefix(bad):
    with pytest.raises(ValueError, match="integer tensor"):
        _check(bad)


@pytest.mark.parametrize("shape", [(3, 2), (1, 2), (2,), (2, 2, 1)])
def test_wrong_batch(shape):
    with pytest.raises(ValueError, match="shape"):
        _check(torch.ones(shape, dtype=torch.int64))


def test_nonzero_after_zero():
    with pytest.raises(ValueError, match="follows a 0"):
        _check(torch.tensor([[5, 0, 6], [5, 6, 7]]))


@pytest.mark.parametrize("j", [-1, V + 10, V + 11, 10 ** 6])
def test_label_out_of_range(j):
    with pytest.raises(ValueError, match=r"\[0, V \+ S"):
        _check(torch.tensor([[5, j], [5, 6]]))


@pytest.mark.parametrize("s", [4, 5, 8, 9])       # diff padding (sou == pad) and sub-token padding (sub_token == 0)
def test_copy_label_at_a_masked_memory_position(s):
    with pytest.raises(ValueError, match="masked memory position"):
        _check(torch.tensor([[5, V + s], [5, 6]]))


def test_pad_label():
    with pytest.raises(ValueError, match="pad_id"):
        _check(torch.tensor([[5, 3], [5, 6]]), pad_id=3)


def test_eos_rules_differ_by_decoder():
    with pytest.raises(ValueError, match="last prefix label"):
        _check(torch.tensor([[EOS, 5], [5, 6]]), eos_last=True)
    with pytest.raises(ValueError, match="cannot contain <eos>"):
        _check(torch.tensor([[5, EOS], [5, 6]]), eos_last=False)


def test_longest_prefix_differs_by_decoder():
    full = torch.full((2, T - 1), 5, dtype=torch.int64)                 # tar_len - 1 labels
    _check(full, eos_last=True)
    with pytest.raises(ValueError, match="at most 6"):
        _check(full, eos_last=False)
    _check(full[:, :T - 2], eos_last=False)
    with pytest.raises(ValueError, match="at most 7"):
        _check(torch.full((2, T), 5, dtype=torch.int64), eos_last=True)


def test_score_prefix_needs_eos_within_tar_len():
    from fira_icse_b200.sample import score_prefix
    lab = torch.tensor([[1, 5, 6, EOS, 0, 0, 0, 0], [1, 5, EOS, 9, 9, 0, 0, 0]])
    pre = score_prefix(lab, T, EOS)
    assert pre.tolist() == [[5, 6, EOS, 0, 0, 0, 0], [5, EOS, 0, 0, 0, 0, 0]]
    with pytest.raises(ValueError, match="<eos>"):
        score_prefix(torch.tensor([[1, 5, 6, 7, 8, 9, 10, 11, EOS]]), T, EOS)      # <eos> only after tar_len


def test_prefix_labels_equal_build_commit_tar_label():
    from fira_icse_b200.data import build_commit, prefix_labels
    raw = load_raw_golden()
    vocab, upper = raw["word_vocab"], set(raw["VOCAB_UPPER_CASE"])
    compared = copies = 0
    for i in range(len(raw["raw"]["msg"])):
        words = raw["raw"]["msg"][i]
        tar_label = build_commit(raw["raw"], i, vocab, raw["ast_change_vocab"], upper)["tar_label"]
        for n in range(min(len(words), len(tar_label) - 1) + 1):
            got = prefix_labels(raw["raw"], i, words[:n], vocab, upper)
            assert got == list(tar_label[1:1 + n]), (i, n)
            compared += 1
        copies += sum(j >= len(vocab) for j in tar_label)
    assert compared > 128 and copies > 0
