"""The minimum-Bayes-risk rule (float64 restatement, tests/mbr_rule.py), the id-level versus text-level BLEU of the
golden vocabulary, and the argument checks of fira_icse_b200.mbr, on CPU.  The kernel is compared with the restatement
in tests/test_gpu_mbr.py."""
import random

import pytest

from fira_icse_b200.bleu import sentence_bleu_method2
from fira_testlib import load_raw_golden
from mbr_rule import select, words

START, EOS, PAD = 2, 1, 0
MARKERS = ("<start>", "<eos>", "<pad>")


def test_cleaning_drops_markers_anywhere_and_stops_at_length():
    assert words([START, 5, PAD, 6, START, 7, EOS, 9], 7, START, EOS, PAD) == [5, 6, 7]
    assert words([START, 5, 6], 1, START, EOS, PAD) == []
    assert words([START, EOS, PAD], 3, START, EOS, PAD) == []


def test_rule_picks_the_consensus_and_breaks_ties_by_index():
    a = [START, 5, 6, 7, 8, 9, EOS]
    near_a = [START, 5, 6, 7, 8, 3, EOS]
    other = [START, 4, 4, EOS, PAD, PAD, PAD]
    pairs, u, best = select([other, a, near_a, a], [4, 7, 7, 7], START, EOS, PAD)
    assert best == 1 and u[1] == u[3] > u[2] > u[0]              # duplicates: identical utilities, smaller index
    assert pairs[1][3] == pairs[3][1] == 1.0 and pairs[0][1] == 0.0
    assert u[1] == (pairs[1][0] + pairs[1][2] + pairs[1][3]) / 3
    _, u, best = select([a, a], [7, 7], START, EOS, PAD)
    assert u == [1.0, 1.0] and best == 0
    _, u, best = select([[START, EOS], [START, PAD]], [2, 1], START, EOS, PAD)   # empty candidates score 0
    assert u == [0.0, 0.0] and best == 0


def _ids_to_text():
    import run_model
    return run_model.ids_to_text


def test_id_level_bleu_is_text_level_bleu_except_for_import_static():
    """One id is one text token of run_model.ids_to_text for every golden vocabulary word but `import static`, so the
    id-level BLEU of messages over the other words equals the text-level BLEU run_model.py reports."""
    ids_to_text = _ids_to_text()
    vocab = load_raw_golden()["word_vocab"]
    r_vocab = {i: w for w, i in vocab.items()}
    start, eos, pad = (vocab[m] for m in MARKERS)

    def one_token(i):
        toks = ids_to_text([i], r_vocab)
        return len(toks) == 1 and not any(m in toks[0] for m in MARKERS)

    others = [i for w, i in vocab.items() if w not in MARKERS]
    assert [r_vocab[i] for i in others if not one_token(i)] == ["import static"]
    plain = [i for i in others if r_vocab[i] != "import static"]
    assert len({ids_to_text([i], r_vocab)[0] for i in plain}) == len(plain)          # no two ids share a token
    rng = random.Random(0)
    pool = rng.sample(plain, 12) + [vocab["<unkm>"]]                                  # small pool: n-grams repeat
    for _ in range(400):
        seqs = []
        for _ in range(2):
            n = rng.randint(0, 28)
            body = [rng.choice(pool) if rng.random() > 0.15 else rng.choice((pad, start)) for _ in range(n)]
            seqs.append([start] + body + [eos])
        hyp, ref = seqs
        at_id = sentence_bleu_method2([words(ref, len(ref), start, eos, pad)], words(hyp, len(hyp), start, eos, pad))
        at_text = sentence_bleu_method2([ids_to_text(ref, r_vocab)], ids_to_text(hyp, r_vocab))
        assert at_id == at_text, (hyp, ref)


@pytest.mark.parametrize("kw", [dict(num_samples=1), dict(num_samples=33), dict(num_samples=2.0), dict(tar_len=33),
                                dict(tar_len=64), dict(tar_len=1), dict(temperature=0.0), dict(top_k=-1),
                                dict(top_p=0.0), dict(seed=-1), dict(first_index=-1)])
def test_invalid_arguments_raise_before_any_device_work(kw):
    from fira_icse_b200.mbr import mbr
    args = dict(num_samples=4, temperature=1.0, top_k=0, top_p=1.0, seed=0, first_index=0, tar_len=30)
    args.update(kw)
    with pytest.raises(ValueError):
        mbr(None, None, None, None, None, None, start_id=START, eos_id=EOS, **args)    # no model, no tensors needed
