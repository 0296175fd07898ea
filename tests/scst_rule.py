"""Float64 restatement of the self-critical reward rule of fira_icse_b200.scst / fira_bleu_reward (test infrastructure):
each sample's sentence BLEU against the commit's reference through bleu.sentence_bleu_method2, and its leave-one-out
advantage: the differences to the other samples' rewards, summed in ascending order, over N - 1."""
from fira_icse_b200.bleu import sentence_bleu_method2

from mbr_rule import words


def reference(tar, T, start_id, eos_id, pad_id):
    """tar[1:e] without start / pad ids, e = the first column >= 1 holding <eos> (T if none before column T)."""
    ids = [int(x) for x in list(tar)[:T]]
    e = ids.index(eos_id, 1) if eos_id in ids[1:] else T
    return [x for x in ids[1:e] if x not in (start_id, pad_id)]


def rewards(seq, length, tar, start_id, eos_id, pad_id):
    """One commit: seq [N, T] ids, length [N], its reference ids tar -> (reward [N], advantage [N])."""
    T = len(seq[0])
    ref = reference(tar, T, start_id, eos_id, pad_id)
    r = [sentence_bleu_method2([ref], words(s, min(max(int(n), 1), T), start_id, eos_id, pad_id))
         for s, n in zip(seq, length)]
    N = len(r)
    adv = []
    for n in range(N):
        total = 0.0
        for m in range(N):
            if m != n:
                total += r[n] - r[m]
        adv.append(total / (N - 1))
    return r, adv
