"""Float64 restatement of the minimum-Bayes-risk rule of fira_icse_b200.mbr / fira_mbr_select (test infrastructure):
clean every candidate, score every ordered pair with bleu.sentence_bleu_method2, average each row over the other
candidates in ascending order, take the smallest index of the largest utility."""
from fira_icse_b200.bleu import sentence_bleu_method2


def words(ids, length, start_id, eos_id, pad_id):
    """ids[1:length] without the three marker ids."""
    return [int(x) for x in list(ids)[1:int(length)] if int(x) not in (start_id, eos_id, pad_id)]


def select(seq, length, start_id, eos_id, pad_id):
    """One commit: seq [N, T] ids, length [N] -> (pair BLEU [N][N], utility [N], chosen index)."""
    cands = [words(s, n, start_id, eos_id, pad_id) for s, n in zip(seq, length)]
    pairs = [[sentence_bleu_method2([cj], ci) for cj in cands] for ci in cands]
    N = len(cands)
    utility = []
    for i in range(N):
        total = 0.0
        for j in range(N):
            if j != i:
                total += pairs[i][j]
        utility.append(total / (N - 1))
    return pairs, utility, utility.index(max(utility))
