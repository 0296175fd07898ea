"""Float64 restatement of offline distillation's stored targets (fira_pointer_mix_topk) and of the loss against them
(fira_pointer_mix_kd_sparse_fwd / _bwd) (test infrastructure).

topk(P, mem_mask, V, k) takes one row's teacher probabilities P [V + S] (sample_rule.mixture of its triple):
    candidates  every j < V and every unmasked copy position j = V + s with P_j > 0 in fp32
    kept        the k candidates first in (P_j descending, then j ascending) order, in that order
    mass        sum of the kept P_j in that order;  t~_i = P_i / mass
    -> (labels [k] with -1 for missing slots, t~ [k] with 0 for them, mass)
row(x, c, gl, mem_mask, labels, probs, y, alpha) is kd_rule.row against the dense vector holding probs at labels and 0
elsewhere (label -1 adds nothing)."""
import numpy as np

from kd_rule import row as kd_row


def topk(P, mem_mask, V, k):
    P = np.asarray(P, np.float64)
    mk = np.asarray(mem_mask) != 0
    ok = P.astype(np.float32) > 0
    ok[V:] &= mk
    cand = np.nonzero(ok)[0]
    order = cand[np.lexsort((cand, -P[cand]))][:k]
    mass = 0.0
    for j in order:
        mass += P[j]
    labels = np.full(k, -1, np.int64)
    probs = np.zeros(k)
    labels[:len(order)] = order
    probs[:len(order)] = P[order] / mass if len(order) else 0.0
    return labels, probs, mass


def dense(labels, probs, n):
    t = np.zeros(n)
    for j, p in zip(labels, probs):
        if j >= 0:
            t[int(j)] = p
    return t


def row(x, c, gl, mem_mask, labels, probs, y, alpha):
    return kd_row(x, c, gl, mem_mask, dense(labels, probs, len(x) + len(c)), y, alpha)
