"""Float64 restatement of one position of the n-best rule of fira_icse_b200.beam.nbest / fira_pointer_mix_beam_step
(test infrastructure).

step(L, n, status, P, copy_ok, V, K, alpha) takes one commit's slot state (L: log-probability sums, n: generated
tokens, status: 0 live / 1 finished / 2 inactive, one entry per slot) and its slots' mixtures P [K, V + S] (rows of
mixture.mixture; rows of slots that are not live are ignored) and returns the new slots best first as
(parent i, j, L, n, score), with j = C = V + S for a carried finished slot.  `gap` is the relative float64 distance
between the K-th and the (K+1)-th score (inf when there is no (K+1)-th), where an fp32 evaluation may pick the other.
"""
import numpy as np


def token_logprob(P):
    return np.log(np.clip(np.asarray(P, np.float64), 1e-10, 1.0))


def candidates(L, n, status, P, copy_ok, V, K, alpha, prefilter=True):
    """every (score, i * (C + 1) + j, i, j, L, n) of the position; prefilter=True proposes only each live row's top K
    by (lp descending, j ascending), as the kernel's row stage does; False proposes every candidate (brute force)"""
    P = np.asarray(P, np.float64)
    C = P.shape[1]
    ok = np.ones(C, bool)
    ok[V:] = np.asarray(copy_ok, bool)
    out = []
    for i, st in enumerate(status):
        if st == 1:
            out.append((L[i] / ((5.0 + n[i]) / 6.0) ** alpha, i * (C + 1) + C, i, C, L[i], n[i]))
        if st != 0:
            continue
        js = np.nonzero(ok)[0]
        lp = token_logprob(P[i, js])
        if prefilter:
            order = np.lexsort((js, -lp))[:K]
            js, lp = js[order], lp[order]
        for j, l in zip(js, lp):
            Lj, nj = L[i] + l, n[i] + 1
            out.append((Lj / ((5.0 + nj) / 6.0) ** alpha, i * (C + 1) + int(j), i, int(j), Lj, nj))
    return out


def step(L, n, status, P, copy_ok, V, K, alpha, prefilter=True):
    cand = candidates(L, n, status, P, copy_ok, V, K, alpha, prefilter)
    cand.sort(key=lambda c: (-c[0], c[1]))
    sel = [(c[2], c[3], c[4], c[5], c[0]) for c in cand[:K]]
    gap = np.inf
    if len(cand) > K:
        a, b = cand[K - 1][0], cand[K][0]
        gap = abs(a - b) / max(1e-30, abs(a))
    return sel, gap
