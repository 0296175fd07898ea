"""Float64 restatement of one position of diverse n-best beam search (fira_icse_b200.beam.nbest with groups > 1 /
fira_pointer_mix_diverse_beam_step), on top of the n-best rule of tests/beam_rule.py (test infrastructure).

One commit: slot state L, n, status (as beam_rule.step), the slots' mixtures P [K, V + S], copy_ok [S] and copy_src
[S] (copy position -> vocabulary id).  The K slots form G groups of Kg = K / G; group g owns slots g*Kg..(g+1)*Kg-1.
Group g proposes beam_rule's candidates of its own slots and ranks them by

    value = score - diversity * h(token of j),   h(w) = how many earlier-group slots grew with w at this position

(token of j: j, or copy_src[j - V] for a copy; a carried finished slot proposes its score unpenalised and counts
nothing).  Candidates are (value, i * (C + 1) + j, i, j, L, n, score), j = C = V + S for a carried finished slot.
step() runs the groups in order and returns, per group, its new slots best first as (i, j, L, n, score, value) and the
relative float64 gap between its Kg-th and (Kg+1)-th value (inf when there is none), plus the token every slot grew with
(-1 when carried or left empty).
"""
import numpy as np

from beam_rule import candidates as nbest_candidates
from beam_rule import token_logprob


def token_ids(V, copy_src):
    """the word behind every candidate index j < C"""
    return np.concatenate([np.arange(V), np.asarray(copy_src, np.int64)])


def penalty(tok, prev):
    """h for every token in `tok`: how many of the earlier groups' tokens `prev` (-1 = none) equal it"""
    h = np.zeros(len(tok))
    for w in prev:
        if w >= 0:
            h += tok == w
    return h


def group_candidates(L, n, status, P, copy_ok, copy_src, V, G, g, alpha, diversity, prev, prefilter=True, keep=None):
    """group g's candidates; prefilter=True keeps each live row's Kg (or `keep`) best by (value descending, j
    ascending), as the kernel's row stage does, False every candidate (brute force through beam_rule.candidates)"""
    P = np.asarray(P, np.float64)
    K, C = P.shape
    Kg = K // G
    own = np.full(K, 2)
    own[g * Kg:(g + 1) * Kg] = np.asarray(status)[g * Kg:(g + 1) * Kg]
    h = penalty(token_ids(V, copy_src), prev)
    if not prefilter:
        return [(sc if j == C else sc - diversity * h[j], idx, i, j, Lj, nj, sc)
                for sc, idx, i, j, Lj, nj in nbest_candidates(L, n, own, P, copy_ok, V, Kg, alpha, prefilter=False)]
    ok = np.ones(C, bool)
    ok[V:] = np.asarray(copy_ok, bool)
    js = np.nonzero(ok)[0]
    out = []
    for i in range(g * Kg, (g + 1) * Kg):
        if own[i] == 1:
            sc = L[i] / ((5.0 + n[i]) / 6.0) ** alpha
            out.append((sc, i * (C + 1) + C, i, C, L[i], n[i], sc))
        if own[i] != 0:
            continue
        Lj, nj = L[i] + token_logprob(P[i, js]), n[i] + 1
        sc = Lj / ((5.0 + nj) / 6.0) ** alpha
        v = sc - diversity * h[js]
        for o in np.lexsort((js, -v))[:keep or Kg]:
            out.append((v[o], i * (C + 1) + int(js[o]), i, int(js[o]), Lj[o], nj, sc[o]))
    return out


def group_step(L, n, status, P, copy_ok, copy_src, V, G, g, alpha, diversity, prev, prefilter=True):
    """-> (group g's new slots best first as (i, j, L, n, score, value), gap)"""
    Kg = np.asarray(P).shape[0] // G
    cand = group_candidates(L, n, status, P, copy_ok, copy_src, V, G, g, alpha, diversity, prev, prefilter)
    cand.sort(key=lambda c: (-c[0], c[1]))
    sel = [(c[2], c[3], c[4], c[5], c[6], c[0]) for c in cand[:Kg]]
    gap = np.inf
    if len(cand) > Kg:
        a, b = cand[Kg - 1][0], cand[Kg][0]
        gap = abs(a - b) / max(1e-30, abs(a))
    return sel, gap


def grown_tokens(sel, Kg, C, V, copy_src):
    """the token each of the group's Kg new slots grew with (-1: carried, or no candidate filled it)"""
    tok = [-1] * Kg
    for k, s in enumerate(sel):
        if s[1] != C:
            tok[k] = s[1] if s[1] < V else int(copy_src[s[1] - V])
    return tok


def step(L, n, status, P, copy_ok, copy_src, V, G, alpha, diversity, prefilter=True):
    """-> ([(sel, gap) per group], chosen [K])"""
    K, C = np.asarray(P).shape
    Kg = K // G
    groups, chosen = [], []
    for g in range(G):
        sel, gap = group_step(L, n, status, P, copy_ok, copy_src, V, G, g, alpha, diversity, chosen, prefilter)
        groups.append((sel, gap))
        chosen += grown_tokens(sel, Kg, C, V, copy_src)
    return groups, chosen
