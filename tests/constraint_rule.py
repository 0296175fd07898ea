"""Restatement of n-gram repeat blocking and minimum length (fira_icse_b200 `no_repeat_ngram=` / `min_length=`, the
fira_pointer_mix_*_rules step kernels), and the wrappers that run the existing float64 rules (tests/sample_rule.py,
tests/beam_rule.py, tests/diverse_rule.py) with the banned labels removed (test infrastructure).

banned(words, n, m, eos_id, length): the words of a row are its tokens after <start> (a copy as its word copy_src),
length counts <start>.  A word w may not be appended when, with n >= 1, words[i .. i+n-2] == the last n - 1 words and
words[i+n-1] == w for some i (n = 1: every word already there), or when w == eos_id and length - 1 < m.  A label j is
banned when its word (j, or copy_src[j - V]) is.
"""
import numpy as np

from beam_rule import token_logprob
from diverse_rule import penalty, token_ids
from sample_rule import draw


def banned(words, n, m, eos_id, length):
    """-> the set of banned words"""
    words = [int(w) for w in words]
    out = set()
    if n >= 1:
        tail = words[len(words) - n + 1:] if n > 1 else []
        for i in range(len(words) - n + 1):
            if words[i:i + n - 1] == tail:
                out.add(words[i + n - 1])
    if m and length - 1 < m:
        out.add(int(eos_id))
    return out


def allowed(ban, V, copy_src, copy_ok):
    """bool [V + S]: the labels a row may still take (masked copy positions never)"""
    ok = ~np.isin(token_ids(V, copy_src), np.fromiter(ban, np.int64, len(ban)))
    ok[V:] &= np.asarray(copy_ok, bool)
    return ok


def sample_draw(P, copy_ok, copy_src, ban, V, temperature, top_k, top_p, u, tol=1e-5):
    """sample_rule.draw with the banned labels taken out of the candidates (P = 0 is not a candidate there)"""
    P = np.array(P, np.float64)
    P[~allowed(ban, V, copy_src, np.ones(len(copy_ok), bool))] = 0.0
    return draw(P, copy_ok, V, temperature, top_k, top_p, u, tol)


def candidates(L, n, status, P, ok, copy_src, V, G, g, alpha, diversity, prev, keep=None):
    """group g's candidates as diverse_rule.group_candidates forms them (G = 1, diversity 0: beam_rule's n-best
    candidates, value = score), but over each live slot's own allowed labels ok[i] ([K, V + S], from `allowed`):
    (value, i * (C + 1) + j, i, j, L, n, score), each live row's Kg (or `keep`) best by (value descending, j ascending)"""
    P = np.asarray(P, np.float64)
    K, C = P.shape
    Kg = K // G
    h = penalty(token_ids(V, copy_src), prev)
    out = []
    for i in range(g * Kg, (g + 1) * Kg):
        if status[i] == 1:
            sc = L[i] / ((5.0 + n[i]) / 6.0) ** alpha
            out.append((sc, i * (C + 1) + C, i, C, L[i], n[i], sc))
        if status[i] != 0:
            continue
        js = np.nonzero(ok[i])[0]
        Lj, nj = L[i] + token_logprob(P[i, js]), n[i] + 1
        sc = Lj / ((5.0 + nj) / 6.0) ** alpha
        v = sc - diversity * h[js]
        for o in np.lexsort((js, -v))[:keep or Kg]:
            out.append((v[o], i * (C + 1) + int(js[o]), i, int(js[o]), Lj[o], nj, sc[o]))
    return out


def select(cand, Kg):
    """the Kg best candidates by (value descending, then index ascending) as (i, j, L, n, score, value), and the
    relative gap between the Kg-th and the (Kg+1)-th value (inf when there is none), as diverse_rule.group_step"""
    cand = sorted(cand, key=lambda c: (-c[0], c[1]))
    sel = [(c[2], c[3], c[4], c[5], c[6], c[0]) for c in cand[:Kg]]
    gap = np.inf
    if len(cand) > Kg:
        a, b = cand[Kg - 1][0], cand[Kg][0]
        gap = abs(a - b) / max(1e-30, abs(a))
    return sel, gap


def repeats_ngram(words, n, start=0):
    """True when some word at index >= start completes an n-gram that already ended at an earlier index"""
    words = [int(w) for w in words]
    seen = set()
    for t in range(n - 1, len(words)):
        g = tuple(words[t - n + 1:t + 1])
        if g in seen and t >= start:
            return True
        seen.add(g)
    return False
