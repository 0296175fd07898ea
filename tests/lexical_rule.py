"""Float64 restatement of one position of lexically constrained n-best (fira_icse_b200.beam.nbest `constraints=`,
fira_pointer_mix_beam_step_lexical; test infrastructure).

phrases: one commit's phrases, lists of vocabulary ids (empty lists and 0 padding dropped by `phrases_of`); Tc = the
number of their words.  words: a row's words, its seq ids after <start> (a copy as its word copy_src).
  progress(words, c) = len(c) when c occurs contiguously in words, else the largest m < len(c) with words ending in
  c[:m] (0 if none); a row meets its constraints when the sum over the phrases is Tc.
candidates(...) forms one commit's candidates as the kernels' row stage does (beam_rule's n-best candidates, the rules
of constraint_rule, <eos> banned below Tc, one extra label per unmet phrase), each with its bank; select(...) takes the
K new slots (Tc = 0: beam_rule's order; Tc > 0: carried finished slots first, then the striping over the banks).
"""
import numpy as np

from beam_rule import token_logprob
from constraint_rule import allowed
from diverse_rule import token_ids


def phrases_of(con):
    """[P, L] ids with 0 = padding -> list of phrases (lists of ids), empty ones dropped"""
    out = [[int(w) for w in row if int(w) != 0] for row in np.asarray(con).reshape(-1, np.asarray(con).shape[-1])]
    return [c for c in out if c]


def progress(words, c):
    words, c = [int(w) for w in words], [int(w) for w in c]
    L = len(c)
    if any(words[a:a + L] == c for a in range(len(words) - L + 1)):
        return L
    return max([m for m in range(1, L) if m <= len(words) and words[len(words) - m:] == c[:m]], default=0)


def row_progress(words, phrases):
    return sum(progress(words, c) for c in phrases)


def meets(words, phrases):
    return row_progress(words, phrases) == sum(len(c) for c in phrases)


def candidates(L, n, status, P, copy_ok, copy_src, words, bans, phrases, V, K, alpha, eos_id, forced=None):
    """every (score, i * (C + 1) + j, i, j, L, n, bank) of one commit at one position; words[i] / bans[i] the history
    and the rule-banned words (constraint_rule.banned) of slot i, forced = the prefix label of a commit inside its
    prefix (None: free).  A carried finished slot has j = C and bank -1."""
    P = np.asarray(P, np.float64)
    C = P.shape[1]
    tc = sum(len(c) for c in phrases)
    tok = token_ids(V, copy_src)
    out = []
    for i, st in enumerate(status):
        if st == 1:
            out.append((L[i] / ((5.0 + n[i]) / 6.0) ** alpha, i * (C + 1) + C, i, C, L[i], n[i], -1))
        if st != 0:
            continue
        lp = token_logprob(P[i])
        if forced is not None:
            props = [forced]
        else:
            ban = set(bans[i])
            if row_progress(words[i], phrases) < tc:
                ban.add(int(eos_id))
            js = np.nonzero(allowed(ban, V, copy_src, copy_ok))[0]
            props = [int(j) for j in js[np.lexsort((js, -lp[js]))[:K]]]
            seen = set()
            top = list(props)
            for c in phrases:
                m = progress(words[i], c)
                if m == len(c):
                    continue
                w = c[m]
                if w in ban or w in seen:
                    seen.add(w)
                    continue
                seen.add(w)
                labels = [w] + [V + s for s in range(C - V) if copy_ok[s] and copy_src[s] == w]
                best = min(labels, key=lambda j: (-lp[j], j))
                if best not in top:
                    props.append(best)
        for j in props:
            Lj, nj = L[i] + lp[j], n[i] + 1
            bank = row_progress(list(words[i]) + [int(tok[j])], phrases)
            out.append((Lj / ((5.0 + nj) / 6.0) ** alpha, i * (C + 1) + j, i, j, Lj, nj, bank))
    return out


def select(cand, K, tc):
    """the K new slots as (i, j, L, n, score, bank), in slot order"""
    if tc == 0:
        order = sorted(cand, key=lambda c: (-c[0], c[1]))
    else:
        fin = sorted((c for c in cand if c[6] < 0), key=lambda c: (-c[0], c[1]))
        live = [c for c in cand if c[6] >= 0]
        rank = {}
        for bank in {c[6] for c in live}:
            for r, c in enumerate(sorted((c for c in live if c[6] == bank), key=lambda c: (-c[0], c[1]))):
                rank[c[1]] = r
        order = fin + sorted(live, key=lambda c: (rank[c[1]], -c[6], -c[0], c[1]))
    return [(c[2], c[3], c[4], c[5], c[0], c[6]) for c in order[:K]]
