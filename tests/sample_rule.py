"""Float64 restatement of the sampling rule of fira_icse_b200.sample / fira_pointer_mix_sample (test infrastructure).

draw(P, copy_ok, ...) takes one row's mixture probabilities P [V + S] (float64) and returns the index the rule picks
for the uniform u, plus `near`: True when the row sits within `tol` of a decision boundary (the top-k cut between two
distinct scores, the top-p cut, or u * Z against the running weight), where an fp32 evaluation may legitimately pick a
neighbour."""
import numpy as np


def mixture(logits, copy_scores, gate_logits, mem_mask):
    """Float64 P of one row: g0 * softmax(logits) || g1 * softmax(copy scores, masked positions at -1e9)."""
    x = np.asarray(logits, np.float64)
    c = np.where(np.asarray(mem_mask) != 0, np.asarray(copy_scores, np.float64), -1e9)
    g = np.exp(np.asarray(gate_logits, np.float64) - np.max(gate_logits))
    g = g / g.sum()
    pv = np.exp(x - x.max())
    pc = np.exp(c - c.max())
    return np.concatenate((g[0] * pv / pv.sum(), g[1] * pc / pc.sum()))


def draw(P, copy_ok, V, temperature, top_k, top_p, u, tol=1e-5):
    P = np.asarray(P, np.float64)
    cand = P > 0
    cand[V:] &= np.asarray(copy_ok, bool)
    idx = np.nonzero(cand)[0]
    if len(idx) == 0:
        return 0, False
    s = np.log(np.minimum(P[idx], 1.0)) / temperature
    order = np.lexsort((idx, -s))                       # score descending, then index ascending
    ranked, rs = idx[order], s[order]
    near = False
    if 0 < top_k < len(ranked):
        a, b = rs[top_k - 1], rs[top_k]
        near |= bool(a != b and abs(a - b) <= tol * max(1.0, abs(a)))
        ranked, rs = ranked[:top_k], rs[:top_k]
    smax = rs[0]
    w = np.where(rs == smax, 1.0, np.exp(rs - smax))
    if top_p < 1.0:
        c = np.cumsum(w)
        target = top_p * c[-1]
        m = int(np.argmax(c >= target)) + 1             # shortest prefix whose weight reaches p * W
        near |= bool(np.any(np.abs(c - target) <= tol * c[-1]))
        ranked, w = ranked[:m], w[:m]
    o = np.argsort(ranked)
    ji, wi = ranked[o], w[o]
    c = np.cumsum(wi)
    target = u * c[-1]
    hit = np.nonzero((c > target) & (wi > 0))[0]
    j = ji[hit[0]] if len(hit) else ji[wi > 0][-1]
    near |= bool(np.any(np.abs(c - target) <= tol * c[-1]))
    return int(j), near
