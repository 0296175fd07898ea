"""Float64 restatement of fira_pointer_mix_ensemble (test infrastructure): M members' rows rewritten into one triple
whose mixture (sample_rule.mixture) is sum_m w_m P^m.

rewrite(rows, weights, mem_mask) takes rows = [(logits [V], copy scores [S], gate logits [2]) per member] and the
normalised weights, and returns (x' [V], c' [S], gl' [2]) by the kernel's formula:
    G0 = sum_m w_m g0^m, G1 = sum_m w_m g1^m
    x'_j = LSE over m with w_m g0^m > 0 of [log(w_m g0^m / G0) + x^m_j - vmax^m - log vsum^m]   (G0 = 0: log w_m)
    c'_s = the same with g1, the masked copy scores (-1e9 at masked s), cmax, csum; masked s: -1e9
    gl'  = (log G0, log G1)"""
import numpy as np

MASK_FILL = -1e9


def _stats(x, c, gl):
    x, c, gl = (np.asarray(a, np.float64) for a in (x, c, gl))
    e = np.exp(gl - gl.max())
    g = e / e.sum()
    vmax, cmax = x.max(), c.max()
    return g, vmax, np.log(np.exp(x - vmax).sum()), cmax, np.log(np.exp(c - cmax).sum())


def _lse(terms):
    t = np.stack(terms)
    m = t.max(0)
    return m + np.log(np.exp(t - m).sum(0))


def rewrite(rows, weights, mem_mask):
    mk = np.asarray(mem_mask) != 0
    w = np.asarray(weights, np.float64)
    st = []
    for x, c, gl in rows:
        cm = np.where(mk, np.asarray(c, np.float64), MASK_FILL)
        st.append((np.asarray(x, np.float64), cm) + _stats(x, cm, gl))
    G = sum(wm * s[2] for wm, s in zip(w, st))
    with np.errstate(divide="ignore"):
        lG = np.log(G)
    out = []
    for side, (val, mx, ls) in enumerate(((0, 3, 4), (1, 5, 6))):
        terms = []
        for wm, s in zip(w, st):
            a = wm * s[2][side]
            if G[side] > 0:
                if a == 0:
                    continue
                off = np.log(a) - lG[side]
            else:
                off = np.log(wm)
            terms.append(off + s[val] - s[mx] - s[ls])
        out.append(_lse(terms))
    x, c = out
    c = np.where(mk, c, MASK_FILL)
    return x, c, lG


def average(rows, weights, mem_mask, mixture):
    """sum_m w_m P^m in float64 (mixture: sample_rule.mixture)."""
    return sum(w * mixture(x, c, gl, mem_mask) for w, (x, c, gl) in zip(weights, rows))
