"""Float64 restatement of the distillation loss of fira_pointer_mix_kd_fwd / _bwd (test infrastructure).

row(x, c, gl, mem_mask, t, y, alpha) takes one row's student logits [V], copy scores [S], gate logits [2], the commit's
mem_mask [S], the teacher's probabilities t [V + S] (sample_rule.mixture of its triple) and the shifted label y, and
returns (nll, kd, loss, dx [V], dc [S], dgl [2]), the gradients for upstream 1:
    P      = sample_rule.mixture(x, c, gl, mem_mask), live_j = (1e-10 <= P_j <= 1)
    nll    = -log clamp(P_y, 1e-10, 1)          (P_y = 0 for a copy label beyond S)
    kd     = -sum_j t_j log clamp(P_j, 1e-10, 1)
    loss   = (1 - alpha) nll + alpha kd
    a_j    = [(1 - alpha) [j == y] + alpha t_j] live_j,  A_V = sum_{j<V} a_j,  A_C = sum_s a_{V+s}
    dx     = softmax(x) A_V - a[:V],  dc = softmax(masked c) A_C - a[V:] (0 at masked s),  dgl = g (A_V + A_C) - (A_V, A_C)
A row with y = 0 gives zeros everywhere."""
import numpy as np

from sample_rule import mixture

FLOOR = 1e-10


def row(x, c, gl, mem_mask, t, y, alpha):
    x, c, gl, t = (np.asarray(a, np.float64) for a in (x, c, gl, t))
    V, S = len(x), len(c)
    mk = np.asarray(mem_mask) != 0
    if y == 0:
        return 0.0, 0.0, 0.0, np.zeros(V), np.zeros(S), np.zeros(2)
    P = mixture(x, c, gl, mem_mask)
    live = (P >= FLOOR) & (P <= 1.0)
    p_y = P[y] if y < V + S else 0.0
    nll = -np.log(min(max(p_y, FLOOR), 1.0))
    pos = t > 0
    kd = -float(np.sum(t[pos] * np.log(np.clip(P[pos], FLOOR, 1.0))))
    a = alpha * t
    if y < V + S:
        a[y] += 1.0 - alpha
    a = np.where(live, a, 0.0)
    A_V, A_C = a[:V].sum(), a[V:].sum()
    p = np.exp(x - x.max())
    p /= p.sum()
    cm = np.where(mk, c, -1e9)
    q = np.exp(cm - cm.max())
    q /= q.sum()
    g = np.exp(gl - gl.max())
    g /= g.sum()
    dx = p * A_V - a[:V]
    dc = np.where(mk, q * A_C - a[V:], 0.0)
    dgl = g * (A_V + A_C) - np.array([A_V, A_C])
    return nll, kd, (1.0 - alpha) * nll + alpha * kd, dx, dc, dgl
