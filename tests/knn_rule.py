"""Float64 restatement of nearest-neighbour decoding (fira_icse_b200/knn.py, include/fira_b200.h): the exact search
over the bf16-rounded operands in (d, i) order, the neighbour distribution q and the mixture P'."""
import numpy as np
import torch


def bf16(x):
    """x rounded to bf16, as float64"""
    return torch.as_tensor(np.asarray(x, dtype=np.float32)).to(torch.bfloat16).double().numpy()


def distances(queries, keys):
    """d [R, N] float64 over the bf16-rounded queries and keys: |q|^2 + |key|^2 - 2 q . key"""
    q, k = bf16(queries), bf16(keys)
    return (q * q).sum(1)[:, None] + (k * k).sum(1)[None, :] - 2.0 * q @ k.T


def search(queries, keys, k):
    """(idx [R, k], d [R, k]): the k smallest (d_i, i) of every row, ascending"""
    d = distances(queries, keys)
    idx = np.lexsort((np.broadcast_to(np.arange(d.shape[1]), d.shape), d), axis=1)[:, :k]
    return idx, np.take_along_axis(d, idx, 1)


def neighbour_q(words, dist, tau, V):
    """q [V] of one row: sum over neighbours with word w of exp(-(d_i - d_1) / tau), normalised"""
    d = np.asarray(dist, dtype=np.float64)
    e = np.exp(-(d - d[0]) / tau)
    q = np.zeros(V)
    np.add.at(q, np.asarray(words), e)
    return q / e.sum()


def mix(P, q, lam, V):
    """P' of one row: (1 - lam) P_j + lam q_j for j < V, (1 - lam) P_j for the copy labels"""
    out = (1.0 - lam) * np.asarray(P, dtype=np.float64)
    out[:V] += lam * q
    return out
