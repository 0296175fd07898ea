"""The error bound of the bf16 training step against a float64 reference -- test infrastructure.

One number per stage, eps, sets three bounds on a kernel output g and its float64 reference r:

  * element-wise:  |g - r| <= 2 eps |r| + eps max|r|;
  * per row (row-structured tensors: activations and their gradients, embedding-gradient rows):
        ||g_i - r_i|| <= 2 eps ||r_i|| + eps max_j ||r_j||,
    which catches a zeroed or misrouted row even when its norm is small next to the tensor's largest row;
  * gradients that vanish in exact arithmetic (fc_k.bias of every attention, copy_net.LinearRes.bias: softmax shift
    invariance): max|g| <= eps * the scale of a gradient of the same block.

So eps is the global (ε_glob) and 2 eps the relative and per-row (ε_rel, ε_row) factor of tests/test_gpu_bf16_step.py;
each check prints its worst error as a fraction of its bound."""
import math

import torch


def _frac(err, bound):
    """max over elements of err / bound (0 / 0 = 0, x / 0 = inf)"""
    if err.numel() == 0:
        return 0.0
    out = torch.zeros_like(err)
    pos = bound > 0
    out[pos] = err[pos] / bound[pos]
    out[~pos & (err > 0)] = math.inf
    return out.max().item()


def close(what, g, r, eps, rows=False, allow=None):
    """assert g (kernel) is within eps of r (float64 reference) element-wise, and per row (last dim) with rows=True;
    allow: a further element-wise allowance (tests/test_gpu_bf16_step.py: ReLU gates at a rounding of zero)
    -> the worst error as a fraction of its bound"""
    g, r = g.detach().cpu().double(), r.detach().cpu().double()
    assert g.shape == r.shape, (what, tuple(g.shape), tuple(r.shape))
    assert torch.isfinite(g).all(), f"{what}: non-finite values"
    a = r.abs()
    err = (g - r).abs() if allow is None else ((g - r).abs() - allow.detach().cpu().double()).clamp(min=0)
    fe = _frac(err, 2 * eps * a + eps * a.max())
    fr = 0.0
    if rows:
        g2, r2 = g.reshape(-1, g.shape[-1]), r.reshape(-1, r.shape[-1])
        n = r2.norm(dim=1)
        fr = _frac((g2 - r2).norm(dim=1), 2 * eps * n + eps * n.max())
    worst = max(fe, fr)
    print(f"[bf16 bound] {what}: {worst:.3f} of eps = 2^{math.log2(eps):.0f} (element {fe:.3f}, row {fr:.3f})")
    assert fe <= 1.0, f"{what}: element error {fe:.3f} x its bound (eps = {eps})"
    assert fr <= 1.0, f"{what}: row error {fr:.3f} x its bound (eps = {eps})"
    return worst


def small(what, g, scale, eps):
    """a gradient that vanishes in exact arithmetic: max|g| <= eps * scale"""
    g = g.detach().cpu().double()
    assert torch.isfinite(g).all(), f"{what}: non-finite values"
    f = _frac(g.abs().max().reshape(1), torch.tensor([eps * float(scale)], dtype=torch.float64))
    print(f"[bf16 bound] {what} (vanishing): {f:.3f} of eps = 2^{math.log2(eps):.0f}")
    assert f <= 1.0, f"{what}: {f:.3f} x its bound (eps = {eps})"
    return f


def vanishing(name):
    """parameters whose gradient is zero in exact arithmetic"""
    return name.endswith("fc_k.bias") or name == "copy_net.LinearRes.bias"
