"""float64 restatement of global-norm gradient clipping with the non-finite guard (optim.ClipGroup: fira_grad_sumsq,
fira_grad_clip_finalize, fira_adam_flat_clip in csrc/optim.cu, include/fira_b200.h), for a group of members that each
hold (p, m, v[, e]) and one gradient per step:

    S = sum of g^2 over every member (float64);  norm = sqrt(S) / s      (s = grad_scale, 1 without one)
    S not finite: the step is skipped -- no member's p, m, v, e or step count t changes; skipped += 1
    else:  coef = fl32(min(1, c / (norm + 1e-6)))  (clip_grad_norm_'s formula in float64, rounded once);
           clipped += (coef < 1);  t += 1;  g' = fl32(fl32(g * fl32(1 / s)) * coef);  Adam (ema_rule.adam) on g'

c = inf never clips.  The fp32 roundings of g' are the kernel's (exact in numpy's float32 arithmetic), everything
after them is float64, so the kernel's result is this one up to Adam's own fp32 roundings."""
import numpy as np

import ema_rule

f32 = ema_rule.f32


def norm(grads, grad_scale=None):
    """-> (S, norm) of the group's gradients (a list of arrays)"""
    S = float(sum(np.sum(np.square(np.asarray(g, np.float64))) for g in grads))
    s = f32(grad_scale) if grad_scale is not None else 1.0
    with np.errstate(invalid="ignore", over="ignore"):
        return S, np.sqrt(S) / s


def coefficient(nrm, c):
    """fl32(min(1, c / (norm + 1e-6))) as a float64"""
    return f32(min(1.0, c / (nrm + 1e-6)))


def scaled_grad(g, coef, grad_scale=None):
    """g' = fl32(fl32(g * fl32(1 / s)) * coef) in the kernel's fp32 order (float64 out)"""
    g = np.asarray(g, np.float32)
    if grad_scale is not None:
        g = g * (np.float32(1.0) / np.float32(grad_scale))
    return (g * np.float32(coef)).astype(np.float64)


def new_state(params, ema=False):
    """the group's state before the first step: members (p, m = v = 0[, e = p]), t = 0, no clipped or skipped step"""
    members = [dict(p=np.asarray(p, np.float64).copy(), m=np.zeros(np.shape(p)), v=np.zeros(np.shape(p)))
               for p in params]
    if ema:
        for mb in members:
            mb["e"] = mb["p"].copy()
    return dict(members=members, t=0, clipped=0, skipped=0, norm=0.0)


def step(state, grads, c, lr, b1, b2, eps, grad_scale=None, ema_decay=None):
    """one clipped step of the group, in place; -> (taken, norm, coef or None)"""
    S, nrm = norm(grads, grad_scale)
    state["norm"] = nrm
    if not np.isfinite(S):
        state["skipped"] += 1
        return False, nrm, None
    coef = coefficient(nrm, c)
    state["clipped"] += int(coef < 1.0)
    state["t"] += 1
    for mb, g in zip(state["members"], grads):
        gp = scaled_grad(g, coef, grad_scale)
        mb["p"], mb["m"], mb["v"] = ema_rule.adam(mb["p"], gp, mb["m"], mb["v"], state["t"], lr, b1, b2, eps)
        if ema_decay is not None:
            mb["e"] = ema_rule.ema(mb["e"], mb["p"], ema_decay)
    return True, nrm, coef
