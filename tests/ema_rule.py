"""float64 restatement of fira_adam_flat with the exponential moving average of the weights (csrc/optim.cu,
include/fira_b200.h), in the kernel's evaluation order:

    g' = g / grad_scale;  m = b1 m + (1 - b1) g';  v = b2 v + (1 - b2) g'^2
    p -= (lr / (1 - b1^t)) * (m / (sqrt(v) * (1 / sqrt(1 - b2^t)) + eps))
    c = fl32(1 - d);  e = d e + fl32(c p)           (the kernel: one fused multiply-add, d and c fp32 constants)

Every input is taken as the fp32 value the kernel sees (the scalars rounded to fp32 first) and everything after that
is float64, so the kernel's result is this one up to its own fp32 roundings."""
import numpy as np


def f32(x):
    return np.float64(np.float32(x))


def ema_coefficients(d):
    """(d, c) as the kernel holds them: d rounded to fp32, c = fl32(1 - d)"""
    d = f32(d)
    return d, f32(np.float32(1.0) - np.float32(d))


def ema(e, p, d):
    """one EMA update e = d e + fl32(c p) of the stored parameters p (arrays, float64 out)"""
    d, c = ema_coefficients(d)
    cp = np.asarray(p, np.float64) * c
    return d * np.asarray(e, np.float64) + cp.astype(np.float32).astype(np.float64)


def adam(p, g, m, v, t, lr, b1, b2, eps, grad_scale=None):
    """one Adam step (torch.optim.Adam semantics: no weight decay, no amsgrad) -> (p, m, v) float64"""
    p, g, m, v = (np.asarray(x, np.float64) for x in (p, g, m, v))
    lr, b1, b2, eps, t = f32(lr), f32(b1), f32(b2), f32(eps), f32(t)
    if grad_scale is not None:
        g = g / f32(grad_scale)
    m = b1 * m + (1.0 - b1) * g
    v = b2 * v + (1.0 - b2) * g * g
    step_size = lr / (1.0 - b1 ** t)
    denom = np.sqrt(v) / np.sqrt(1.0 - b2 ** t) + eps
    return p - step_size * (m / denom), m, v


def adam_ema(p, g, m, v, e, t, lr, b1, b2, eps, d, grad_scale=None):
    """Adam, then the EMA of the updated parameters -> (p, m, v, e) float64"""
    p, m, v = adam(p, g, m, v, t, lr, b1, b2, eps, grad_scale)
    return p, m, v, ema(e, p, d)
