"""Word-level knowledge distillation (Hinton et al. 2015; Kim & Rush 2016): train one model on a teacher's full
distribution at every teacher-forced target position, so that it approaches an ensemble's quality at one model's
decoding cost.

For a padded batch, row r = (commit b, position t) with shifted label y = TransModel.shifted_label(tar_label) (y = 0:
no loss), the student's dual-copy mixture P (Model.py:54-86) and the teacher's mixture t (ensemble.py: P = sum_m w_m P^m
over its members, or one model's own):

    nll_r  = -log clamp(P_y, 1e-10, 1)                         (the training loss's own term)
    kd_r   = -sum_{j < V+S} t_j log clamp(P_j, 1e-10, 1)      (cross-entropy against the teacher)
    loss_r = (1 - alpha) nll_r + alpha kd_r,   step loss = sum_r loss_r / sum_r [y != 0]

Where it runs: teacher_targets runs every teacher member's teacher-forced forward (encoder, decoder, the head's three
products, ops.head_products) under no_grad in eval mode, then one fira_pointer_mix_ensemble launch with N = T turns
the M triples into one fp32 triple whose mixture is t.  The student's head (ops.HeadFn with a teacher) forms the loss
and its gradient through both softmaxes, the gate and the clamp in fira_pointer_mix_kd_fwd / _bwd (include/fira_b200.h),
so the 25,020-wide distributions are never stored.  distill_step is the eager padded-batch path, as scst.scst_step:
the kernels' dropout in the student, an eager optim.FlatAdam step and scst.bump_weights.  The teacher keeps M member
triples and their fp32 average on the device, about (M s + 4) B T ld_logits bytes (s = 4 fp32, 2 bf16).
"""
import ctypes
import math
import numbers
from typing import NamedTuple

import torch

from . import ops
from . import optim as _optim
from ._lib import FIRA_BF16, FIRA_F32, call
from .ensemble import Ensemble, refuse
from .model import TransModel
from .modules import _i32, _u8
from .scst import bump_weights


class Step(NamedTuple):
    loss: float           # sum_r loss_r / tokens
    nll: float            # sum_r nll_r / tokens
    kd: float             # sum_r kd_r / tokens
    tokens: int           # rows with y != 0


def check_alpha(alpha):
    """TypeError / ValueError unless alpha is a finite number in [0, 1] (host only)."""
    if isinstance(alpha, bool) or not isinstance(alpha, numbers.Real):
        raise TypeError(f"alpha must be a number in [0, 1], got {alpha!r}")
    if not (math.isfinite(float(alpha)) and 0.0 <= float(alpha) <= 1.0):
        raise ValueError(f"alpha must be a finite number in [0, 1], got {alpha!r}")


def teacher_members(teacher, student=None):
    """teacher: a TransModel or an Ensemble -> (its models, log weights).  TypeError for anything else; with the
    student, ValueError for a member that is the student itself (the optimizer would move the teacher) or a vocabulary
    or device that differs from the student's (host only)."""
    if isinstance(teacher, TransModel):
        models, log_w = (teacher,), (0.0,)
    elif isinstance(teacher, Ensemble):
        models, log_w = teacher.models, teacher.log_weights
    else:
        raise TypeError(f"the teacher must be a TransModel or an Ensemble, got {type(teacher).__name__}")
    if student is not None:
        for i, m in enumerate(models):
            if m is student:
                raise ValueError(f"teacher member {i} is the student itself: distil from a separate copy")
        if models[0].vocab_size != student.vocab_size:
            raise ValueError(f"the teacher has vocab_size {models[0].vocab_size}, the student {student.vocab_size}")
        t_dev, s_dev = models[0].out_fc.weight.device, student.out_fc.weight.device
        if t_dev != s_dev:
            raise ValueError(f"the teacher is on {t_dev}, the student on {s_dev}")
    return models, log_w


def teacher_targets(teacher, batch, label):
    """The teacher's fp32 triple for the padded batch (the 8-tuple of run_model.py) and its shifted labels [B, T]:
    (logits [B*T, ld_logits], copy scores [B, T, S], gate logits [B*T, 2]) whose mixture is the teacher's distribution
    at every position (a single model is an ensemble of one).  Leaves the members in eval mode.  Rows with label 0 are
    not meaningful: the loss never reads them."""
    models, log_w = teacher_members(teacher)
    first = models[0]
    dev = first.out_fc.weight.device
    sou, tar, _, mark, ast_change, edge, _, sub_token = batch
    sou, tar, mark, ast_change, sub_token = (t.to(dev) for t in (sou, tar, mark, ast_change, sub_token))
    label = label.to(dev)
    B, T = label.shape
    mem_mask = torch.cat((sou != 0, sub_token != 0), dim=1)
    S, V, Mt = mem_mask.shape[1], first.vocab_size, B * T
    mm = _u8(mem_mask)
    row_mask = _u8(label != 0).view(-1)                   # the rows a loss reads
    triples = []
    with torch.no_grad():
        for m in models:
            m.eval()
            bf16 = m.precision == "bf16"
            if bf16:
                _optim.ensure_fresh(m)
            memory = m.encoder.encode_memory(sou, mark, ast_change, edge, sub_token)
            dec = m.decoder(tar, memory, mem_mask, tar != 0)
            pr = ops.Prec(bf16)
            dec2 = dec.contiguous().to(pr.tdt).view(Mt, ops.D)
            logits, _, _, sc, gl = ops.head_products(
                pr, memory.contiguous().to(pr.tdt).view(-1, ops.D), dec2, dec2.float() if bf16 else dec2, dec2, Mt,
                m.out_fc.weight, m.out_fc.bias, *m.copy_net.flat_params(), B, T, S, mm, row_mask)
            triples.append((logits, sc, gl))
    M = len(models)
    ld = triples[0][0].shape[1]
    f32 = dict(dtype=torch.float32, device=dev)
    out, sc_out, gl_out = torch.empty((Mt, ld), **f32), torch.empty((B, T, S), **f32), torch.empty((Mt, 2), **f32)
    lw = torch.tensor(log_w, **f32)
    arrs = [(ctypes.c_void_p * M)(*[ops._ptr(t[k]) for t in triples]) for k in range(3)]
    call("fira_pointer_mix_ensemble", ctypes.addressof(arrs[0]), ld, ctypes.addressof(arrs[1]),
         ctypes.addressof(arrs[2]), M, ops._ptr(lw), ops._ptr(mm), ops._ptr(out), ld, ops._ptr(sc_out),
         ops._ptr(gl_out), B, T, V, S, FIRA_BF16 if first.precision == "bf16" else FIRA_F32, ops._stream())
    return out, sc_out, gl_out


def distill_loss(model, batch, targets, label, alpha):
    """sum_r loss_r under autograd in the model's current mode -> (loss_sum, nll [B, T], kd [B*T]).  targets: the
    teacher's triple of teacher_targets; label: the shifted labels [B, T] on the model's device."""
    m = model
    dev = m.out_fc.weight.device
    sou, tar, _, mark, ast_change, edge, _, sub_token = batch
    sou, tar, mark, ast_change, sub_token = (t.to(dev) for t in (sou, tar, mark, ast_change, sub_token))
    bf16 = m.precision == "bf16"
    if bf16:
        _optim.ensure_fresh(m)
    m.decoder.prefetch_weights()
    pf_head = ops.prefetch_head(bf16, m.out_fc.weight, m.copy_net.LinearSource.weight, m.copy_net.LinearTarget.weight)
    memory = m.encoder.encode_memory(sou, mark, ast_change, edge, sub_token)
    mem_mask = torch.cat((sou != 0, sub_token != 0), dim=1)
    dec = m.decoder(tar, memory, mem_mask, tar != 0)
    kd = torch.empty(label.numel(), dtype=torch.float32, device=dev)
    loss, nll, _ = ops.HeadFn.apply(False, bf16, pf_head, memory, dec, _u8(mem_mask), _i32(label).view(-1),
                                    m.out_fc.weight, m.out_fc.bias, *m.copy_net.flat_params(), None, None,
                                    (*targets, float(alpha), kd))
    return loss, nll, kd


def distill_step(model, optimizer, batch, teacher, *, alpha):
    """One distillation step on the padded batch (the 8-tuple of run_model.py on the model's device) -> Step(per-token
    loss, nll and kd, tokens).  The student runs in training mode (the kernels' dropout) and stays in it; the
    teacher's members are left in eval mode.  Settings and teacher are checked on the host before any device work."""
    check_alpha(alpha)
    refuse(model, "distill_step")
    teacher_members(teacher, model)
    dev = model.out_fc.weight.device
    label = model.shifted_label(batch[6].to(dev))
    targets = teacher_targets(teacher, batch, label)
    model.train()
    optimizer.zero_grad()
    loss_sum, nll, kd = distill_loss(model, batch, targets, label, alpha)
    tokens = (label != 0).sum()
    (loss_sum / tokens).backward()
    optimizer.step()
    bump_weights(model)                   # the decoding loops' cached weight operands follow the eager step
    n = int(tokens.item())
    d = max(n, 1)
    return Step(loss_sum.item() / d, float(nll.sum().item()) / d, float(kd.sum().item()) / d, n)
