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

Offline distillation: the teacher is frozen and teacher-forced, so its distributions are the same every epoch.
build_targets runs it once over a split and keeps, per loss row, its k most probable labels (fira_pointer_mix_topk:
P descending, then label ascending; Tan et al., ICLR 2019 keep 8) renormalised to t~_i = P_i / mass, mass = the kept
P summed in key order.  A KDTargets holds them; KDTargets.batch gathers a batch's [B*T, k] labels and probabilities,
and distill_step trains against them with fira_pointer_mix_kd_sparse_fwd / _bwd: the loss above with t = t~ at the
kept labels and 0 elsewhere, no teacher run and no teacher memory.
"""
import ctypes
import math
import numbers
from typing import NamedTuple

import numpy as np

import torch

from . import ops
from . import optim as _optim
from ._lib import FIRA_BF16, FIRA_F32, call
from .ensemble import Ensemble, refuse
from .knn import fingerprint
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


MAX_TOPK = 64             # fira_pointer_mix_topk / fira_pointer_mix_kd_sparse_*
FORMAT = "fira-kd-targets-1"


class SparseTargets(NamedTuple):
    """One padded batch's stored teacher targets (KDTargets.batch), on the student's device."""
    t_label: torch.Tensor     # int32 [B*T, k]: vocabulary id j < V or V + copy position; -1 = no entry
    t_prob: torch.Tensor      # fp32 [B*T, k]: t~ of each label (0 for -1)


def check_topk(k):
    """ValueError unless k is an integer in [1, MAX_TOPK] (host only)."""
    if isinstance(k, bool) or not isinstance(k, numbers.Integral) or not 1 <= int(k) <= MAX_TOPK:
        raise ValueError(f"k must be an integer in [1, {MAX_TOPK}], got {k!r}")


def topk_targets(targets, mem_mask, label, V, k):
    """fira_pointer_mix_topk of the teacher's triple (teacher_targets) -> (t_label int32 [B*T, k], t_prob fp32
    [B*T, k], mass fp32 [B*T]) on its device; mem_mask [B, S] uint8, label the shifted labels [B, T]."""
    check_topk(k)
    logits, sc, gl = targets
    B, T, S = sc.shape
    dev = logits.device
    t_label = torch.empty((B * T, k), dtype=torch.int32, device=dev)
    t_prob = torch.empty((B * T, k), dtype=torch.float32, device=dev)
    mass = torch.empty((B * T,), dtype=torch.float32, device=dev)
    lab = _i32(label).reshape(-1).contiguous()
    call("fira_pointer_mix_topk", ops._ptr(logits), logits.stride(0), ops._ptr(sc), ops._ptr(gl), ops._ptr(mem_mask),
         ops._ptr(lab), int(k), ops._ptr(t_label), ops._ptr(t_prob), ops._ptr(mass), B * T, T, V, S, ops._stream())
    return t_label, t_prob, mass


class KDTargets:
    """A split's stored top-k teacher targets (build_targets).  Commit i of the split (dataset position first + i)
    owns rows row_off[i] .. row_off[i + 1] - 1, its loss rows (shifted label y != 0) in position order; per row: pos
    (the target position t) and y, kept to check that a batch is the one the rows were built from, and the kept labels
    t_label [R, k] int32 (-1: none), their renormalised probabilities t_prob [R, k] fp32 and the kept teacher mass
    [R] fp32.  All on the host.  provenance: the teacher members' knn.state_fingerprint, their weights, the precision
    the teacher ran in and the split size.  ValueError for inconsistent shapes or dtypes."""

    def __init__(self, row_off, pos, y, t_label, t_prob, mass, *, vocab_size, k, first, provenance):
        check_topk(k)
        for name, t, dt in (("row_off", row_off, torch.int64), ("pos", pos, torch.int16), ("y", y, torch.int32),
                            ("t_label", t_label, torch.int32), ("t_prob", t_prob, torch.float32),
                            ("mass", mass, torch.float32)):
            if not torch.is_tensor(t) or t.dtype != dt or t.device.type != "cpu":
                raise ValueError(f"KDTargets {name} must be a host {dt} tensor, got {getattr(t, 'dtype', type(t))}")
        R = pos.numel()
        if row_off.dim() != 1 or row_off.numel() < 1 or int(row_off[0]) != 0 or int(row_off[-1]) != R or \
                bool((row_off[1:] < row_off[:-1]).any()):
            raise ValueError("KDTargets row_off must rise from 0 to the row count")
        if tuple(y.shape) != (R,) or tuple(mass.shape) != (R,) or tuple(t_label.shape) != (R, k) or \
                tuple(t_prob.shape) != (R, k):
            raise ValueError(f"KDTargets rows: pos / y / mass [{R}], t_label / t_prob [{R}, {k}], got "
                             f"{tuple(y.shape)}, {tuple(mass.shape)}, {tuple(t_label.shape)}, {tuple(t_prob.shape)}")
        if isinstance(vocab_size, bool) or not isinstance(vocab_size, int) or vocab_size < 1:
            raise ValueError(f"vocab_size must be a positive integer, got {vocab_size!r}")
        self.row_off, self.pos, self.y = row_off.contiguous(), pos.contiguous(), y.contiguous()
        self.t_label, self.t_prob, self.mass = t_label.contiguous(), t_prob.contiguous(), mass.contiguous()
        self.vocab_size, self.k, self.first = vocab_size, int(k), int(first)
        self.provenance = dict(provenance)

    @property
    def n(self):
        """number of commits"""
        return self.row_off.numel() - 1

    @property
    def rows(self):
        return self.pos.numel()

    @property
    def nbytes(self):
        return sum(t.numel() * t.element_size() for t in (self.row_off, self.pos, self.y, self.t_label, self.t_prob,
                                                          self.mass))

    def save(self, path):
        torch.save({"format": FORMAT, "vocab_size": self.vocab_size, "k": self.k, "first": self.first,
                    "provenance": self.provenance, "row_off": self.row_off, "pos": self.pos, "y": self.y,
                    "t_label": self.t_label, "t_prob": self.t_prob, "mass": self.mass}, path)

    @classmethod
    def load(cls, path, *, vocab_size=None, k=None, commits=None):
        """The targets saved at `path`.  ValueError for another file format and a vocabulary size, k or commit count
        other than the given ones (None: not checked)."""
        s = torch.load(path, map_location="cpu", weights_only=True)
        if not isinstance(s, dict) or s.get("format") != FORMAT:
            raise ValueError(f"{path} is not a distillation target file ({FORMAT})")
        n = s["row_off"].numel() - 1
        for name, want, got in (("vocab_size", vocab_size, s["vocab_size"]), ("k", k, s["k"]), ("commits", commits, n)):
            if want is not None and want != got:
                raise ValueError(f"{path}: {name} {got}, expected {want}")
        return cls(*(s[f] for f in ("row_off", "pos", "y", "t_label", "t_prob", "mass")), vocab_size=s["vocab_size"],
                   k=s["k"], first=s["first"], provenance=s["provenance"])

    def batch(self, indices, label, device=None):
        """SparseTargets of the padded batch holding the commits at dataset positions `indices` (in batch order) with
        shifted labels `label` [B, T] (TransModel.shifted_label of its tar_label; host tensors avoid a device
        read-back) -> [B*T, k] labels and probabilities on `device` (default: label's).  ValueError, before anything is
        sent to the device, for a position outside the stored commits or stored rows other than the batch's loss rows
        (another split, order or label encoding)."""
        idx = torch.as_tensor(np.asarray(indices, dtype=np.int64)).view(-1) - self.first
        lab = label.detach().to("cpu")
        B, T = lab.shape
        if idx.numel() != B:
            raise ValueError(f"KDTargets.batch: {idx.numel()} positions for a batch of {B} commits")
        if idx.numel() and (int(idx.min()) < 0 or int(idx.max()) >= self.n):
            raise ValueError(f"KDTargets.batch: a position outside the stored commits {self.first}.."
                             f"{self.first + self.n - 1}")
        live = lab != 0
        lo, hi = self.row_off[idx], self.row_off[idx + 1]
        if not torch.equal(hi - lo, live.sum(1)):
            raise ValueError("KDTargets.batch: the stored row counts differ from the batch's loss rows (a file built "
                             "for another split or order?)")
        src = torch.cat([torch.arange(int(a), int(z)) for a, z in zip(lo, hi)] + [torch.zeros(0, dtype=torch.int64)])
        b, t = live.nonzero(as_tuple=True)
        if not torch.equal(self.pos[src].long(), t) or not torch.equal(self.y[src], lab[b, t].to(torch.int32)):
            raise ValueError("KDTargets.batch: the stored positions or labels differ from the batch's (a file built "
                             "for another split or order?)")
        t_label = torch.full((B * T, self.k), -1, dtype=torch.int32)
        t_prob = torch.zeros((B * T, self.k), dtype=torch.float32)
        dst = b * T + t
        t_label[dst] = self.t_label[src]
        t_prob[dst] = self.t_prob[src]
        dev = label.device if device is None else device
        return SparseTargets(t_label.to(dev), t_prob.to(dev))


@torch.no_grad()
def build_targets(teacher, batches, *, k, first_index):
    """KDTargets from padded batches (the 8-tuples of run_model.py on the teacher's device) that follow one another
    from dataset position first_index: teacher_targets, then fira_pointer_mix_topk, per batch.  Only rows with y != 0
    are stored."""
    check_topk(k)
    models, _ = teacher_members(teacher)
    weights = teacher.weights if isinstance(teacher, Ensemble) else (1.0,)
    V = models[0].vocab_size
    dev = models[0].out_fc.weight.device
    parts, counts = [], []
    for batch in batches:
        label = TransModel.shifted_label(batch[6].to(dev))
        targets = teacher_targets(teacher, batch, label)
        mem_mask = _u8(torch.cat((batch[0] != 0, batch[7] != 0), dim=1).to(dev))
        t_label, t_prob, mass = topk_targets(targets, mem_mask, label, V, k)
        live = (label != 0).view(-1)
        t = torch.arange(label.shape[1], device=dev).expand_as(label).reshape(-1)
        parts.append(tuple(a[live].cpu() for a in (t.to(torch.int16), _i32(label).view(-1), t_label, t_prob, mass)))
        counts.append((label != 0).sum(1).cpu())
    if not parts:
        raise ValueError("build_targets: no batches")
    pos, y, t_label, t_prob, mass = (torch.cat(x) for x in zip(*parts))
    counts = torch.cat(counts)
    row_off = torch.zeros(counts.numel() + 1, dtype=torch.int64)
    row_off[1:] = torch.cumsum(counts, 0)
    provenance = dict(fingerprints=[fingerprint(m) for m in models], weights=[float(w) for w in weights],
                      precision=models[0].precision, commits=counts.numel())
    return KDTargets(row_off, pos, y, t_label, t_prob, mass, vocab_size=V, k=k, first=first_index,
                     provenance=provenance)


def distill_loss(model, batch, targets, label, alpha):
    """sum_r loss_r under autograd in the model's current mode -> (loss_sum, nll [B, T], kd [B*T]).  targets: the
    teacher's triple of teacher_targets, or the batch's SparseTargets; label: the shifted labels [B, T] on the model's
    device."""
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
    if isinstance(targets, SparseTargets):
        dense, sparse = None, (targets.t_label, targets.t_prob, float(alpha), kd)
    else:
        dense, sparse = (*targets, float(alpha), kd), None
    loss, nll, _ = ops.HeadFn.apply(False, bf16, pf_head, memory, dec, _u8(mem_mask), _i32(label).view(-1),
                                    m.out_fc.weight, m.out_fc.bias, *m.copy_net.flat_params(), None, None, dense,
                                    sparse)
    return loss, nll, kd


def check_sparse(targets, model, rows):
    """ValueError unless targets are SparseTargets of `rows` rows and 1..MAX_TOPK labels on the model's device (host
    only)."""
    dev = model.out_fc.weight.device
    a, p = targets
    ok = torch.is_tensor(a) and torch.is_tensor(p) and a.dtype == torch.int32 and p.dtype == torch.float32 and \
        a.dim() == 2 and p.shape == a.shape and a.shape[0] == rows and 1 <= a.shape[1] <= MAX_TOPK
    if not ok:
        raise ValueError(f"sparse targets must be int32 labels and fp32 probabilities [{rows}, k], 1 <= k <= "
                         f"{MAX_TOPK}")
    if a.device != dev or p.device != dev:
        raise ValueError(f"the sparse targets are on {a.device}, the student on {dev}")


def distill_step(model, optimizer, batch, teacher, *, alpha):
    """One distillation step on the padded batch (the 8-tuple of run_model.py on the model's device) -> Step(per-token
    loss, nll and kd, tokens).  teacher: a TransModel or an Ensemble, run on the batch (its members are left in eval
    mode), or the batch's SparseTargets (KDTargets.batch): then no teacher runs.  The student runs in training mode
    (the kernels' dropout) and stays in it.  Settings and teacher are checked on the host before any device work."""
    check_alpha(alpha)
    refuse(model, "distill_step")
    sparse = isinstance(teacher, SparseTargets)
    if sparse:
        check_sparse(teacher, model, batch[6].shape[0] * batch[6].shape[1])
    else:
        teacher_members(teacher, model)
    dev = model.out_fc.weight.device
    label = model.shifted_label(batch[6].to(dev))
    targets = teacher if sparse else teacher_targets(teacher, batch, label)
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
