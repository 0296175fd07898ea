"""The on-device decoding loop shared by seeded sampling (sample.py) and n-best beam search (beam.nbest), and the batch
front end every decoder shares (`encode`, also used by beam.beam_search).

Per batch the encoder, the cross-attention K/V of the memory and LinearSource(memory) run once (`start`).  The N rows
of a commit (samples or beam slots) are the N query rows of an incremental.IncrementalDecoder.  Per position:
newest decoder row -> out_fc -> target projection and gate -> copy scores (`head`), then the decoder's own kernel,
which writes the next input tokens straight into the decoder's token buffer and keeps every row's slot state
(`position`, defined by each decoder).  A position is captured once into a CUDA graph and replayed for every later
batch of the same shape; the loop reads back nothing but an all-finished flag, once every POLL_EVERY positions.
Every position also passes the per-commit prefix buffers (`check_prefix`): a commit still inside its prefix takes the
given label at that position instead of choosing one, inside the step kernel.  The n-gram repeat blocking and minimum
length settings (`check_rules`) are part of a position's cfg key, so each setting replays its own graphs.
"""
import ctypes
import weakref

import torch

from . import ops
from . import optim as _optim
from ._lib import call
from .incremental import IncrementalDecoder, replay_or_capture, weights_key

D = ops.D
POLL_EVERY = 8            # positions between two reads of the all-finished flag


def _f32(x):
    return ctypes.c_float(x).value


def is_int(v):
    return isinstance(v, int) and not isinstance(v, bool)


def check_tar_len(model, tar_len):
    """ValueError when the decoder has fewer than tar_len positions (called before any device work)."""
    if tar_len > model.decoder.pos_encode.shape[0]:
        raise ValueError(f"tar_len {tar_len} exceeds the decoder's {model.decoder.pos_encode.shape[0]} positions")


MAX_RULES_TAR_LEN = 32    # the step kernels hold a row's history in a fixed shared-memory list (head.cu TMAX)


def check_rules(no_repeat_ngram, min_length, tar_len):
    """ValueError for n-gram blocking / minimum length settings the step kernels cannot honour (called before any device
    work).  no_repeat_ngram = n >= 1 bans every word that would repeat an n-gram of the row's history, min_length = m
    bans <eos> while the row has fewer than m words; 0 turns either off.  n > tar_len - 1 or m > tar_len - 2 could never
    apply, or would leave no position for <eos>, so they are refused rather than silently ignored."""
    for name, v in (("no_repeat_ngram", no_repeat_ngram), ("min_length", min_length)):
        if not is_int(v) or v < 0:
            raise ValueError(f"{name} must be an integer >= 0 (0 = off), got {v!r}")
    if no_repeat_ngram > tar_len - 1:
        raise ValueError(f"no_repeat_ngram must be <= tar_len - 1 = {tar_len - 1}, got {no_repeat_ngram}")
    if min_length > tar_len - 2:
        raise ValueError(f"min_length must be <= tar_len - 2 = {tar_len - 2}, got {min_length}")
    if (no_repeat_ngram or min_length) and tar_len > MAX_RULES_TAR_LEN:
        raise ValueError(f"no_repeat_ngram / min_length need tar_len <= {MAX_RULES_TAR_LEN}, got {tar_len}")


def check_prefix(prefix, sou, sub_token, *, V, tar_len, eos_id, pad_id, eos_last):
    """Validates a prefix (called before any device work) -> (prefix int32 [B, tar_len], prefix_len int32 [B]) on the
    host, or None for prefix=None.

    prefix: an integer tensor [B, P] of labels in the tar_label encoding (j < V a vocabulary id, V + s memory position
    s of cat(sou, sub_token)) without <start>; a 0 ends a commit's prefix.  ValueError for a wrong dtype or B, a nonzero
    entry after a 0, a label outside [0, V + S), a copy label at a masked memory position (mem_mask = cat(sou != pad_id,
    sub_token != 0), as `encode` forms it), a pad_id label, and, with eos_last (sample / mbr), <eos> anywhere but as a
    commit's last entry or more than tar_len - 1 entries; without it (nbest), any <eos> or more than tar_len - 2 entries,
    so that every commit has a free position to branch at.  sou / sub_token are read once on the host."""
    if prefix is None:
        return None
    B = sou.shape[0]
    if not torch.is_tensor(prefix) or prefix.dtype == torch.bool or prefix.is_floating_point() or prefix.is_complex():
        raise ValueError(f"prefix must be an integer tensor, got {getattr(prefix, 'dtype', type(prefix))}")
    if prefix.dim() != 2 or prefix.shape[0] != B:
        raise ValueError(f"prefix must have shape [B={B}, P], got {tuple(prefix.shape)}")
    pre = prefix.detach().to("cpu", torch.int64)
    P = pre.shape[1]
    nz = pre != 0
    n = nz.sum(1)                                                           # entries before the first 0, if valid
    if (nz & (torch.arange(P).unsqueeze(0) >= n.unsqueeze(1))).any():
        raise ValueError("prefix: a nonzero label follows a 0 (a 0 ends a commit's prefix)")
    mem_mask = torch.cat((sou.detach().cpu() != pad_id, sub_token.detach().cpu() != 0), dim=1)
    S = mem_mask.shape[1]
    if ((pre < 0) | (pre >= V + S)).any():
        raise ValueError(f"prefix: labels must be in [0, V + S = {V + S})")
    copy = nz & (pre >= V)
    rows = torch.arange(B).unsqueeze(1).expand(B, P)
    if (copy & ~mem_mask[rows, (pre - V).clamp(0, S - 1)]).any():
        raise ValueError("prefix: a copy label points at a masked memory position")
    if pad_id != 0 and (nz & (pre == pad_id)).any():
        raise ValueError(f"prefix: pad_id {pad_id} is not a label")
    eos = nz & (pre == eos_id)
    if eos_last:
        last = torch.arange(P).unsqueeze(0) == (n - 1).unsqueeze(1)
        if (eos & ~last).any():
            raise ValueError("prefix: <eos> may only be a commit's last prefix label")
        longest = tar_len - 1
    else:
        if eos.any():
            raise ValueError("prefix: n-best prefixes cannot contain <eos>")
        longest = tar_len - 2
    if (n > longest).any():
        raise ValueError(f"prefix: at most {longest} labels per commit with tar_len {tar_len}, got {int(n.max())}")
    out = torch.zeros((B, tar_len), dtype=torch.int32)
    w = min(P, tar_len)
    out[:, :w] = pre[:, :w].to(torch.int32)
    return out, n.to(torch.int32)


def encode(model, sou, mark, ast_change, edge, sub_token, pad_id):
    """Encoder memory [B, S, D] on the model's device, once per batch, with the copy mask mem_mask [B, S] (bool) and
    copy_src [B, S] (copy position -> vocabulary id)."""
    dev = model.out_fc.weight.device
    sou, mark, ast_change, sub_token = (t.to(dev) for t in (sou, mark, ast_change, sub_token))
    memory = model.encoder.encode_memory(sou, mark, ast_change, edge, sub_token)
    mem_mask = torch.cat((sou != pad_id, sub_token != 0), dim=1)
    copy_src = torch.cat((sou, sub_token), dim=1)
    return memory, mem_mask, copy_src


class PositionLoop:
    """Static buffers, slot state and captured position graphs of one (model, B, N, tar_len, S, precision).

    Slot state: seq, raw, tlp [halves, R, T] and length, lp, status [halves, R] (status 0 live, 1 finished); position t
    reads half t % halves.  Subclasses set `halves` and define position(t, *cfg) (head(t), then their own launches;
    every launch on the current stream)."""

    halves = 1

    def __init__(self, model, B, N, T, S):
        self.model, self.B, self.N, self.T, self.S = model, B, N, T, S
        self.inc = IncrementalDecoder(model.decoder, B, N, T, S, graphs=False)   # its launches go into our graphs
        self.pr = ops.Prec(self.inc.be.bf16)
        self.dev = dev = model.out_fc.weight.device
        R = self.R = B * N
        tdt = self.inc.be.tdt
        self.V = model.vocab_size
        self.ldl = ops._ld_logits(self.V)
        self.mem_mask = torch.zeros((B, S), dtype=torch.uint8, device=dev)
        self.copy_src = torch.zeros((B, S), dtype=torch.int32, device=dev)
        self.src = torch.empty((B * S, D), dtype=tdt, device=dev)
        self.logits = torch.empty((R, self.ldl), dtype=tdt, device=dev)
        self.tgt = torch.empty((R, D), dtype=tdt, device=dev)
        self.gl = torch.empty((R, 2), dtype=torch.float32, device=dev)
        self.sc = torch.empty((B, N, S), dtype=torch.float32, device=dev)
        H = self.halves
        i32 = dict(dtype=torch.int32, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)
        self.seq = torch.empty((H, R, T), **i32)
        self.raw = torch.empty((H, R, T), **i32)
        self.tlp = torch.empty((H, R, T), **f32)
        self.length = torch.empty((H, R), **i32)
        self.lp = torch.empty((H, R), **f32)
        self.status = torch.empty((H, R), dtype=torch.uint8, device=dev)
        # forced labels per commit (check_prefix); every position passes them to the step kernel, so a batch without a
        # prefix (prefix_len 0) replays the same graphs
        self.prefix = torch.zeros((B, T), **i32)
        self.prefix_len = torch.zeros(B, **i32)
        self.graphs = {}

    def start(self, memory, mem_mask, copy_src, start_id, pad_id, prefix=None):
        """prefix: None or check_prefix's host pair (prefix [B, T], prefix_len [B])."""
        inc = self.inc
        if prefix is None:
            self.prefix.zero_()
            self.prefix_len.zero_()
        else:
            self.prefix.copy_(prefix[0])
            self.prefix_len.copy_(prefix[1])
        inc.start(memory, mem_mask)
        mem2 = memory.contiguous().to(inc.be.tdt).view(self.B * self.S, D)
        self.pr.linear(mem2, self.model.copy_net.LinearSource.weight, out=self.src)     # once per batch, not per row
        self.mem_mask.copy_(mem_mask)
        self.copy_src.copy_(copy_src)
        inc.tok[:self.R].fill_(start_id)
        inc.tok_mask[:, 0].fill_(int(start_id != pad_id))
        for x in (self.seq, self.raw):        # n-best's half 1 is written whole at position 0 (columns > 1 from half 0)
            x[0].fill_(pad_id)
            x[0, :, 0] = start_id
        self.tlp[0].zero_()
        self.length[0].fill_(1)
        self.lp[0].zero_()
        self.status[0].zero_()

    def refresh_weights(self):
        """The parameters changed in place (an optimizer step): refresh the operand copies the captured graphs read, so
        they replay with the new weights.  The decoder's concatenated weights follow in start() (IncrementalDecoder
        compares weights_key); here the bf16 mirror and the bf16 copies of the head's weights.  fp32 mode reads the
        parameters themselves."""
        if self.pr.bf16:
            _optim.ensure_fresh(self.model)
            for W, W16 in self.pr.wcache.values():
                W16.copy_(W.detach())

    def unfinished(self, t):
        """A device bool: some row still decodes after t positions."""
        return self.status[t % self.halves].eq(0).any()

    def slots(self, t):
        """The slot state after t positions: seq, raw [B, N, T] int64, length [B, N] int64, lp [B, N] and
        token log-probabilities [B, N, T] (copies), and status [B, N] (a view)."""
        h, B, N, T = t % self.halves, self.B, self.N, self.T
        return (self.seq[h].view(B, N, T).long(), self.raw[h].view(B, N, T).long(), self.length[h].view(B, N).long(),
                self.lp[h].view(B, N).clone(), self.tlp[h].view(B, N, T).clone(), self.status[h].view(B, N))

    def head(self, t):
        """logits, copy scores and gate logits of decoder row t (every launch on the current stream: capturable)."""
        m, pr, B, N, S = self.model, self.pr, self.B, self.N, self.S
        cn = m.copy_net
        x = self.inc.advance(t)                                                  # [R, D]
        pr.linear(x, m.out_fc.weight, m.out_fc.bias, out=self.logits, ld_out=self.ldl)
        pr.linear(x, cn.LinearTarget.weight, out=self.tgt)
        ops.linear(x.float() if pr.bf16 else x, cn.LinearProb.weight, cn.LinearProb.bias, out=self.gl)   # fp32 gate
        p = ops._ptr
        call("fira_copy_scores_fwd", p(self.src), p(self.tgt), p(cn.LinearRes.weight), p(cn.LinearRes.bias),
             p(self.mem_mask), None, p(self.sc), B, N, S, D, pr.code, ops._stream())

    def run(self, cfg):
        """Positions 0..T-2 (fewer once every row has finished) -> the number of positions run."""
        t = 0
        while t < self.T - 1:
            if t and t % POLL_EVERY == 0 and not bool(self.unfinished(t)):
                break
            replay_or_capture(self.graphs, (cfg, t), lambda: self.position(t, *cfg))
            t += 1
        return t


_LOOPS = weakref.WeakKeyDictionary()   # model -> {(class, B, N, T, S, precision): (weights key, addresses, loop)}


def loop_for(cls, model, B, N, T, S):
    """The cached `cls` instance of this shape.  Weights updated in place (a new weights_key, every parameter at the
    address the graphs captured) are refreshed inside the loop, whose position graphs keep replaying: a training loop
    that samples after every optimizer step (scst.py) does not recapture them.  A parameter that moved rebuilds the
    loop (fresh operand copies and graphs)."""
    store = _LOOPS.setdefault(model, {})
    key = (cls, B, N, T, S, model.precision)
    wkey = weights_key(model, model.decoder)
    addr = tuple(p.data_ptr() for p in model.parameters())
    cur = store.get(key)
    if cur is None or cur[1] != addr:
        store[key] = (wkey, addr, cls(model, B, N, T, S))
    elif cur[0] != wkey:
        cur[2].refresh_weights()
        store[key] = (wkey, addr, cur[2])
    return store[key][2]
