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
from ._lib import FIRA_F32, call
from .ensemble import Ensemble, members
from .incremental import IncrementalDecoder, replay_or_capture, weights_key
from .knn import KNNModel, base_model, search_into, workspace_bytes

D = ops.D
POLL_EVERY = 8            # positions between two reads of the all-finished flag


def _f32(x):
    return ctypes.c_float(x).value


def is_int(v):
    return isinstance(v, int) and not isinstance(v, bool)


def check_tar_len(model, tar_len):
    """ValueError when the decoder (of any member of an ensemble) has fewer than tar_len positions (called before any
    device work)."""
    for m in members(base_model(model)):
        if tar_len > m.decoder.pos_encode.shape[0]:
            raise ValueError(f"tar_len {tar_len} exceeds the decoder's {m.decoder.pos_encode.shape[0]} positions")


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


MAX_PHRASES = MAX_PHRASE_LEN = 4    # head.cu kPhrases / kPhraseLen


def check_constraints(constraints, B, *, V, tar_len, start_id, eos_id, pad_id, groups=1):
    """Validates lexical constraints (called before any device work) -> int32 [B, 4, 4] on the host (zero-padded), or
    None for constraints=None.

    constraints: an integer tensor [B, P <= 4, L <= 4] of vocabulary ids, commit b's phrases; 0 ends a phrase (an
    all-zero phrase is none).  ValueError for a wrong dtype or shape, a nonzero id after a 0 inside a phrase, an id
    outside [0, V), <start>, <eos> or pad_id, more than tar_len - 2 words in one commit (every word needs a position
    before <eos>), tar_len > 32 (the step keeps a row's history in shared memory) and groups > 1 (diverse groups take no
    constraints)."""
    if constraints is None:
        return None
    if not is_int(groups) or groups != 1:
        raise ValueError(f"constraints apply to plain n-best only (groups = 1), got groups={groups!r}")
    if tar_len > MAX_RULES_TAR_LEN:
        raise ValueError(f"constraints need tar_len <= {MAX_RULES_TAR_LEN}, got {tar_len}")
    if not torch.is_tensor(constraints) or constraints.dtype == torch.bool or constraints.is_floating_point() or \
            constraints.is_complex():
        raise ValueError(f"constraints must be an integer tensor, got {getattr(constraints, 'dtype', type(constraints))}")
    if constraints.dim() != 3 or constraints.shape[0] != B or not 1 <= constraints.shape[1] <= MAX_PHRASES or \
            not 1 <= constraints.shape[2] <= MAX_PHRASE_LEN:
        raise ValueError(f"constraints must have shape [B={B}, P <= {MAX_PHRASES}, L <= {MAX_PHRASE_LEN}], got "
                         f"{tuple(constraints.shape)}")
    c = constraints.detach().to("cpu", torch.int64)
    nz = c != 0
    if (nz[:, :, 1:] & ~nz[:, :, :-1]).any():
        raise ValueError("constraints: a nonzero id follows a 0 inside a phrase (a 0 ends a phrase)")
    if ((c < 0) | (c >= V)).any():
        raise ValueError(f"constraints: ids must be in [0, V = {V})")
    for name, i in (("<start>", start_id), ("<eos>", eos_id), ("pad_id", pad_id)):
        if i != 0 and (c == i).any():
            raise ValueError(f"constraints: {name} ({i}) cannot be required")
    tc = nz.sum((1, 2))
    if (tc > tar_len - 2).any():
        raise ValueError(f"constraints: at most tar_len - 2 = {tar_len - 2} words per commit, got {int(tc.max())}")
    out = torch.zeros((B, MAX_PHRASES, MAX_PHRASE_LEN), dtype=torch.int32)
    out[:, :c.shape[1], :c.shape[2]] = c.to(torch.int32)
    return out


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


def encode_members(model, sou, mark, ast_change, edge, sub_token, pad_id):
    """encode() with every member of an ensemble (one model: itself) -> ([memory per member], mem_mask, copy_src)."""
    out = [encode(m, sou, mark, ast_change, edge, sub_token, pad_id) for m in members(base_model(model))]
    return [o[0] for o in out], out[0][1], out[0][2]


class _Head:
    """One model's part of a position: its IncrementalDecoder and the buffers its output head writes (src = the
    memory's LinearSource projection, logits, tgt, gate logits gl, copy scores sc)."""

    def __init__(self, model, B, N, T, S, share=None):
        self.model = model
        self.inc = IncrementalDecoder(model.decoder, B, N, T, S, graphs=False, share=share)   # launches go into our graphs
        self.pr = ops.Prec(self.inc.be.bf16)
        dev = model.out_fc.weight.device
        R, tdt = B * N, self.inc.be.tdt
        self.src = torch.empty((B * S, D), dtype=tdt, device=dev)
        self.logits = torch.empty((R, ops._ld_logits(model.vocab_size)), dtype=tdt, device=dev)
        self.tgt = torch.empty((R, D), dtype=tdt, device=dev)
        self.gl = torch.empty((R, 2), dtype=torch.float32, device=dev)
        self.sc = torch.empty((B, N, S), dtype=torch.float32, device=dev)

    def start(self, memory, mem_mask):
        self.inc.start(memory, mem_mask)
        mem2 = memory.contiguous().to(self.inc.be.tdt).view(self.src.shape[0], D)
        self.pr.linear(mem2, self.model.copy_net.LinearSource.weight, out=self.src)     # once per batch, not per row

    def run(self, t, mem_mask, B, N, S):
        """logits, copy scores and gate logits of decoder row t (every launch on the current stream: capturable)."""
        m, pr = self.model, self.pr
        cn = m.copy_net
        x = self.x = self.inc.advance(t)                                         # [R, D]; a kNN loop's queries
        pr.linear(x, m.out_fc.weight, m.out_fc.bias, out=self.logits, ld_out=self.logits.shape[1])
        pr.linear(x, cn.LinearTarget.weight, out=self.tgt)
        ops.linear(x.float() if pr.bf16 else x, cn.LinearProb.weight, cn.LinearProb.bias, out=self.gl)   # fp32 gate
        p = ops._ptr
        call("fira_copy_scores_fwd", p(self.src), p(self.tgt), p(cn.LinearRes.weight), p(cn.LinearRes.bias),
             p(mem_mask), None, p(self.sc), B, N, S, D, pr.code, ops._stream())

    def refresh_weights(self):
        if self.pr.bf16:
            _optim.ensure_fresh(self.model)
            for W, W16 in self.pr.wcache.values():
                W16.copy_(W.detach())


class PositionLoop:
    """Static buffers, slot state and captured position graphs of one (model, B, N, tar_len, S, precision).

    Slot state: seq, raw, tlp [halves, R, T] and length, lp, status [halves, R] (status 0 live, 1 finished); position t
    reads half t % halves.  Subclasses set `halves` and define position(t, *cfg) (head(t), then their own launches;
    every launch on the current stream), passing logits / sc / gl with dtype code `code` to their step kernel.

    An ensemble.Ensemble gets one _Head per member.  The members decode the same tokens, so their decoders share the
    first one's token buffer and pad mask (`inc`, which the step kernels write); reorder() moves every member's KV
    cache and the shared mask once.  head(t) runs the members one after another, then fira_pointer_mix_ensemble writes
    the averaged triple into the loop's own fp32 logits / sc / gl.  One model is one _Head whose buffers are the
    loop's, with no combine.  A knn.KNNModel is its model's _Head, then fira_knn_search of the decoder row and
    fira_pointer_mix_knn into the loop's own fp32 triple, with lam / tau in a device buffer written at start()."""

    halves = 1

    def __init__(self, model, B, N, T, S):
        self.model, self.B, self.N, self.T, self.S = model, B, N, T, S
        ms = members(base_model(model))
        self.heads = [_Head(ms[0], B, N, T, S)]
        self.heads += [_Head(m, B, N, T, S, share=self.heads[0].inc) for m in ms[1:]]
        h0 = self.heads[0]
        self.inc, self.pr = h0.inc, h0.pr
        self.dev = dev = ms[0].out_fc.weight.device
        R = self.R = B * N
        self.V = model.vocab_size
        self.ldl = ops._ld_logits(self.V)
        self.mem_mask = torch.zeros((B, S), dtype=torch.uint8, device=dev)
        self.copy_src = torch.zeros((B, S), dtype=torch.int32, device=dev)
        self.ensemble = isinstance(model, Ensemble)
        self.knn = isinstance(model, KNNModel)
        if self.knn:
            f32 = dict(dtype=torch.float32, device=dev)
            self.logits = torch.empty((R, self.ldl), **f32)
            self.gl = torch.empty((R, 2), **f32)
            self.sc = torch.empty((B, N, S), **f32)
            self.code = FIRA_F32
            self.store, self.k = model.datastore, model.k      # the loop holds the datastore its graphs read
            self.knn_idx = torch.empty((R, self.k), dtype=torch.int32, device=dev)
            self.knn_dist = torch.empty((R, self.k), **f32)
            self.knn_ws = torch.empty(workspace_bytes(R, self.k, dev), dtype=torch.uint8, device=dev)
            self.knn_params = torch.zeros(2, **f32)           # (lam, tau), read by the captured combine
            self.knn_settings = (model.lam, model.temperature)  # loop_for sets the calling KNNModel's
        elif self.ensemble:
            f32 = dict(dtype=torch.float32, device=dev)
            self.logits = torch.empty((R, self.ldl), **f32)
            self.gl = torch.empty((R, 2), **f32)
            self.sc = torch.empty((B, N, S), **f32)
            self.code = FIRA_F32
            self.log_w = torch.zeros(len(ms), **f32)
            self.log_weights = model.log_weights           # loop_for sets the calling ensemble's; start() writes them
            M = len(ms)
            self._members = tuple((ctypes.c_void_p * M)(*[ops._ptr(getattr(h, k)) for h in self.heads])
                                  for k in ("logits", "sc", "gl"))
        else:
            self.logits, self.gl, self.sc, self.code = h0.logits, h0.gl, h0.sc, self.pr.code
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
        """memory: encode_members' list (one encoder memory per member); prefix: None or check_prefix's host pair
        (prefix [B, T], prefix_len [B])."""
        inc = self.inc
        if prefix is None:
            self.prefix.zero_()
            self.prefix_len.zero_()
        else:
            self.prefix.copy_(prefix[0])
            self.prefix_len.copy_(prefix[1])
        for h, mem in zip(self.heads, memory):
            h.start(mem, mem_mask)
        if self.knn:
            self.knn_params.copy_(torch.tensor(self.knn_settings, dtype=torch.float32))
        if self.ensemble:
            self.log_w.copy_(torch.tensor(self.log_weights, dtype=torch.float32))
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
        for h in self.heads:
            h.refresh_weights()

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
        B, N, S = self.B, self.N, self.S
        for h in self.heads:
            h.run(t, self.mem_mask, B, N, S)
        if self.ensemble:
            lg, sc, gl = self._members
            p = ops._ptr
            call("fira_pointer_mix_ensemble", ctypes.addressof(lg), self.heads[0].logits.shape[1], ctypes.addressof(sc),
                 ctypes.addressof(gl), len(self.heads), p(self.log_w), p(self.mem_mask), p(self.logits), self.ldl,
                 p(self.sc), p(self.gl), B, N, self.V, S, self.pr.code, ops._stream())
        elif self.knn:
            h, p = self.heads[0], ops._ptr
            search_into(self.store, h.x, self.k, self.knn_ws, self.knn_idx, self.knn_dist)
            call("fira_pointer_mix_knn", p(h.logits), h.logits.shape[1], p(h.sc), p(h.gl), p(self.mem_mask),
                 p(self.knn_idx), p(self.knn_dist), p(self.store.words), self.k, p(self.knn_params), p(self.logits),
                 self.ldl, p(self.sc), p(self.gl), B, N, self.V, S, self.pr.code, ops._stream())

    def reorder(self, parent):
        """Row r of every member's KV cache and of the shared pad mask continues row parent[r] (n-best)."""
        self.inc.reorder(parent)
        for h in self.heads[1:]:
            h.inc.reorder(parent, tok_mask=False)       # the mask is the first decoder's, already moved

    def run(self, cfg):
        """Positions 0..T-2 (fewer once every row has finished) -> the number of positions run."""
        t = 0
        while t < self.T - 1:
            if t and t % POLL_EVERY == 0 and not bool(self.unfinished(t)):
                break
            replay_or_capture(self.graphs, (cfg, t), lambda: self.position(t, *cfg))
            t += 1
        return t


def drop_loops(model):
    """Forget the cached loops (buffers and captured graphs) of `model`: a TransModel or an Ensemble drops every loop
    of its first member, a KNNModel only the loops over its datastore, which releases the datastore and the search
    workspace those loops hold.  The next decode captures its graphs again."""
    ms = members(base_model(model))
    store = _LOOPS.get(ms[0])
    if store is None:
        return
    if isinstance(model, KNNModel):
        for key in [k for k in store if "knn" in k and k[k.index("knn") + 1] == id(model.datastore)]:
            del store[key]
    else:
        del _LOOPS[ms[0]]


_LOOPS = weakref.WeakKeyDictionary()   # model (an ensemble's first member) -> {key: (weights keys, addresses, loop)}


def loop_for(cls, model, B, N, T, S):
    """The cached `cls` instance of this shape.  Weights updated in place (a new weights_key, every parameter at the
    address the graphs captured) are refreshed inside the loop, whose position graphs keep replaying: a training loop
    that samples after every optimizer step (scst.py) does not recapture them.  A parameter that moved rebuilds the
    loop (fresh operand copies and graphs).  An ensemble is keyed by its members, not by the Ensemble object: a new
    Ensemble of the same models replays the same graphs, with its own weights written at start().  A KNNModel is keyed
    by its model, its Datastore object (with the addresses of the keys, norms and words its graphs read) and k: a new
    KNNModel over the same model and datastore replays the same graphs, with its own lam / tau written at start().
    A cached kNN loop holds its datastore and search workspace for as long as the model lives; drop_loops releases
    them."""
    ms = members(base_model(model))
    store = _LOOPS.setdefault(ms[0], {})
    key = (cls, B, N, T, S, ms[0].precision)
    if isinstance(model, Ensemble):        # the loop holds its members, so their ids stay theirs while it is cached
        key += (tuple(id(m) for m in ms),)
    if isinstance(model, KNNModel):        # the loop holds the datastore, so its id stays its own while cached
        st = model.datastore
        key += ("knn", id(st), st.keys.data_ptr(), st.norms.data_ptr(), st.words.data_ptr(), st.N, model.k)
    wkey = tuple(weights_key(m, m.decoder) for m in ms)
    addr = tuple(p.data_ptr() for m in ms for p in m.parameters())
    cur = store.get(key)
    if cur is None or cur[1] != addr:
        store[key] = (wkey, addr, cls(model, B, N, T, S))
    elif cur[0] != wkey:
        cur[2].refresh_weights()
        store[key] = (wkey, addr, cur[2])
    loop = store[key][2]
    if isinstance(model, Ensemble):
        loop.log_weights = model.log_weights
    if isinstance(model, KNNModel):
        loop.knn_settings = (model.lam, model.temperature)
    return loop
