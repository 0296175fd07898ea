"""Beam search with the reference's exact ranking semantics (run_model.py:187-380), batched on the GPU.

What is kept from the reference:
  * beam 0 starts with probability 1, the others 0; scores are PRODUCTS of probabilities in fp32;
  * a finished beam (last token <eos>) re-enters the ranking with its stored probability through
    `beam_size` extra candidate slots (-1 when absent), unfinished rows of finished samples are -1;
  * candidates = [live beams x (vocab + 210 + 160)] ++ [finished-beam slots], ranked by
    torch.sort(descending=True), top `beam_size` kept; copy ids are mapped back to vocabulary ids
    through the commit's own diff / sub-token ids; the loop stops when every beam of every sample ended.
What changes: the encoder memory is computed once, ALL live beams go through the decoder in one
batched call, and only position `step` is pushed through the output head (the reference recomputes the
full 30 x 25,020 distribution per beam and reads one row of it).  mode="graph" evaluates only the newest decoder row
per step against cached keys/values (incremental.IncrementalDecoder), replaying each step's kernels as a CUDA graph
(the first batch of a shape runs them eagerly and captures them); mode="full" re-runs the 30-position decoder every
step, and is the only mode for beam sizes above 32 (the incremental cross-attention has at most 32 query rows).
The default comes from FIRA_BEAM_MODE (default "graph").  Ranking keeps the reference's candidate layout; only
the first `beam_size` entries of its descending sort are ever used, so the sort is a device top-k.

`nbest` is beam search in log space with length normalisation, decoded on the device, returning every commit's K
hypotheses with their scores (`beam_search` stays the reference-exact default):

    lp_j = log(clamp(P_j, 1e-10, 1))   (P_j the dual-copy mixture; = -nll of the training loss for label j)
    candidates: every vocabulary entry and every unmasked copy position (masked copy positions never)
    position 0: only slot 0 is live (L = 0); slots 1..K-1 are inactive and propose nothing
    a live slot i (log-probability sum L_i, n_i generated tokens) proposes (i, j): L = L_i + lp_j (fp32), n = n_i + 1;
    a finished slot (its last token <eos>) proposes itself unchanged, once, as j = C = V + S
    score = L / ((5 + n) / 6) ** length_penalty (fp32, powf): length_penalty = 0 ranks by L, the reference's
    ranking in log space, so it cannot underflow to 0 the way products of probabilities do
    the K best by (score descending, then i * (C + 1) + j ascending) become the new slots, in that order
    copies become vocabulary ids through the commit's own sou / sub_token; stop when every slot of every commit has
    finished, or after tar_len - 1 positions.
A vocabulary candidate and a copy candidate that spell the same word stay two candidates (as in the reference), so an
n-best list can hold the same message twice.

Diverse n-best (`groups` G > 1, `diversity` lambda; diverse beam search, Vijayakumar et al., 2018): the K slots form G
groups of Kg = K / G, group g owning slots g * Kg .. (g + 1) * Kg - 1; at position 0 slot g * Kg of every group is live.
At every position the groups choose in order, each with the rule above restricted to its own slots (the Kg best become
its slots, parents inside the group), ranking by score - lambda * h_g(token) where h_g(w) counts the slots of groups
0..g-1 that grew at this position with word w (a copy's word is copy_src[b, j - V], so a copy and the vocabulary entry
spelling the same word are penalised alike; a carried finished slot counts nothing and proposes its stored score
unpenalised).  The penalty only ranks: logprob, token_logprob and score are the quantities above.  Each commit's K
hypotheses are returned stably sorted by score, best first.  groups = 1 is plain n-best (the same code path);
diversity = 0 makes every group an independent nbest(beam_size=Kg).

Prefix-constrained n-best (`prefix`): while a commit is inside its prefix, each live slot's row stage proposes only
the prefix label (with its true lp); since only slot 0 (each group's first slot) is live at position 0, that slot
grows with the prefix and the search branches at the commit's first free position.  logprob, token_logprob and
score cover the prefix, and the length penalty's n counts it.  A prefix may not hold <eos> and leaves at least one
free position: a commit that never branched would keep K - 1 inactive slots with score 0.

n-gram repeat blocking and minimum length (`no_repeat_ngram` n, `min_length` m; 0 = off; DESIGN.md §9): at position
pos a live, non-forced slot's words are its history after <start> (a copy counts as its word, prefix words count); a
candidate whose word would complete an n-gram already in that history, or is <eos> while the slot has fewer than m
words, is never offered to the row stage's top K.  The select stage is unchanged, lp and score stay the model's, and a
slot with fewer than K allowed entries proposes fewer.  A hypothesis can still end unfinished at tar_len.

Lexically constrained n-best (`constraints`; dynamic beam allocation, Post & Vilar, 2018; DESIGN.md §9): each commit
requires up to 4 phrases of up to 4 vocabulary ids (Tc words in all).  A phrase's progress on a slot's words (its
history after <start>, copies as their words, prefix words included) is its length when it occurs contiguously, else
the longest start of it the words end with; a slot meets its constraints when the progress summed over the phrases is
Tc, and <eos> is banned until it does.  Besides its K best allowed labels, a live slot proposes, per phrase it has not
met, the best label spelling that phrase's next word (the vocabulary entry or a copy of it).  Each candidate's bank is
the progress with its word appended.  With Tc > 0 the carried finished slots are kept first, then the other slots are
filled by striping over the banks: within each bank the candidates are ranked by (score, index), and the ranks are
taken in order, higher banks first on a tie.  Tc = 0 is plain n-best.  Every finished hypothesis meets its
constraints; one that reaches tar_len unfinished may not.  Each commit's K hypotheses are returned stably sorted by
(meets its constraints, score), best first (`constraints_met`).

The loop is decode_loop.PositionLoop (described there); a position ends with fira_pointer_mix_beam_step (per live slot
row its top K, then per commit the merge, writing the new slots, their parents and the next tokens), the KV-cache
reorder to the parents and the pad mask of the next tokens.  Slot state is double-buffered by the parity of the
position (a slot's new history comes from another row).
"""
import math
import os
import weakref
from typing import NamedTuple

import torch

from . import ops
from ._lib import call
from .decode_loop import (MAX_PHRASE_LEN, MAX_PHRASES, PositionLoop, _f32, check_constraints, check_prefix, check_rules,
                          check_tar_len, encode, encode_members, is_int, loop_for)
from .ensemble import refuse
from .incremental import IncrementalDecoder

MAX_BEAM = 16             # the row stage keeps a per-thread top K in registers


_DECODERS = weakref.WeakKeyDictionary()          # model -> {(B, K, ...): IncrementalDecoder}


def _incremental_decoder(model, B, K, tar_len, mem_len):
    """IncrementalDecoder instances (static buffers, captured graphs) are kept per model and shape."""
    store = _DECODERS.setdefault(model, {})
    key = (B, K, tar_len, mem_len, model.precision)
    if key not in store:
        store[key] = IncrementalDecoder(model.decoder, B, K, tar_len, mem_len, graphs=True)
    return store[key]


@torch.no_grad()
def beam_search(model, sou, mark, ast_change, edge, sub_token, *, beam_size=3, tar_len=30, start_id, eos_id,
                pad_id=0, mode=None):
    """-> (sequences [B, beam, tar_len] int64 padded with pad_id, lengths [B, beam], probs [B, beam])."""
    refuse(model, "beam_search")
    mode = mode or os.environ.get("FIRA_BEAM_MODE", "graph")
    if mode not in ("full", "graph"):
        raise ValueError("beam search mode must be 'full' or 'graph'")
    memory, mem_mask, copy_src = encode(model, sou, mark, ast_change, edge, sub_token, pad_id)
    dev = memory.device
    B, K = memory.shape[0], beam_size
    V = model.vocab_size
    C = V + copy_src.shape[1]

    seq = torch.full((B, K, tar_len), pad_id, dtype=torch.long, device=dev)
    seq[:, :, 0] = start_id
    length = torch.ones((B, K), dtype=torch.long, device=dev)
    prob = torch.zeros((B, K), dtype=torch.float32, device=dev)
    prob[:, 0] = 1.0
    ar = torch.arange(B, device=dev)
    inc = None
    if mode == "graph":
        inc = _incremental_decoder(model, B, K, tar_len, memory.shape[1]).start(memory, mem_mask)

    for step in range(tar_len - 1):
        last = seq.gather(2, (length - 1).unsqueeze(-1)).squeeze(-1)
        finished = last == eos_id                                                       # [B, K]
        live = [j for j, done in enumerate(finished.all(0).tolist()) if not done]      # one host sync per step
        if not live:
            break
        n_live = len(live)
        live_t = torch.tensor(live, device=dev)
        mem_rep = memory.unsqueeze(1).expand(B, n_live, -1, -1).reshape(B * n_live, memory.shape[1], -1)
        mask_rep = mem_mask.unsqueeze(1).expand(B, n_live, -1).reshape(B * n_live, -1)
        if inc is None:
            tokens = seq[:, live_t].reshape(B * n_live, tar_len)
            dec = model.decoder(tokens, mem_rep, mask_rep, tokens != pad_id)[:, step:step + 1]   # only row `step`
        else:                                          # newest row of every beam against the K/V caches
            row = inc.step(seq[:, :, step].reshape(B * K), step, pad_id)
            dec = row.view(B, K, -1)[:, live_t].reshape(B * n_live, 1, -1)
        gen = torch.softmax(model.out_fc(dec), dim=-1)
        copy, gate = model.copy_net(mem_rep, dec)
        copy = torch.softmax(copy.masked_fill(~mask_rep.unsqueeze(1), -1e9), dim=-1)
        dist = torch.cat((gate[:, :, 0:1] * gen, gate[:, :, 1:2] * copy), dim=-1).view(B, n_live, C)
        dist = dist * prob[:, live_t].unsqueeze(-1)
        dist = dist.masked_fill(finished[:, live_t].unsqueeze(-1), -1.0)
        # finished beams, in beam order, padded with -1 (run_model.py:284-298)
        order = torch.argsort((~finished).to(torch.int8), dim=1, stable=True)            # finished first, stable
        n_fin = finished.sum(1, keepdim=True)
        slot_ok = torch.arange(K, device=dev).unsqueeze(0) < n_fin
        ends_prob = torch.where(slot_ok, prob.gather(1, order), torch.full_like(prob, -1.0))
        cand = torch.cat((dist.view(B, n_live * C), ends_prob), dim=1)
        top_p, top_i = torch.topk(cand, K, dim=-1)          # == sort(descending=True)[:K] (run_model.py:300-303)
        which_beam = top_i // C
        which_tok = top_i % C
        carried = which_beam == n_live                                                   # "keep a finished beam"
        src_beam = torch.where(carried, order.gather(1, which_tok.clamp(max=K - 1)),
                               live_t[which_beam.clamp(max=n_live - 1)])
        tok = torch.where(which_tok >= V, copy_src.gather(1, (which_tok - V).clamp(min=0, max=copy_src.shape[1] - 1)),
                          which_tok)
        new_seq = seq[ar.unsqueeze(1), src_beam]                                         # [B, K, T]
        new_len = length.gather(1, src_beam)
        grow = ~carried
        pos = new_len.clamp(max=tar_len - 1)
        cur = new_seq.gather(2, pos.unsqueeze(-1)).squeeze(-1)
        new_seq.scatter_(2, pos.unsqueeze(-1), torch.where(grow, tok, cur).unsqueeze(-1))
        seq, length, prob = new_seq, new_len + grow.long(), top_p
        if inc is not None:
            inc.reorder((ar.unsqueeze(1) * K + src_beam).reshape(-1))
    return seq, length, prob


def best_sequences(seq, length, prob):
    """run_model.py:351: the beam with the largest probability (first one on ties, like np.argmax)."""
    best = torch.argmax(prob, dim=1)
    ar = torch.arange(seq.shape[0], device=seq.device)
    return seq[ar, best], length[ar, best]


class Hypotheses(NamedTuple):
    seq: torch.Tensor             # [B, K, T] int64 vocabulary ids: <start>, the tokens, pad after <eos>; best first
    raw: torch.Tensor             # [B, K, T] int64 raw indices (label encoding: V + memory position for a copy)
    length: torch.Tensor          # [B, K] int64 tokens including <start> and <eos>
    logprob: torch.Tensor         # [B, K] fp32 sum of token_logprob
    score: torch.Tensor           # [B, K] fp32 logprob / ((5 + length - 1) / 6) ** length_penalty, non-increasing
    token_logprob: torch.Tensor   # [B, K, T] fp32 log(clamp(P, 1e-10, 1)) of each token, 0 at 0 and after <eos>
    finished: torch.Tensor        # [B, K] bool: the hypothesis ends with <eos>


def _finite_f32(x):
    return not isinstance(x, bool) and isinstance(x, (int, float)) and 0.0 <= _f32(x) < math.inf


def check_nbest_args(beam_size, length_penalty, tar_len, groups=1, diversity=0.0):
    """ValueError for any parameter nbest cannot honour (called before any device work)."""
    if not is_int(beam_size) or not 1 <= beam_size <= MAX_BEAM:
        raise ValueError(f"beam_size must be an integer in [1, {MAX_BEAM}], got {beam_size!r}")
    if not _finite_f32(length_penalty):
        raise ValueError(f"length_penalty must be a finite number >= 0 (in fp32), got {length_penalty!r}")
    if not is_int(tar_len) or tar_len < 2:
        raise ValueError(f"tar_len must be an integer >= 2, got {tar_len!r}")
    if not is_int(groups) or groups < 1 or beam_size % groups:
        raise ValueError(f"groups must be an integer >= 1 that divides beam_size {beam_size}, got {groups!r}")
    if not _finite_f32(diversity):
        raise ValueError(f"diversity must be a finite number >= 0 (in fp32), got {diversity!r}")


class _NBest(PositionLoop):
    """Double-buffered slot state (half t & 1 read at position t; status 2: inactive) on top of the shared position
    loop, with each slot's score, its parent row and the row stage's workspace."""

    halves = 2

    def __init__(self, model, B, K, T, S):
        super().__init__(model, B, K, T, S)
        R, dev = self.R, self.dev
        self.score = torch.empty((2, R), dtype=torch.float32, device=dev)
        self.parent = torch.empty(R, dtype=torch.int64, device=dev)
        self.work = torch.empty(R * K, dtype=torch.int64, device=dev)         # per-row top K rank keys (uint64)

    def start(self, memory, mem_mask, copy_src, start_id, pad_id, prefix=None):
        super().start(memory, mem_mask, copy_src, start_id, pad_id, prefix)
        self.score[0].zero_()
        self.status[0].view(self.B, self.N)[:, 1:] = 2          # beam 0 has probability 1, the others 0

    def position(self, t, length_penalty, eos_id, pad_id, no_repeat_ngram, min_length):
        """Slots of position t + 1 from decoder row t (every launch on the current stream: capturable)."""
        self.head(t)
        p = ops._ptr
        inc = self.inc
        call("fira_pointer_mix_beam_step_rules", p(self.logits), self.ldl, p(self.sc), p(self.gl), p(self.mem_mask),
             p(self.copy_src), float(length_penalty), int(eos_id), int(pad_id), p(self.work), p(self.seq), p(self.raw),
             p(self.tlp), p(self.length), p(self.lp), p(self.score), p(self.status), p(self.parent), p(inc.tok),
             self.T, t, self.B, self.N, self.V, self.S, self.code, ops._stream(), p(self.prefix), self.T,
             p(self.prefix_len), int(no_repeat_ngram), int(min_length))
        # caches follow the parents BEFORE the pad mask of the new tokens is written (reorder moves tok_mask rows too)
        self.reorder(self.parent)
        inc.tok_mask[:, t + 1].copy_(inc.tok[:self.R] != pad_id)


class _LexicalNBest(_NBest):
    """_NBest with lexical constraints: the commits' phrases in a static buffer (written at start, read by every captured
    position) and a row-stage workspace of K + 4 keys per row (the K best labels, then one per unmet phrase)."""

    def __init__(self, model, B, K, T, S):
        super().__init__(model, B, K, T, S)
        self.work = torch.empty(self.R * (K + MAX_PHRASES), dtype=torch.int64, device=self.dev)
        self.constraints = torch.zeros((B, MAX_PHRASES, MAX_PHRASE_LEN), dtype=torch.int32, device=self.dev)

    def start(self, memory, mem_mask, copy_src, start_id, pad_id, constraints, prefix=None):
        super().start(memory, mem_mask, copy_src, start_id, pad_id, prefix)
        self.constraints.copy_(constraints)

    def position(self, t, length_penalty, eos_id, pad_id, no_repeat_ngram, min_length):
        self.head(t)
        p = ops._ptr
        inc = self.inc
        call("fira_pointer_mix_beam_step_lexical", p(self.logits), self.ldl, p(self.sc), p(self.gl), p(self.mem_mask),
             p(self.copy_src), float(length_penalty), int(eos_id), int(pad_id), p(self.work), p(self.seq), p(self.raw),
             p(self.tlp), p(self.length), p(self.lp), p(self.score), p(self.status), p(self.parent), p(inc.tok),
             self.T, t, self.B, self.N, self.V, self.S, self.code, ops._stream(), p(self.prefix), self.T,
             p(self.prefix_len), int(no_repeat_ngram), int(min_length), p(self.constraints))
        self.reorder(self.parent)
        inc.tok_mask[:, t + 1].copy_(inc.tok[:self.R] != pad_id)


def constraints_met(seq, length, constraints):
    """bool [B, K] on seq's device: hypothesis (b, k) contains every phrase of commit b contiguously among its words
    seq[b, k, 1:length[b, k]].  seq [B, K, T] vocabulary ids (Hypotheses.seq), length [B, K], constraints [B, P, L]
    vocabulary ids with 0 = padding (check_constraints); a commit without phrases meets them."""
    dev = seq.device
    con = constraints.to(dev, torch.long)
    B, K, T = seq.shape
    P, Lc = con.shape[1:]
    col = torch.arange(T, device=dev)
    words = torch.where((col >= 1) & (col < length.to(dev).unsqueeze(-1)), seq.long(), -1)       # -1: no word
    win = torch.cat((words, words.new_full((B, K, Lc - 1), -1)), 2).unfold(2, Lc, 1)          # [B, K, T, Lc]
    care = con != 0                                                                             # [B, P, Lc]
    hit = (win.unsqueeze(2) == con[:, None, :, None, :]) | ~care[:, None, :, None, :]           # [B, K, P, T, Lc]
    return (hit.all(-1).any(-1) | ~care.any(-1).unsqueeze(1)).all(-1)


class _DiverseNBest(_NBest):
    """_NBest with beam groups: the token every slot grew with at the current position (`chosen`, read by the later
    groups' penalty) and the true lp of every row winner next to its rank key."""

    def __init__(self, model, B, K, T, S):
        super().__init__(model, B, K, T, S)
        self.chosen = torch.empty(self.R, dtype=torch.int32, device=self.dev)
        self.work_lp = torch.empty(self.R * K, dtype=torch.float32, device=self.dev)

    def start(self, memory, mem_mask, copy_src, start_id, pad_id, groups, prefix=None):
        super().start(memory, mem_mask, copy_src, start_id, pad_id, prefix)
        status = self.status[0].view(self.B, self.N)
        status.fill_(2)
        status[:, ::self.N // groups] = 0               # slot g * Kg of every group starts live (L = 0)

    def position(self, t, length_penalty, eos_id, pad_id, no_repeat_ngram, min_length, groups, diversity):
        """Slots of position t + 1 from decoder row t: one call, 2 * groups launches on the current stream."""
        self.head(t)
        p = ops._ptr
        inc = self.inc
        call("fira_pointer_mix_diverse_beam_step_rules", p(self.logits), self.ldl, p(self.sc), p(self.gl),
             p(self.mem_mask), p(self.copy_src), float(length_penalty), int(eos_id), int(pad_id), p(self.work),
             p(self.seq), p(self.raw), p(self.tlp), p(self.length), p(self.lp), p(self.score), p(self.status),
             p(self.parent), p(inc.tok), self.T, t, self.B, self.N, self.V, self.S, int(groups), float(diversity),
             p(self.chosen), p(self.work_lp), self.code, ops._stream(), p(self.prefix), self.T, p(self.prefix_len),
             int(no_repeat_ngram), int(min_length))
        self.reorder(self.parent)
        inc.tok_mask[:, t + 1].copy_(inc.tok[:self.R] != pad_id)


@torch.no_grad()
def nbest(model, sou, mark, ast_change, edge, sub_token, *, beam_size=3, length_penalty=0.0, tar_len=30, start_id,
          eos_id, pad_id=0, groups=1, diversity=0.0, prefix=None, no_repeat_ngram=0, min_length=0, constraints=None):
    """Log-space beam search with length normalisation -> Hypotheses, each commit's K best first (module docstring).
    model: a TransModel, or an ensemble.Ensemble (ranked by its averaged distribution).
    groups > 1 splits the K slots into diverse beam groups penalised by `diversity` per earlier-group repeat.
    prefix: None, or labels [B, P] every hypothesis of a commit starts with (decode_loop.check_prefix: the tar_label
    encoding without <start>, a 0 ends a commit's prefix, no <eos>, at most tar_len - 2 labels).
    no_repeat_ngram = n >= 1 / min_length = m >= 1: a slot never extends with a word that completes an n-gram already
    in its hypothesis, nor with <eos> before m words (0 = off; module docstring).
    constraints: None, or vocabulary ids [B, P <= 4, L <= 4] (0 = padding), phrases every finished hypothesis of a
    commit contains (decode_loop.check_constraints; plain n-best only); the hypotheses come sorted by (meets its
    constraints, score), best first (module docstring)."""
    check_nbest_args(beam_size, length_penalty, tar_len, groups, diversity)
    check_rules(no_repeat_ngram, min_length, tar_len)
    con = check_constraints(constraints, sou.shape[0], V=model.vocab_size, tar_len=tar_len, start_id=start_id,
                            eos_id=eos_id, pad_id=pad_id, groups=groups)
    if beam_size > model.vocab_size:
        raise ValueError(f"beam_size {beam_size} exceeds the vocabulary ({model.vocab_size})")
    check_tar_len(model, tar_len)
    pre = check_prefix(prefix, sou, sub_token, V=model.vocab_size, tar_len=tar_len, eos_id=eos_id, pad_id=pad_id,
                       eos_last=False)
    memory, mem_mask, copy_src = encode_members(model, sou, mark, ast_change, edge, sub_token, pad_id)
    B, S = memory[0].shape[:2]
    if con is not None:
        st = loop_for(_LexicalNBest, model, B, beam_size, tar_len, S)
        st.start(memory, mem_mask, copy_src, start_id, pad_id, con, pre)
        t = st.run((float(length_penalty), int(eos_id), int(pad_id), no_repeat_ngram, min_length))
        seq, raw, length, lp, tlp, status = st.slots(t)
        score = st.score[t & 1].view(B, beam_size)
        met = constraints_met(seq, length, st.constraints)
        # (meets descending, score descending), stable: score first, then a stable sort on met
        score, order = torch.sort(score, dim=1, descending=True, stable=True)
        _, o2 = torch.sort(met.gather(1, order).to(torch.int8), dim=1, descending=True, stable=True)
        order, score = order.gather(1, o2), score.gather(1, o2)
        o2, o3 = order, order.unsqueeze(-1).expand_as(seq)
        return Hypotheses(seq.gather(1, o3), raw.gather(1, o3), length.gather(1, o2), lp.gather(1, o2), score,
                          tlp.gather(1, o3), (status == 1).gather(1, o2))
    if groups == 1:
        st = loop_for(_NBest, model, B, beam_size, tar_len, S)
        st.start(memory, mem_mask, copy_src, start_id, pad_id, pre)
        t = st.run((float(length_penalty), int(eos_id), int(pad_id), no_repeat_ngram, min_length))
        seq, raw, length, lp, tlp, status = st.slots(t)
        return Hypotheses(seq, raw, length, lp, st.score[t & 1].view(B, beam_size).clone(), tlp, status == 1)
    st = loop_for(_DiverseNBest, model, B, beam_size, tar_len, S)
    st.start(memory, mem_mask, copy_src, start_id, pad_id, groups, pre)
    t = st.run((float(length_penalty), int(eos_id), int(pad_id), no_repeat_ngram, min_length, int(groups),
                _f32(diversity)))
    seq, raw, length, lp, tlp, status = st.slots(t)
    score = st.score[t & 1].view(B, beam_size)
    score, order = torch.sort(score, dim=1, descending=True, stable=True)        # best first across the groups
    o2, o3 = order, order.unsqueeze(-1).expand_as(seq)
    return Hypotheses(seq.gather(1, o3), raw.gather(1, o3), length.gather(1, o2), lp.gather(1, o2), score,
                      tlp.gather(1, o3), (status == 1).gather(1, o2))
