"""Seeded sampling decoding: temperature, top-k and top-p draws from the dual-copy mixture (Model.py:54-86).

Where beam search keeps the most probable continuations, `sample` draws N independent messages per commit from the
model's distribution and reports the model's own log-probability of every drawn token:

    P_j = g0 * softmax(vocab logits)_j  (j < V)   ||   g1 * softmax(masked copy scores)_s  (j = V + s)
    candidates: P_j > 0 in fp32 and, for copies, mem_mask[b, s] != 0;  s_j = log P_j / temperature
    top_k > 0 keeps the top_k highest s_j (ties: smaller j first); top_p < 1 then keeps the shortest such rank prefix
    whose weight sum(exp(s_j - max s)) reaches top_p of the kept weight; the draw u in [0, 1) picks the smallest kept
    j whose running weight in index order exceeds u * (total kept weight).

u comes from Philox4x32-7 keyed by `seed` with the counter (first_index + b, n, position), so a commit's samples depend
on its position in the dataset, not on the batch it was decoded in or the GPU count.  The emitted log-probability is
log(clamp(P_j, 1e-10, 1)) whatever temperature, top_k and top_p are: it is -nll of the training loss for label j.

The loop is decode_loop.PositionLoop (described there); a position ends with fira_pointer_mix_sample_rules, which also
writes the next input token straight into the decoder's token buffer and keeps each row's finished flag, length and
log-probability sum.  A commit still inside its `prefix` at a position takes the given label there instead of drawing
one (same log-probability expression, same bookkeeping); `score` forces the whole message to return log p(message).
`no_repeat_ngram` / `min_length` remove the labels that would repeat an n-gram of the sample or end it before m words
from the candidates of that position, inside the same kernel (DESIGN.md §9).
"""
from typing import NamedTuple

import torch

from . import ops
from ._lib import call
from .decode_loop import (PositionLoop, _f32, check_prefix, check_rules, check_tar_len, encode_members, is_int,
                          loop_for)

MAX_SAMPLES = 32          # the N samples of a commit are its query rows in fira_attn_fwd / fira_copy_scores_fwd (<= 32)


class Samples(NamedTuple):
    seq: torch.Tensor             # [B, N, T] int64 vocabulary ids: <start>, the drawn tokens, pad after <eos>
    raw: torch.Tensor             # [B, N, T] int64 raw indices (label encoding: V + memory position for a copy)
    length: torch.Tensor          # [B, N] int64 tokens including <start> and <eos>
    logprob: torch.Tensor         # [B, N] fp32 sum of token_logprob
    token_logprob: torch.Tensor   # [B, N, T] fp32 log(clamp(P, 1e-10, 1)) of each drawn token, 0 at 0 and after <eos>


def check_args(num_samples, temperature, top_k, top_p, seed, first_index, tar_len):
    """ValueError for any parameter the sampler cannot honour (called before any device work)."""
    if not is_int(num_samples) or not 1 <= num_samples <= MAX_SAMPLES:
        raise ValueError(f"num_samples must be an integer in [1, {MAX_SAMPLES}], got {num_samples!r}")
    if not isinstance(temperature, (int, float)) or not 0.0 < _f32(temperature) < float("inf"):
        raise ValueError(f"temperature must be a positive finite number (in fp32), got {temperature!r}")
    if not is_int(top_k) or top_k < 0:
        raise ValueError(f"top_k must be an integer >= 0 (0 = off), got {top_k!r}")
    if not isinstance(top_p, (int, float)) or not 0.0 < _f32(top_p) <= 1.0:
        raise ValueError(f"top_p must be in (0, 1] (1 = off), got {top_p!r}")
    if not is_int(seed) or not 0 <= seed < 2 ** 64:
        raise ValueError(f"seed must be an integer in [0, 2**64), got {seed!r}")
    if not is_int(first_index) or not 0 <= first_index < 2 ** 31:
        raise ValueError(f"first_index must be an integer in [0, 2**31), got {first_index!r}")
    if not is_int(tar_len) or tar_len < 2:
        raise ValueError(f"tar_len must be an integer >= 2, got {tar_len!r}")


class _Sampler(PositionLoop):
    """The sampler's seed and first index on top of the shared position loop (status: the finished flag)."""

    def __init__(self, model, B, N, T, S):
        super().__init__(model, B, N, T, S)
        self.seed = torch.zeros(1, dtype=torch.int64, device=self.dev)      # read by the kernel as uint64
        self.first = torch.zeros(1, dtype=torch.int32, device=self.dev)

    def start(self, memory, mem_mask, copy_src, seed, first_index, start_id, pad_id, prefix=None):
        super().start(memory, mem_mask, copy_src, start_id, pad_id, prefix)
        self.seed.fill_(seed - 2 ** 64 if seed >= 2 ** 63 else seed)
        self.first.fill_(first_index)

    def position(self, t, temperature, top_k, top_p, eos_id, pad_id, no_repeat_ngram, min_length):
        """Draw position t + 1 from decoder row t, or take a commit's prefix label there (every launch on the current
        stream: capturable)."""
        self.head(t)
        p = ops._ptr
        call("fira_pointer_mix_sample_rules", p(self.logits), self.ldl, p(self.sc), p(self.gl), p(self.mem_mask),
             p(self.copy_src), p(self.seed), p(self.first), None, float(temperature), int(top_k), float(top_p),
             int(eos_id), int(pad_id), p(self.inc.tok), p(self.seq), p(self.raw), p(self.tlp), p(self.inc.tok_mask),
             self.T, t, p(self.status), p(self.length), p(self.lp), self.B, self.N, self.V, self.S, self.code,
             ops._stream(), p(self.prefix), self.T, p(self.prefix_len), int(no_repeat_ngram), int(min_length))


@torch.no_grad()
def sample(model, sou, mark, ast_change, edge, sub_token, *, num_samples=1, temperature=1.0, top_k=0, top_p=1.0,
           seed=0, first_index=0, tar_len=30, start_id, eos_id, pad_id=0, prefix=None, no_repeat_ngram=0,
           min_length=0):
    """Draw `num_samples` messages per commit -> Samples(seq, raw, length, logprob, token_logprob).

    model: a TransModel, or an ensemble.Ensemble (its averaged distribution; token_logprob is the ensemble's).
    first_index: dataset position of the batch's first commit (the Philox counter uses first_index + b).
    prefix: None, or labels [B, P] every sample of a commit starts with (decode_loop.check_prefix: the tar_label
    encoding without <start>, a 0 ends a commit's prefix, <eos> only as its last label).  The positions after a prefix
    draw with the Philox numbers they would draw without it; logprob and token_logprob cover the prefix too.
    no_repeat_ngram = n >= 1: no drawn word completes an n-gram already in the sample (n = 1: no word twice; a copy
    counts as its word).  min_length = m >= 1: no <eos> before m words.  Banned labels are dropped from the candidates
    before the top-k / top-p cuts, nothing is renormalised and token_logprob keeps the model's log-probability; prefix
    positions are exempt.  0 turns either off (decode_loop.check_rules)."""
    check_args(num_samples, temperature, top_k, top_p, seed, first_index, tar_len)
    check_rules(no_repeat_ngram, min_length, tar_len)
    check_tar_len(model, tar_len)
    if first_index + sou.shape[0] > 2 ** 31:
        raise ValueError("first_index + batch size must stay below 2**31")
    pre = check_prefix(prefix, sou, sub_token, V=model.vocab_size, tar_len=tar_len, eos_id=eos_id, pad_id=pad_id,
                       eos_last=True)
    memory, mem_mask, copy_src = encode_members(model, sou, mark, ast_change, edge, sub_token, pad_id)
    B, S = memory[0].shape[:2]
    st = loop_for(_Sampler, model, B, num_samples, tar_len, S)
    st.start(memory, mem_mask, copy_src, seed, first_index, start_id, pad_id, pre)
    t = st.run((float(temperature), int(top_k), float(top_p), int(eos_id), int(pad_id), no_repeat_ngram, min_length))
    seq, raw, length, lp, tlp, _ = st.slots(t)
    return Samples(seq, raw, length, lp, tlp)


class Scores(NamedTuple):
    token_logprob: torch.Tensor   # [B, T] fp32 log(clamp(P, 1e-10, 1)) of each label, 0 at 0 and after <eos>
    logprob: torch.Tensor         # [B] fp32 sum of token_logprob: log p(message | commit)
    length: torch.Tensor          # [B] int64 tokens including <start> and <eos>


def score_prefix(tar_label, tar_len, eos_id):
    """The labels of tar_label [B, >= tar_len] after <start> up to and including each row's first <eos> -> a prefix
    [B, tar_len - 1] (zeros after <eos>); ValueError for a row without <eos> within tar_len (host only)."""
    lab = tar_label.detach().to("cpu", torch.int64)[:, 1:tar_len]
    is_eos = lab == eos_id
    if lab.shape[1] < tar_len - 1 or not is_eos.any(1).all():
        raise ValueError(f"every row of tar_label needs <eos> within its first tar_len = {tar_len} labels")
    after = is_eos.to(torch.int64).cumsum(1) - is_eos.to(torch.int64) > 0       # strictly after the first <eos>
    return lab.masked_fill(after, 0)


@torch.no_grad()
def score(model, sou, mark, ast_change, edge, sub_token, tar_label, *, tar_len=30, start_id, eos_id, pad_id=0):
    """log p(message | commit) of each commit's given message -> Scores(token_logprob, logprob, length).
    model: a TransModel or an ensemble.Ensemble (then log of the averaged probability).

    tar_label [B, >= tar_len]: <start>, the labels (tar_label encoding), <eos> within tar_len, anything after.  The
    sampler with one sample per commit and the whole message forced, so token_logprob[:, t] is the -nll the training
    loss gives label tar_label[:, t] after the labels before it."""
    if not is_int(tar_len) or tar_len < 2:
        raise ValueError(f"tar_len must be an integer >= 2, got {tar_len!r}")
    prefix = score_prefix(tar_label, tar_len, eos_id)
    s = sample(model, sou, mark, ast_change, edge, sub_token, num_samples=1, tar_len=tar_len, start_id=start_id,
               eos_id=eos_id, pad_id=pad_id, prefix=prefix)
    return Scores(s.token_logprob[:, 0], s.logprob[:, 0], s.length[:, 0])
