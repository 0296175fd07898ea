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

The loop is decode_loop.PositionLoop (described there); a position ends with fira_pointer_mix_sample, which also writes
the next input token straight into the decoder's token buffer and keeps each row's finished flag, length and
log-probability sum.
"""
from typing import NamedTuple

import torch

from . import ops
from ._lib import call
from .decode_loop import PositionLoop, _f32, check_tar_len, encode, is_int, loop_for

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

    def start(self, memory, mem_mask, copy_src, seed, first_index, start_id, pad_id):
        super().start(memory, mem_mask, copy_src, start_id, pad_id)
        self.seed.fill_(seed - 2 ** 64 if seed >= 2 ** 63 else seed)
        self.first.fill_(first_index)

    def position(self, t, temperature, top_k, top_p, eos_id, pad_id):
        """Draw position t + 1 from decoder row t (every launch on the current stream: capturable)."""
        self.head(t)
        p = ops._ptr
        call("fira_pointer_mix_sample", p(self.logits), self.ldl, p(self.sc), p(self.gl), p(self.mem_mask),
             p(self.copy_src), p(self.seed), p(self.first), None, float(temperature), int(top_k), float(top_p),
             int(eos_id), int(pad_id), p(self.inc.tok), p(self.seq), p(self.raw), p(self.tlp), p(self.inc.tok_mask),
             self.T, t, p(self.status), p(self.length), p(self.lp), self.B, self.N, self.V, self.S, self.pr.code,
             ops._stream())


@torch.no_grad()
def sample(model, sou, mark, ast_change, edge, sub_token, *, num_samples=1, temperature=1.0, top_k=0, top_p=1.0,
           seed=0, first_index=0, tar_len=30, start_id, eos_id, pad_id=0):
    """Draw `num_samples` messages per commit -> Samples(seq, raw, length, logprob, token_logprob).

    first_index: dataset position of the batch's first commit (the Philox counter uses first_index + b)."""
    check_args(num_samples, temperature, top_k, top_p, seed, first_index, tar_len)
    check_tar_len(model, tar_len)
    if first_index + sou.shape[0] > 2 ** 31:
        raise ValueError("first_index + batch size must stay below 2**31")
    memory, mem_mask, copy_src = encode(model, sou, mark, ast_change, edge, sub_token, pad_id)
    B, S = memory.shape[:2]
    st = loop_for(_Sampler, model, B, num_samples, tar_len, S)
    st.start(memory, mem_mask, copy_src, seed, first_index, start_id, pad_id)
    t = st.run((float(temperature), int(top_k), float(top_p), int(eos_id), int(pad_id)))
    seq, raw, length, lp, tlp, _ = st.slots(t)
    return Samples(seq, raw, length, lp, tlp)
