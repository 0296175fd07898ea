"""Minimum-Bayes-risk decoding: among each commit's N seeded samples (sample.py), the one with the highest expected
sentence BLEU, every other sample serving as a pseudo-reference.

    words_n   = seq[b, n, 1:length[b, n]] without every id equal to start_id, eos_id or pad_id, wherever it occurs
    BLEU(i,j) = bleu.sentence_bleu_method2([words_j], words_i) over the vocabulary ids, in float64 (n = 1..4, clipped
                matches, denominator floored at 1, method-2 +1 smoothing for n >= 2, 0 for an empty hypothesis or no
                unigram match, brevity penalty with r = len(words_j))
    U_i       = (sum over j != i, j ascending, of BLEU(i, j)) / (N - 1)
    chosen    = the smallest i with the largest U_i

For a word that is non-empty, whitespace-free and contains none of the three markers, one id is one text token of
run_model.ids_to_text (<unkm> becomes one token too), so for messages made of such words the id-level BLEU equals the
text-level BLEU that run_model.py reports.  The golden vocabulary has one word that is not: `import static`, which is
two text tokens and one id here.  U is only the selection criterion; the reported BLEU stays text-level.

The candidates are sample()'s, so a commit's choice depends only on the seed, the sampling parameters and its dataset
position, whatever the batch or GPU count.  The pairwise scoring is one fira_mbr_select launch per batch
(csrc/mbr.cu, one CTA per commit).
"""
from typing import NamedTuple

import torch

from . import ops
from ._lib import call
from .sample import Samples, check_args, sample

MAX_TAR_LEN = 32          # fira_mbr_select: at most 31 words per candidate, one per lane of a warp


class MBR(NamedTuple):
    seq: torch.Tensor             # [B, T] int64 the chosen sample (vocabulary ids, <start> first, pad after <eos>)
    length: torch.Tensor          # [B] int64 its tokens including <start> and <eos>
    logprob: torch.Tensor         # [B] fp32 its log-probability (Samples.logprob)
    index: torch.Tensor           # [B] int64 which of the N samples it is
    utility: torch.Tensor         # [B, N] float64 U_i of every sample
    samples: Samples              # every candidate


@torch.no_grad()
def mbr(model, sou, mark, ast_change, edge, sub_token, *, num_samples=16, temperature=1.0, top_k=0, top_p=1.0,
        seed=0, first_index=0, tar_len=30, start_id, eos_id, pad_id=0, prefix=None, no_repeat_ngram=0, min_length=0):
    """Draw `num_samples` messages per commit with sample() and keep the one of highest expected BLEU -> MBR.
    prefix, no_repeat_ngram, min_length: passed to sample(), so every candidate obeys them.  model: a TransModel or an
    ensemble.Ensemble (the candidates are drawn from its averaged distribution)."""
    check_args(num_samples, temperature, top_k, top_p, seed, first_index, tar_len)
    if num_samples < 2:
        raise ValueError(f"MBR needs num_samples >= 2, got {num_samples!r}")
    if tar_len > MAX_TAR_LEN:
        raise ValueError(f"MBR needs tar_len <= {MAX_TAR_LEN}, got {tar_len!r}")
    s = sample(model, sou, mark, ast_change, edge, sub_token, num_samples=num_samples, temperature=temperature,
               top_k=top_k, top_p=top_p, seed=seed, first_index=first_index, tar_len=tar_len, start_id=start_id,
               eos_id=eos_id, pad_id=pad_id, prefix=prefix, no_repeat_ngram=no_repeat_ngram, min_length=min_length)
    B, N, T = s.seq.shape
    dev = s.seq.device
    seq, length = s.seq.to(torch.int32), s.length.to(torch.int32)
    utility = torch.empty((B, N), dtype=torch.float64, device=dev)
    best = torch.empty(B, dtype=torch.int32, device=dev)
    p = ops._ptr
    call("fira_mbr_select", p(seq), p(length), T, int(start_id), int(eos_id), int(pad_id), None, p(utility), p(best),
         B, N, T, ops._stream())
    index = best.long()
    rows = torch.arange(B, device=dev)
    return MBR(s.seq[rows, index], s.length[rows, index], s.logprob[rows, index], index, utility, s)
