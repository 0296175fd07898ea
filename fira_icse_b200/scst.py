"""Self-critical sequence training (SCST, Rennie et al. 2017) on sentence BLEU: fine-tune a trained model towards the
measure run_model.py selects checkpoints and reports results by.

For a padded batch of B commits, one step draws N >= 2 seeded messages per commit with sample() (eval mode), scores
each against the commit's reference and raises the log-probability of the samples that beat their baseline:

    words(x)  = ids in columns 1..len-1 without start / eos / pad ids                     (as mbr.py)
    ref_b     = the words of tar[b] in columns 1.. before its first <eos>                (run_model.reference_words)
    r[b,n]    = bleu.sentence_bleu_method2([ref_b], words(seq[b,n])) over the ids, float64
    A[b,n]    = (sum over m != n, m ascending, of (r[b,n] - r[b,m])) / (N - 1)        leave-one-out baseline:
                r[b,n] minus the mean of the commit's other rewards, exactly 0 for tied rewards
    L         = (1 / (B*N)) * sum_{b,n} A[b,n] * sum_t nll[b,n,t]

nll is the training loss's own per-position NLL (ops.HeadFn) of the sampled message: tar = seq (a copy as its word id),
tar_label = raw, shifted as TransModel.shifted_label does, so the gradient pass conditions on exactly the tokens the
sampler conditioned on.  The reward is id-level like MBR's utility (mbr.py: `import static` is the one golden word where
it differs from the text-level BLEU run_model.py reports).

Where it runs: the rewards and advantages are one fira_bleu_reward launch (csrc/mbr.cu, one CTA per commit, one warp per
sample).  The gradient pass encodes the batch once, in training mode with the kernels' dropout, and replicates the memory
N-fold along the batch under autograd (the encoder's gradient is the sum over the copies); the decoder and the head then
run on the B*N sampled targets with seq_weight = A / (B*N) (fira_pointer_mix_nll_bwd_rows_weighted; a sample whose
advantage is exactly 0 costs the head's backward nothing).  The cross-attention K/V projection of the memory is paid N
times.  This is the eager padded-batch path: no CUDA graph of the step, no packed layout.

After the optimizer step the decoder's weights_epoch is bumped: an eager FlatAdam step writes the parameters through a raw
kernel that moves neither their version counters nor their addresses, and the next sample() must decode with the new
weights.  decode_loop.loop_for then refreshes the cached loop's weight operands in place and keeps replaying its
captured position graphs.
"""
from typing import NamedTuple

import torch

from . import ops
from . import optim as _optim
from ._lib import call
from .decode_loop import check_rules, check_tar_len, is_int
from .ensemble import refuse
from .modules import _i32, _u8
from .sample import MAX_SAMPLES, check_args, sample

MAX_TAR_LEN = 32          # fira_bleu_reward: at most 31 words per message, one per lane of a warp


class Step(NamedTuple):
    reward: float         # mean r over the B*N samples
    advantage: float      # mean |A|
    loss: float           # L


def check_step(tar, *, num_samples, temperature, top_k, top_p, seed, first_index, no_repeat_ngram, min_length,
               tar_len, eos_id, model=None):
    """ValueError for any setting or reference (tar [B, >= tar_len], None: settings only) scst_step cannot honour
    (host only, before any device work)."""
    if not is_int(num_samples) or not 2 <= num_samples <= MAX_SAMPLES:
        raise ValueError(f"SCST needs num_samples in [2, {MAX_SAMPLES}], got {num_samples!r}")
    if is_int(tar_len) and tar_len > MAX_TAR_LEN:
        raise ValueError(f"SCST needs tar_len <= {MAX_TAR_LEN}, got {tar_len!r}")
    check_args(num_samples, temperature, top_k, top_p, seed, first_index, tar_len)
    check_rules(no_repeat_ngram, min_length, tar_len)
    if model is not None:
        check_tar_len(model, tar_len)
    if tar is None:
        return
    ref = tar.detach().to("cpu", torch.int64)
    if ref.dim() != 2 or ref.shape[1] < tar_len or not (ref[:, 1:tar_len] == eos_id).any(1).all():
        raise ValueError(f"every reference row of tar needs <eos> within its first tar_len = {tar_len} ids")


def rewards(seq, length, tar, *, start_id, eos_id, pad_id):
    """seq [B, N, T] / length [B, N] of sample() against the references tar [B, >= T] (<start> first) -> reward and
    advantage [B, N] float64 on the device (fira_bleu_reward)."""
    B, N, T = seq.shape
    dev = seq.device
    s = seq.to(torch.int32).contiguous()
    n = length.to(torch.int32).contiguous()
    ref = tar.to(dev, torch.int32).contiguous()
    reward = torch.empty((B, N), dtype=torch.float64, device=dev)
    advantage = torch.empty((B, N), dtype=torch.float64, device=dev)
    p = ops._ptr
    call("fira_bleu_reward", p(s), p(n), T, p(ref), ref.shape[1], int(start_id), int(eos_id), int(pad_id), p(reward),
         p(advantage), B, N, T, ops._stream())
    return reward, advantage


def policy_loss(model, batch, seq, raw, seq_weight, pad_id=0):
    """sum over the B*N sampled messages of seq_weight[b*N + n] * their NLL, under autograd, in the model's current
    mode -> (loss, per-position nll [B*N, T]).  batch: the padded 8-tuple; seq / raw [B, N, T] of sample()."""
    sou, _, _, mark, ast_change, edge, _, sub_token = batch
    m = model
    dev = m.out_fc.weight.device
    sou, mark, ast_change, sub_token = (t.to(dev) for t in (sou, mark, ast_change, sub_token))
    B, N, T = seq.shape
    bf16 = m.precision == "bf16"
    if bf16:
        _optim.ensure_fresh(m)
    m.decoder.prefetch_weights()
    pf_head = ops.prefetch_head(bf16, m.out_fc.weight, m.copy_net.LinearSource.weight, m.copy_net.LinearTarget.weight)
    memory = m.encoder.encode_memory(sou, mark, ast_change, edge, sub_token)
    mem_mask = torch.cat((sou != pad_id, sub_token != 0), dim=1)       # as decode_loop.encode forms it for the sampler

    def rep(x):                                                         # commit b -> rows b*N .. b*N + N-1
        return x.unsqueeze(1).expand(B, N, *x.shape[1:]).reshape(B * N, *x.shape[1:])
    memory_r, mem_mask_r = rep(memory), rep(mem_mask)
    tar = seq.reshape(B * N, T)
    label = m.shifted_label(raw.reshape(B * N, T))
    dec = m.decoder(tar, memory_r, mem_mask_r, tar != pad_id)
    loss, nll, _ = ops.HeadFn.apply(False, bf16, pf_head, memory_r, dec, _u8(mem_mask_r), _i32(label).view(-1),
                                    m.out_fc.weight, m.out_fc.bias, *m.copy_net.flat_params(), None, seq_weight)
    return loss, nll


def bump_weights(model):
    """Tell the decoding loops' weight caches that the parameters moved (decode_loop.loop_for)."""
    model.decoder.weights_epoch = getattr(model.decoder, "weights_epoch", 0) + 1


def scst_step(model, optimizer, batch, *, num_samples, temperature=1.0, top_k=0, top_p=1.0, seed=0, first_index=0,
              no_repeat_ngram=0, min_length=0, tar_len=30, start_id, eos_id, pad_id=0):
    """One self-critical step on the padded batch (the 8-tuple of run_model.py on the model's device) -> Step(mean
    reward, mean |advantage|, loss).  Sampling settings as sample(); leaves the model in training mode."""
    refuse(model, "scst_step")
    check_step(batch[1], num_samples=num_samples, temperature=temperature, top_k=top_k, top_p=top_p, seed=seed,
               first_index=first_index, no_repeat_ngram=no_repeat_ngram, min_length=min_length, tar_len=tar_len,
               eos_id=eos_id, model=model)
    sou, tar, _, mark, ast_change, edge, _, sub_token = batch
    model.eval()
    s = sample(model, sou, mark, ast_change, edge, sub_token, num_samples=num_samples, temperature=temperature,
               top_k=top_k, top_p=top_p, seed=seed, first_index=first_index, tar_len=tar_len, start_id=start_id,
               eos_id=eos_id, pad_id=pad_id, no_repeat_ngram=no_repeat_ngram, min_length=min_length)
    reward, advantage = rewards(s.seq, s.length, tar, start_id=start_id, eos_id=eos_id, pad_id=pad_id)
    B, N = reward.shape
    weight = (advantage / (B * N)).to(torch.float32).reshape(-1)
    model.train()
    optimizer.zero_grad()
    loss, _ = policy_loss(model, batch, s.seq, s.raw, weight, pad_id)
    loss.backward()
    optimizer.step()
    bump_weights(model)
    return Step(reward.mean().item(), advantage.abs().mean().item(), loss.item())
