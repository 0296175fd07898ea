#!/usr/bin/env python
"""`python run_model.py train|test|finetune|distill|kd-targets` -- the reference's CLI (run_model.py:417-425) on the CUDA path.

Same CWD-relative files (DataSet/*.json, all_index, VOCAB_UPPER_CASE, best_model.pt,
OUTPUT/{output_fira,train_process,dev_output}), same hyper-parameters (run_model.py:27-46), same
training loop semantics (Adam 1e-4, loss = sum(loss)/sum(tokens), dev BLEU every 10 batches from
epoch 15, best checkpoint saved as a plain state_dict with the reference's 338 keys) and the same
beam search ranking.  Differences, all below the module surface:
  * one process per GPU (launch with torchrun for N > 1) with an NCCL gradient all-reduce instead of
    nn.DataParallel; batch 170 PER GPU like upstream (run_model.py:40);
  * training batches come from the native loader (data.PackedBatchLoader: C++ gather + padding trim + CSR
    packing into pinned memory) instead of dense float64 650x650 through DataLoader workers;
  * the training step (zero-grad, forward, backward, Adam) is replayed as a CUDA graph per batch shape
    (engine.GraphedTrainStep); FIRA_ENGINE=eager issues the same kernels launch by launch;
  * optional env overrides, defaults unchanged: FIRA_BATCH, FIRA_TEST_BATCH, FIRA_EPOCHS, FIRA_BEAM,
    FIRA_MAX_BATCHES (smoke runs), FIRA_WORKERS, FIRA_PRECISION (fp32 parity mode | bf16 throughput mode),
    FIRA_MAX_SHAPES (bound on distinct trimmed batch shapes = captured graphs, default 24), FIRA_BUCKET (0 = the
    reference's uniform batching; K > 1 = size-bucketed batches within windows of K batches, see PackedBatchLoader).
  * FIRA_EMA=d (`train`, default unset = off; 0 < d < 1, e.g. 0.999): keep an exponential moving average of the weights,
    e = d e + (1 - d) p after every Adam step, updated inside the optimizer kernel (optim.FlatAdam, DESIGN.md §9).  Every
    dev gate first scores and saves the trained weights as without it, then scores the EMA weights with the same dev()
    and keeps their own best: best_model_ema.pt, OUTPUT/dev_output_ema and `ema epoch: ...` lines in
    OUTPUT/train_process.  This doubles the time spent at dev gates.  `test`, `datastore`, `finetune` and `distill` read
    the EMA checkpoint with FIRA_CHECKPOINT=best_model_ema.pt, a teacher or ensemble with FIRA_ENSEMBLE=best_model_ema.pt.
    FIRA_ENGINE=eager (torch's fused Adam) with FIRA_EMA exits with an error.
  * FIRA_CLIP_NORM=c (`train`, `finetune` and `distill`; default unset = off; a positive number or inf): clip the
    gradient's global norm to c before every Adam step (torch.nn.utils.clip_grad_norm_'s rule) and skip steps whose
    gradient is not finite, on the device (optim.FlatAdam(max_grad_norm), DESIGN.md §9); inf only monitors the norm and
    skips non-finite steps.  The 10-batch progress line then also prints the window's mean gradient norm and the
    clipped / skipped step counts.  Bad values, and FIRA_ENGINE=eager in `train`, exit with an error.
  * `test` decoding: FIRA_DECODE=beam (default, the reference's beam search -> OUTPUT/output_fira) or sample (seeded
    sampling, fira_icse_b200.sample -> OUTPUT/output_fira_samples: FIRA_SAMPLES consecutive lines per commit in test
    order, `<log-probability>\\t<message>`; prints the mean sentence BLEU over all samples).  Sampling parameters:
    FIRA_SAMPLES (default 3), FIRA_TEMPERATURE (1.0), FIRA_TOP_K (0 = off), FIRA_TOP_P (1.0 = off), FIRA_SEED (0).
    A commit's samples depend on the seed and its position in the test split only, so sharded runs draw the same.
    FIRA_DECODE=nbest: log-space beam search with length normalisation (fira_icse_b200.beam.nbest) ->
    OUTPUT/output_fira_nbest: FIRA_BEAM consecutive lines per commit in test order, best first,
    `<score>\t<log-probability>\t<message>`; FIRA_LENGTH_PENALTY (default 0 = rank by log-probability) sets the
    penalty alpha of score = logprob / ((5 + n) / 6) ** alpha; prints the mean sentence BLEU of the top hypothesis.
    FIRA_BEAM_GROUPS (default 1 = plain n-best) splits the FIRA_BEAM hypotheses into that many diverse beam groups
    (it must divide FIRA_BEAM); a group's candidates are ranked down by FIRA_DIVERSITY (default 0.5, used only when
    FIRA_BEAM_GROUPS > 1) per earlier-group hypothesis that chose the same word at that position.
    FIRA_DECODE=mbr: minimum-Bayes-risk decoding (fira_icse_b200.mbr) -> OUTPUT/output_fira_mbr: one line per commit in
    test order, `<expected BLEU>\\t<log-probability>\\t<message>`, the commit's sample with the highest mean id-level
    sentence BLEU against its other samples; FIRA_SAMPLES (default 16 here), FIRA_TEMPERATURE, FIRA_TOP_K, FIRA_TOP_P
    and FIRA_SEED as for sampling; prints the mean sentence BLEU of the chosen messages.
    FIRA_PREFIX_WORDS=k (default 0 = off; FIRA_DECODE=sample, nbest or mbr): prefix-constrained completion, every test
    commit's message starts with the first min(k, message words) words of its own reference (their labels, never
    <eos>) and the decoder completes it -> OUTPUT/<name>_prefix<k> (output_fira_samples_prefix2, ...), so the full
    decoding outputs stay.  Lines hold the whole message, prefix included, and the printed BLEU is of the whole
    message against the reference.  FIRA_DECODE=beam with k > 0 exits with an error.
    FIRA_NO_REPEAT_NGRAM=n and FIRA_MIN_LENGTH=m (default 0 = off; FIRA_DECODE=sample, nbest or mbr): no generated word
    completes an n-gram already in its message (n = 1: no word twice), and no message ends before m words (DESIGN.md
    §9).  A nonzero value appends _norepeat<n> / _minlen<m> to the output name, after any _prefix<k>
    (output_fira_nbest_norepeat2_minlen3, ...), so the outputs without them stay.  FIRA_DECODE=beam with either set
    exits with an error.
    FIRA_CONSTRAINT_WORDS=k (default 0 = off, at most 4; FIRA_DECODE=nbest with FIRA_BEAM_GROUPS=1 only): lexically
    constrained n-best (DESIGN.md §9), every test commit's message must contain the first k distinct words of its
    reference that also occur among its diff ids (sou or sub_token, never <unkm>), each a one-word phrase: the
    oracle-constraint evaluation of the constrained-decoding papers.  Appends _lex<k> to the output name after the other
    tags (output_fira_nbest_lex1, ...) and prints, after the mean BLEU, the share of commits whose top hypothesis meets
    its constraints.  Any other decoding mode, or FIRA_BEAM_GROUPS > 1, with k > 0 exits with an error.
    FIRA_CHECKPOINT (default best_model.pt): the state_dict `test` decodes with (best_model_scst.pt after finetune).
    FIRA_ENSEMBLE=a.pt,b.pt[,...] (FIRA_DECODE=sample, nbest or mbr; up to 8 state_dicts, not with FIRA_CHECKPOINT):
    decode with the ensemble of those checkpoints (fira_icse_b200.ensemble: the weighted average of their
    distributions at every position), weighted by FIRA_ENSEMBLE_WEIGHTS=w1,w2,... (positive, one per checkpoint;
    default uniform).  Appends _ens<M> to the output name after the other tags (output_fira_nbest_norepeat2_ens2, ...),
    so single-model outputs stay.  FIRA_DECODE=beam with an ensemble exits with an error.
    FIRA_KNN=datastore.pt (FIRA_DECODE=sample, nbest or mbr; not with FIRA_ENSEMBLE): nearest-neighbour decoding
    (fira_icse_b200.knn, DESIGN.md §9) with the datastore `datastore` built from this checkpoint: each position mixes the
    model's distribution with the next words of the FIRA_KNN_K (default 8) nearest training positions, at temperature
    FIRA_KNN_TEMPERATURE (default 10) and weight FIRA_KNN_LAMBDA (default 0.25).  The defaults are common starting
    points of the kNN-MT papers, not tuned on this data.  Appends _knn<k> to the output name after the other tags.
    FIRA_DECODE=beam, an ensemble, bad settings and a datastore built by another checkpoint exit with an error before
    any device work.
  * `datastore`: builds the kNN datastore of `test`'s FIRA_KNN from the train split with FIRA_CHECKPOINT (default
    best_model.pt) in padded batches of FIRA_BATCH commits (FIRA_PRECISION: the precision it is built and used in) and
    writes FIRA_DATASTORE (default datastore.pt): one entry per target position (decoder state -> next word).  Prints
    the entry count and bytes.  One GPU.
  * `finetune`: self-critical fine-tuning on sentence BLEU (fira_icse_b200.scst, DESIGN.md §9), one GPU.  Loads
    best_model.pt and runs FIRA_SCST_EPOCHS (default 1) epochs of scst_step with optim.FlatAdam at FIRA_SCST_LR
    (default 1e-5) over padded batches of FIRA_BATCH commits (FIRA_MAX_BATCHES bounds an epoch): FIRA_SAMPLES (default
    5, 2..32) seeded samples per commit with FIRA_TEMPERATURE, FIRA_TOP_K, FIRA_TOP_P, FIRA_SEED (epoch e draws with
    seed FIRA_SEED + e), FIRA_NO_REPEAT_NGRAM and FIRA_MIN_LENGTH, each rewarded with its id-level sentence BLEU
    against the reference and weighted by its leave-one-out advantage.  Prints the mean reward every 10 batches, runs
    dev() after every epoch and saves the state_dict of the best dev BLEU to best_model_scst.pt; best_model.pt is never
    overwritten.  WORLD_SIZE > 1 exits with an error.
  * `distill`: word-level knowledge distillation from an ensemble (fira_icse_b200.distill, DESIGN.md §9), one GPU.  The
    student is FIRA_CHECKPOINT (default best_model.pt), the teacher the Ensemble of FIRA_ENSEMBLE=a.pt[,b.pt,...]
    weighted by FIRA_ENSEMBLE_WEIGHTS (as for `test`; both are needed here).  Runs FIRA_KD_EPOCHS (default 1) epochs of
    distill_step with optim.FlatAdam at FIRA_KD_LR (default 1e-4, the reference's rate) over padded batches of
    FIRA_BATCH commits (FIRA_MAX_BATCHES bounds an epoch), on the loss (1 - FIRA_KD_ALPHA) NLL + FIRA_KD_ALPHA
    cross-entropy against the teacher's distribution (FIRA_KD_ALPHA in [0, 1], default 0.5).  Prints loss / nll / kd
    every 10 batches, runs dev() after every epoch and saves the state_dict of the best dev BLEU to best_model_kd.pt
    (dev output: OUTPUT/dev_output_kd); best_model.pt and the teacher checkpoints are never overwritten.  WORLD_SIZE > 1
    exits with an error.  With FIRA_KD_TARGETS=path (not with FIRA_ENSEMBLE) the teacher is the file `kd-targets`
    wrote: no teacher is loaded or run, and each epoch e visits the train split in the seeded permutation FIRA_SEED + e
    (the file's rows are found by dataset position).  The file's vocabulary size and commit count are checked against
    the data before any device work.
  * `kd-targets`: runs the teacher of FIRA_ENSEMBLE / FIRA_ENSEMBLE_WEIGHTS (one checkpoint is allowed) once over the
    train split in dataset order, in padded batches of FIRA_BATCH commits and FIRA_PRECISION, and writes its
    FIRA_KD_TOPK (default 8, 1..64) most probable labels per target position, renormalised, to FIRA_KD_TARGETS (default
    kd_targets.pt) for `distill`.  Prints the rows, the bytes and the mean kept teacher mass.  One GPU.
"""
import json
import os
import random
import sys
import time

import numpy as np
import torch
import torch.distributed as dist
from torch.optim import Adam
from torch.utils.data import DataLoader

from fira_icse_b200 import TransModel
from fira_icse_b200.beam import beam_search, best_sequences, constraints_met, nbest
from fira_icse_b200.bleu import sentence_bleu_method2
from fira_icse_b200.decode_loop import MAX_PHRASES
from fira_icse_b200.distill import MAX_TOPK, KDTargets, build_targets, distill_step
from fira_icse_b200.data import PackedBatchLoader, TransDataset, batch_to_device, collate_packed
from fira_icse_b200.engine import GraphedTrainStep
from fira_icse_b200.ensemble import MAX_MEMBERS, Ensemble
from fira_icse_b200.knn import Datastore, KNNModel, build_datastore, check_settings, state_fingerprint
from fira_icse_b200.mbr import mbr
from fira_icse_b200.parallel import DataParallelStep, shard_range
from fira_icse_b200.sample import sample
from fira_icse_b200.scst import check_step, scst_step


class DotDict(dict):
    def __getattr__(self, attr):
        return self[attr]


WORLD = int(os.environ.get("WORLD_SIZE", "1"))
RANK = int(os.environ.get("RANK", "0"))
LOCAL_RANK = int(os.environ.get("LOCAL_RANK", "0"))

args = DotDict({
    'sou_len': 210, 'tar_len': 30, 'att_len': 25, 'ast_change_len': 280, 'sub_token_len': 160,
    'lr': 1e-4, 'dropout_rate': 0.1, 'num_head': 8, 'embedding_dim': 256,
    'batch_size': int(os.environ.get("FIRA_BATCH", 170)),           # per GPU, as upstream (170 * n_gpu global)
    'test_batch_size': int(os.environ.get("FIRA_TEST_BATCH", 20)),
    'epoches': int(os.environ.get("FIRA_EPOCHS", 150)),
    'beam_size': int(os.environ.get("FIRA_BEAM", 3)),
    'vocab_size': 0, 'ast_change_vocab_size': 0,
})


def load_globals():
    g = {}
    g["vocab"] = json.load(open('DataSet/word_vocab.json'))
    g["r_vocab"] = {v: k for k, v in g["vocab"].items()}
    args.vocab_size = len(g["vocab"])
    args.ast_change_vocab_size = len(json.load(open('DataSet/ast_change_vocab.json')))
    g["var_maps"] = json.load(open("DataSet/variable.json"))
    return g


def seed_everything(seed=0):
    random.seed(seed)
    os.environ['PYTHONHASHSEED'] = str(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    torch.cuda.manual_seed_all(seed)


def device():
    if not torch.cuda.is_available():
        raise SystemExit("run_model.py: no CUDA device. This build has no CPU path; the CPU reference is "
                         "the upstream repository (or oracle/ for tests).")
    torch.cuda.set_device(LOCAL_RANK)
    return torch.device("cuda", LOCAL_RANK)


def ids_to_text(ids, r_vocab):
    s = ' '.join(r_vocab[i] for i in ids)
    return s.replace('<start>', "").replace('<eos>', "").replace('<pad>', "").replace('<unkm>', "😅").strip().split()


def deanonymise(tokens, var_map):
    rev = {v: k for k, v in var_map.items()}
    return [rev.get(t, t) for t in tokens]


def reference_words(tar, vocab, r_vocab):
    """The reference message of one commit (its target ids between <start> and <eos>) as words."""
    ref = tar.tolist()
    return [r_vocab[x] for x in ref[1:ref.index(vocab['<eos>'])]]


def reference_prefix(b, k, eos_id, pad_id):
    """The first min(k, message words) labels of each commit's tar_label (b[6]) after <start>, never <eos> -> [B, k]
    (zeros after a message's last word), the decoders' `prefix`.  A copy label the truncated diff no longer holds (its
    memory position is padding) ends the commit's prefix early."""
    lab = b[6][:, 1:1 + k]
    mem_mask = torch.cat((b[0] != pad_id, b[7] != 0), dim=1)
    V = args.vocab_size
    gone = (lab >= V) & ~mem_mask.gather(1, (lab - V).clamp(0, mem_mask.shape[1] - 1))
    return lab.masked_fill(((lab == eos_id) | gone).long().cumsum(1) > 0, 0)


def oracle_constraints(b, k, vocab):
    """Each commit's first k distinct reference words (b[1] after <start>, up to <eos>) that also occur among its diff ids
    (sou b[0] or sub_token b[7]), never <unkm> or a special id, as one-word phrases -> [B, k, 1] (zeros where a commit
    has fewer), nbest's `constraints`."""
    special = {vocab[w] for w in ("<start>", "<eos>", "<pad>", "<unkm>") if w in vocab} | {0}
    tar, sou, sub = b[1].tolist(), b[0].tolist(), b[7].tolist()
    out = torch.zeros((len(tar), k, 1), dtype=torch.long)
    for i, ref in enumerate(tar):
        ref = ref[1:ref.index(vocab['<eos>'])] if vocab['<eos>'] in ref else ref[1:]
        diff, words = set(sou[i]) | set(sub[i]), []
        for w in ref:
            if w in diff and w not in special and w not in words and len(words) < k:
                words.append(w)
        out[i, :len(words), 0] = torch.tensor(words, dtype=torch.long)
    return out


def loader(ds, batch_size, shuffle, indices=None):
    sampler = None
    if indices is not None:
        ds = torch.utils.data.Subset(ds, indices)
    return DataLoader(ds, batch_size=batch_size, shuffle=shuffle, sampler=sampler,
                      num_workers=int(os.environ.get("FIRA_WORKERS", 2)),
                      collate_fn=lambda items: collate_packed(items, pin=False), pin_memory=True)


def dev(model, dev_loader, g, valid_index, epoch, dev):
    """Teacher-forced argmax + sentence BLEU (run_model.py:118-184)."""
    vocab, r_vocab, var_maps = g["vocab"], g["r_vocab"], g["var_maps"]
    model.eval()
    out_str, bleus, total = '', 0.0, 0
    with torch.no_grad():
        for idx, batch in enumerate(dev_loader):
            b = batch_to_device(batch, dev)
            out = model(*b, 'dev').cpu().numpy()
            whole, sub, tar = batch[0].numpy(), batch[7].numpy(), batch[1].numpy()
            for i in range(len(out)):
                sen = out[i].tolist()
                if vocab['<eos>'] in sen:
                    sen = sen[:sen.index(vocab['<eos>'])]
                for t in range(len(sen)):
                    if sen[t] >= args.vocab_size + args.sou_len:
                        sen[t] = int(sub[i][sen[t] - args.vocab_size - args.sou_len])
                    elif sen[t] >= args.vocab_size:
                        sen[t] = int(whole[i][sen[t] - args.vocab_size])
                hyp = ' '.join(r_vocab[x] for x in sen).replace('<pad>', "").replace('<unkm>', "😅").strip().split()
                ref = reference_words(tar[i], vocab, r_vocab)
                bleu = sentence_bleu_method2([ref], hyp)
                bleus += bleu
                out_str += ' '.join(deanonymise(hyp, var_maps[valid_index[total + i]])) + ',' + str(bleu) + '\n'
            total += len(out)
            if idx % 10 == 0:
                print("epoch: %d data: %d/%d bleu: %.4f" % (epoch, total, len(dev_loader.dataset), bleus / total))
    return bleus / max(1, len(dev_loader.dataset)), out_str


class ClipLog:
    """The gradient fields of the 10-batch progress line under FIRA_CLIP_NORM: the window's mean norm, summed on the
    device after every step, and the clipped / skipped step counts, all read where the line reads the loss.
    `group()` returns the optim.ClipGroup, or None before it exists."""

    def __init__(self, group):
        self.group, self.sum, self.n = group, None, 0

    def add(self):
        c = self.group()
        if c is not None:
            self.sum = c.grad_norm.clone() if self.sum is None else self.sum + c.grad_norm
            self.n += 1

    def text(self):
        c = self.group()
        if c is None:
            return ""
        mean = float(self.sum) / self.n if self.n else float("nan")
        self.sum, self.n = None, 0
        return " grad_norm: %.4f clipped: %d skipped: %d" % (mean, int(c.clipped.item()), int(c.skipped.item()))


def keep_best(model, scored, best_bleu, progress, checkpoint, dev_output):
    """Appends `<progress> dev bleu: <bleu> is better: <bool>` to OUTPUT/train_process for dev()'s (bleu, output); when
    the BLEU beats best_bleu, saves the model's state_dict to `checkpoint` and the output to OUTPUT/<dev_output> -> the
    best dev BLEU so far."""
    bleu, output_str = scored
    open('OUTPUT/train_process', 'a').write('{} dev bleu: {} is better: {}\n'.format(progress, bleu, bleu > best_bleu))
    if not bleu > best_bleu:
        return best_bleu
    torch.save(model.state_dict(), checkpoint)
    open('OUTPUT/' + dev_output, 'w').write(output_str)
    return bleu


def train_epoch(dp, model, train_loader, epoch, best_bleu, dev_loader, g, valid_index, dev_, ema=None, clip_log=None):
    """ema: None, or {"best": best dev BLEU of the EMA weights so far} when FIRA_EMA is set (updated in place);
    clip_log: a ClipLog when FIRA_CLIP_NORM is set"""
    model.train()
    graphed = isinstance(dp, GraphedTrainStep)
    total_data, total_loss = 0, (torch.zeros((), device=dev_) if graphed else 0.0)
    max_batches = int(os.environ.get("FIRA_MAX_BATCHES", 0))
    for idx, batch in enumerate(train_loader):
        if max_batches and idx >= max_batches:
            break
        if epoch >= 15 and idx % 10 == 0:
            if RANK == 0:
                best_bleu = keep_best(model, dev(model, dev_loader, g, valid_index, epoch, dev_), best_bleu,
                                      f"epoch: {epoch} batch: {idx}", "best_model.pt", "dev_output")
                if ema is not None and dp.opt_ready:
                    # the EMA weights, scored and kept on their own; building the shadow model and the dev loader's
                    # iterator draw from torch's CPU generator, which also shuffles and seeds dropout: fork it, so
                    # training goes on exactly as without FIRA_EMA
                    with torch.random.fork_rng(devices=[]):
                        shadow = dp.ema_model()
                        scored = dev(shadow, dev_loader, g, valid_index, epoch, dev_)
                    ema["best"] = keep_best(shadow, scored, ema["best"], f"ema epoch: {epoch} batch: {idx}",
                                            EMA_CHECKPOINT, "dev_output_ema")
            if WORLD > 1:
                dist.barrier()
            model.train()
        if graphed:
            loss_sum, n_tok = dp.step(batch)              # pinned host batch -> static buffers -> graph replay
            total_loss += loss_sum / n_tok                # stays on the device: no sync per step
        else:
            loss, _ = dp.step(batch_to_device(batch, dev_))
            total_loss += loss.item()
        total_data += (batch.B if hasattr(batch, "shape_key") else len(batch[0])) * WORLD
        if clip_log is not None:
            clip_log.add()
        if idx % 10 == 0 and RANK == 0:
            print("epoch: %d batch: %d/%d  data: %d/%d loss: %.4f" % (
                epoch, idx, len(train_loader), total_data, n_train_total(train_loader) * WORLD, float(total_loss) / 10)
                + (clip_log.text() if clip_log is not None else ""))
            total_loss = torch.zeros((), device=dev_) if graphed else 0.0
    return best_bleu


def n_train_total(train_loader):
    return len(train_loader.indices) if isinstance(train_loader, PackedBatchLoader) else len(train_loader.dataset)


EMA_CHECKPOINT = "best_model_ema.pt"


def ema_settings():
    """FIRA_EMA -> the EMA decay, or None when unset; checked before any device work (SystemExit on an error)."""
    spec = os.environ.get("FIRA_EMA", "")
    if not spec:
        return None
    try:
        d = float(spec)
    except ValueError:
        raise SystemExit(f"FIRA_EMA must be a number in (0, 1), got {spec!r}")
    if not 0.0 < d < 1.0:
        raise SystemExit(f"FIRA_EMA must be a number in (0, 1), got {spec!r}")
    if os.environ.get("FIRA_ENGINE", "graph") != "graph":
        raise SystemExit("FIRA_EMA is kept by the graph engine's flat Adam kernel: unset FIRA_ENGINE=eager")
    return d


def clip_settings(engine_checked=False):
    """FIRA_CLIP_NORM -> the clipping threshold (a positive float, inf allowed), or None when unset; checked before any
    device work (SystemExit on an error).  engine_checked: `train`, where clipping needs the graph engine."""
    spec = os.environ.get("FIRA_CLIP_NORM", "")
    if not spec:
        return None
    try:
        c = float(spec)
    except ValueError:
        raise SystemExit(f"FIRA_CLIP_NORM must be a positive number or inf, got {spec!r}")
    if not c > 0.0:                                              # NaN fails the comparison
        raise SystemExit(f"FIRA_CLIP_NORM must be a positive number or inf, got {spec!r}")
    if engine_checked and os.environ.get("FIRA_ENGINE", "graph") != "graph":
        raise SystemExit("FIRA_CLIP_NORM is applied by the graph engine's flat Adam kernels: unset FIRA_ENGINE=eager")
    return c


def main_train():
    max_grad_norm = clip_settings(engine_checked=True)
    ema_decay = ema_settings()
    dev_ = device()
    if WORLD > 1:
        dist.init_process_group("nccl", device_id=dev_)
    g = load_globals()
    train_set = TransDataset(args, 'train')
    dev_set = TransDataset(args, 'valid')
    all_index = json.load(open('all_index'))
    lo, hi = shard_range(len(train_set), RANK, WORLD)               # graphs shard by commit
    if WORLD > 1:                                                   # equal step counts on every rank: floor-sized
        per = len(train_set) // WORLD                               # contiguous shards (never past the end)
        lo, hi = RANK * per, RANK * per + per
    dev_loader = loader(dev_set, args.batch_size, False)
    model = TransModel(args).to(dev_)
    if os.environ.get("FIRA_ENGINE", "graph") == "graph":
        train_loader = PackedBatchLoader(train_set, args.batch_size, args.vocab_size, shuffle=True,
                                         indices=range(lo, hi) if WORLD > 1 else None, multiples=(8, 16, 16),
                                         max_shapes=int(os.environ.get("FIRA_MAX_SHAPES", 24)), drop_last=WORLD > 1,
                                         bucket=int(os.environ.get("FIRA_BUCKET", 0)),
                                         # per-commit packed node rows (packed.py) by default; FIRA_LAYOUT=trimmed keeps
                                         # the padded batches cut to the batch maximum
                                         packed=os.environ.get("FIRA_LAYOUT", "packed") == "packed")
        from fira_icse_b200.optim import FlatAdam
        dp = GraphedTrainStep(model, args.batch_size,
                              lambda ps: FlatAdam(ps, lr=args.lr, groups=model.flat_groups(), ema_decay=ema_decay,
                                                  max_grad_norm=max_grad_norm),
                              edge_capacity=train_loader.edge_cap)
    else:
        train_loader = loader(train_set, args.batch_size, True, list(range(lo, hi)) if WORLD > 1 else None)
        dp = DataParallelStep(model, lambda ps: Adam(ps, args.lr, fused=True))
    best_bleu = -1
    ema = None if ema_decay is None else {"best": -1}
    clip_log = None if max_grad_norm is None else ClipLog(lambda: dp.clip)
    for epoch in range(args.epoches):
        best_bleu = train_epoch(dp, model, train_loader, epoch, best_bleu, dev_loader, g, all_index['valid'], dev_, ema,
                                clip_log)
    if RANK == 0 and not os.path.exists("best_model.pt"):
        torch.save(model.state_dict(), "best_model.pt")             # short runs never reach the epoch-15 dev gate
    if RANK == 0 and ema is not None and not os.path.exists(EMA_CHECKPOINT):
        # as for best_model.pt; before the first step the average is the initial weights
        torch.save((dp.ema_model() if dp.opt_ready else model).state_dict(), EMA_CHECKPOINT)
    if WORLD > 1:
        dist.destroy_process_group()


_UNCHECKED = object()


def decoder(mode, vocab, knn=_UNCHECKED):
    """FIRA_DECODE -> (output file, decode(model, batch, dataset position of its first commit) -> seq [B, N, T],
    length [B, N] and the numeric columns [B, N] written before each message, how many leading hypotheses of a commit
    count towards the BLEU).  knn: knn_settings' result when the caller has already checked it."""
    ids = dict(tar_len=args.tar_len, start_id=vocab['<start>'], eos_id=vocab['<eos>'], pad_id=vocab['<pad>'])
    k = int(os.environ.get("FIRA_PREFIX_WORDS", 0))
    if k and mode == "beam":
        raise SystemExit("FIRA_PREFIX_WORDS applies to FIRA_DECODE=sample, nbest and mbr; the reference beam search "
                         "takes no prefix")
    no_repeat = int(os.environ.get("FIRA_NO_REPEAT_NGRAM", 0))
    min_len = int(os.environ.get("FIRA_MIN_LENGTH", 0))
    if (no_repeat or min_len) and mode == "beam":
        raise SystemExit("FIRA_NO_REPEAT_NGRAM and FIRA_MIN_LENGTH apply to FIRA_DECODE=sample, nbest and mbr; the "
                         "reference beam search takes no rules")
    rules = dict(no_repeat_ngram=no_repeat, min_length=min_len)
    ens = ensemble_settings(mode)
    n_lex = int(os.environ.get("FIRA_CONSTRAINT_WORDS", 0))
    if n_lex and (mode != "nbest" or int(os.environ.get("FIRA_BEAM_GROUPS", 1)) != 1):
        raise SystemExit("FIRA_CONSTRAINT_WORDS applies to FIRA_DECODE=nbest with FIRA_BEAM_GROUPS=1 only")
    if not 0 <= n_lex <= MAX_PHRASES:
        raise SystemExit(f"FIRA_CONSTRAINT_WORDS must be in [0, {MAX_PHRASES}], got {n_lex}")
    if knn is _UNCHECKED:
        knn = knn_settings(mode, ens)
    tag = (f"_prefix{k}" if k else "") + (f"_norepeat{no_repeat}" if no_repeat else "") + \
        (f"_minlen{min_len}" if min_len else "") + (f"_ens{len(ens[0])}" if ens else "") + \
        (f"_lex{n_lex}" if n_lex else "") + (f"_knn{knn['k']}" if knn else "")

    def pre(b):                         # each commit's own first k reference labels, or no prefix
        return reference_prefix(b, k, vocab['<eos>'], vocab['<pad>']) if k else None
    if mode == "beam":                  # the reference's beam search: its best beam, `<message>`
        def decode(model, b, first_index):
            beams = beam_search(model, b[0], b[3], b[4], b[5], b[7], beam_size=args.beam_size, **ids)
            best, blen = best_sequences(*beams)
            return best.unsqueeze(1), blen.unsqueeze(1), ()
        return "output_fira", decode, 1
    if mode in ("sample", "mbr"):       # FIRA_SAMPLES seeded samples per commit
        n = int(os.environ.get("FIRA_SAMPLES", 16 if mode == "mbr" else 3))
        opts = dict(num_samples=n, temperature=float(os.environ.get("FIRA_TEMPERATURE", 1.0)),
                    top_k=int(os.environ.get("FIRA_TOP_K", 0)), top_p=float(os.environ.get("FIRA_TOP_P", 1.0)),
                    seed=int(os.environ.get("FIRA_SEED", 0)))
    if mode == "sample":                # every sample, `<log-prob>\t<message>`
        def decode(model, b, first_index):
            out = sample(model, b[0], b[3], b[4], b[5], b[7], first_index=first_index, prefix=pre(b), **rules, **opts,
                         **ids)
            return out.seq, out.length, (out.logprob,)
        return "output_fira_samples" + tag, decode, n
    if mode == "mbr":                   # the sample of highest expected BLEU, `<expected BLEU>\t<log-prob>\t<message>`
        def decode(model, b, first_index):
            out = mbr(model, b[0], b[3], b[4], b[5], b[7], first_index=first_index, prefix=pre(b), **rules, **opts,
                      **ids)
            expected = out.utility.gather(1, out.index.unsqueeze(1))
            return out.seq.unsqueeze(1), out.length.unsqueeze(1), (expected, out.logprob.unsqueeze(1))
        return "output_fira_mbr" + tag, decode, 1
    if mode == "nbest":                 # FIRA_BEAM hypotheses best first, `<score>\t<log-prob>\t<message>`
        alpha = float(os.environ.get("FIRA_LENGTH_PENALTY", 0.0))
        groups = int(os.environ.get("FIRA_BEAM_GROUPS", 1))
        diverse = dict(groups=groups, diversity=float(os.environ.get("FIRA_DIVERSITY", 0.5))) if groups != 1 else {}

        def decode(model, b, first_index):
            con = oracle_constraints(b, n_lex, vocab) if n_lex else None
            out = nbest(model, b[0], b[3], b[4], b[5], b[7], beam_size=args.beam_size, length_penalty=alpha, **diverse,
                        prefix=pre(b), **rules, constraints=con, **ids)
            if n_lex:                   # commits whose top hypothesis meets its constraints, commits
                decode.met[0] += int(constraints_met(out.seq[:, :1], out.length[:, :1], con).sum())
                decode.met[1] += out.seq.shape[0]
            return out.seq, out.length, (out.score, out.logprob)
        if n_lex:
            decode.met = [0, 0]
        return "output_fira_nbest" + tag, decode, 1
    raise SystemExit("FIRA_DECODE must be 'beam', 'sample', 'nbest' or 'mbr'")


def test(model, test_loader, g, test_index, dev_, first_index, decode, n_bleu, out_path):
    """Decodes the test split (run_model.py:187-380): N lines per commit in test order, the numeric columns then the
    message -> mean sentence BLEU over the first n_bleu hypotheses of every commit."""
    vocab, r_vocab, var_maps = g["vocab"], g["r_vocab"], g["var_maps"]
    model.eval()
    total, bleus = 0, 0.0
    with open(out_path, 'w') as f:
        for batch in test_loader:
            b = batch_to_device(batch, dev_)
            seq, length, cols = decode(model, b, first_index + total)
            seq, length, cols = seq.cpu().numpy(), length.cpu().numpy(), [c.cpu().numpy() for c in cols]
            tar = batch[1].numpy()
            bleu_batch = 0.0
            for i in range(len(seq)):
                ref = reference_words(tar[i], vocab, r_vocab)
                for k in range(seq.shape[1]):
                    hyp = ids_to_text(seq[i, k][:length[i, k]].tolist(), r_vocab)
                    if k < n_bleu:
                        bl = sentence_bleu_method2([ref], hyp)
                        bleus += bl; bleu_batch += bl
                    f.write(''.join('%.6f\t' % c[i, k] for c in cols) +
                            ' '.join(deanonymise(hyp, var_maps[test_index[total + i]])) + '\n')
            f.flush()
            total += len(seq)
            print("data: %d/%d bleu: %f" % (total, len(test_loader.dataset), bleu_batch / (len(seq) * n_bleu)))
    return bleus / max(1, total * n_bleu)


def ensemble_settings(mode):
    """`test`'s FIRA_ENSEMBLE / FIRA_ENSEMBLE_WEIGHTS -> (checkpoint paths, weights or None for uniform), or None without
    an ensemble; checked before any device work (SystemExit on an error)."""
    if os.environ.get("FIRA_ENSEMBLE", ""):
        if mode == "beam":
            raise SystemExit("FIRA_ENSEMBLE applies to FIRA_DECODE=sample, nbest and mbr; the reference beam search "
                             "decodes one model")
        if "FIRA_CHECKPOINT" in os.environ:
            raise SystemExit("FIRA_ENSEMBLE names the checkpoints itself: unset FIRA_CHECKPOINT")
    return ensemble_checkpoints()


def ensemble_checkpoints():
    """FIRA_ENSEMBLE / FIRA_ENSEMBLE_WEIGHTS -> (checkpoint paths, weights or None for uniform), or None without an
    ensemble (SystemExit on an error)."""
    spec, wspec = os.environ.get("FIRA_ENSEMBLE", ""), os.environ.get("FIRA_ENSEMBLE_WEIGHTS", "")
    if not spec:
        if wspec:
            raise SystemExit("FIRA_ENSEMBLE_WEIGHTS needs FIRA_ENSEMBLE")
        return None
    paths = [p.strip() for p in spec.split(",")]
    if not all(paths) or not 1 <= len(paths) <= MAX_MEMBERS:
        raise SystemExit(f"FIRA_ENSEMBLE must list 1 to {MAX_MEMBERS} checkpoints separated by commas, got {spec!r}")
    weights = None
    if wspec:
        try:
            weights = [float(w) for w in wspec.split(",")]
        except ValueError:
            raise SystemExit(f"FIRA_ENSEMBLE_WEIGHTS must be numbers separated by commas, got {wspec!r}")
        if len(weights) != len(paths):
            raise SystemExit(f"FIRA_ENSEMBLE_WEIGHTS has {len(weights)} weights for {len(paths)} checkpoints")
        if not all(0.0 < w < float("inf") for w in weights):
            raise SystemExit(f"FIRA_ENSEMBLE_WEIGHTS must be positive finite numbers, got {wspec!r}")
    for p in paths:
        if not os.path.isfile(p):
            raise SystemExit(f"FIRA_ENSEMBLE: checkpoint {p} not found")
    return paths, weights


def knn_settings(mode, ens):
    """`test`'s FIRA_KNN / FIRA_KNN_K / FIRA_KNN_TEMPERATURE / FIRA_KNN_LAMBDA -> dict(path, k, temperature, lam, store),
    or None without FIRA_KNN; store is the datastore on the host, loaded once.  Checked before any device work, the
    datastore against the checkpoint on the host (SystemExit on an error)."""
    path = os.environ.get("FIRA_KNN", "")
    if not path:
        return None
    if mode == "beam":
        raise SystemExit("FIRA_KNN applies to FIRA_DECODE=sample, nbest and mbr; the reference beam search decodes the "
                         "model alone")
    if ens:
        raise SystemExit("FIRA_KNN decodes one checkpoint: unset FIRA_ENSEMBLE")
    try:
        s = dict(path=path, k=int(os.environ.get("FIRA_KNN_K", 8)),
                 temperature=float(os.environ.get("FIRA_KNN_TEMPERATURE", 10.0)),
                 lam=float(os.environ.get("FIRA_KNN_LAMBDA", 0.25)))
        check_settings(s["k"], s["temperature"], s["lam"])
    except ValueError as e:
        raise SystemExit(f"FIRA_KNN settings: {e}")
    ckpt = os.environ.get("FIRA_CHECKPOINT", "best_model.pt")
    for p in (path, ckpt):
        if not os.path.isfile(p):
            raise SystemExit(f"FIRA_KNN: {p} not found")
    try:
        store = Datastore.load(path, "cpu", precision=os.environ.get("FIRA_PRECISION", "fp32"))
        check_settings(s["k"], s["temperature"], s["lam"], store.N)
    except ValueError as e:
        raise SystemExit(f"FIRA_KNN: {e}")
    if store.fingerprint != state_fingerprint(torch.load(ckpt, map_location="cpu")):
        raise SystemExit(f"FIRA_KNN: {path} was built by other weights than {ckpt} (fingerprint mismatch)")
    s["store"] = store
    return s


def load_model(path, dev_):
    model = TransModel(args)
    model.load_state_dict(torch.load(path, map_location="cpu"))
    return model.to(dev_)


def main_test():
    mode = os.environ.get("FIRA_DECODE", "beam")
    ens = ensemble_settings(mode)
    knn = knn_settings(mode, ens)                                   # the datastore is read once, on the host
    dev_ = device()
    g = load_globals()
    test_set = TransDataset(args, 'test')
    all_index = json.load(open('all_index'))
    name, decode, n_bleu = decoder(mode, g["vocab"], knn)           # every setting is checked before the models load
    if ens:
        model = Ensemble([load_model(p, dev_) for p in ens[0]], ens[1])
    else:
        model = load_model(os.environ.get("FIRA_CHECKPOINT", "best_model.pt"), dev_)
    if knn:
        model = KNNModel(model, knn.pop("store").to(dev_), k=knn["k"], temperature=knn["temperature"],
                         lam=knn["lam"])
    lo, hi = shard_range(len(test_set), RANK, WORLD)                # replicas only: index ranges, files concatenated
    idx = list(range(lo, hi)) if WORLD > 1 else None
    test_loader = loader(test_set, args.test_batch_size, False, idx)
    out = f"OUTPUT/{name}" if WORLD == 1 else f"OUTPUT/{name}.part{RANK:02d}"
    bleu = test(model, test_loader, g, all_index['test'][lo:hi], dev_, lo, decode, n_bleu, out)
    print("mean sentence bleu: %f" % bleu)
    if hasattr(decode, "met"):
        print("constraints met by the top hypothesis: %f" % (decode.met[0] / max(1, decode.met[1])))


def one_gpu(stage):
    """SystemExit when launched with torchrun: `stage` runs on one GPU."""
    if WORLD > 1:
        raise SystemExit(f"run_model.py {stage} runs on one GPU: launch it without torchrun (WORLD_SIZE=1)")


def finetune_epochs(stage, model, lr, max_grad_norm, epochs, batches, step, progress, checkpoint, dev_output, g, dev_):
    """The epoch loop of `finetune` and `distill`: optim.FlatAdam at `lr` over the model's live parameters, clipped at
    max_grad_norm (FIRA_CLIP_NORM); per epoch e, step(optimizer, e, idx, batch) on every batch of batches(e)
    (FIRA_MAX_BATCHES bounds an epoch), and every 10 batches a progress line ending in progress(the step results since
    the last line); then dev(), keeping the best dev BLEU's weights in `checkpoint` and its output in
    OUTPUT/<dev_output>."""
    from fira_icse_b200 import optim
    opt = optim.FlatAdam(model.live_parameters(), lr=lr, groups=model.flat_groups(), max_grad_norm=max_grad_norm)
    optim.attach(model, [opt])
    clip_log = None if max_grad_norm is None else ClipLog(lambda: opt.clip)
    dev_loader = loader(TransDataset(args, 'valid'), args.batch_size, False)
    valid_index = json.load(open('all_index'))['valid']
    max_batches = int(os.environ.get("FIRA_MAX_BATCHES", 0))
    best_bleu = -1.0
    for epoch in range(epochs):
        train_loader, steps = batches(epoch), []
        for idx, batch in enumerate(train_loader):
            if max_batches and idx >= max_batches:
                break
            steps.append(step(opt, epoch, idx, batch))
            if clip_log is not None:
                clip_log.add()
            if idx % 10 == 0:
                print("%s epoch: %d batch: %d/%d " % (stage, epoch, idx, len(train_loader)) + progress(steps)
                      + (clip_log.text() if clip_log is not None else ""))
                steps = []
        best_bleu = keep_best(model, dev(model, dev_loader, g, valid_index, epoch, dev_), best_bleu,
                              f"{stage} epoch: {epoch}", checkpoint, dev_output)
    print("best dev bleu: %f" % best_bleu)


def finetune_settings():
    """The finetune stage's settings from the environment, checked before any device work (SystemExit on an error)."""
    one_gpu("finetune")
    try:
        s = dict(epochs=int(os.environ.get("FIRA_SCST_EPOCHS", 1)), lr=float(os.environ.get("FIRA_SCST_LR", 1e-5)),
                 num_samples=int(os.environ.get("FIRA_SAMPLES", 5)),
                 temperature=float(os.environ.get("FIRA_TEMPERATURE", 1.0)), top_k=int(os.environ.get("FIRA_TOP_K", 0)),
                 top_p=float(os.environ.get("FIRA_TOP_P", 1.0)), seed=int(os.environ.get("FIRA_SEED", 0)),
                 no_repeat_ngram=int(os.environ.get("FIRA_NO_REPEAT_NGRAM", 0)),
                 min_length=int(os.environ.get("FIRA_MIN_LENGTH", 0)))
    except ValueError as e:
        raise SystemExit(f"run_model.py finetune: {e}")
    if s["epochs"] < 1:
        raise SystemExit(f"FIRA_SCST_EPOCHS must be >= 1, got {s['epochs']}")
    if not 0.0 < s["lr"] < float("inf"):
        raise SystemExit(f"FIRA_SCST_LR must be a positive finite number, got {s['lr']}")
    sampling = {k: s[k] for k in ("num_samples", "temperature", "top_k", "top_p", "seed", "no_repeat_ngram",
                                  "min_length")}
    try:                # the batches' references are checked per step
        check_step(None, **sampling, first_index=0, tar_len=args.tar_len, eos_id=None)
    except ValueError as e:
        raise SystemExit(f"run_model.py finetune: {e}")
    return s, sampling


def main_finetune():
    max_grad_norm = clip_settings()
    s, sampling = finetune_settings()
    dev_ = device()
    g = load_globals()
    vocab = g["vocab"]
    ids = dict(tar_len=args.tar_len, start_id=vocab['<start>'], eos_id=vocab['<eos>'], pad_id=vocab['<pad>'])
    train_loader = loader(TransDataset(args, 'train'), args.batch_size, True)
    model = load_model("best_model.pt", dev_)

    def step(opt, epoch, idx, batch):          # every batch but an epoch's last holds batch_size commits
        return scst_step(model, opt, batch_to_device(batch, dev_), **dict(sampling, seed=sampling["seed"] + epoch),
                         first_index=idx * args.batch_size, **ids)

    def progress(steps):
        return "reward: %.4f |advantage|: %.4f loss: %.6f" % (
            sum(x.reward for x in steps) / len(steps), steps[-1].advantage, steps[-1].loss)
    finetune_epochs("scst", model, s["lr"], max_grad_norm, s["epochs"], lambda epoch: train_loader, step, progress,
                    "best_model_scst.pt", "dev_output_scst", g, dev_)


KD_CHECKPOINT = "best_model_kd.pt"


def distill_settings():
    """The distill stage's settings from the environment, checked before any device work (SystemExit on an error) ->
    (settings, student checkpoint, (teacher checkpoints, weights or None))."""
    one_gpu("distill")
    try:
        s = dict(alpha=float(os.environ.get("FIRA_KD_ALPHA", 0.5)), epochs=int(os.environ.get("FIRA_KD_EPOCHS", 1)),
                 lr=float(os.environ.get("FIRA_KD_LR", 1e-4)))
    except ValueError as e:
        raise SystemExit(f"run_model.py distill: {e}")
    if not 0.0 <= s["alpha"] <= 1.0:
        raise SystemExit(f"FIRA_KD_ALPHA must be a number in [0, 1], got {s['alpha']}")
    if s["epochs"] < 1:
        raise SystemExit(f"FIRA_KD_EPOCHS must be >= 1, got {s['epochs']}")
    if not 0.0 < s["lr"] < float("inf"):
        raise SystemExit(f"FIRA_KD_LR must be a positive finite number, got {s['lr']}")
    targets = os.environ.get("FIRA_KD_TARGETS", "")
    if targets:
        if os.environ.get("FIRA_ENSEMBLE", ""):
            raise SystemExit("FIRA_KD_TARGETS is the teacher: unset FIRA_ENSEMBLE")
        if not os.path.isfile(targets):
            raise SystemExit(f"FIRA_KD_TARGETS: {targets} not found")
        teacher = targets
    else:
        teacher = ensemble_checkpoints()
        if teacher is None:
            raise SystemExit("run_model.py distill needs the teacher: FIRA_ENSEMBLE=a.pt[,b.pt,...] or "
                             "FIRA_KD_TARGETS=kd_targets.pt")
    student = os.environ.get("FIRA_CHECKPOINT", "best_model.pt")
    if not os.path.isfile(student):
        raise SystemExit(f"FIRA_CHECKPOINT: student checkpoint {student} not found")
    out = os.path.realpath(KD_CHECKPOINT)
    if not targets and any(os.path.realpath(p) == out for p in teacher[0]):
        raise SystemExit(f"FIRA_ENSEMBLE names {KD_CHECKPOINT}, which distill writes: copy the teacher elsewhere")
    return s, student, teacher


def load_targets(path, train_set):
    """The KDTargets file of FIRA_KD_TARGETS, checked against the vocabulary and the train split on the host
    (SystemExit on an error)."""
    try:
        return KDTargets.load(path, vocab_size=args.vocab_size, commits=len(train_set))
    except (ValueError, RuntimeError, OSError, KeyError) as e:
        raise SystemExit(f"FIRA_KD_TARGETS: {e}")


def main_distill():
    max_grad_norm = clip_settings()
    s, student, teacher_spec = distill_settings()
    if isinstance(teacher_spec, str):
        g = load_globals()
        train_set = TransDataset(args, 'train')
        targets = load_targets(teacher_spec, train_set)       # before any device work
        seed = int(os.environ.get("FIRA_SEED", 0))
        dev_ = device()
    else:
        targets = None
        dev_ = device()
        g = load_globals()
        train_set = TransDataset(args, 'train')
        train_loader = loader(train_set, args.batch_size, True)
    model = load_model(student, dev_)
    teacher = Ensemble([load_model(p, dev_) for p in teacher_spec[0]], teacher_spec[1]) if targets is None else None
    perm = None

    def batches(epoch):
        nonlocal perm
        if targets is None:
            return train_loader
        # a seeded permutation: each batch's dataset positions are known
        perm = torch.randperm(len(train_set), generator=torch.Generator().manual_seed(seed + epoch)).tolist()
        return loader(train_set, args.batch_size, False, indices=perm)

    def step(opt, epoch, idx, batch):
        t = teacher
        if targets is not None:
            pos = perm[idx * args.batch_size: idx * args.batch_size + batch[6].shape[0]]
            t = targets.batch(pos, TransModel.shifted_label(batch[6]), device=dev_)
        return distill_step(model, opt, batch_to_device(batch, dev_), t, alpha=s["alpha"])

    def progress(steps):
        return "loss: %.4f nll: %.4f kd: %.4f tokens: %d" % (steps[-1].loss, steps[-1].nll, steps[-1].kd,
                                                             steps[-1].tokens)
    finetune_epochs("kd", model, s["lr"], max_grad_norm, s["epochs"], batches, step, progress, KD_CHECKPOINT,
                    "dev_output_kd", g, dev_)


def kd_targets_settings():
    """`kd-targets`' settings, checked before any device work (SystemExit on an error) -> (k, (teacher checkpoints,
    weights or None), output path)."""
    one_gpu("kd-targets")
    try:
        k = int(os.environ.get("FIRA_KD_TOPK", 8))
    except ValueError as e:
        raise SystemExit(f"FIRA_KD_TOPK: {e}")
    if not 1 <= k <= MAX_TOPK:
        raise SystemExit(f"FIRA_KD_TOPK must be in [1, {MAX_TOPK}], got {k}")
    teacher = ensemble_checkpoints()
    if teacher is None:
        raise SystemExit("run_model.py kd-targets needs the teacher: FIRA_ENSEMBLE=a.pt[,b.pt,...]")
    return k, teacher, os.environ.get("FIRA_KD_TARGETS", "kd_targets.pt")


def main_kd_targets():
    k, (paths, weights), out = kd_targets_settings()
    dev_ = device()
    load_globals()
    train_set = TransDataset(args, 'train')
    teacher = Ensemble([load_model(p, dev_) for p in paths], weights)
    batches = (batch_to_device(b, dev_) for b in loader(train_set, args.batch_size, False))
    t0 = time.perf_counter()
    targets = build_targets(teacher, batches, k=k, first_index=0)
    dt = time.perf_counter() - t0
    targets.save(out)
    print("kd-targets: %d commits, %d rows, k = %d, %d bytes, mean kept mass %.4f, %.1f commits/s -> %s" % (
        targets.n, targets.rows, k, targets.nbytes, float(targets.mass.double().mean()) if targets.rows else 0.0,
        targets.n / dt, out))


def main_datastore():
    one_gpu("datastore")
    ckpt = os.environ.get("FIRA_CHECKPOINT", "best_model.pt")
    out = os.environ.get("FIRA_DATASTORE", "datastore.pt")
    if not os.path.isfile(ckpt):
        raise SystemExit(f"FIRA_CHECKPOINT: {ckpt} not found")
    dev_ = device()
    g = load_globals()
    vocab = g["vocab"]
    train_set = TransDataset(args, 'train')
    model = load_model(ckpt, dev_)
    batches = (batch_to_device(b, dev_) for b in loader(train_set, args.batch_size, False))
    store = build_datastore(model, batches, first_index=0, start_id=vocab['<start>'], eos_id=vocab['<eos>'],
                            pad_id=vocab['<pad>'], unk_id=vocab['<unkm>'])
    store.save(out)
    print("datastore: %d entries, %d bytes -> %s" % (store.N, store.nbytes, out))


if __name__ == '__main__':
    stage = str(sys.argv[1])
    seed_everything()
    os.makedirs('OUTPUT', exist_ok=True)
    if stage == 'train':
        main_train()
    elif stage == 'test':
        main_test()
    elif stage == 'finetune':
        main_finetune()
    elif stage == 'distill':
        main_distill()
    elif stage == 'datastore':
        main_datastore()
    elif stage == 'kd-targets':
        main_kd_targets()
    else:
        raise SystemExit("usage: python run_model.py train|test|finetune|distill|datastore|kd-targets")
