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


def train_epoch(dp, model, train_loader, epoch, best_bleu, dev_loader, g, valid_index, dev_):
    model.train()
    graphed = isinstance(dp, GraphedTrainStep)
    total_data, total_loss = 0, (torch.zeros((), device=dev_) if graphed else 0.0)
    max_batches = int(os.environ.get("FIRA_MAX_BATCHES", 0))
    for idx, batch in enumerate(train_loader):
        if max_batches and idx >= max_batches:
            break
        if epoch >= 15 and idx % 10 == 0:
            if RANK == 0:
                cur_bleu, output_str = dev(model, dev_loader, g, valid_index, epoch, dev_)
                open('OUTPUT/train_process', 'a').write(
                    'epoch: {} batch: {} dev bleu: {} is better: {}\n'.format(epoch, idx, cur_bleu, cur_bleu > best_bleu))
                if cur_bleu > best_bleu:
                    best_bleu = cur_bleu
                    torch.save(model.state_dict(), "best_model.pt")
                    open('OUTPUT/dev_output', 'w').write(output_str)
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
        if idx % 10 == 0 and RANK == 0:
            print("epoch: %d batch: %d/%d  data: %d/%d loss: %.4f" % (
                epoch, idx, len(train_loader), total_data, n_train_total(train_loader) * WORLD, float(total_loss) / 10))
            total_loss = torch.zeros((), device=dev_) if graphed else 0.0
    return best_bleu


def n_train_total(train_loader):
    return len(train_loader.indices) if isinstance(train_loader, PackedBatchLoader) else len(train_loader.dataset)


def main_train():
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
        dp = GraphedTrainStep(model, args.batch_size, lambda ps: FlatAdam(ps, lr=args.lr, groups=model.flat_groups()),
                              edge_capacity=train_loader.edge_cap)
    else:
        train_loader = loader(train_set, args.batch_size, True, list(range(lo, hi)) if WORLD > 1 else None)
        dp = DataParallelStep(model, lambda ps: Adam(ps, args.lr, fused=True))
    best_bleu = -1
    for epoch in range(args.epoches):
        best_bleu = train_epoch(dp, model, train_loader, epoch, best_bleu, dev_loader, g, all_index['valid'], dev_)
    if RANK == 0 and not os.path.exists("best_model.pt"):
        torch.save(model.state_dict(), "best_model.pt")             # short runs never reach the epoch-15 dev gate
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


def finetune_settings():
    """The finetune stage's settings from the environment, checked before any device work (SystemExit on an error)."""
    if WORLD > 1:
        raise SystemExit("run_model.py finetune runs on one GPU: launch it without torchrun (WORLD_SIZE=1)")
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
    s, sampling = finetune_settings()
    dev_ = device()
    g = load_globals()
    vocab = g["vocab"]
    ids = dict(tar_len=args.tar_len, start_id=vocab['<start>'], eos_id=vocab['<eos>'], pad_id=vocab['<pad>'])
    train_set = TransDataset(args, 'train')
    dev_set = TransDataset(args, 'valid')
    all_index = json.load(open('all_index'))
    model = TransModel(args)
    model.load_state_dict(torch.load("best_model.pt", map_location="cpu"))
    model = model.to(dev_)
    from fira_icse_b200 import optim
    opt = optim.FlatAdam(model.live_parameters(), lr=s["lr"], groups=model.flat_groups())
    optim.attach(model, [opt])
    train_loader = loader(train_set, args.batch_size, True)
    dev_loader = loader(dev_set, args.batch_size, False)
    max_batches = int(os.environ.get("FIRA_MAX_BATCHES", 0))
    best_bleu = -1.0
    for epoch in range(s["epochs"]):
        total, rewards = 0, []
        for idx, batch in enumerate(train_loader):
            if max_batches and idx >= max_batches:
                break
            b = batch_to_device(batch, dev_)
            step = scst_step(model, opt, b, **dict(sampling, seed=sampling["seed"] + epoch), first_index=total, **ids)
            rewards.append(step.reward)
            total += len(b[0])
            if idx % 10 == 0:
                print("scst epoch: %d batch: %d/%d reward: %.4f |advantage|: %.4f loss: %.6f" % (
                    epoch, idx, len(train_loader), sum(rewards) / len(rewards), step.advantage, step.loss))
                rewards = []
        cur_bleu, output_str = dev(model, dev_loader, g, all_index['valid'], epoch, dev_)
        open('OUTPUT/train_process', 'a').write(
            'scst epoch: {} dev bleu: {} is better: {}\n'.format(epoch, cur_bleu, cur_bleu > best_bleu))
        if cur_bleu > best_bleu:
            best_bleu = cur_bleu
            torch.save(model.state_dict(), "best_model_scst.pt")
            open('OUTPUT/dev_output_scst', 'w').write(output_str)
    print("best dev bleu: %f" % best_bleu)


KD_CHECKPOINT = "best_model_kd.pt"


def distill_settings():
    """The distill stage's settings from the environment, checked before any device work (SystemExit on an error) ->
    (settings, student checkpoint, (teacher checkpoints, weights or None))."""
    if WORLD > 1:
        raise SystemExit("run_model.py distill runs on one GPU: launch it without torchrun (WORLD_SIZE=1)")
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
    dev_set = TransDataset(args, 'valid')
    all_index = json.load(open('all_index'))
    model = load_model(student, dev_)
    teacher = Ensemble([load_model(p, dev_) for p in teacher_spec[0]], teacher_spec[1]) if targets is None else None
    from fira_icse_b200 import optim
    opt = optim.FlatAdam(model.live_parameters(), lr=s["lr"], groups=model.flat_groups())
    optim.attach(model, [opt])
    train_loader = loader(train_set, args.batch_size, True) if targets is None else None
    dev_loader = loader(dev_set, args.batch_size, False)
    max_batches = int(os.environ.get("FIRA_MAX_BATCHES", 0))
    best_bleu = -1.0
    for epoch in range(s["epochs"]):
        if targets is not None:                 # a seeded permutation: each batch's dataset positions are known
            perm = torch.randperm(len(train_set), generator=torch.Generator().manual_seed(seed + epoch)).tolist()
            train_loader = loader(train_set, args.batch_size, False, indices=perm)
        for idx, batch in enumerate(train_loader):
            if max_batches and idx >= max_batches:
                break
            if targets is not None:
                pos = perm[idx * args.batch_size: idx * args.batch_size + batch[6].shape[0]]
                teacher = targets.batch(pos, TransModel.shifted_label(batch[6]), device=dev_)
            step = distill_step(model, opt, batch_to_device(batch, dev_), teacher, alpha=s["alpha"])
            if idx % 10 == 0:
                print("kd epoch: %d batch: %d/%d loss: %.4f nll: %.4f kd: %.4f tokens: %d" % (
                    epoch, idx, len(train_loader), step.loss, step.nll, step.kd, step.tokens))
        cur_bleu, output_str = dev(model, dev_loader, g, all_index['valid'], epoch, dev_)
        open('OUTPUT/train_process', 'a').write(
            'kd epoch: {} dev bleu: {} is better: {}\n'.format(epoch, cur_bleu, cur_bleu > best_bleu))
        if cur_bleu > best_bleu:
            best_bleu = cur_bleu
            torch.save(model.state_dict(), KD_CHECKPOINT)
            open('OUTPUT/dev_output_kd', 'w').write(output_str)
    print("best dev bleu: %f" % best_bleu)


def kd_targets_settings():
    """`kd-targets`' settings, checked before any device work (SystemExit on an error) -> (k, (teacher checkpoints,
    weights or None), output path)."""
    if WORLD > 1:
        raise SystemExit("run_model.py kd-targets runs on one GPU: launch it without torchrun (WORLD_SIZE=1)")
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
    if WORLD > 1:
        raise SystemExit("run_model.py datastore runs on one GPU: launch it without torchrun (WORLD_SIZE=1)")
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
