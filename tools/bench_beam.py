#!/usr/bin/env python
"""Beam-search inference throughput (BASELINE.json config 4: `run_model.py test`, beam 3 / 5).

Synthetic commits with the DataSet node/edge distribution, random-initialised weights.  With random
weights no beam emits <eos>, so every batch runs all tar_len-1 = 29 decoding steps: the worst case the
reference's own loop was timed on in BASELINE.md (72 s for 32 commits on CPU).  One JSON line per
(batch, beam) configuration; timing with CUDA events around whole batches, inputs resident on the device.

    python tools/bench_beam.py [--batches 20,128] [--beams 3,5] [--precision fp32|bf16] [--reps 3]
                               [--modes full,graph,sample,nbest,diverse,mbr] [--diversity 0.5]
                               (sample: N = the beam width;
                               nbest: beam.nbest, log-space n-best beam search with length_penalty 0;
                               diverse: beam.nbest with groups = the beam width and --diversity;
                               mbr: mbr.mbr over N = the beam width samples)
                               [--prefix-words k]
                               (k > 0: sample, nbest, diverse and mbr are also timed with each commit's first k
                               reference labels (tar_label, never <eos>) as a prefix, next to the same mode without
                               one; those lines carry prefix_words = k)
                               [--no-repeat-ngram n] [--min-length m]
                               (either > 0: sample, nbest, diverse and mbr are also timed with n-gram repeat blocking
                               and the minimum length, next to the same mode without them; every line of those modes
                               carries repeat_share, the share of returned hypotheses (mbr: the chosen ones) in which
                               a word repeats an n-gram, n = repeat_share_n = n or 2, and mean_length (tokens with
                               <start> and <eos>); the lines with the rules carry no_repeat_ngram and min_length)

    python tools/bench_beam.py --ensemble 1,2,4 [--batches ...] [--beams ...] [--precision ...] [--reps ...]
                               (ensemble decoding instead of the modes above: for each member count M, an
                               ensemble.Ensemble of the bench model and M - 1 copies whose out_fc / copy_net weights
                               carry their own seeded perturbation; sample, nbest and mbr per batch at the first beam
                               width, then fira_pointer_mix_ensemble alone with its algorithmic bytes per row
                               M * 2 * (V * s + S * 4) + (V + S) * 4 (s = 2 bytes in bf16, 4 in fp32: each member row is
                               read twice, the fp32 triple written once) and the share of HBM peak that implies)

    python tools/bench_beam.py --constraint-words k [--batches ...] [--beams ...] [--precision ...] [--reps ...]
                               (lexically constrained n-best instead of the modes above: nbest per batch and beam
                               width without and with each commit's first k distinct reference words that occur in
                               its diff as one-word phrases (run_model.oracle_constraints), in the same run, each line
                               with met_share, the share of commits whose top hypothesis meets the constraints; then
                               one step call, fira_pointer_mix_beam_step_lexical against fira_pointer_mix_beam_step_rules,
                               at B = 128, pos = 20 with every slot live)

nbest and diverse lines also carry `self_bleu`: the mean pairwise id-level sentence BLEU among each commit's K
hypotheses (one fira_mbr_select launch with pair_bleu, off-diagonal entries averaged over the batch); lower means a
more diverse list.

mbr also prints one line for fira_mbr_select alone on the batch's own samples: the median device time per launch
(bench.time_launches: launches replayed from a CUDA graph between CUDA events), next to the host time of the same
selection with bleu.sentence_bleu_method2 (tests/mbr_rule.py, one pass over the batch) and the largest utility difference
between the two.
"""
import argparse
import ctypes
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))     # mbr_rule: the host restatement the selection is compared with


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="20,128")
    ap.add_argument("--beams", default="3,5")
    ap.add_argument("--precision", default="fp32")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--trim", action="store_true", help="loader-side padding trimming (data.trim_batch_host)")
    ap.add_argument("--modes", default="full,graph")
    ap.add_argument("--diversity", type=float, default=0.5, help="diverse mode's penalty per repeated word")
    ap.add_argument("--prefix-words", type=int, default=0, help="also time the decoders with k-label reference prefixes")
    ap.add_argument("--no-repeat-ngram", type=int, default=0, help="also time the decoders with n-gram repeat blocking")
    ap.add_argument("--min-length", type=int, default=0, help="also time the decoders with a minimum message length")
    ap.add_argument("--ensemble", default="", help="member counts M to time ensemble decoding at (e.g. 1,2,4)")
    ap.add_argument("--constraint-words", type=int, default=0, help="time nbest with k oracle constraint words")
    a = ap.parse_args()
    rules = (a.no_repeat_ngram, a.min_length)
    import torch
    import __graft_entry__
    __graft_entry__.build()
    import bench
    import fira_icse_b200 as F
    from fira_icse_b200 import _lib
    from fira_icse_b200.beam import beam_search, nbest
    from fira_icse_b200.mbr import mbr
    from fira_icse_b200.sample import sample
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = F.TransModel(bench.model_args()).to(dev)
    model.set_precision(a.precision)
    model.eval()
    if a.ensemble:
        return bench_ensemble(a, model, dev)
    if a.constraint_words:
        return bench_lexical(a, model, dev)
    for B in (int(x) for x in a.batches.split(",")):
        hb = bench.host_batch(10_000, B, pin=False, trim=a.trim)
        b = bench.device_batch(hb, dev, B)
        lab = b[6][:, 1:1 + a.prefix_words]                         # the reference prefixes: never <eos> (id 2)
        ref_prefix = lab.masked_fill((lab == 2).long().cumsum(1) > 0, 0)
        decoders = ("sample", "nbest", "diverse", "mbr")
        cases = [(int(x), m, pw, rl) for x in a.beams.split(",") for m in a.modes.split(",")
                 for pw in ((0, a.prefix_words) if a.prefix_words and m in decoders else (0,))
                 for rl in (((0, 0), rules) if any(rules) and m in decoders else ((0, 0),))]
        for K, mode, pw, rl in cases:
            pre = dict(prefix=ref_prefix) if pw else {}
            if any(rl):
                pre.update(no_repeat_ngram=rl[0], min_length=rl[1])

            def run():
                if mode == "sample":                                 # N = the beam width, default T / k / p
                    return sample(model, b[0], b[3], b[4], b[5], b[7], num_samples=K, tar_len=30, start_id=1, eos_id=2,
                                  pad_id=0, **pre)
                if mode == "mbr":
                    return mbr(model, b[0], b[3], b[4], b[5], b[7], num_samples=K, tar_len=30, start_id=1, eos_id=2,
                               pad_id=0, **pre)
                if mode == "nbest":
                    return nbest(model, b[0], b[3], b[4], b[5], b[7], beam_size=K, tar_len=30, start_id=1, eos_id=2,
                                 pad_id=0, **pre)
                if mode == "diverse":
                    return nbest(model, b[0], b[3], b[4], b[5], b[7], beam_size=K, tar_len=30, start_id=1, eos_id=2,
                                 pad_id=0, groups=K, diversity=a.diversity, **pre)
                return beam_search(model, b[0], b[3], b[4], b[5], b[7], beam_size=K, tar_len=30, start_id=1, eos_id=2,
                                   pad_id=0, mode=mode)
            ref = run()                                              # warm-up (lazy CUDA state, graph capture)
            if mode == "full":
                ref_full = ref
            same = bool(torch.equal(ref[0], ref_full[0])) if "full" in a.modes.split(",") and mode not in ("sample", "nbest", "mbr") else None
            torch.cuda.synchronize()
            n0 = _lib.LAUNCH_COUNT
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.reps):
                out = run()
            length = out.samples.length if mode == "mbr" else out.length if mode in ("sample", "nbest", "diverse") else out[1]
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / a.reps
            metric = {"sample": "sampling", "mbr": "mbr"}.get(mode, "beam-search") + " inference throughput"
            extra = {"prefix_words": pw} if a.prefix_words else {}
            if a.prefix_words:
                extra.update(card=torch.cuda.get_device_name(dev), power_limit_w=power_limit())
            if any(rules) and mode in decoders:
                seq, ln = (out.seq.unsqueeze(1), out.length.unsqueeze(1)) if mode == "mbr" else (out.seq, out.length)
                count_n = a.no_repeat_ngram or 2
                extra.update(card=torch.cuda.get_device_name(dev), power_limit_w=power_limit(),
                             repeat_share=repeat_share(seq, ln, count_n), repeat_share_n=count_n,
                             mean_length=ln.double().mean().item())
                if any(rl):
                    extra.update(no_repeat_ngram=rl[0], min_length=rl[1])
            if mode in ("nbest", "diverse"):
                extra.update(self_bleu=self_bleu(out, B, K), card=torch.cuda.get_device_name(dev),
                             power_limit_w=power_limit())
                if mode == "diverse":
                    extra.update(groups=K, diversity=a.diversity)
            print(json.dumps({**extra,
                "metric": metric, "unit": "commits/s", "value": B / ms * 1e3,
                "ms_per_batch": ms, "batch": B, "beam": K, "decoded_steps": int(length.max().item()) - 1,
                "precision": a.precision, "mode": mode, "ids_equal_full_mode": same, "trimmed": bool(a.trim), "data": "synthetic (DataSet distribution), random weights",
                "c_abi_calls_per_batch": (_lib.LAUNCH_COUNT - n0) // a.reps,
                "note": "encoder once per batch; full = 30-position decoder re-run per step over all live beams, "
                        "graph = newest row against K/V caches as CUDA-graph replays, "
                        "sample = beam-width seeded samples per commit (T = 1, no top-k / top-p), one graph per position, "
                        "nbest = log-space n-best beam search (length_penalty 0), one graph per position, "
                        "diverse = nbest with groups = K and the given diversity, one graph per position, "
                        "mbr = sample + one fira_mbr_select launch"}),
                  flush=True)
            if mode == "mbr":
                print(json.dumps(mbr_select_timing(out.samples, B, K)), flush=True)


HBM_PEAK_GBS = 3350.0     # H100 SXM5 80 GB HBM3 peak


def bench_ensemble(a, model, dev):
    """--ensemble: decoders and the combine kernel at each member count (module docstring)."""
    import copy
    import torch
    import bench
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import FIRA_BF16, FIRA_F32, call
    from fira_icse_b200.beam import nbest
    from fira_icse_b200.ensemble import Ensemble
    from fira_icse_b200.mbr import mbr
    from fira_icse_b200.sample import sample
    counts = [int(x) for x in a.ensemble.split(",")]
    K = int(a.beams.split(",")[0])
    pool = [model]
    for i in range(1, max(counts)):
        m = copy.deepcopy(model)
        g = torch.Generator(device=dev).manual_seed(i)
        with torch.no_grad():
            for p in (m.out_fc.weight, m.copy_net.LinearRes.weight, m.copy_net.LinearProb.weight):
                p.add_(torch.randn(p.shape, generator=g, device=dev) * p.std() * 0.1)
        pool.append(m.set_precision(a.precision).eval())
    card, watts = torch.cuda.get_device_name(dev), power_limit()
    ids = dict(tar_len=30, start_id=1, eos_id=2, pad_id=0)
    for B in (int(x) for x in a.batches.split(",")):
        b = bench.device_batch(bench.host_batch(10_000, B, pin=False, trim=a.trim), dev, B)
        S = b[0].shape[1] + b[7].shape[1]
        for M in counts:
            ens = Ensemble(pool[:M])
            runs = {"sample": lambda: sample(ens, b[0], b[3], b[4], b[5], b[7], num_samples=K, **ids),
                    "nbest": lambda: nbest(ens, b[0], b[3], b[4], b[5], b[7], beam_size=K, **ids),
                    "mbr": lambda: mbr(ens, b[0], b[3], b[4], b[5], b[7], num_samples=K, **ids)}
            for mode, run in runs.items():
                out = run()                                              # warm-up (graph capture)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.reps):
                    out = run()
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / a.reps
                length = out.samples.length if mode == "mbr" else out.length
                print(json.dumps({"metric": "ensemble decoding throughput", "unit": "commits/s", "value": B / ms * 1e3,
                                  "ms_per_batch": ms, "batch": B, "beam": K, "members": M, "mode": mode,
                                  "decoded_steps": int(length.max().item()) - 1, "precision": a.precision,
                                  "card": card, "power_limit_w": watts,
                                  "data": "synthetic (DataSet distribution), random weights, perturbed copies"}),
                      flush=True)
            # the combine alone: rotating member buffers (more than L2 in all), launches replayed from a CUDA graph
            V, R = model.vocab_size, B * K
            ldl = ops._ld_logits(V)
            tdt = torch.bfloat16 if a.precision == "bf16" else torch.float32
            es = 2 if a.precision == "bf16" else 4
            set_bytes = M * R * (ldl * es + S * 4 + 8)
            n_rot = max(2, -(-200 * 2 ** 20 // set_bytes))
            gen = torch.Generator(device=dev).manual_seed(M)
            sets = []
            for _ in range(n_rot):
                mem = [(torch.randn((R, ldl), generator=gen, device=dev).to(tdt),
                        torch.randn((B, K, S), generator=gen, device=dev), torch.randn((R, 2), generator=gen, device=dev))
                       for _ in range(M)]
                arr = [(ctypes.c_void_p * M)(*[ops._ptr(t[k]) for t in mem]) for k in range(3)]
                sets.append((mem, arr))
            mask = torch.ones((B, S), dtype=torch.uint8, device=dev)
            lw = torch.full((M,), -math.log(M), dtype=torch.float32, device=dev)
            x = torch.empty((R, ldl), dtype=torch.float32, device=dev)
            c = torch.empty((B, K, S), dtype=torch.float32, device=dev)
            gl = torch.empty((R, 2), dtype=torch.float32, device=dev)

            def launch(i):
                arr = sets[i % n_rot][1]
                call("fira_pointer_mix_ensemble", ctypes.addressof(arr[0]), ldl, ctypes.addressof(arr[1]),
                     ctypes.addressof(arr[2]), M, ops._ptr(lw), ops._ptr(mask), ops._ptr(x), ldl, ops._ptr(c),
                     ops._ptr(gl), B, K, V, S, FIRA_BF16 if a.precision == "bf16" else FIRA_F32, ops._stream())
            _, med_ms, launches = bench.time_launches(launch, n_rot)
            row_bytes = M * 2 * (V * es + S * 4) + (V + S) * 4
            gbs = row_bytes * R / (med_ms * 1e-3) / 1e9
            print(json.dumps({"metric": "fira_pointer_mix_ensemble time", "unit": "us", "value": med_ms * 1e3,
                              "batch": B, "rows": R, "members": M, "V": V, "S": S, "precision": a.precision,
                              "algorithmic_bytes_per_row": row_bytes, "algorithmic_GB_per_s": gbs,
                              "share_of_hbm_peak": gbs / HBM_PEAK_GBS, "hbm_peak_GB_per_s": HBM_PEAK_GBS,
                              "timed_launches": launches, "rotating_sets": n_rot, "card": card, "power_limit_w": watts,
                              "note": "median device time per launch, launches replayed from one CUDA graph between "
                                      "CUDA events; bytes count each member row twice (the second read is meant to "
                                      "come from L2)"}), flush=True)
            del sets


def bench_lexical(a, model, dev):
    """--constraint-words: nbest without and with oracle constraints, then one step call of each kernel (module
    docstring)."""
    import torch
    import bench
    import run_model
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import FIRA_BF16, FIRA_F32, call
    from fira_icse_b200.beam import constraints_met, nbest
    card, watts = torch.cuda.get_device_name(dev), power_limit()
    ids = dict(tar_len=30, start_id=1, eos_id=2, pad_id=0)
    vocab = {"<start>": 1, "<eos>": 2, "<pad>": 0}
    for B in (int(x) for x in a.batches.split(",")):
        b = bench.device_batch(bench.host_batch(10_000, B, pin=False, trim=a.trim), dev, B)
        con = run_model.oracle_constraints(b, a.constraint_words, vocab)
        for K in (int(x) for x in a.beams.split(",")):
            for c in (None, con):
                def run():
                    return nbest(model, b[0], b[3], b[4], b[5], b[7], beam_size=K, constraints=c, **ids)
                out = run()                                              # warm-up (graph capture)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.reps):
                    out = run()
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / a.reps
                met = constraints_met(out.seq[:, :1], out.length[:, :1], con)
                print(json.dumps({"metric": "lexically constrained n-best throughput", "unit": "commits/s",
                                  "value": B / ms * 1e3, "ms_per_batch": ms, "batch": B, "beam": K,
                                  "constraint_words": a.constraint_words if c is not None else 0,
                                  "commits_with_constraints": int((con != 0).any(-1).any(-1).sum()),
                                  "met_share": met.float().mean().item(), "mean_length": out.length.double().mean().item(),
                                  "decoded_steps": int(out.length.max().item()) - 1, "precision": a.precision,
                                  "card": card, "power_limit_w": watts,
                                  "data": "synthetic (DataSet distribution), random weights"}), flush=True)
    # one step call at B = 128, pos = 20: every slot live, random histories, the bench model's V and S = 370
    gen = torch.Generator(device=dev).manual_seed(5)
    B, K, T, pos, S, V = 128, int(a.beams.split(",")[0]), 30, 20, 370, model.vocab_size
    R = B * K
    ldl = ops._ld_logits(V)
    tdt = torch.bfloat16 if a.precision == "bf16" else torch.float32
    logits = (torch.randn((R, ldl), generator=gen, device=dev) * 3).to(tdt)
    sc = torch.randn((B, K, S), generator=gen, device=dev) * 2
    gl = torch.randn((R, 2), generator=gen, device=dev)
    mask = torch.ones((B, S), dtype=torch.uint8, device=dev)
    src = torch.randint(3, V, (B, S), generator=gen, device=dev, dtype=torch.int32)
    seq = torch.randint(3, V, (2, R, T), generator=gen, device=dev, dtype=torch.int32)
    raw, tlp = seq.clone(), torch.zeros((2, R, T), device=dev)
    length = torch.full((2, R), pos + 1, dtype=torch.int32, device=dev)
    lp, score = -torch.rand((2, R), generator=gen, device=dev), torch.zeros((2, R), device=dev)
    status = torch.zeros((2, R), dtype=torch.uint8, device=dev)
    parent = torch.empty(R, dtype=torch.int64, device=dev)
    nxt = torch.empty(R, dtype=torch.int32, device=dev)
    work = torch.empty(R * (K + 4), dtype=torch.int64, device=dev)
    cons = torch.zeros((B, 4, 4), dtype=torch.int32, device=dev)
    k = a.constraint_words
    cons[:, :k, 0] = src[:, :k]                                      # one-word phrases the copies can spell
    pre = torch.zeros((B, T), dtype=torch.int32, device=dev)
    pre_len = torch.zeros(B, dtype=torch.int32, device=dev)
    P = ops._ptr
    args = [P(logits), ldl, P(sc), P(gl), P(mask), P(src), 0.0, 2, 0, P(work), P(seq), P(raw), P(tlp), P(length),
            P(lp), P(score), P(status), P(parent), P(nxt), T, pos, B, K, V, S,
            FIRA_BF16 if a.precision == "bf16" else FIRA_F32]
    tail = [P(pre), T, P(pre_len), 0, 0]
    times = {}
    for name, extra in (("fira_pointer_mix_beam_step_rules", []), ("fira_pointer_mix_beam_step_lexical", [P(cons)]),
                        ("fira_pointer_mix_beam_step_rules", []), ("fira_pointer_mix_beam_step_lexical", [P(cons)])):
        # the stream is read per launch: time_launches captures on its own stream
        _, med_ms, launches = bench.time_launches(lambda i: call(name, *args, ops._stream(), *tail, *extra), 1, reps=20)
        times.setdefault(name, []).append(med_ms)                    # alternated: two measurements each
    for name, t in times.items():
        print(json.dumps({"metric": name + " time", "unit": "us", "value": min(t) * 1e3, "runs_us": [x * 1e3 for x in t],
                          "batch": B, "beam": K, "pos": pos, "V": V, "S": S, "constraint_words": k,
                          "precision": a.precision, "card": card, "power_limit_w": watts,
                          "note": "median device time per call (row + select launches), calls replayed from one CUDA "
                                  "graph between CUDA events, the two kernels alternated"}), flush=True)


def self_bleu(h, B, K):
    """mean pairwise id-level sentence BLEU among each commit's K hypotheses `h` (one fira_mbr_select launch with
    pair_bleu; the diagonal is left out)"""
    import torch
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import call
    T = h.seq.shape[2]
    seq, length = h.seq.to(torch.int32).contiguous(), h.length.to(torch.int32).contiguous()
    pair = torch.empty((B, K, K), dtype=torch.float64, device=seq.device)
    utility = torch.empty((B, K), dtype=torch.float64, device=seq.device)
    best = torch.empty(B, dtype=torch.int32, device=seq.device)
    call("fira_mbr_select", ops._ptr(seq), ops._ptr(length), T, 1, 2, 0, ops._ptr(pair), ops._ptr(utility),
         ops._ptr(best), B, K, T, ops._stream())
    off = ~torch.eye(K, dtype=torch.bool, device=seq.device)
    return pair[:, off].mean().item()


def repeat_share(seq, length, n):
    """the share of hypotheses seq [B, K, T] (length [B, K], <start> counted) in which some word after <start>
    completes an n-gram that already occurred in it (counted on the host)"""
    seq, length = seq.cpu().tolist(), length.cpu().tolist()
    hits = total = 0
    for rows, lens in zip(seq, length):
        for s, ln in zip(rows, lens):
            grams = [tuple(s[t - n + 1:t + 1]) for t in range(n, ln)]
            hits += len(set(grams)) < len(grams)
            total += 1
    return hits / max(1, total)


def power_limit():
    """the card's power limit in W as nvidia-smi reports it (None when nvidia-smi is unavailable)"""
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def mbr_select_timing(s, B, N):
    """fira_mbr_select alone on the samples `s` of one batch, against the host restatement of the same selection."""
    import torch
    import bench
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import call
    from mbr_rule import select
    T = s.seq.shape[2]
    seq, length = s.seq.to(torch.int32), s.length.to(torch.int32)
    utility = torch.empty((B, N), dtype=torch.float64, device=seq.device)
    best = torch.empty(B, dtype=torch.int32, device=seq.device)

    def launch(_):
        call("fira_mbr_select", ops._ptr(seq), ops._ptr(length), T, 1, 2, 0, None, ops._ptr(utility), ops._ptr(best),
             B, N, T, ops._stream())
    _, med_ms, launches = bench.time_launches(launch, 1, reps=20)
    host_seq, host_len = s.seq.cpu().tolist(), s.length.cpu().tolist()
    t0 = time.perf_counter()
    host = [select(host_seq[c], host_len[c], 1, 2, 0) for c in range(B)]
    host_s = time.perf_counter() - t0
    diff = max(abs(u - h) for c in range(B) for u, h in zip(utility[c].tolist(), host[c][1]))
    return {"metric": "fira_mbr_select time", "unit": "us", "value": med_ms * 1e3, "batch": B, "samples": N,
            "timed_launches": launches, "host_sentence_bleu_method2_us": host_s * 1e6,
            "host_pair_evaluations": B * N * N, "max_abs_utility_diff_vs_host": diff,
            "same_choice_as_host": all(int(best[c]) == host[c][2] for c in range(B)),
            "note": "median device time per launch, launches replayed from one CUDA graph between CUDA events; host = "
                    "the float64 restatement (tests/mbr_rule.py) over the same batch, one pass, one host thread"}


if __name__ == "__main__":
    main()
