#!/usr/bin/env python
"""Knowledge distillation (fira_icse_b200.distill) on one GPU: time per step split into its parts, next to the plain
eager MLE step, and the two loss kernels against the NLL kernels on the same rows.

    python tools/bench_distill.py [--batch 64] [--members 1 2 4] [--steps 10] [--warmup 3] [--topk 8 32]
                                  [--json out.json]

Step: synthetic commits (fira_icse_b200.synth), B = --batch, fp32 and bf16; the teacher is M copies of the seeded model,
each but the first with the seeded perturbation of tools/bench_beam.py --ensemble.  CUDA events around the teacher's
forward (all members), the combine (fira_pointer_mix_ensemble) and the student's step (optim.eager_step: forward +
backward in training mode with dropout, then FlatAdam); the median of each over --steps after --warmup.  The MLE step
is model(..., 'train'), backward and FlatAdam on the same batch, eager.
Kernels: microseconds per launch of fira_pointer_mix_kd_fwd / _bwd and fira_pointer_mix_nll_fwd_rows / _bwd_rows on the
same rows (the batch's shifted labels), replayed from a CUDA graph over buffer sets larger than L2
(bench.time_launches).  Algorithmic bytes per loss row (y != 0): the kd forward reads the student row (V s + S 4) and
the teacher row (V 4 + S 4) twice; the kd backward reads each once and writes V s + S 4 + 8; the NLL forward reads the
one softmax the label lives in, the NLL backward reads it and writes both gradient rows; both backward kernels also
write zero gradient rows for the rows without a loss.  Share of the 3,350 GB/s data-sheet peak.
--topk K...: offline distillation with stored top-K targets (distill.KDTargets), per precision and K: the step with
SparseTargets (student forward + backward, FlatAdam; no teacher), fira_pointer_mix_topk per launch on the M = 1 teacher's
triple, the sparse kernels next to the dense kd and NLL kernels on the same rows (the sparse forward reads the student
row once and the targets, 8 K bytes per row; the backward reads it once and writes the gradient rows), the targets'
production rate (teacher forward + combine + top-K, commits/s), stored bytes per commit and the mean kept teacher mass.
One JSON object on stdout, with the card name and power limit read in the same run."""
import argparse
import copy
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench_scst import card, mle_loss, new_model, synthetic_batch  # noqa: E402

PEAK_GBS = 3350.0
L2_BYTES = 50 * 2 ** 20


def teacher(precision, dev, M):
    from fira_icse_b200.ensemble import Ensemble
    base, _ = new_model(precision, dev, 1e-4)
    pool = [base.eval()]
    for i in range(1, M):
        m = copy.deepcopy(base)
        g = torch.Generator(device=dev).manual_seed(i)
        with torch.no_grad():
            for p in (m.out_fc.weight, m.copy_net.LinearRes.weight, m.copy_net.LinearProb.weight):
                p.add_(torch.randn(p.shape, generator=g, device=dev) * p.std() * 0.1)
        pool.append(m.eval())
    return Ensemble(pool)


def timed_step(m, opt, batch, ens, alpha=0.5):
    """one distill_step, its parts between CUDA events -> milliseconds per part"""
    from fira_icse_b200 import distill, optim
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    label = m.shifted_label(batch[6])
    ev[0].record()
    models, log_w = distill.teacher_members(ens, m)
    triples, mm = distill.member_triples(models, batch, label)
    ev[1].record()
    targets = distill.combine(triples, log_w, mm, m.vocab_size)
    ev[2].record()
    tokens = (label != 0).sum()
    optim.eager_step(m, opt, lambda: (distill.distill_loss(m, batch, targets, label, alpha)[0] / tokens,))
    ev[3].record()
    torch.cuda.synchronize()
    return [ev[i].elapsed_time(ev[i + 1]) for i in range(3)], targets


def mle_step(m, opt, batch):
    from fira_icse_b200 import optim
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    optim.eager_step(m, opt, lambda: mle_loss(m, batch))
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1])


def kernel_times(m, batch, targets):
    """µs per launch of the kd and NLL kernels on this batch's rows, with the student's head products"""
    import bench
    from fira_icse_b200 import distill, ops
    from fira_icse_b200._lib import call
    label = m.shifted_label(batch[6])
    B, T = label.shape
    [(lg, sc, gl)], mm = distill.member_triples([m], batch, label)
    lab = label.to(torch.int32).contiguous().view(-1)
    S, V, R = mm.shape[1], m.vocab_size, B * T
    bf16 = m.precision == "bf16"
    pr = ops.Prec(bf16)
    tx, tsc, tgl = targets
    s = 2 if bf16 else 4
    ld = lg.shape[1]
    per_set = R * ld * (s + 4 + s) + R * S * 4 * 3
    n_rot = max(2, -(-2 * L2_BYTES // per_set))
    f32 = dict(dtype=torch.float32, device=lg.device)
    sets = []
    for _ in range(n_rot):
        sets.append(dict(lg=lg.clone(), tx=tx.clone(), dl=torch.empty_like(lg), dsc=torch.empty((B, T, S), **f32),
                         st=torch.empty((R, 16), **f32), st8=torch.empty((R, 8), **f32), o=torch.empty((R, 3), **f32)))
    u = torch.ones(1, **f32)
    p, code = ops._ptr, pr.code
    dgl, act = torch.empty((R, 2), **f32), torch.empty(R, dtype=torch.uint8, device=lg.device)

    def kd_fwd(i):
        z = sets[i % n_rot]
        call("fira_pointer_mix_kd_fwd", p(z["lg"]), ld, p(sc), p(gl), p(mm), p(lab), p(z["tx"]), ld, p(tsc), p(tgl), 0.5,
             p(z["st"]), p(z["o"]), p(z["o"], R), p(z["o"], 2 * R), R, T, V, S, code, ops._stream())

    def kd_bwd(i):
        z = sets[i % n_rot]
        call("fira_pointer_mix_kd_bwd", p(z["lg"]), ld, p(sc), p(mm), p(lab), p(z["tx"]), ld, p(tsc), 0.5, p(z["st"]),
             p(u), p(z["dl"]), p(z["dsc"]), p(dgl), p(act), R, T, V, S, code, ops._stream())

    def nll_fwd(i):
        z = sets[i % n_rot]
        call("fira_pointer_mix_nll_fwd_rows", p(z["lg"]), ld, p(sc), p(gl), p(mm), p(lab), None, p(z["st8"]), p(z["o"]),
             None, R, T, V, S, code, ops._stream())

    def nll_bwd(i):
        z = sets[i % n_rot]
        call("fira_pointer_mix_nll_bwd_rows", p(z["lg"]), ld, p(sc), p(mm), p(lab), None, None, 0, p(z["st8"]), p(u),
             p(z["dl"]), p(z["dsc"]), p(dgl), p(act), R, T, V, S, code, ops._stream())

    for i in range(n_rot):                 # the stats rows the backward launches read
        kd_fwd(i)
    out = {}
    y = lab.long()
    n_loss = int((y != 0).sum())
    n_vocab = int(((y != 0) & (y < V)).sum())
    n_copy = n_loss - n_vocab
    row_kd = V * s + S * 4 + V * 4 + S * 4
    zero = (R - n_loss) * (V * s + S * 4 + 8)           # the zeros both backward kernels write on the other rows
    bytes_ = {"kd_fwd": 2 * row_kd * n_loss,
              "kd_bwd": (row_kd + V * s + S * 4 + 8) * n_loss + zero,
              "nll_fwd": n_vocab * V * s + n_loss * S * 4,
              "nll_bwd": n_vocab * 2 * V * s + n_copy * (V * s + 2 * S * 4 + 8) + zero}
    for name, fn in (("kd_fwd", kd_fwd), ("nll_fwd", nll_fwd), ("kd_bwd", kd_bwd)):
        if name == "kd_bwd":
            for i in range(n_rot):
                kd_fwd(i)
        mean, med, n = bench.time_launches(fn, n_rot)
        out[name] = {"us": med * 1e3, "bytes": bytes_[name], "GB_s": bytes_[name] / (med * 1e-3) / 1e9}
    for i in range(n_rot):
        nll_fwd(i)
    mean, med, n = bench.time_launches(nll_bwd, n_rot)
    out["nll_bwd"] = {"us": med * 1e3, "bytes": bytes_["nll_bwd"], "GB_s": bytes_["nll_bwd"] / (med * 1e-3) / 1e9}
    for v in out.values():
        v["share_of_peak"] = v["GB_s"] / PEAK_GBS
    out["rows"] = {"all": R, "loss": n_loss, "vocabulary_label": n_vocab, "copy_label": n_copy}
    return out


def sparse_times(m, opt, batch, targets, k, steps, warmup):
    """offline distillation at top-k: step time, kernel µs per launch, rate and bytes of the stored targets"""
    import bench
    from fira_icse_b200 import distill, ops, optim
    from fira_icse_b200._lib import call
    label = m.shifted_label(batch[6])
    B, T = label.shape
    sou, _, _, _, _, _, _, sub_token = batch
    mm = torch.cat((sou != 0, sub_token != 0), 1).to(torch.uint8).contiguous()
    S, V, R = mm.shape[1], m.vocab_size, B * T
    lab = label.to(torch.int32).contiguous().view(-1)
    tl, tp, mass = distill.topk_targets(targets, mm, label, V, k)
    sparse = distill.SparseTargets(tl, tp)
    tokens = (label != 0).sum()
    times = []
    for i in range(warmup + steps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        optim.eager_step(m, opt, lambda: (distill.distill_loss(m, batch, sparse, label, 0.5)[0] / tokens,))
        ev[1].record()
        torch.cuda.synchronize()
        if i >= warmup:
            times.append(ev[0].elapsed_time(ev[1]))
    # the kernels on the student's head products of this batch
    [(lg, sc, gl)], _ = distill.member_triples([m], batch, label)
    bf16 = m.precision == "bf16"
    pr = ops.Prec(bf16)
    s = 2 if bf16 else 4
    ld = lg.shape[1]
    n_rot = max(2, -(-2 * L2_BYTES // (R * ld * 2 * s + R * S * 8)))
    f32 = dict(dtype=torch.float32, device=lg.device)
    sets = [dict(lg=lg.clone(), dl=torch.empty_like(lg), dsc=torch.empty((B, T, S), **f32),
                 st=torch.empty((R, 10), **f32), o=torch.empty((R, 3), **f32)) for _ in range(n_rot)]
    u = torch.ones(1, **f32)
    p, code = ops._ptr, pr.code
    dgl, act = torch.empty((R, 2), **f32), torch.empty(R, dtype=torch.uint8, device=lg.device)

    def fwd(i):
        z = sets[i % n_rot]
        call("fira_pointer_mix_kd_sparse_fwd", p(z["lg"]), ld, p(sc), p(gl), p(mm), p(lab), p(tl), p(tp), k, 0.5,
             p(z["st"]), p(z["o"]), p(z["o"], R), p(z["o"], 2 * R), R, T, V, S, code, ops._stream())

    def bwd(i):
        z = sets[i % n_rot]
        call("fira_pointer_mix_kd_sparse_bwd", p(z["lg"]), ld, p(sc), p(mm), p(lab), p(tl), p(tp), k, 0.5, p(z["st"]),
             p(u), p(z["dl"]), p(z["dsc"]), p(dgl), p(act), R, T, V, S, code, ops._stream())

    tx, tsc, tgl = targets
    outs = [(torch.empty((R, k), dtype=torch.int32, device=lg.device), torch.empty((R, k), **f32),
             torch.empty(R, **f32), tx.clone()) for _ in range(max(2, -(-2 * L2_BYTES // (R * ld * 4))))]

    def topk(i):
        a, b, c, x = outs[i % len(outs)]
        call("fira_pointer_mix_topk", p(x), ld, p(tsc), p(tgl), p(mm), p(lab), k, p(a), p(b), p(c), R, T, V, S,
             ops._stream())

    y = lab.long()
    n_loss = int((y != 0).sum())
    zero = (R - n_loss) * (V * s + S * 4 + 8)
    row = V * s + S * 4
    bytes_ = {"sparse_fwd": (row + 8 * k) * n_loss, "sparse_bwd": (2 * row + 8 + 8 * k) * n_loss + zero,
              "topk": (V * 4 + S * 4 + 8 * k) * n_loss}
    kern = {}
    for i in range(n_rot):
        fwd(i)
    for name, fn, n in (("sparse_fwd", fwd, n_rot), ("sparse_bwd", bwd, n_rot), ("topk", topk, len(outs))):
        _, med_ms, _ = bench.time_launches(fn, n)
        kern[name] = {"us": med_ms * 1e3, "bytes": bytes_[name], "GB_s": bytes_[name] / (med_ms * 1e-3) / 1e9,
                      "share_of_peak": bytes_[name] / (med_ms * 1e-3) / 1e9 / PEAK_GBS}
    live = y != 0
    per_commit = (n_loss * (2 + 4 + 8 * k + 4) + 8 * B) / B
    return {"ms_step": statistics.median(times), "kernels": kern, "bytes_per_commit": per_commit,
            "mean_kept_mass": float(mass[live].double().mean())}


def targets_rate(ens, batch, k, steps):
    """commits/s of teacher_targets + fira_pointer_mix_topk (what `run_model.py kd-targets` runs per batch)"""
    from fira_icse_b200 import distill
    m = ens.models[0]
    label = m.shifted_label(batch[6])
    mm = torch.cat((batch[0] != 0, batch[7] != 0), 1).to(torch.uint8).contiguous()
    times = []
    for i in range(steps + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        distill.topk_targets(distill.teacher_targets(ens, batch, label), mm, label, m.vocab_size, k)
        ev[1].record()
        torch.cuda.synchronize()
        if i:
            times.append(ev[0].elapsed_time(ev[1]))
    return batch[0].shape[0] / (statistics.median(times) * 1e-3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--members", type=int, nargs="+", default=[1, 2, 4])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--topk", type=int, nargs="*", default=[], help="stored top-k targets at these k")
    ap.add_argument("--json", default=None, help="also write the result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_distill.py needs a CUDA device")
    dev = torch.device("cuda:0")
    batch = synthetic_batch(args.batch, dev)
    rows = []
    for precision in ("fp32", "bf16"):
        m, opt = new_model(precision, dev, 1e-4)
        mle = [mle_step(m, opt, batch) for _ in range(args.warmup + args.steps)][args.warmup:]
        del m, opt
        for M in args.members:
            ens = teacher(precision, dev, M)
            m, opt = new_model(precision, dev, 1e-4)
            parts = []
            for i in range(args.warmup + args.steps):
                t, targets = timed_step(m, opt, batch, ens)
                if i >= args.warmup:
                    parts.append(t)
            med = [statistics.median(x[k] for x in parts) for k in range(3)]
            steps = [sum(x) for x in parts]
            row = {"precision": precision, "B": args.batch, "M": M,
                   "ms": dict(zip(("teacher_forward", "combine", "student_step"), med)),
                   "ms_step": statistics.median(steps), "ms_mle_step": statistics.median(mle)}
            if M == args.members[0]:
                row["kernels"] = kernel_times(m, batch, targets)
            if M == 1:
                row["topk"] = {}
                for k in args.topk:
                    r = sparse_times(m, opt, batch, targets, k, args.steps, args.warmup)
                    r["kd_targets_commits_s"] = targets_rate(ens, batch, k, args.steps)
                    row["topk"][k] = r
            rows.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
            del m, opt, ens, targets
            torch.cuda.empty_cache()
    out = {"card": card(), "timing": rows, "peak_GB_s": PEAK_GBS}
    line = json.dumps(out)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
