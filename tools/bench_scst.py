#!/usr/bin/env python
"""Self-critical fine-tuning (fira_icse_b200.scst) on one GPU: time per step split into its four parts, and the mean
reward of a model first trained with the MLE loss.

    python tools/bench_scst.py [--batch 32] [--samples 4 8] [--steps 10] [--warmup 3] [--mle-steps 300]
                               [--reward-steps 50] [--json out.json]

Timing: synthetic commits (fira_icse_b200.synth), B = --batch, each N of --samples, fp32 and bf16; per step, CUDA events
around sampling (eval mode, sample()), the rewards (fira_bleu_reward) and the training step (optim.eager_step:
policy_loss forward + backward in training mode with dropout, then FlatAdam); the median over --steps after --warmup.
The cross-attention K/V projection of the memory runs on the N replicas (scst.py): its forward product is timed on B and
on B*N memory rows.
Reward: the seeded model trained for --mle-steps Adam steps (lr 1e-4, bf16, batches of 16 golden commits), then
--reward-steps SCST steps (N = 4, lr 1e-5) on the same commits; the mean reward over those steps.
One JSON object on stdout, with the card name and power limit read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

VOCAB, AST_VOCAB = 24650, 71
D = 256


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return {"name": name, "power_limit_and_max_sm_clock": q}


def synthetic_batch(B, dev):
    from fira_icse_b200.graph import PackedEdges
    from fira_icse_b200.synth import N_NODES, synth_batch
    ids, coo = synth_batch(0, B, VOCAB, AST_VOCAB)
    t = {k: torch.from_numpy(v).to(dev) for k, v in ids.items()}
    edge = PackedEdges.from_coo_lists(coo, N_NODES, dev)
    return [t["sou"], t["tar"], torch.zeros(B, 1, dtype=torch.int64, device=dev), t["mark"], t["ast_change"], edge,
            t["tar_label"], t["sub_token"]]


def new_model(precision, dev, lr):
    from fira_icse_b200 import TransModel, optim
    from fira_testlib import reference_args
    torch.manual_seed(0)
    m = TransModel(reference_args()).to(dev).set_precision(precision)
    opt = optim.FlatAdam(m.live_parameters(), lr=lr, groups=m.flat_groups())
    optim.attach(m, [opt])
    return m, opt


def mle_loss(m, batch):
    """the training loss of model(..., 'train') per token, as optim.eager_step takes it"""
    ls, nt = m(*batch, "train")
    return (ls / nt,)


def timed_step(m, opt, batch, N, ids, seed):
    """one scst_step, its three parts between CUDA events -> milliseconds per part"""
    from fira_icse_b200 import optim, scst
    from fira_icse_b200.sample import sample
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    sou, tar, _, mark, ast_change, edge, _, sub_token = batch
    ev[0].record()
    m.eval()
    s = sample(m, sou, mark, ast_change, edge, sub_token, num_samples=N, seed=seed, tar_len=30, **ids)
    ev[1].record()
    reward, adv = scst.rewards(s.seq, s.length, tar, **ids)
    B = reward.shape[0]
    w = (adv / (B * N)).float().reshape(-1)
    ev[2].record()
    optim.eager_step(m, opt, lambda: scst.policy_loss(m, batch, s.seq, s.raw, w, ids["pad_id"]))
    ev[3].record()
    torch.cuda.synchronize()
    return [ev[i].elapsed_time(ev[i + 1]) for i in range(3)]


def kv_projection_ms(m, memory, N, reps=20):
    """forward of the six layers' cross-attention K/V projection on memory [B, S, D] and on its N replicas"""
    from fira_icse_b200 import ops
    pr = ops.Prec(m.precision == "bf16")
    W = torch.cat([t for c in m.decoder.cross_attention_list for t in (c.fc_k.weight, c.fc_v.weight)], 0).detach()
    b = torch.cat([t for c in m.decoder.cross_attention_list for t in (c.fc_k.bias, c.fc_v.bias)], 0).detach()
    out = {}
    for name, x in (("once", memory), ("replicated", memory.repeat_interleave(N, 0))):
        x2 = x.reshape(-1, D).to(pr.tdt).contiguous()
        pr.linear(x2, W, b)
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            pr.linear(x2, W, b)
        e.record()
        torch.cuda.synchronize()
        out[name] = a.elapsed_time(e) / reps
    return out


def timing(args, dev):
    from fira_icse_b200.synth import EOS, START
    ids = dict(start_id=START, eos_id=EOS, pad_id=0)
    batch = synthetic_batch(args.batch, dev)
    rows = []
    for precision in ("fp32", "bf16"):
        for N in args.samples:
            m, opt = new_model(precision, dev, 1e-5)
            parts = []
            for i in range(args.warmup + args.steps):
                t = timed_step(m, opt, batch, N, ids, seed=i)
                if i >= args.warmup:
                    parts.append(t)
            med = [statistics.median(p[k] for p in parts) for k in range(3)]
            with torch.no_grad():
                m.eval()
                memory = m.teacher_forced(*(batch[i] for i in (0, 1, 3, 4, 5, 7)))[1]
            rows.append({"precision": precision, "B": args.batch, "N": N,
                         "ms": dict(zip(("sampling", "reward", "train_step"), med)),
                         "ms_step": sum(med), "kv_projection_fwd_ms": kv_projection_ms(m, memory, N)})
            print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
            del m, opt
            torch.cuda.empty_cache()
    return rows


def reward_after_mle(args, dev):
    from fira_icse_b200 import optim, scst
    from fira_testlib import golden_batch, load_raw_golden
    v = load_raw_golden()["word_vocab"]
    ids = dict(start_id=v["<start>"], eos_id=v["<eos>"], pad_id=v["<pad>"])
    batches = [[t.to(dev) for t in golden_batch(lo, lo + 16)] for lo in range(0, 128, 16)]
    m, opt = new_model("bf16", dev, 1e-4)
    for i in range(args.mle_steps):
        optim.eager_step(m, opt, lambda: mle_loss(m, batches[i % len(batches)]))
    ft = optim.FlatAdam(m.live_parameters(), lr=1e-5, groups=m.flat_groups())
    optim.attach(m, [ft])
    steps = []
    for i in range(args.reward_steps):
        b = batches[i % len(batches)]
        steps.append(scst.scst_step(m, ft, b, num_samples=4, seed=i, first_index=16 * (i % len(batches)), **ids))
    r = [s.reward for s in steps]
    return {"mle_steps": args.mle_steps, "scst_steps": args.reward_steps, "N": 4, "B": 16,
            "mean_reward": sum(r) / len(r), "mean_reward_first10": sum(r[:10]) / len(r[:10]),
            "mean_reward_last10": sum(r[-10:]) / len(r[-10:]),
            "mean_abs_advantage": sum(s.advantage for s in steps) / len(steps)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--samples", type=int, nargs="+", default=[4, 8])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mle-steps", type=int, default=300)
    ap.add_argument("--reward-steps", type=int, default=50)
    ap.add_argument("--json", default=None, help="also write the result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_scst.py needs a CUDA device")
    dev = torch.device("cuda:0")
    out = {"card": card(), "timing": timing(args, dev), "reward": reward_after_mle(args, dev)}
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
