#!/usr/bin/env python
"""What the exponential moving average of the weights (optim.FlatAdam(..., ema_decay=d)) costs on one GPU.

    python tools/bench_ema.py [--launches 200] [--steps 50] [--windows 3] [--json out.json]

(a) fira_adam_flat alone on the flat layout of the bench model (27,802,189 live parameters, n = the padded layout
    length), with and without `ema`, launches alternated: the median microseconds per launch (a CUDA event pair around
    each launch) and the achieved GB/s from 30 B per parameter (reads p, g, m, v; writes p, m, v and the bf16 mirror)
    and 38 B with the EMA (also reads and writes e).  Share of the 3,350 GB/s data-sheet peak.
(b) The graphed bf16 packed training step at batch 64 as bench.py builds it (synthetic commits, GraphedTrainStep,
    FlatAdam lr 1e-4 in the default single-GPU mode), once with the EMA off and once with d = 0.999, two engines in
    one process.  --windows timed windows of --steps replays each, alternating off / on; commits/s per window, the
    median and the spread (max - min) / median of each.
One JSON object on stdout, with the card name and power limit read in the same run."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench_scst import card  # noqa: E402

PEAK_GBS = 3350.0
DECAY = 0.999


def kernel_times(dev, launches):
    """(a): µs per fira_adam_flat launch without / with the EMA buffer, alternated"""
    import bench
    from fira_icse_b200 import TransModel, _lib
    from fira_icse_b200.optim import FlatAdam
    torch.manual_seed(0)
    m = TransModel(bench.model_args()).to(dev)
    opt = FlatAdam(m.live_parameters(), lr=1e-4, groups=m.flat_groups(), ema_decay=DECAY)
    n_live = sum(p.numel() for p in opt.params)
    opt.g.normal_()
    opt.step_t.fill_(10.0)
    stream = torch.cuda.current_stream().cuda_stream

    def launch(ema):
        _lib.call("fira_adam_flat", opt.p.data_ptr(), opt.g.data_ptr(), opt.m.data_ptr(), opt.v.data_ptr(),
                  opt.p16.data_ptr(), opt.n, opt.lr, opt.betas[0], opt.betas[1], opt.eps, opt.step_t.data_ptr(), None,
                  opt.ema.data_ptr() if ema else None, DECAY if ema else 0.0, stream)
    for _ in range(10):
        launch(False)
        launch(True)
    torch.cuda.synchronize()
    ev = {k: [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(launches)]
          for k in (False, True)}
    for i in range(launches):
        for k in (False, True):
            ev[k][i][0].record()
            launch(k)
            ev[k][i][1].record()
    torch.cuda.synchronize()
    out = {"n_live": n_live, "n_layout": opt.n, "launches": launches}
    for k, name, bpp in ((False, "without_ema", 30), (True, "with_ema", 38)):
        us = statistics.median(a.elapsed_time(b) for a, b in ev[k]) * 1e3
        gbs = bpp * opt.n / (us * 1e-6) / 1e9
        out[name] = {"us_median": us, "bytes": bpp * opt.n, "GB_s": gbs, "share_of_peak": gbs / PEAK_GBS}
    out["extra_us"] = out["with_ema"]["us_median"] - out["without_ema"]["us_median"]
    del m, opt
    torch.cuda.empty_cache()
    return out


def step_rates(dev, steps, windows, warmup=5):
    """(b): commits/s of the graphed bf16 packed step at batch 64 without / with the EMA, windows alternated"""
    import numpy as np
    import bench
    from fira_icse_b200 import TransModel
    from fira_icse_b200.engine import GraphedTrainStep
    from fira_icse_b200.optim import FlatAdam
    from fira_icse_b200.packed import PackedTables, pack_from_dataset
    from fira_icse_b200.synth import SynthDataset
    B = bench.PER_GPU_BATCH
    ds = SynthDataset(0, bench.N_POOL * B, bench.VOCAB, bench.AST_VOCAB)
    tables = PackedTables(ds)
    host = [pack_from_dataset(tables, np.arange(i * B, (i + 1) * B), bench.VOCAB, pin=True) for i in range(bench.N_POOL)]
    pool = [pb.to(dev) for pb in host]
    cap = (max(pb.nnz for pb in host) + 4095) // 4096 * 4096 * 2
    engines = {}
    for name, decay in (("off", None), ("on", DECAY)):
        torch.manual_seed(0)
        m = TransModel(bench.model_args()).to(dev)
        m.train()
        m.set_precision("bf16")
        eng = GraphedTrainStep(m, B, lambda ps, m=m, decay=decay: FlatAdam(ps, lr=1e-4, groups=m.flat_groups(),
                                                                           ema_decay=decay), edge_capacity=cap)
        eng.load(pool[0])
        eng.capture()
        for pb in pool[1:]:
            eng.step(pb)
        for i in range(warmup):
            eng.step(pool[i % len(pool)])
        engines[name] = eng
    assert all(o.ema is not None for o in engines["on"].flat_optims)
    assert all(o.ema is None for o in engines["off"].flat_optims)
    rates = {"off": [], "on": []}
    for _ in range(windows):
        for name in ("off", "on"):
            eng = engines[name]
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(steps):
                eng.step(pool[i % len(pool)])
            e1.record()
            torch.cuda.synchronize()
            rates[name].append(B * steps / (e0.elapsed_time(e1) * 1e-3))
    out = {"B": B, "steps_per_window": steps, "windows": windows, "ema_decay": DECAY}
    for name in ("off", "on"):
        r = rates[name]
        med = statistics.median(r)
        out[name] = {"commits_s": r, "median": med, "spread": (max(r) - min(r)) / med}
    out["on_over_off"] = out["on"]["median"] / out["off"]["median"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ema.py needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    dev = torch.device("cuda:0")
    out = {"card": card(), "kernel": kernel_times(dev, args.launches)}
    print(json.dumps(out["kernel"]), file=sys.stderr, flush=True)
    out["step"] = step_rates(dev, args.steps, args.windows)
    out["peak_GB_s"] = PEAK_GBS
    line = json.dumps(out)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
