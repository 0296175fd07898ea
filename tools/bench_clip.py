#!/usr/bin/env python
"""What global-norm gradient clipping (optim.FlatAdam(..., max_grad_norm=c)) costs on one GPU.

    python tools/bench_clip.py [--launches 200] [--steps 50] [--windows 3] [--json out.json]

(a) The norm on the flat layout of the bench model (one buffer over every live parameter): fira_grad_sumsq alone, and
    fira_grad_sumsq + fira_grad_clip_finalize as a step runs them, median microseconds (a CUDA event pair around each
    pair of launches) and the achieved GB/s from 4 B read per element.  Share of the 3,350 GB/s data-sheet peak.
(b) fira_adam_flat_clip against fira_adam_flat on the same layout, without and with the EMA, launches alternated:
    median microseconds and GB/s from 30 B per parameter (38 B with the EMA).
(c) The graphed bf16 packed training step at batch 64 as bench.py builds it (synthetic commits, GraphedTrainStep,
    FlatAdam lr 1e-4) with clipping off and on (c = 1, which clips every step here), in the default overlap mode and
    with FIRA_OPT_OVERLAP=0: four engines in one process.  --windows timed windows of --steps replays each, the four
    alternated; commits/s per window, the median and the spread (max - min) / median of each.
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
CLIP = 1.0


def _timed(fns, launches):
    """median µs per call of each fn in `fns` (dict name -> fn), calls alternated"""
    for _ in range(10):
        for fn in fns.values():
            fn()
    torch.cuda.synchronize()
    ev = {k: [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(launches)]
          for k in fns}
    for i in range(launches):
        for k, fn in fns.items():
            ev[k][i][0].record()
            fn()
            ev[k][i][1].record()
    torch.cuda.synchronize()
    return {k: statistics.median(a.elapsed_time(b) for a, b in ev[k]) * 1e3 for k in fns}


def kernel_times(dev, launches):
    """(a) and (b)"""
    import bench
    from fira_icse_b200 import TransModel, _lib
    from fira_icse_b200.optim import FlatAdam
    torch.manual_seed(0)
    m = TransModel(bench.model_args()).to(dev)
    opt = FlatAdam(m.live_parameters(), lr=1e-4, groups=m.flat_groups(), ema_decay=DECAY, max_grad_norm=CLIP)
    grp = opt.clip
    n_live = sum(p.numel() for p in opt.params)
    opt.g.normal_()
    opt.step_t.fill_(10.0)
    stream = torch.cuda.current_stream().cuda_stream
    taken = torch.tensor([0.0, 0.5, 1.0, 0.0, 0.0], dtype=torch.float64, device=dev)     # a taken step, coef 0.5

    def sumsq():
        _lib.call("fira_grad_sumsq", opt.g.data_ptr(), opt.n, grp.partials.data_ptr(), stream)

    def norm():
        sumsq()
        _lib.call("fira_grad_clip_finalize", grp.partials.data_ptr(), grp.partials.numel(), None, CLIP,
                  grp.state.data_ptr(), grp.steps.data_ptr(), 0, stream)

    def adam(clip, ema):
        args = [opt.p.data_ptr(), opt.g.data_ptr(), opt.m.data_ptr(), opt.v.data_ptr(), opt.p16.data_ptr(), opt.n,
                opt.lr, opt.betas[0], opt.betas[1], opt.eps, opt.step_t.data_ptr(), None,
                opt.ema.data_ptr() if ema else None, DECAY if ema else 0.0]
        if clip:
            _lib.call("fira_adam_flat_clip", *args, taken.data_ptr(), stream)
        else:
            _lib.call("fira_adam_flat", *args, stream)

    us = _timed({"sumsq": sumsq, "sumsq_finalize": norm}, launches)
    out = {"n_live": n_live, "n_layout": opt.n, "partials": grp.partials.numel(), "launches": launches}
    for k in ("sumsq", "sumsq_finalize"):
        gbs = 4 * opt.n / (us[k] * 1e-6) / 1e9
        out[k] = {"us_median": us[k], "bytes": 4 * opt.n, "GB_s": gbs, "share_of_peak": gbs / PEAK_GBS}
    fns = {f"{'clip' if c else 'flat'}_{'ema' if e else 'plain'}": (lambda c=c, e=e: adam(c, e))
           for e in (False, True) for c in (False, True)}
    us = _timed(fns, launches)
    for k, v in us.items():
        bpp = 38 if k.endswith("ema") else 30
        gbs = bpp * opt.n / (v * 1e-6) / 1e9
        out[k] = {"us_median": v, "bytes": bpp * opt.n, "GB_s": gbs, "share_of_peak": gbs / PEAK_GBS}
    del m, opt, grp
    torch.cuda.empty_cache()
    return out


def step_rates(dev, steps, windows, warmup=5):
    """(c): commits/s of the graphed bf16 packed step at batch 64, clipping off / on, overlap / FIRA_OPT_OVERLAP=0"""
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
    saved = os.environ.get("FIRA_OPT_OVERLAP")
    try:
        for mode in ("overlap", "single_opt"):
            os.environ["FIRA_OPT_OVERLAP"] = "1" if mode == "overlap" else "0"       # read by GraphedTrainStep()
            for clip in ("off", "on"):
                torch.manual_seed(0)
                m = TransModel(bench.model_args()).to(dev)
                m.train()
                m.set_precision("bf16")
                c = CLIP if clip == "on" else None
                eng = GraphedTrainStep(m, B, lambda ps, m=m, c=c: FlatAdam(ps, lr=1e-4, groups=m.flat_groups(),
                                                                           max_grad_norm=c), edge_capacity=cap)
                eng.load(pool[0])
                eng.capture()
                for pb in pool[1:]:
                    eng.step(pb)
                for i in range(warmup):
                    eng.step(pool[i % len(pool)])
                assert (eng.clip is not None) == (clip == "on") and eng.opt_overlap == (mode == "overlap")
                engines[f"{mode}_{clip}"] = eng
    finally:
        if saved is None:
            os.environ.pop("FIRA_OPT_OVERLAP", None)
        else:
            os.environ["FIRA_OPT_OVERLAP"] = saved
    rates = {k: [] for k in engines}
    for _ in range(windows):
        for name, eng in engines.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(steps):
                eng.step(pool[i % len(pool)])
            e1.record()
            torch.cuda.synchronize()
            rates[name].append(B * steps / (e0.elapsed_time(e1) * 1e-3))
    out = {"B": B, "steps_per_window": steps, "windows": windows, "max_grad_norm": CLIP}
    for name, r in rates.items():
        med = statistics.median(r)
        out[name] = {"commits_s": r, "median": med, "spread": (max(r) - min(r)) / med,
                     "ms_per_step": B / med * 1e3}
    for mode in ("overlap", "single_opt"):
        out[f"{mode}_on_over_off"] = out[f"{mode}_on"]["median"] / out[f"{mode}_off"]["median"]
    out["clipped_steps"] = {k: int(e.clipped.item()) for k, e in engines.items() if e.clip is not None}
    out["skipped_steps"] = {k: int(e.skipped.item()) for k, e in engines.items() if e.clip is not None}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_clip.py needs a CUDA device")
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
