#!/usr/bin/env python
"""Micro-benchmark of the GNN scatter kernel (fira_gcn_aggregate) alone, cold L2 (rotating buffers).
Prints one JSON line per workload: DataSet-like graphs (B=64/256) and the config-5 stress graphs."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fira_icse_b200 import _lib  # noqa: E402
from fira_icse_b200.graph import PackedEdges  # noqa: E402
from fira_icse_b200.synth import synth_batch, synth_stress_graphs  # noqa: E402


def run(name, coo, N, segs, dtype_code=0):
    dev = torch.device("cuda:0")
    B = len(coo)
    pe = PackedEdges.from_coo_lists(coo, N, dev)
    R = B * N
    tdt = torch.float32 if dtype_code == 0 else torch.bfloat16
    esz = 4 if dtype_code == 0 else 2
    n_pairs = max(3, int(400e6 // (2 * R * 256 * esz)) + 1)
    xs = [torch.randn(R, 256, device=dev).to(tdt) for _ in range(n_pairs)]
    ys = [torch.empty(R, 256, device=dev, dtype=tdt) for _ in range(n_pairs)]
    st = torch.cuda.current_stream()

    def launch(i):
        _lib.call("fira_gcn_aggregate", pe.rowptr.data_ptr(), pe.col.data_ptr(), pe.val.data_ptr(),
                  xs[i % n_pairs].data_ptr(), None, ys[i % n_pairs].data_ptr(), B, *segs, 256, dtype_code, st.cuda_stream)
    for i in range(5):
        launch(i)
    iters = 30
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    torch.cuda.synchronize()
    for i in range(iters):
        ev[i][0].record(st); launch(i); ev[i][1].record(st)
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in ev)
    avg = sum(ms) / len(ms)
    # size-matched plain copy (same rotation): what a pure stream of these bytes achieves on this box
    for i in range(iters):
        ev[i][0].record(st); ys[i % n_pairs].copy_(xs[i % n_pairs]); ev[i][1].record(st)
    torch.cuda.synchronize()
    copy_ms = sorted(a.elapsed_time(b) for a, b in ev)
    copy_avg = sum(copy_ms) / len(copy_ms)
    alg = 2 * R * 256 * esz + (R + 1) * 4 + pe.nnz * 8
    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(
        os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0     # H100 SXM data-sheet HBM3 bandwidth
    print(json.dumps({"workload": name, "dtype": "f32" if dtype_code == 0 else "bf16", "rows": R, "nnz": pe.nnz,
                      "avg_us": round(avg * 1e3, 2), "min_us": round(ms[0] * 1e3, 2),
                      "alg_MB": round(alg / 1e6, 2), "GBps": round(alg / avg / 1e6, 1),
                      "frac_of_measured_peak": round(alg / avg / 1e6 / peak, 3),
                      "same_size_copy_us": round(copy_avg * 1e3, 2),
                      "same_size_copy_GBps": round(2 * R * 256 * esz / copy_avg / 1e6, 1)}), flush=True)


if __name__ == "__main__":
    if "--stress-sweep" in sys.argv:           # BASELINE.json config 5: per-GPU batch sweep 32 ... 256 graphs of 2048 nodes
        for B in (32, 64, 128, 256):
            g = synth_stress_graphs(0, B)
            run(f"stress N=2048 16k edges/relation B={B}", g, 2048, (2048, 0, 0), 0)
            run(f"stress N=2048 16k edges/relation B={B}", g, 2048, (2048, 0, 0), 1)
        sys.exit(0)
    for B in ((64,) if "--b64-only" in sys.argv else (64, 256)):
        _, coo = synth_batch(0, B)
        run(f"dataset-like B={B}", coo, 650, (210, 160, 280), 0)
        run(f"dataset-like B={B}", coo, 650, (210, 160, 280), 1)
    if "--b64-only" in sys.argv:
        sys.exit(0)
    g = synth_stress_graphs(0, 32)
    run("stress N=2048 16k edges/relation B=32", g, 2048, (2048, 0, 0), 0)
    run("stress N=2048 16k edges/relation B=32", g, 2048, (2048, 0, 0), 1)
