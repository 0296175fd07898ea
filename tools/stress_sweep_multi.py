#!/usr/bin/env python
"""BASELINE.json config 5 on N GPUs: "synthetic stress: 2048-node graphs, 16k edges/relation, batch 256, 8xH100
roofline sweep".  Graphs shard by rank (no data-path collective: message passing never crosses a graph); every rank
times the GNN scatter (fira_gcn_aggregate, fp32 and bf16) and the fused GCN layer (fira_gcn_layer_fwd, bf16) on ITS
shard for per-GPU batches 32 ... 256, cold L2 (rotating buffers), CUDA events; the time of a configuration is the MAX
over ranks, the aggregate is N x per-GPU work / that time.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29511 \
        tools/stress_sweep_multi.py            # (also runs as a plain single-GPU script)
"""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    from fira_icse_b200 import _lib
    from fira_icse_b200.graph import PackedEdges
    from fira_icse_b200.synth import synth_stress_graphs
    peak = 3350.0                        # H100 SXM data-sheet HBM3 bandwidth unless MEASURED_PEAKS.json says otherwise
    pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(pk):
        peak = float(json.load(open(pk))["hbm_gbs"])
    N = 2048
    st = torch.cuda.current_stream()

    def timed(launch, iters=12):
        for i in range(3):
            launch(i)
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        for i in range(iters):
            ev[i][0].record(st); launch(i); ev[i][1].record(st)
        torch.cuda.synchronize()
        ms = sum(a.elapsed_time(b) for a, b in ev) / iters
        t = torch.tensor([ms], device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return t.item()

    for B in (32, 64, 128, 256):
        graphs = synth_stress_graphs(rank * 1000 + 0, B)
        pe = PackedEdges.from_coo_lists(graphs, N, dev)
        R = B * N
        er = pe.rows_csr(N, 0, 0)
        for code, tdt, esz in ((0, torch.float32, 4), (1, torch.bfloat16, 2)):
            n_pairs = max(3, int(400e6 // (2 * R * 256 * esz)) + 1)
            xs = [torch.randn(R, 256, device=dev).to(tdt) for _ in range(n_pairs)]
            ys = [torch.empty(R, 256, device=dev, dtype=tdt) for _ in range(n_pairs)]

            def scatter(i):
                _lib.call("fira_gcn_aggregate", pe.rowptr.data_ptr(), pe.col.data_ptr(), pe.val.data_ptr(),
                          xs[i % n_pairs].data_ptr(), None, ys[i % n_pairs].data_ptr(), B, N, 0, 0, 256, code, st.cuda_stream)
            ms = timed(scatter)
            alg = 2 * R * 256 * esz + (R + 1) * 4 + pe.nnz * 8
            if rank == 0:
                print(json.dumps({"config": "stress N=2048, 4 x 16,384 edges/relation", "kernel": "fira_gcn_aggregate",
                                  "dtype": "f32" if code == 0 else "bf16", "n_gpus": world, "per_gpu_batch": B,
                                  "rows_per_gpu": R, "nnz_per_gpu": pe.nnz, "ms_max_over_ranks": round(ms, 4),
                                  "graph_layers_per_s_all_gpus": round(world * B / (ms * 1e-3), 1),
                                  "algorithmic_GBps_per_gpu": round(alg / ms / 1e6, 1),
                                  "frac_of_measured_hbm_peak": round(alg / ms / 1e6 / peak, 4)}), flush=True)
            if code == 1:
                W = (torch.randn(256, 256, device=dev) / 16).to(torch.bfloat16)
                b2, c1 = torch.zeros(256, device=dev), torch.zeros(256, device=dev)
                gamma, beta = torch.ones(256, device=dev), torch.zeros(256, device=dev)
                zs = [torch.empty(R, 256, device=dev, dtype=tdt) for _ in range(n_pairs)]
                stats = torch.empty(2, R, device=dev)

                def fused(i):
                    _lib.call("fira_gcn_layer_fwd", er[0].data_ptr(), er[1].data_ptr(), er[2].data_ptr(),
                              xs[i % n_pairs].data_ptr(), W.data_ptr(), b2.data_ptr(), c1.data_ptr(), gamma.data_ptr(),
                              beta.data_ptr(), zs[i % n_pairs].data_ptr(), ys[i % n_pairs].data_ptr(),
                              ys[i % n_pairs].data_ptr(), 0, stats.data_ptr(), stats.data_ptr() + 4 * R, R, 256, 0.2, 7,
                              None, 1, st.cuda_stream)
                ms = timed(fused)
                alg = 3 * R * 256 * 2 + (R + 1) * 4 + pe.nnz * 8 + 256 * 256 * 2
                if rank == 0:
                    print(json.dumps({"config": "stress N=2048, 4 x 16,384 edges/relation",
                                      "kernel": "fira_gcn_layer_fwd (gather -> wgmma -> LayerNorm, one launch)",
                                      "dtype": "bf16", "n_gpus": world, "per_gpu_batch": B, "rows_per_gpu": R,
                                      "ms_max_over_ranks": round(ms, 4),
                                      "graph_layers_per_s_all_gpus": round(world * B / (ms * 1e-3), 1),
                                      "algorithmic_GBps_per_gpu": round(alg / ms / 1e6, 1),
                                      "frac_of_measured_hbm_peak": round(alg / ms / 1e6 / peak, 4)}), flush=True)
            del xs, ys
        del pe
        torch.cuda.empty_cache()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
