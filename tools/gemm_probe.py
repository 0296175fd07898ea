#!/usr/bin/env python
"""Where does a small wgmma GEMM launch spend its time?  fira_debug_set_probe makes CTA (0,0,0) of fira_gemm_bf16_tc
stamp %globaltimer at its phase boundaries; this tool replays a CUDA graph of 8 dependent launches (each reads the previous
output, like the decoder's chain) and prints the phase deltas of the LAST one, plus the per-launch time of the chain.

    python tools/gemm_probe.py            # one JSON line per (shape, PDL on/off)
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PHASES = ["prologue", "dep_wait", "tma_issue", "first_stage_landed(from dep)", "mma_issued(from landed)",
          "acc_visible(from mma_issued)", "epilogue_stores", "exit"]


def main():
    import __graft_entry__
    __graft_entry__.build()
    from fira_icse_b200 import _lib, ops
    dev = "cuda:0"
    L = _lib.lib()
    probe = torch.zeros(16, dtype=torch.int64, device=dev)
    shapes = [(1920, 256, 256), (1920, 768, 256), (1920, 1024, 256), (1920, 256, 1024), (3584, 512, 256), (11264, 256, 256)]
    for pdl in (0, 1):
        L.fira_set_pdl(pdl)
        for M, N, K in shapes:
            W = (torch.randn(N, K, device=dev) / 16).to(torch.bfloat16)
            W2 = (torch.randn(K, N, device=dev) / 16).to(torch.bfloat16)
            bias = torch.randn(N, device=dev)
            bias2 = torch.randn(K, device=dev)
            x = torch.randn(M, K, device=dev).to(torch.bfloat16)
            y = torch.empty(M, N, device=dev, dtype=torch.bfloat16)

            def chain():
                for _ in range(4):          # x -> y -> x ... : every launch depends on the previous one
                    ops.gemm_tc(x, K, 1, W, K, 1, y, N, M, N, K, bias=bias)
                    ops.gemm_tc(y, N, 1, W2, N, 1, x, K, M, K, N, bias=bias2)
            L.fira_debug_set_probe(probe.data_ptr())
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                chain()
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                chain()
            best = None
            times = []
            for _ in range(20):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                g.replay()
                e1.record()
                torch.cuda.synchronize()
                times.append(1e3 * e0.elapsed_time(e1) / 8)
                t = probe.cpu().tolist()
                d = {"prologue": t[1] - t[0], "dep_wait": t[2] - t[1], "tma_issue": t[3] - t[2],
                     "first_stage_landed(from dep)": t[4] - t[2], "mma_issued(from landed)": t[5] - t[4],
                     "acc_visible(from mma_issued)": t[6] - t[5], "epilogue_stores": t[7] - t[6], "exit": t[8] - t[7],
                     "total_cta0": t[8] - t[0]}
                if best is None or d["total_cta0"] < best["total_cta0"]:
                    best = d
            L.fira_debug_set_probe(None)
            times.sort()
            print(json.dumps({"shape": [M, N, K], "pdl": pdl, "chain_us_per_launch_median": round(times[len(times) // 2], 2),
                              "chain_us_per_launch_min": round(times[0], 2), "cta0_phase_ns": best}), flush=True)
    L.fira_set_pdl(0)


if __name__ == "__main__":
    main()
