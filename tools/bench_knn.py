"""Nearest-neighbour decoding timings (fira_icse_b200/knn.py) on one GPU.

  * fira_knn_search: CUDA events over graph-replayed launches at N in {2^18, 2^20, 2^22}, R in {60, 384, 2048},
    k in {8, 64}, against both bounds -- one read of the datastore (N (512 + 8) B at 3.35 TB/s) and the distance
    product (2 R N 256 bf16 FLOP at 989 TFLOP/s); the larger is named and the kernel's share of it reported.
    Breakdown: the same search over a store of N identical keys, where every distance ties and a later index never
    beats the k-th key, so the only insertions are the k that fill each (split, row) list: that time is the product,
    the key stream, the fill and the merge; the rest of the random-key time is the insertions past the fill.
  * fira_pointer_mix_knn: time and algorithmic bytes per row (the model's triple read once, the fp32 triple written).
  * sample and nbest per batch (B = 128 commits, N = K = 3, bf16) with and without a datastore (N = 2^20, k = 8).
The card's name and power limit are read in the same run.  Prints a markdown table and one JSON line.

    python tools/bench_knn.py [--quick]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM = 3.35e12
BF16 = 989e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # noqa: BLE001 -- the table still names the device torch reports
        out = f"{torch.cuda.get_device_name()} (nvidia-smi: {e})"
    return out


def graph_time(fn, reps=50):
    """mean ms of one replay of a graph of `fn` (CUDA events over `reps` replays after warm-up)"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    for _ in range(3):
        g.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def bench_search(quick):
    from fira_icse_b200.knn import Datastore, search_into, workspace_bytes
    rows = []
    dev = "cuda:0"
    for N in ([2 ** 20] if quick else [2 ** 18, 2 ** 20, 2 ** 22]):
        keys = torch.randn((N, 256), device=dev).to(torch.bfloat16)
        st = Datastore(keys, keys.float().square().sum(1), torch.zeros(N, dtype=torch.int32, device=dev),
                       torch.zeros((N, 2), dtype=torch.int32, device=dev), vocab_size=1, precision="bf16",
                       fingerprint="bench")
        same = keys[:1].expand(N, 256).contiguous()
        flat = Datastore(same, same.float().square().sum(1), st.words, st.source, vocab_size=1, precision="bf16",
                         fingerprint="bench")
        for R in (60, 384, 2048):
            q = (keys[torch.randint(0, N, (R,), device=dev)].float() + 0.3 * torch.randn((R, 256), device=dev)).to(
                torch.bfloat16)
            for k in (8, 64):
                ws = torch.empty(workspace_bytes(R, k, dev), dtype=torch.uint8, device=dev)
                idx = torch.empty((R, k), dtype=torch.int32, device=dev)
                dist = torch.empty((R, k), dtype=torch.float32, device=dev)
                ms = graph_time(lambda: search_into(st, q, k, ws, idx, dist))
                ms_fill = graph_time(lambda: search_into(flat, q, k, ws, idx, dist))
                t_mem = N * (512 + 8) / HBM * 1e3
                t_flop = 2.0 * R * N * 256 / BF16 * 1e3
                bound, name = (t_mem, "HBM") if t_mem >= t_flop else (t_flop, "bf16")
                rows.append(dict(N=N, R=R, k=k, ms=ms, fill_only_ms=ms_fill, hbm_bound_ms=t_mem, flop_bound_ms=t_flop,
                                 bound=name, share=bound / ms, tflops=2.0 * R * N * 256 / ms / 1e9))
        del keys, st, same, flat
        torch.cuda.empty_cache()
    return rows


def bench_combine():
    from fira_icse_b200 import ops
    from fira_icse_b200._lib import FIRA_BF16, call
    dev = "cuda:0"
    B, N, V, S, k = 128, 3, 24650, 370, 8
    R, ld = B * N, ops._ld_logits(24650)
    logits = torch.randn((R, ld), device=dev).to(torch.bfloat16)
    sc = torch.randn((B, N, S), device=dev)
    gl = torch.randn((R, 2), device=dev)
    mask = torch.ones((B, S), dtype=torch.uint8, device=dev)
    idx = torch.randint(0, 1000, (R, k), dtype=torch.int32, device=dev)
    dist = torch.sort(torch.rand((R, k), device=dev), 1).values
    words = torch.randint(0, V, (1000,), dtype=torch.int32, device=dev)
    params = torch.tensor([0.25, 10.0], device=dev)
    out = torch.empty((R, ld), device=dev)
    sco, glo = torch.empty((B, N, S), device=dev), torch.empty((R, 2), device=dev)
    p = ops._ptr

    def run():
        call("fira_pointer_mix_knn", p(logits), ld, p(sc), p(gl), p(mask), p(idx), p(dist), p(words), k, p(params),
             p(out), ld, p(sco), p(glo), B, N, V, S, FIRA_BF16, ops._stream())
    ms = graph_time(run, reps=200)
    per_row = V * 2 + S * 4 + 8 + S + k * 12 + V * 4 + S * 4 + 8       # triple + mask + neighbours in, fp32 triple out
    return dict(B=B, N=N, ms=ms, bytes_per_row=per_row, hbm_share=R * per_row / HBM * 1e3 / ms)


def bench_decode(quick):
    from fira_testlib import golden_batch
    from test_gpu_sample import _model, _vocab
    from fira_icse_b200.beam import nbest
    from fira_icse_b200.knn import Datastore, KNNModel, fingerprint
    from fira_icse_b200.sample import sample
    dev = "cuda:0"
    m = _model("bf16")
    b = golden_batch(0, 128)
    v = _vocab()
    ids = dict(start_id=v["<start>"], eos_id=v["<eos>"], pad_id=v["<pad>"])
    Nst = 2 ** 20
    keys = (torch.randn((Nst, 256), device=dev) * 0.5).to(torch.bfloat16)
    st = Datastore(keys, keys.float().square().sum(1), torch.randint(3, m.vocab_size, (Nst,), dtype=torch.int32,
                   device=dev), torch.zeros((Nst, 2), dtype=torch.int32, device=dev), vocab_size=m.vocab_size,
                   precision="bf16", fingerprint=fingerprint(m))
    km = KNNModel(m, st, k=8)
    g = b[0], b[3], b[4], b[5].to(dev), b[7]
    out = {}
    for name, model in (("plain", m), ("knn", km)):
        for dec, fn in (("sample", lambda mm: sample(mm, *g, num_samples=3, seed=0, **ids)),
                        ("nbest", lambda mm: nbest(mm, *g, beam_size=3, **ids))):
            fn(model)
            fn(model)
            torch.cuda.synchronize()
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 2 if quick else 5
            a.record()
            for _ in range(reps):
                fn(model)
            e.record()
            torch.cuda.synchronize()
            out[f"{dec}_{name}_ms"] = a.elapsed_time(e) / reps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_knn.py needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    res = dict(card=card(), sms=torch.cuda.get_device_properties(0).multi_processor_count)
    res["search"] = bench_search(a.quick)
    res["combine"] = bench_combine()
    res["decode"] = bench_decode(a.quick)
    print(f"card: {res['card']}")
    print("| N | R | k | search (ms) | fill-only search (ms) | insertions past the fill | HBM bound (ms) | "
          "bf16 bound (ms) | larger bound | share of it | TFLOP/s |")
    print("|---|---|---|---|---|---|---|---|---|---|---|")
    for r in res["search"]:
        print(f"| {r['N']} | {r['R']} | {r['k']} | {r['ms']:.3f} | {r['fill_only_ms']:.3f} | "
              f"{100 * (1 - r['fill_only_ms'] / r['ms']):.0f} % | {r['hbm_bound_ms']:.3f} | {r['flop_bound_ms']:.3f} "
              f"| {r['bound']} | {100 * r['share']:.0f} % | {r['tflops']:.0f} |")
    c = res["combine"]
    print(f"combine B={c['B']} N={c['N']}: {1e3 * c['ms']:.1f} us, {c['bytes_per_row']} B/row, "
          f"{100 * c['hbm_share']:.0f} % of HBM peak")
    print("decode per batch (ms):", json.dumps({k: round(v, 2) for k, v in res["decode"].items()}))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
