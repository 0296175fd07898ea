#!/usr/bin/env python
"""Per-kernel GPU time of one eager training step via torch.profiler (CUPTI) -- the cheap iteration tool.
usage: python tools/profile_step.py [bf16|fp32] [B]"""
import collections
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import fira_icse_b200 as F  # noqa: E402
from fira_icse_b200.parallel import DataParallelStep  # noqa: E402

prec = sys.argv[1] if len(sys.argv) > 1 else "bf16"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 64
dev = torch.device("cuda:0")
torch.manual_seed(0)
model = F.TransModel(bench.model_args()).to(dev).train().set_precision(prec)
dp = DataParallelStep(model, lambda ps: torch.optim.Adam(ps, lr=1e-4, fused=True))
batches = [bench.device_batch(bench.host_batch(i * B, B, pin=False), dev, B) for i in range(2)]
for i in range(3):
    dp.step(batches[i % 2])
torch.cuda.synchronize()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    dp.step(batches[0])
    torch.cuda.synchronize()
agg = collections.defaultdict(lambda: [0, 0.0])
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA:
        k = e.name.replace("void ", "").replace("(anonymous namespace)::", "").replace("at::native::", "")
        k = k.split("(")[0][:80]
        agg[k][0] += 1
        agg[k][1] += e.device_time
tot = sum(v[1] for v in agg.values())
print(f"precision={prec} B={B}: {sum(v[0] for v in agg.values())} kernels, {tot / 1e3:.2f} ms GPU time")
for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:32]:
    print(f"{t:9.1f} us {100 * t / tot:5.1f}% n={c:4d}  {k}")

# per-launch detail for one kernel family (grid sizes come from the chrome trace)
if len(sys.argv) > 3:
    import json
    import tempfile
    pat = sys.argv[3]
    path = os.path.join(tempfile.mkdtemp(), "trace.json")
    prof.export_chrome_trace(path)
    ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel" and pat in e.get("name", "")]
    groups = collections.defaultdict(list)
    for e in ev:
        a = e.get("args", {})
        groups[(tuple(a.get("grid", [])), tuple(a.get("block", [])))].append(e["dur"])
    print(f"--- {pat}: {len(ev)} launches")
    for k, v in sorted(groups.items(), key=lambda kv: -sum(kv[1])):
        print(f"grid={k[0]} block={k[1]} n={len(v)} total={sum(v):8.1f} us  avg={sum(v) / len(v):7.1f}  min={min(v):7.1f} max={max(v):7.1f}")
