"""Tower throughput vs views per pass (workspace chunk): smaller chunks keep more of the activations in the 50 MB L2
at the price of fewer tiles per GEMM launch.  Same weights and pixels for every setting, alternating, CUDA events."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pigeon_b200 import synthetic  # noqa: E402
from pigeon_b200.vit_engine import VitDims, VitEngine  # noqa: E402

dev = torch.device("cuda:0")
dims = VitDims()
sd = synthetic.random_vit_state_dict(dims, seed=0)
views = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
px = torch.randn(views, 3, 336, 336, device=dev).half()
res = {}
engines = {c: VitEngine(sd, dims, device=dev, max_views_per_pass=c) for c in (256, 128, 64, 32, 16)}
for rep in range(2):
    for c, eng in engines.items():
        for _ in range(2):
            eng.forward(px)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        for _ in range(3):
            eng.forward(px)
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e) / 3
        res.setdefault(c, []).append(ms)
        print(f"chunk {c:4d} views: {ms:8.2f} ms per {views} views  ({views / ms * 1000 / 4:.1f} four-view images/s)", flush=True)
json.dump(res, open("gpurun_out/chunk_sweep.json", "w"))
