"""Experiment: fixed cost of the kernel chain.  Forward time at small batches, with / without PDL
(YB_NO_PDL=1) and with / without CUDA graph (flags=2).  python tools/exp_fixed_cost.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import yolosharp_b200 as y  # noqa: E402
from tests.util import oracle_model, synth_image  # noqa: E402

m = oracle_model("v8", "detect", "n")
sd = m.state_dict()
for B in (1, 32):
    for flags, label in ((0, "graph"), (2, "eager"), (8, "graph, no concurrency")):
        e = y.Engine("v8", "n", "detect", 80, "f16", 0, B, 640, 640, flags=flags)
        e.load_state_dict(sd)
        e.finalize()
        x = synth_image(B, 640, 640, dtype=torch.float16).cuda()
        out = torch.empty((B, e.pred_channels, e.anchors), dtype=torch.float32, device="cuda")
        for _ in range(5):
            e.forward(x, out_pred=out)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(50):
            e.forward(x, out_pred=out)
        b.record()
        torch.cuda.synchronize()
        print(f"B={B:2d} {label:24s} pdl={'off' if os.environ.get('YB_NO_PDL') else 'on '} forward {a.elapsed_time(b) / 50:.4f} ms", flush=True)
        del e
