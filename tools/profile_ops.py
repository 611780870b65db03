"""Per-op device times of one eager forward (CUDA events around every launch) with the
algorithmic bytes/FLOPs of each op and the fraction of its own roofline bound.
    python tools/profile_ops.py [v8n|v8s|v8x] [batch] > ops_<model>.txt"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import yolosharp_b200 as y  # noqa: E402
from bench import MODELS, load_peaks  # noqa: E402
from tests.util import oracle_model, synth_image  # noqa: E402

model = sys.argv[1] if len(sys.argv) > 1 else "v8n"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 32
arch, size, task, gflop = MODELS[model]
peaks = load_peaks()
m = oracle_model(arch, task, size)
e = y.Engine(arch, size, task, 80, "f16", 0, B, 640, 640)
e.load_state_dict(m.state_dict())
e.finalize()
in_dt = {"f16": torch.float16, "u8": torch.uint8, "f32": torch.float32}[sys.argv[3] if len(sys.argv) > 3 else "f16"]
x = synth_image(B, 640, 640, dtype=in_dt).cuda()
best = None
for _ in range(5):
    rows = e.profile(x)
    if best is None:
        best = rows
    else:
        for a, b in zip(best, rows):
            a["ms"] = min(a["ms"], b["ms"])
kinds = {0: "tc", 1: "cc", 2: "stem", 3: "dw", 4: "pool", 5: "up", 6: "decode", 7: "other"}
tot = sum(r["ms"] for r in best)
print(f"# {model} B={B} fp16; peaks: HBM {peaks['hbm']} GB/s, TC {peaks['tc']} TFLOP/s ({peaks['src']}); "
      f"sum of op times {tot:.3f} ms -> {B / tot * 1e3:.0f} img/s if serialised")
print(f"{'idx':>3} {'kind':6} {'name':26} {'ms':>8} {'share':>6} {'GFLOP':>8} {'MB':>8} {'TFLOP/s':>8} {'GB/s':>8} {'bound':>6} {'frac':>6}")
for r in best:
    ms = max(r["ms"], 1e-6)
    tf = r["flops"] / ms / 1e9
    gb = r["bytes"] / ms / 1e6
    t_tc = r["flops"] / (peaks["tc"] * 1e12) * 1e3
    t_hb = r["bytes"] / (peaks["hbm"] * 1e9) * 1e3
    bound, frac = ("tc", t_tc / ms) if t_tc > t_hb else ("hbm", t_hb / ms)
    print(f"{r['index']:3d} {kinds[r['kind']]:6} {r['name']:26} {ms:8.4f} {ms / tot:6.1%} {r['flops'] / 1e9:8.2f} "
          f"{r['bytes'] / 1e6:8.1f} {tf:8.1f} {gb:8.0f} {bound:>6} {frac:6.1%}")
floor = sum(max(r["flops"] / (peaks["tc"] * 1e12), r["bytes"] / (peaks["hbm"] * 1e9)) for r in best) * 1e3
print(f"# layer-wise roofline floor {floor:.3f} ms ({B / floor * 1e3:.0f} img/s); achieved/floor = {floor / tot:.1%}")
