"""Timeline of one tensor-core conv launch (CTA 0): per tile, cycles relative to the first stamp.
cols (thread 0 of the first consumer warpgroup): [tile start, accumulator complete (main loop done), epilogue done]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import torch
import yolosharp_b200 as y
from yolosharp_b200 import _lib as L
from tests.util import oracle_model, synth_image
size = os.environ.get("YB_TL_SIZE", "n")
m = oracle_model("v8", "detect", size)
B = int(os.environ.get("YB_TL_BATCH", "32"))
e = y.Engine("v8", size, "detect", 80, "f16", 0, B, 640, 640, flags=2 | 8)
e.load_state_dict(m.state_dict()); e.finalize()
x = synth_image(B, 640, 640, dtype=torch.float16).cuda()
e.forward(x); torch.cuda.synchronize()
for idx in [int(a) for a in sys.argv[1:]] or [44]:
    buf = torch.zeros(128, dtype=torch.int64, device="cuda")
    L.lib().yb_debug_timeline(C.c_void_p(buf.data_ptr()), idx)
    e.forward(x); torch.cuda.synchronize()
    t = buf.cpu().view(16, 8)
    t0 = int(t[0, 0])
    print(f"--- conv_tc launch #{idx}")
    for i in range(16):
        if int(t[i, 0]) == 0: break
        print(i, [int(t[i, k]) - t0 if int(t[i, k]) else 0 for k in (0, 3, 6)])
