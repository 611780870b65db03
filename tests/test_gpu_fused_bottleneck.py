"""Fused Bottleneck launches (DESIGN 4.1): both 3x3 convolutions of a Bottleneck in one kernel, the intermediate in shared
memory.  Every fused pair is checked against the fp16-emulating oracle: the Bottleneck output that the fused launch
stores, and the intermediate that yb_debug_read_activation materialises for the absorbed first conv."""
import ctypes as C

import pytest
import torch

from oracle import emul16
from tests.test_gpu_fp16_pinned import EMUL_LAYER_RMS, EMUL_LAYER_TOL
from tests.test_gpu_parity import make_engine, y  # noqa: F401  (fixture)
from tests.util import expected_for_op, oracle_activations, oracle_model, rel_err, synth_image

pytestmark = pytest.mark.gpu


def fused_pairs(e, B):
    """(absorbed op, fused op) index pairs: an absorbed tensor-core conv reports its FLOPs and no bytes of its own."""
    from yolosharp_b200 import _lib as L
    lib, pairs = L.lib(), []
    for i in range(lib.yb_num_ops(e._h)):
        fl, by = C.c_double(), C.c_double()
        L.check(lib.yb_op_cost(e._h, i, B, C.byref(fl), C.byref(by)))
        if lib.yb_op_kind(e._h, i) == 0 and fl.value > 0 and by.value == 0:
            pairs.append((i, i + 1))
    return pairs


def launches_without_fusion(e):
    from yolosharp_b200 import _lib as L
    lib = L.lib()
    return sum(1 for i in range(lib.yb_num_ops(e._h)) if lib.yb_op_kind(e._h, i) != 6)  # Detect decodes are fused


def check_fused(y, arch, size, B, H, W, expect):
    m = oracle_model(arch, "detect", size)
    m16 = emul16.convert(m)
    u8 = synth_image(B, H, W, dtype=torch.uint8)
    e = make_engine(y, m, "f16", B, H, W, size=size, arch=arch)
    try:
        names = e.op_names()
        pairs = fused_pairs(e, B)
        got_blocks = sorted(names[j].rsplit(".", 1)[0] for _, j in pairs)
        assert got_blocks == sorted(expect), got_blocks
        for i, j in pairs:
            assert names[i].endswith(".cv1") and names[j].endswith(".cv2")
        assert e.launches_per_forward() == launches_without_fusion(e) - len(pairs)
        e.forward(u8.cuda())
        torch.cuda.synchronize()
        (_, _), acts = oracle_activations(m16, emul16.input_u8(u8))
        bad = []
        for i, j in pairs:
            for k in (j, i):  # the Bottleneck output first: reading the absorbed op writes its arena buffer
                exp = expected_for_op(m16, acts, names[k])
                got = e.read_activation(k, B)
                assert tuple(got.shape) == tuple(exp.shape), names[k]
                err = rel_err(got, exp)
                rms = float(((got - exp.float()) ** 2).mean().sqrt() / exp.float().abs().max().clamp(min=1e-12))
                if not (err < EMUL_LAYER_TOL and rms < EMUL_LAYER_RMS):
                    bad.append((names[k], f"{err:.3e}", f"{rms:.3e}"))
        assert not bad, bad
    finally:
        e.close()


# c = 128 (model.8 / 21) does not fit; c = 64 without shortcut (model.12 / 18) runs one CTA per SM and stays unfused
V8N_FUSED = [f"model.{l}.m.{i}" for l, n in ((2, 1), (4, 2), (6, 2), (15, 1)) for i in range(n)]


@pytest.mark.parametrize("B,H,W", [(2, 224, 288), (3, 96, 160)])
def test_fused_bottleneck_v8n_partial_tiles(y, B, H, W):
    """YOLOv8n: shortcut on (model.2 / 4 / 6) and off (model.15); 8x16 tiles that end mid-image and touch all four
    image edges at every level."""
    check_fused(y, "v8", "n", B, H, W, V8N_FUSED)


def test_fused_bottleneck_v11s_cmid_differs(y):
    """YOLOv11s: the C3k2 Bottlenecks (e = 0.5: cin = cout = 2 cmid) and the two Bottlenecks inside model.6's C3k
    (e = 1.0); the c = 128 ones stay unfused."""
    check_fused(y, "v11", "s", 2, 96, 160, ["model.2.m.0", "model.4.m.0", "model.6.m.0.m.0", "model.6.m.0.m.1", "model.16.m.0"])


def test_fused_bottleneck_v8m_c48(y):
    """YOLOv8m model.2: 48 -> 48 -> 48 with shortcut, so channels 48..63 of the 64-channel slabs are K padding (the
    wider Bottlenecks of v8m stay unfused)."""
    check_fused(y, "v8", "m", 2, 96, 160, ["model.2.m.0", "model.2.m.1"])


def test_fused_bottleneck_v8n_benched_shape(y):
    """Batch 32 at 640x640, the benchmark's shape."""
    check_fused(y, "v8", "n", 32, 640, 640, V8N_FUSED)
