"""1x1 fold (DESIGN 4.1): a conv whose only reader is the next op, a 1x1 conv, runs that 1x1 in its own wgmma launch on
the accumulator registers of each tile.  The folded 1x1 issues the unfused launch's k16 steps on the same fp16 operands
with the same rounding points, so an engine with the fold must agree BIT FOR BIT with one built with YB_NO_FOLD1X1=1:
the prediction tensor and every activation both engines store.  The absorbed producers, materialised on demand by the
CUDA-core twin, are checked against the fp16-emulating oracle."""
import ctypes as C
import re

import pytest
import torch

from oracle import emul16
from tests.test_gpu_fp16_pinned import EMUL_LAYER_RMS, EMUL_LAYER_TOL
from tests.test_gpu_parity import make_engine, y  # noqa: F401  (fixture)
from tests.util import expected_for_op, oracle_activations, oracle_model, rel_err, synth_image

pytestmark = pytest.mark.gpu

PLAN_FOLD = re.compile(r"^\[plan\] (\S+) .* \(folds (\S+)\)$")
PLAN_REFUSED = re.compile(r"^\[plan\] (\S+)\s+fold refused \((\S+)\): (.*)$")


def _head(hn, branch, tail_from="1"):
    return [(f"{hn}.{branch}.{l}.{tail_from}", f"{hn}.{branch}.{l}.2") for l in range(3)]


# (producer, 1x1) pairs the planner folds, and the pairs it refuses with (a fragment of) its reason
V8N_FOLDS = [("model.1", "model.2.cv1"), ("model.3", "model.4.cv1"), ("model.5", "model.6.cv1")] + \
    _head("model.22", "cv2") + _head("model.22", "cv3")
V8N_REFUSED = {("model.7", "model.8.cv1"): "shared memory", ("model.8.cv2", "model.9.cv1"): "no fold instantiation"}
V8S_FOLDS = [("model.1", "model.2.cv1"), ("model.3", "model.4.cv1")] + _head("model.22", "cv2") + _head("model.22", "cv3")
V8S_REFUSED = {("model.5", "model.6.cv1"): "shared memory", ("model.7", "model.8.cv1"): "N tiles"}
V11S_FOLDS = [("model.1", "model.2.cv1"), ("model.3", "model.4.cv1")] + _head("model.23", "cv2") + \
    [(f"model.23.cv3.{l}.1.1", f"model.23.cv3.{l}.2") for l in range(3)]


def build_pair(y, monkeypatch, capfd, arch, size, B, H, W):
    """(engine with the fold, engine without it, folded pairs, refused pairs -> reason) from the same weights."""
    m = oracle_model(arch, "detect", size)
    monkeypatch.setenv("YB_DEBUG_PLANS", "1")
    capfd.readouterr()
    on = make_engine(y, m, "f16", B, H, W, size=size, arch=arch)
    log = capfd.readouterr().err.splitlines()
    monkeypatch.setenv("YB_NO_FOLD1X1", "1")
    off = make_engine(y, m, "f16", B, H, W, size=size, arch=arch)
    off_log = capfd.readouterr().err
    monkeypatch.delenv("YB_NO_FOLD1X1")
    monkeypatch.delenv("YB_DEBUG_PLANS")
    assert "folds" not in off_log and "fold refused" not in off_log
    folds = [(mt.group(2), mt.group(1)) for mt in map(PLAN_FOLD.match, log) if mt]
    refused = {(mt.group(2), mt.group(1)): mt.group(3) for mt in map(PLAN_REFUSED.match, log) if mt}
    return m, on, off, folds, refused


def folded_ops(e):
    """Indices of the convs folded into the next op: kind 6 (launch nothing), not a Detect decode."""
    from yolosharp_b200 import _lib as L
    lib, names = L.lib(), e.op_names()
    return [i for i in range(lib.yb_num_ops(e._h)) if lib.yb_op_kind(e._h, i) == 6 and "decode" not in names[i]]


def check_fold(y, monkeypatch, capfd, arch, size, B, H, W, expect, expect_refused=None):
    m, on, off, folds, refused = build_pair(y, monkeypatch, capfd, arch, size, B, H, W)
    try:
        names = on.op_names()
        assert names == off.op_names()  # the op list is the same with the fold on and off
        assert sorted(folds) == sorted(expect), folds
        for pair, why in (expect_refused or {}).items():
            assert pair in refused and why in refused[pair], (pair, refused.get(pair))
        idx = folded_ops(on)
        assert sorted(names[i] for i in idx) == sorted(a for a, _ in expect)
        assert all(names[i + 1] == dict(expect)[names[i]] for i in idx)
        assert folded_ops(off) == []
        assert on.launches_per_forward() == off.launches_per_forward() - len(expect)

        from yolosharp_b200 import _lib as L
        lib = L.lib()
        fl_on = fl_off = 0.0
        for i in range(len(names)):
            for e, acc in ((on, "on"), (off, "off")):
                fl, by = C.c_double(), C.c_double()
                L.check(lib.yb_op_cost(e._h, i, B, C.byref(fl), C.byref(by)))
                if lib.yb_op_kind(e._h, i) == 0:
                    if acc == "on":
                        fl_on += fl.value
                    else:
                        fl_off += fl.value
                if e is on and i in idx:
                    assert fl.value == 0 and by.value == 0, names[i]
        assert fl_on == fl_off  # the 1x1 reports both convs' FLOPs

        u8 = synth_image(B, H, W, dtype=torch.uint8).cuda()
        p_on = on.forward(u8).clone()
        p_off = off.forward(u8).clone()
        torch.cuda.synchronize()
        assert torch.equal(p_on, p_off), float((p_on - p_off).abs().max())
        # every activation both engines store, bit for bit (the 1x1 outputs first: reading an absorbed op writes its buffer)
        for i, name in enumerate(names):
            if "decode" in name or i in idx:
                continue
            try:
                a = on.read_activation(i, B)
            except Exception as ex:
                assert "fused head decode" in str(ex), ex
                continue
            b = off.read_activation(i, B)
            assert torch.equal(a, b), f"{name}: {float((a - b).abs().max()):.3e}"
        # the absorbed producers, materialised by the CUDA-core twin, against the fp16-emulating oracle
        m16 = emul16.convert(m)
        (_, _), acts = oracle_activations(m16, emul16.input_u8(u8.cpu()))
        bad = []
        for i in idx:
            exp = expected_for_op(m16, acts, names[i])
            got = on.read_activation(i, B)
            assert tuple(got.shape) == tuple(exp.shape), names[i]
            err = rel_err(got, exp)
            rms = float(((got - exp.float()) ** 2).mean().sqrt() / exp.float().abs().max().clamp(min=1e-12))
            if not (err < EMUL_LAYER_TOL and rms < EMUL_LAYER_RMS):
                bad.append((names[i], f"{err:.3e}", f"{rms:.3e}"))
        assert not bad, bad
    finally:
        on.close()
        off.close()


@pytest.mark.parametrize("B,H,W", [(2, 224, 288), (3, 96, 160)])
def test_fold_v8n_partial_tiles(y, monkeypatch, capfd, B, H, W):
    """YOLOv8n, tiles that end mid-image at every edge: S2P (model.1 / 3), TAP (model.5) and halo (Detect tails, with the
    DFL and sigmoid epilogues on rectangular tiles) producers."""
    check_fold(y, monkeypatch, capfd, "v8", "n", B, H, W, V8N_FOLDS, V8N_REFUSED)


def test_fold_v8n_benched_shape(y, monkeypatch, capfd):
    """Batch 32 at 640x640, the benchmark's shape."""
    check_fold(y, monkeypatch, capfd, "v8", "n", 32, 640, 640, V8N_FOLDS, V8N_REFUSED)


def test_fold_v8s(y, monkeypatch, capfd):
    """YOLOv8s: 64 -> 64 and 128 -> 128 backbone pairs, 128 -> 80 class tails; the 256-wide pair does not fit."""
    check_fold(y, monkeypatch, capfd, "v8", "s", 2, 96, 160, V8S_FOLDS, V8S_REFUSED)


def test_fold_v11s(y, monkeypatch, capfd):
    """YOLOv11s: C3k2 cv1 consumers, and the class tails' 1x1 -> 1x1 (a flattened producer)."""
    check_fold(y, monkeypatch, capfd, "v11", "s", 2, 96, 160, V11S_FOLDS)
