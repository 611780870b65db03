"""GPU parity of the BENCHED mode (fp16 storage + tensor cores, YB_PREC_F16) against the fp16-emulating oracle
(oracle/emul16.py), at the benched shape and on the reference's shipped checkpoint.

Two gaps are stated separately:
  * engine fp16  vs  fp16-emulating oracle  - same rounding points; what is left is summation order,
    `tanh.approx` in the SiLU (<= 2^-11 relative, one fp16 ulp) and one-ulp flips that propagate.
    Bound asserted here: EMUL_LAYER_TOL of the layer's range per layer, EMUL_BOX_TOL px / EMUL_CLS_TOL on
    the prediction tensor, identical kept sets after NMS.
  * fp16-emulating oracle  vs  fp32 oracle  - the price of fp16 storage itself, a property of the mode (the
    reference's own Float16 path pays it too); measured and bounded loosely (F32_GAP_*), never used as parity.
"""
import os

import numpy as np
import pytest
import torch

from oracle import emul16
from oracle import ops as oops
from tests.test_gpu_parity import make_engine, y  # noqa: F401  (fixture)
from tests.util import (GOLDEN, expected_for_op, oracle_activations, oracle_model, oracle_real_v8n, rel_err,
                        synth_image)

pytestmark = pytest.mark.gpu

# Per stored layer, engine vs emulating oracle.  One fp16 ulp at the top of a layer's range is 2^-10 = 9.8e-4 of that
# range, so ANY one-ulp flip of a large element already costs ~1e-3 on the max metric; the error grows from the stem to
# the deepest head layers as flips propagate - it is the fp16 storage noise floor, not an arithmetic difference.
EMUL_LAYER_TOL = 3e-3   # max |diff| / layer range  (3 fp16 ulps at the top of the range)
EMUL_LAYER_RMS = 3e-4   # rms diff / layer range
# Prediction tensor: the final 1x1 convs (64 / 80 inputs) and the DFL expectation (x stride) amplify that noise on
# low-confidence anchors with flat distributions; detections themselves are compared after NMS at DET_* below.
EMUL_BOX_TOL = 6.0      # max over all 8400 anchors, pixels
EMUL_CLS_TOL = 0.04     # max over all anchors x classes
EMUL_BOX_RMS = 0.08     # observed 0.03-0.04 px
EMUL_CLS_RMS = 1e-4     # observed 3e-6 .. 3e-5
DET_BOX_TOL = 0.75      # kept detections (conf > 0.25): pixels
DET_CLS_TOL = 3e-3      # kept detections: score
F32_GAP_LAYER = 3e-2


def load_test_images():
    z = np.load(os.path.join(GOLDEN, "test_images.npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files}


def letterpad640(img):
    """top-left crop to <= 640, pad right/bottom with 114 (the Detector's padding value) to 640x640"""
    img = img[:, :640, :640]
    out = torch.full((3, 640, 640), 114, dtype=torch.uint8)
    out[:, :img.shape[1], :img.shape[2]] = img
    return out


def image_batch(B):
    """B distinct 640x640 uint8 images built from the reference's five test images (rolled copies)."""
    base = [letterpad640(v) for _, v in sorted(load_test_images().items())]
    out = []
    for i in range(B):
        im = base[i % len(base)]
        k = i // len(base)
        out.append(torch.roll(im, shifts=(37 * k, 53 * k), dims=(1, 2)) if k else im)
    return torch.stack(out)


def check_layers_emul(e, m16, x16, B, tol):
    (inf, _), acts = oracle_activations(m16, x16)
    worst, n, table = ("", 0.0), 0, []
    for i, name in enumerate(e.op_names()):
        exp = expected_for_op(m16, acts, name)
        if exp is None:
            continue
        try:
            got = e.read_activation(i, B)
        except Exception as ex:
            assert "fused head decode" in str(ex), ex
            continue
        if name.endswith(".cv1") and type(m16.get_submodule(name.rsplit(".", 1)[0])).__name__ == "C2PSA":
            got, exp = got[:, :got.shape[1] // 2], exp[:, :exp.shape[1] // 2]
        err = rel_err(got, exp)
        rms = float(((got.float() - exp.float()) ** 2).mean().sqrt() / exp.float().abs().max().clamp(min=1e-12))
        table.append((i, name, err, rms))
        worst = max(worst, (name, err), key=lambda t: t[1])
        n += 1
    if os.environ.get("YB_PRINT_LAYER_TABLE"):
        print("\n".join(f"  op {i:3d} {name:34s} max {err:.3e} rms {rms:.3e}" for i, name, err, rms in table))
    bad = [(i, name, f"{err:.3e}", f"{rms:.3e}") for i, name, err, rms in table if not (err < tol and rms < tol * EMUL_LAYER_RMS / EMUL_LAYER_TOL)]
    assert not bad, f"layers beyond max {tol} / rms {tol * EMUL_LAYER_RMS / EMUL_LAYER_TOL} of their range vs the fp16-emulating oracle: {bad}"
    return inf, worst, n


def assert_pred_close(pred, ref, box_tol, cls_tol, scale=1.0):
    err = (pred - ref).abs()
    eb, ec = float(err[:, :4].max()), float(err[:, 4:84].max())
    rb, rc = float((err[:, :4] ** 2).mean().sqrt()), float((err[:, 4:84] ** 2).mean().sqrt())
    print(f"\n[pred vs emul] boxes max {eb:.4f} px rms {rb:.4f}; scores max {ec:.2e} rms {rc:.2e}")
    assert eb < box_tol * scale and ec < cls_tol * scale, f"boxes {eb:.4f} px (tol {box_tol * scale}), scores {ec:.2e} (tol {cls_tol * scale})"
    assert rb < EMUL_BOX_RMS * scale and rc < EMUL_CLS_RMS * scale, f"rms: boxes {rb:.4f} px, scores {rc:.2e}"
    return eb, ec


def test_fp16_layers_vs_emulating_oracle_real_weights_640(y):
    """Shipped Yolov8n checkpoint, 4 real 640x640 images, uint8 input path: every stored layer of the tensor-core
    engine within EMUL_LAYER_TOL of the emulating oracle; the fp16 -> fp32 gap is reported separately."""
    m, sd = oracle_real_v8n()
    m16 = emul16.convert(m)
    u8 = image_batch(4)
    e = y.Engine("v8", "n", "detect", 80, "f16", 0, 4, 640, 640)
    e.load_state_dict(sd)
    e.finalize()
    pred = e.forward(u8.cuda()).cpu()
    inf, worst, n = check_layers_emul(e, m16, emul16.input_u8(u8), 4, EMUL_LAYER_TOL)
    assert n >= 55
    eb, ec = assert_pred_close(pred, inf["boxes"], EMUL_BOX_TOL, EMUL_CLS_TOL)
    with torch.no_grad():
        ref32 = m(u8.float() / 255.0)[0]["boxes"]
    gap = (inf["boxes"] - ref32).abs()
    print(f"\n[fp16 parity] worst layer {worst[0]} {worst[1]:.2e}; pred vs emul: boxes {eb:.4f} px scores {ec:.2e}; "
          f"emul vs fp32 oracle (mode gap): boxes {float(gap[:, :4].max()):.3f} px scores {float(gap[:, 4:].max()):.2e}")
    assert float(gap[:, :4].max()) < 25.0 and float(gap[:, 4:].max()) < 0.05  # the mode's own gap (observed 11.6 px / 8e-3 on background anchors)
    e.close()


def test_fp16_benched_shape_32x640_real_weights(y):
    """BASELINE configs[1] shape (32x3x640x640, fp16 tensor-core) on the shipped checkpoint: prediction tensor within
    tolerance of the emulating oracle, NMS (conf 0.25 / iou 0.45) keeps the same anchors with the same classes."""
    m, sd = oracle_real_v8n()
    m16 = emul16.convert(m)
    u8 = image_batch(32)
    e = y.Engine("v8", "n", "detect", 80, "f16", 0, 32, 640, 640)
    e.load_state_dict(sd)
    e.finalize()
    pred = e.forward(u8.cuda())
    with torch.no_grad():
        ref = m16(emul16.input_u8(u8))[0]["boxes"]
    assert_pred_close(pred.cpu(), ref, EMUL_BOX_TOL, EMUL_CLS_TOL)
    out, keep = y.Ops.non_max_suppression(pred, 0.25, 0.45)
    oout, okeep = oops.non_max_suppression(ref, 0.25, 0.45)
    total, skipped = 0, 0
    for i in range(32):
        # a candidate within the parity tolerance of the confidence threshold may legitimately fall on either side
        cand = ref[i, 4:].amax(0)
        margin = float((cand - 0.25).abs().min())
        if margin < 2 * DET_CLS_TOL:
            skipped += 1
            continue
        assert torch.equal(keep[i].cpu(), okeep[i]), (i, keep[i].tolist(), okeep[i].tolist())
        assert torch.equal(out[i][:, 5].cpu(), oout[i][:, 5]), i
        np.testing.assert_allclose(out[i][:, :4].cpu().numpy(), oout[i][:, :4].numpy(), atol=DET_BOX_TOL)
        np.testing.assert_allclose(out[i][:, 4].cpu().numpy(), oout[i][:, 4].numpy(), atol=DET_CLS_TOL)
        total += oout[i].shape[0]
    print(f"\n[benched shape] {total} detections compared, {skipped} images skipped (a candidate within {2 * DET_CLS_TOL} of the threshold)")
    assert total >= 40 and skipped <= 10, (total, skipped)  # the batch must exercise NMS
    e.close()


def test_fp16_detector_all_test_images_vs_golden(y):
    """Detector.ImagePredict (Float16) on the reference's five test images at their native sizes (pad-114 to x32,
    uint8 stem) against the committed rows of the emulating oracle (tests/golden/v8n_images.npz) and, as the mode
    gap, against the committed fp32-oracle rows."""
    _, sd = oracle_real_v8n()
    z = np.load(os.path.join(GOLDEN, "v8n_images.npz"))
    det = y.Detector(y.Config(YoloType="Yolov8", YoloSize="n", ScalarType="Float16"))
    det.yolo.load_state_dict(sd)
    seen = 0
    for name, img in sorted(load_test_images().items()):
        res = det.ImagePredict(img, 0.3, 0.7)
        exp = oops.to_yolo_results(torch.from_numpy(z[name + "_rows16"]))
        exp32 = oops.to_yolo_results(torch.from_numpy(z[name + "_rows"]))
        assert len(res) == len(exp) == len(exp32), (name, len(res), len(exp))
        for r, ex, e32 in zip(res, exp, exp32):
            assert r.ClassID == ex["ClassID"] == e32["ClassID"], name
            assert abs(r.Score - ex["Score"]) < DET_CLS_TOL, (name, r.Score, ex["Score"])
            assert abs(r.Score - e32["Score"]) < 0.02
            for k in ("CenterX", "CenterY", "Width", "Height"):  # integer-truncated pixels: +-1 from a 0.25 px shift
                assert abs(getattr(r, k) - ex[k]) <= 1, (name, k, r, ex)
                assert abs(getattr(r, k) - e32[k]) <= 2, (name, k, r, e32)
            seen += 1
    assert seen == 13  # bus 6, tennis 3, zidane 4; daisy and trucks have no detection above 0.3


@pytest.mark.parametrize("size,task", [("x", "detect"), ("s", "segment")])
def test_wide_models_640_both_modes(y, size, task):
    """v8x (configs[2]) and v8s-seg (configs[4]) at 640x640: fp32 parity mode within 1e-3 of the fp32 oracle,
    fp16 tensor-core mode within the emulating-oracle tolerance."""
    m = oracle_model("v8", task, size)
    x = synth_image(1, 640, 640)
    with torch.no_grad():
        ref = m(x)[0]
    m16 = emul16.convert(m)
    with torch.no_grad():
        ref16 = m16(emul16.input_f16(x))[0]
    for prec in ("f32", "f16"):
        e = make_engine(y, m, prec, 1, 640, 640, size=size, task=task)
        out = e.forward(x.cuda() if prec == "f32" else x.half().cuda())
        pred, proto = (out if task == "segment" else (out, None))
        if prec == "f32":
            np.testing.assert_allclose(pred.cpu().numpy(), ref["boxes"].numpy(), rtol=1e-3, atol=1e-3)
            if proto is not None:
                np.testing.assert_allclose(proto.cpu().numpy(), ref["proto"].numpy(), rtol=1e-3, atol=1e-3)
        else:
            # deeper / wider nets accumulate more one-ulp flips: 2x the v8n tolerance
            assert_pred_close(pred.cpu(), ref16["boxes"], EMUL_BOX_TOL, EMUL_CLS_TOL, scale=2.0)
            if proto is not None:
                assert rel_err(proto.cpu(), ref16["proto"]) < 2 * EMUL_LAYER_TOL
                coef = (pred.cpu()[:, 84:] - ref16["boxes"][:, 84:]).abs().max() / ref16["boxes"][:, 84:].abs().max()
                assert float(coef) < 2 * EMUL_LAYER_TOL
        e.close()


def test_fp16_v11n_layers_vs_emulating_oracle(y):
    """YOLOv11n (C3k2 / C2PSA attention / depthwise head) with the shipped yolov11n checkpoint, fp16 mode."""
    from oracle import yolo as oyolo
    z = np.load(os.path.join(GOLDEN, "yolov11n_f16.npz"))
    m = oyolo.build("v11", "detect", "n").eval()
    own = m.state_dict()
    m.load_state_dict({k: torch.from_numpy(z[k].astype(np.float32)).reshape(own[k].shape) for k in z.files if k in own},
                      strict=False)
    m16 = emul16.convert(m)
    u8 = image_batch(2)
    e = y.Engine("v11", "n", "detect", 80, "f16", 0, 2, 640, 640)
    e.load_state_dict({k: torch.from_numpy(z[k]) for k in z.files})
    e.finalize()
    pred = e.forward(u8.cuda()).cpu()
    inf, worst, n = check_layers_emul(e, m16, emul16.input_u8(u8), 2, 2 * EMUL_LAYER_TOL)
    assert n >= 80
    assert_pred_close(pred, inf["boxes"], EMUL_BOX_TOL, EMUL_CLS_TOL, scale=2.0)
    e.close()


# ------------------------------------------------------------------ NMS beyond the shared-memory sort
@pytest.mark.parametrize("A,conf", [(20000, 0.0005), (36000, 0.0005)])
def test_nms_more_than_16384_candidates(y, A, conf):
    """> 16384 simultaneous candidates of one image: the global-memory bitonic sort; 36000 > max_nms = 30000 also
    takes the truncation to the 30000 best (Ops.cs:338-342)."""
    from tests.util import nms_case
    pred = nms_case(77, 1, 3, A, 0, 1.0, None, 1.0)
    pred[:, 4:] = pred[:, 4:].clamp(min=0.001)  # every anchor is a candidate
    out, keepi = oops.non_max_suppression(pred, conf, 0.45, nc=3)
    dets, cnt, keep = y.nms(pred.cuda(), conf, 0.45, 300, 3, 30000)
    c = int(cnt[0])
    assert c == out[0].shape[0] == 300
    assert torch.equal(keep[0, :c].cpu().long(), keepi[0])
    assert torch.equal(dets[0, :c].cpu(), out[0])


# ------------------------------------------------------------------ facade: Segmenter / YoloTask / LoadModel
def seg_state():
    z = np.load(os.path.join(GOLDEN, "yolov8n-seg_f16.npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files}


def oracle_seg():
    from oracle import yolo as oyolo
    sd = seg_state()
    m = oyolo.build("v8", "segment", "n").eval()
    own = m.state_dict()
    m.load_state_dict({k: v.float().reshape(own[k].shape) for k, v in sd.items() if k in own}, strict=False)
    return m, sd


@pytest.mark.parametrize("name", ["bus", "zidane"])
def test_segmenter_image_predict_vs_oracle(y, name):
    """Segmenter.ImagePredict (Segmenter.cs:28-84), fp32 parity mode, shipped yolov8n-seg checkpoint: bus.jpg
    (640x480, no padding) and zidane.jpg (431x767 -> pad-114 to 448x768, masks resized back): same detections,
    boxes clipped to the original image, masks agree with the oracle on > 99.9 % of the pixels."""
    m, sd = oracle_seg()
    img = load_test_images()[name]
    seg = y.Segmenter(y.Config(YoloType="Yolov8", YoloSize="n", TaskType="Segmentation", ScalarType="Float32"))
    seg.yolo.load_state_dict(sd)
    res = seg.ImagePredict(img, 0.3, 0.7)
    rows, masks, exp = oops.segmenter_predict(m, img, 0.3, 0.7)
    assert len(res) == len(exp) >= 3
    for r, ex, mk in zip(res, exp, masks):
        assert (r.ClassID, r.CenterX, r.CenterY, r.Width, r.Height) == \
               (ex["ClassID"], ex["CenterX"], ex["CenterY"], ex["Width"], ex["Height"]), (r, ex)
        assert abs(r.Score - ex["Score"]) < 1e-3
        assert r.Mask.shape == (img.shape[2], img.shape[1])  # byte[width, height]
        agree = float((torch.from_numpy(r.Mask.T.copy()).bool() == mk.bool()).float().mean())
        assert agree > 0.999, (name, agree)
    if name == "bus":
        z = np.load(os.path.join(GOLDEN, "v8nseg_bus.npz"))
        assert len(res) == z["rows"].shape[0]
        for r, px in zip(res, z["mask_pixels"]):
            assert abs(int(r.Mask.sum()) - int(px)) <= max(8, 0.002 * px)


def test_yolotask_loadmodel_bin_and_image_path(y, tmp_path):
    """YoloTask(Config).LoadModel(.bin) + ImagePredict(path) (YoloTask.cs:16-104): the checkpoint goes through the
    reference's TorchSharp .bin format on disk (Utils/Lib.cs:9-54), the image through a file."""
    import torchvision
    from yolosharp_b200 import binfmt
    _, sd = oracle_real_v8n()
    path = str(tmp_path / "Yolov8n.bin")
    code = {torch.float16: 5, torch.float32: 6, torch.int64: 4, torch.int32: 3}
    binfmt.write_bin(path, [(k, code[v.dtype], list(v.shape), v.numpy().tobytes()) for k, v in sd.items()])
    img = load_test_images()["bus"]
    ipath = str(tmp_path / "bus.png")
    torchvision.io.write_png(img, ipath)
    task = y.YoloTask(y.Config(YoloType="Yolov8", YoloSize="n", TaskType="Detection", ScalarType="Float32"))
    task.LoadModel(path)
    res = task.ImagePredict(ipath, 0.3, 0.7)
    z = np.load(os.path.join(GOLDEN, "v8n_bus.npz"))
    exp = oops.to_yolo_results(torch.from_numpy(z["rows"]))
    assert [(r.ClassID, r.CenterX, r.CenterY, r.Width, r.Height) for r in res] == \
           [(e["ClassID"], e["CenterX"], e["CenterY"], e["Width"], e["Height"]) for e in exp]
    with pytest.raises(NotImplementedError):
        y.YoloTask(y.Config(TaskType="Pose"))
    bad = str(tmp_path / "short.bin")
    binfmt.write_bin(bad, [(k, code[v.dtype], list(v.shape), v.numpy().tobytes()) for k, v in list(sd.items())[:10]])
    with pytest.raises(KeyError):
        task.LoadModel(bad)


# ------------------------------------------------------------------ validation matching (f3)
def test_box_iou_and_match_predictions_vs_oracle(y):
    """yb_box_iou bit-exact; yb_match_predictions == the reference's per-image match_predictions on the engine's own
    NMS rows, labels = jittered copies of detections (so that several detections compete for one label and vice versa)."""
    from oracle import val as oval
    from tests.util import nms_case
    g = torch.Generator().manual_seed(5)
    b1, b2 = torch.rand(37, 4, generator=g) * 300, torch.rand(53, 4, generator=g) * 300
    b1[:, 2:] += b1[:, :2]
    b2[:, 2:] += b2[:, :2]
    assert torch.equal(y.engine.box_iou(b1.cuda(), b2.cuda()).cpu(), oval.box_iou(b1, b2))
    pred = nms_case(91, 4, 6, 2500, 0, 1.0, None, 0.5)
    dets, counts, _ = y.nms(pred.cuda(), 0.1, 0.7, 300, 6)
    labels = []
    for b in range(4):
        n = int(counts[b])
        rows = dets[b, :n].cpu()
        pick = rows[torch.randperm(n, generator=g)[:40]]
        boxes = pick[:, :4] + torch.randn(pick.shape[0], 4, generator=g) * 6.0
        cls = pick[:, 5].clone()
        cls[::7] = (cls[::7] + 1) % 6  # some labels of another class
        labels.append(torch.cat((torch.full((pick.shape[0], 1), float(b)), cls[:, None], boxes), 1))
        labels.append(labels[-1][:5] + torch.tensor([0, 0, 3.0, -2.0, 4.0, 1.0]))  # near-duplicate labels
    labels = torch.cat(labels)
    correct = y.engine.match_predictions(dets, counts, labels).cpu().bool()
    total = 0
    for b in range(4):
        n = int(counts[b])
        lb = labels[labels[:, 0] == b]
        rows = dets[b, :n].cpu()
        exp = oval.match_predictions(rows[:, 5], lb[:, 1], oval.box_iou(lb[:, 2:], rows[:, :4]))
        assert torch.equal(correct[b, :n], exp), b
        assert not correct[b, n:].any()
        total += int(exp.sum())
    assert total > 100


def test_predict_seg_u8_end_to_end(y):
    """yb_predict_seg_u8_submit / _wait (Segmenter.ImagePredict for a batch): host uint8 images in, rows + the first
    mask_cap byte masks per image out == forward + nms + masks called one by one."""
    m = oracle_model("v8", "segment", "n")
    B, H, W, CAP = 2, 160, 192, 16
    e = make_engine(y, m, "f32", B, H, W, task="segment")
    u8 = synth_image(B, H, W, dtype=torch.uint8)
    pred, proto = e.forward(u8.cuda())
    dets, counts, _ = y.nms(pred, 0.25, 0.45, 300, 80)
    ref_masks = y.masks(proto, dets, counts, H, W)
    dh = torch.empty((B, 300, 38), dtype=torch.float32).pin_memory()
    ch = torch.empty((B,), dtype=torch.int32).pin_memory()
    mh = torch.zeros((B, CAP, H, W), dtype=torch.uint8).pin_memory()
    for slot in (0, 3):
        e.predict_seg_u8_submit(slot, u8.pin_memory(), dh, ch, mh, 0.25, 0.45, 300)
        e.predict_u8_wait(slot)
        assert torch.equal(ch, counts.cpu()) and torch.equal(dh, dets.cpu())
        for b in range(B):
            n = min(int(counts[b]), CAP)
            assert n > 0 and torch.equal(mh[b, :n], ref_masks[b, :n].cpu())
    with pytest.raises(y.YbError):  # detect entry point on a segment engine
        e.predict_u8_submit(0, u8.pin_memory(), dh, ch, 0.25, 0.45, 300)
