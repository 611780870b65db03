"""GPU parity tests (run with -m gpu on an H100): the CUDA path, called through the C ABI, against
the oracle on the same seeded inputs.

Tolerances (BASELINE.json north_star: 1e-3 fp32, indices bit-exact):
  * NMS (integer/index work + fp32 arithmetic restated op by op): bit-exact rows and indices.
  * fp32 parity mode: prediction tensor within rtol/atol 1e-3 of the fp32 oracle (observed ~1e-5).
  * fp16 tensor-core mode: fp16 storage + fp16 MMA operands perturb activations at the 1e-3..1e-2
    level, so it is checked per layer at 3e-2 of the layer's range and on the detections with set
    matching - it cannot meet 1e-3 and neither does the reference's own fp16 path (SURVEY.md §7).
"""
import os

import numpy as np
import pytest
import torch

from oracle import ops as oops
from tests.util import (GOLDEN, expected_for_op, golden_nms_cases, nms_case, oracle_activations, oracle_model,
                        oracle_real_v8n, rel_err, synth_image)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def y():
    import yolosharp_b200
    assert torch.cuda.is_available(), "GPU tests need an H100"
    from yolosharp_b200 import _lib
    _lib.lib()
    return yolosharp_b200


def make_engine(y, model, prec, B, H, W, size="n", flags=0, arch="v8", task="detect"):
    e = y.Engine(arch, size, task, 80, prec, 0, B, H, W, flags=flags)
    e.load_state_dict(model.state_dict())
    e.finalize()
    return e


# ------------------------------------------------------------------ NMS
def run_nms(y, pred, conf, iou, nc, max_det=300, max_nms=30000):
    dets, cnt, keep = y.nms(pred.cuda(), conf, iou, max_det, nc, max_nms)
    cnt = cnt.cpu().numpy()
    rows = [dets[i, :cnt[i]].cpu() for i in range(len(cnt))]
    keeps = [keep[i, :cnt[i]].cpu().long() for i in range(len(cnt))]
    return cnt, rows, keeps, dets.cpu()


def test_nms_golden_bit_exact(y):
    for tag, pred, nc, conf, iou, counts, rows, keep in golden_nms_cases():
        cnt, r, k, dets = run_nms(y, pred, conf, iou, nc)
        assert cnt.tolist() == counts.tolist(), tag
        np.testing.assert_array_equal(torch.cat(r).numpy(), rows, err_msg=tag)
        np.testing.assert_array_equal(torch.cat(k).numpy(), keep, err_msg=tag)
        for i, c in enumerate(cnt):  # rows past the count stay zero
            assert float(dets[i, c:].abs().max() if c < dets.shape[1] else 0.0) == 0.0


@pytest.mark.parametrize("seed,B,nc,A,frac,quant", [(11, 4, 80, 8400, 0.2, None), (12, 2, 80, 8400, 1.0, None),
                                                   (13, 3, 2, 2100, 0.5, 4), (14, 1, 1, 33, 1.0, None),
                                                   (15, 2, 80, 20000, 0.1, None)])
def test_nms_random_vs_oracle(y, seed, B, nc, A, frac, quant):
    """Ties (quantised scores/boxes), every-anchor-is-a-candidate (8400 > 4096: general path, shared-memory sort),
    single class, 20000 anchors (key capacity above the shared-memory sort size; ~2000 candidates: fast path)."""
    pred = nms_case(seed, B, nc, A, 0, 1.0, quant, frac)
    for conf, iou in ((0.25, 0.45), (0.1, 0.7), (0.6, 0.3)):
        out, keepi = oops.non_max_suppression(pred, conf, iou, nc=nc)
        cnt, r, k, _ = run_nms(y, pred, conf, iou, nc)
        assert cnt.tolist() == [o.shape[0] for o in out]
        for i in range(B):
            assert torch.equal(k[i], keepi[i]), (seed, conf, iou, i)
            assert torch.equal(r[i], out[i]), (seed, conf, iou, i)


def test_nms_max_nms_and_max_det(y):
    pred = nms_case(21, 2, 6, 1500, 0, 1.0, None, 1.0)
    for max_det, max_nms in ((10, 30000), (300, 100), (1, 1)):
        out, keepi = oops.non_max_suppression(pred, 0.25, 0.45, nc=6, max_det=max_det, max_nms=max_nms)
        cnt, r, k, _ = run_nms(y, pred, 0.25, 0.45, 6, max_det, max_nms)
        for i in range(2):
            assert torch.equal(k[i], keepi[i]) and torch.equal(r[i], out[i])


def test_nms_overlapping_class_ranges(y):
    """max_wh smaller than the boxes: the per-class offsets no longer separate the classes (boxes of different
    classes suppress each other), so the kernel must leave its class-wise fast path; also a long single-class
    segment and negative / out-of-range coordinates on the fast path."""
    pred = nms_case(31, 2, 5, 3000, 0, 1.0, None, 0.6)
    for max_wh in (1000, 100, 7680):
        out, keepi = oops.non_max_suppression(pred, 0.25, 0.45, nc=5, max_wh=max_wh)
        dets, cnt, keep = y.nms(pred.cuda(), 0.25, 0.45, 300, 5, 30000, max_wh)
        for i in range(2):
            c = int(cnt[i])
            assert c == out[i].shape[0], (max_wh, i)
            assert torch.equal(keep[i, :c].cpu().long(), keepi[i]) and torch.equal(dets[i, :c].cpu(), out[i]), (max_wh, i)
    shifted = pred.clone()
    shifted[:, 0] -= 500.0  # x centres partly negative: still inside (-0.49, 0.49) * max_wh
    out, keepi = oops.non_max_suppression(shifted, 0.25, 0.45, nc=5)
    cnt, r, k, _ = run_nms(y, shifted, 0.25, 0.45, 5)
    for i in range(2):
        assert torch.equal(k[i], keepi[i]) and torch.equal(r[i], out[i])


def test_nms_errors(y):
    p = torch.zeros(1, 84, 64, device="cuda")
    with pytest.raises(ValueError):
        y.Ops.non_max_suppression(p, conf_thres=1.2)
    with pytest.raises(y.YbError):
        y.nms(p, conf_thres=0.25, iou_thres=2.0)
    out, keep = y.Ops.non_max_suppression(p)
    assert out[0].shape == (0, 6) and keep[0].numel() == 0


# ------------------------------------------------------------------ forward, fp32 parity mode
def check_layers(e, model, x, tol, B, min_ops=55):
    (inf, _), acts = oracle_activations(model, x)
    pred = e.forward(x.cuda())
    if isinstance(pred, tuple):
        pred = pred[0]
    torch.cuda.synchronize()
    worst = ("", 0.0)
    n = 0
    for i, name in enumerate(e.op_names()):
        exp = expected_for_op(model, acts, name)
        if exp is None:
            continue
        try:
            got = e.read_activation(i, B)
        except Exception as ex:  # head convs whose epilogue writes pred directly have no NHWC output
            assert "fused head decode" in str(ex), ex
            continue
        assert tuple(got.shape) == tuple(exp.shape), name
        if name.endswith(".cv1") and type(model.get_submodule(name.rsplit(".", 1)[0])).__name__ == "C2PSA":
            # the second half of this buffer is later overwritten in place by the PSA block output
            got, exp = got[:, :got.shape[1] // 2], exp[:, :exp.shape[1] // 2]
        err = rel_err(got, exp)
        assert err < tol, f"op {i} {name}: rel err {err:.3e}"
        worst = max(worst, (name, err), key=lambda t: t[1])
        n += 1
    assert n >= min_ops
    return pred.cpu(), inf["boxes"], worst


def test_fp32_layers_and_pred_v8n(y):
    m = oracle_model("v8", "detect", "n")
    x = synth_image(2, 256, 320)
    e = make_engine(y, m, "f32", 2, 256, 320)
    pred, ref, worst = check_layers(e, m, x, 1e-4, 2)
    np.testing.assert_allclose(pred.numpy(), ref.numpy(), rtol=1e-3, atol=1e-3)
    # second call goes through the captured CUDA graph: identical bits
    p2 = e.forward(x.cuda()).cpu()
    p3 = e.forward(x.cuda()).cpu()
    assert torch.equal(p2, pred) and torch.equal(p3, pred)


def test_fp32_end_to_end_indices_v8n_640(y):
    """configs[0]-style: 1x3x640x640, fp32: boxes/scores within 1e-3, kept indices and classes exact."""
    m = oracle_model("v8", "detect", "n")
    x = synth_image(1, 640, 640)
    with torch.no_grad():
        ref = m(x)[0]["boxes"]
    net = y.Yolov8(80, yoloSize="n", dtype=torch.float32)
    net.load_state_dict(m.state_dict())
    pred = net.forward(x.cuda())[0]["boxes"]
    np.testing.assert_allclose(pred.cpu().numpy(), ref.numpy(), rtol=1e-3, atol=1e-3)
    out, keep = y.Ops.non_max_suppression(pred, 0.25, 0.45)
    oout, okeep = oops.non_max_suppression(ref, 0.25, 0.45)
    assert oout[0].shape[0] > 50, "synthetic weights must exercise NMS"
    assert torch.equal(keep[0].cpu(), okeep[0])
    assert torch.equal(out[0][:, 5].cpu(), oout[0][:, 5])
    np.testing.assert_allclose(out[0].cpu().numpy(), oout[0].numpy(), rtol=1e-3, atol=1e-3)


def test_fp32_real_weights_bus(y):
    """Shipped Yolov8n checkpoint + bus.jpg through Detector.ImagePredict: same YoloResults as the
    oracle / the committed golden rows."""
    m, sd = oracle_real_v8n()
    img = torch.from_numpy(np.load(os.path.join(GOLDEN, "bus_u8.npy")))
    z = np.load(os.path.join(GOLDEN, "v8n_bus.npz"))
    det = y.Detector(y.Config(YoloType="Yolov8", YoloSize="n", ScalarType="Float32"))
    det.yolo.load_state_dict(sd)
    res = det.ImagePredict(img, 0.3, 0.7)
    exp = oops.to_yolo_results(torch.from_numpy(z["rows"]))
    assert len(res) == len(exp) == 6
    for r, ex in zip(res, exp):
        assert (r.ClassID, r.CenterX, r.CenterY, r.Width, r.Height) == \
               (ex["ClassID"], ex["CenterX"], ex["CenterY"], ex["Width"], ex["Height"])
        assert abs(r.Score - ex["Score"]) < 1e-3
    pred = det.yolo.forward(oops.preprocess(img).cuda())[0]["boxes"].cpu()
    np.testing.assert_allclose(pred[0, :, ::37].numpy(), z["pred_sample"], rtol=1e-3, atol=1e-3)
    out, keep = y.Ops.non_max_suppression(pred.cuda(), 0.3, 0.7)
    np.testing.assert_array_equal(keep[0].cpu().numpy(), z["keep"])


def test_fp32_other_sizes(y):
    """v8s / v8x graphs (configs[2]) on a small input."""
    for size in ("s", "x"):
        m = oracle_model("v8", "detect", size)
        x = synth_image(1, 128, 160)
        e = make_engine(y, m, "f32", 1, 128, 160, size)
        with torch.no_grad():
            ref = m(x)[0]["boxes"]
        pred = e.forward(x.cuda()).cpu()
        np.testing.assert_allclose(pred.numpy(), ref.numpy(), rtol=1e-3, atol=1e-3)
        e.close()


# ------------------------------------------------------------------ forward, fp16 modes
def match_detections(a, b, iou_thr=0.9, score_tol=0.03):
    """fraction of rows of `a` that have a same-class partner in `b` with IoU > thr and close score"""
    if a.shape[0] == 0:
        return 1.0
    import torchvision
    iou = torchvision.ops.box_iou(a[:, :4], b[:, :4]) if b.shape[0] else torch.zeros(a.shape[0], 0)
    ok = 0
    for i in range(a.shape[0]):
        cand = (iou[i] > iou_thr) & (b[:, 5] == a[i, 5]) & ((b[:, 4] - a[i, 4]).abs() < score_tol)
        ok += bool(cand.any())
    return ok / a.shape[0]


@pytest.mark.parametrize("flags,label", [(1, "cuda-core fp16 twin"), (0, "tcgen05")])
def test_fp16_layers_v8n(y, flags, label):
    m = oracle_model("v8", "detect", "n")
    x = synth_image(2, 256, 320)
    e = make_engine(y, m, "f16", 2, 256, 320, flags=flags)
    pred, ref, worst = check_layers(e, m, x, 3e-2, 2)
    err = (pred - ref).abs()
    assert float(err[:, :4].max()) < 4.0, "boxes (pixels)"
    assert float(err[:, 4:].max()) < 0.05, "class probabilities"


@pytest.mark.parametrize("size", ["s", "x"])
def test_fp16_layers_wide_models(y, size):
    """v8s / v8x in tensor-core mode, layer by layer: streamed weights with tile pairs (odd tile counts, several N tiles
    per layer), ragged channel slabs (80 / 160 / 400 channels), dynamic tile queue."""
    m = oracle_model("v8", "detect", size)
    x = synth_image(3, 256, 320)
    e = make_engine(y, m, "f16", 3, 256, 320, size)
    pred, ref, worst = check_layers(e, m, x, 5e-2, 3, min_ops=55)
    err = (pred - ref).abs()
    assert float(err[:, :4].max()) < 6.0, ("boxes (pixels)", worst)
    assert float(err[:, 4:].max()) < 0.08, ("class probabilities", worst)
    e.close()


def test_fp16_tcgen05_matches_cuda_core_twin(y):
    """Same fp16 operands, fp32 accumulation: the tensor-core kernel and its CUDA-core twin may only
    differ by summation order / fp16 rounding of near-ties."""
    for size, hw in (("n", (256, 320)), ("s", (128, 160)), ("x", (64, 96))):
        m = oracle_model("v8", "detect", size)
        x = synth_image(2, *hw).cuda()
        a = make_engine(y, m, "f16", 2, hw[0], hw[1], size, flags=0)
        b = make_engine(y, m, "f16", 2, hw[0], hw[1], size, flags=1)
        pa = a.forward(x).clone()
        pb = b.forward(x).clone()
        torch.cuda.synchronize()
        assert float((pa - pb).abs()[:, :4].max()) < 1.0 and float((pa - pb).abs()[:, 4:].max()) < 0.02
        for i, name in enumerate(a.op_names()):
            if "decode" in name:
                continue
            try:
                ga, gb = a.read_activation(i, 2), b.read_activation(i, 2)
            except Exception as ex:
                assert "fused head decode" in str(ex), ex
                continue
            assert rel_err(ga, gb) < 1e-2, f"v8{size} op {i} {name}: {rel_err(ga, gb):.3e}"
        a.close()
        b.close()


def test_fp16_detections_real_weights(y):
    """Shipped Yolov8n weights + bus.jpg in fp16 tensor-core mode: same detections as the fp32 oracle
    (classes equal, boxes within 2 px, scores within 0.02)."""
    m, sd = oracle_real_v8n()
    img = torch.from_numpy(np.load(os.path.join(GOLDEN, "bus_u8.npy")))
    z = np.load(os.path.join(GOLDEN, "v8n_bus.npz"))
    det = y.Detector(y.Config(YoloType="Yolov8", YoloSize="n", ScalarType="Float16"))
    det.yolo.load_state_dict(sd)
    res = det.ImagePredict(img, 0.3, 0.7)
    rows = z["rows"]
    strong = rows[rows[:, 4] > 0.5]
    assert len(strong) == 4
    for r, ex in zip(res[:4], oops.to_yolo_results(torch.from_numpy(strong))):
        assert r.ClassID == ex["ClassID"]
        assert abs(r.Score - ex["Score"]) < 0.02
        for k in ("CenterX", "CenterY", "Width", "Height"):
            assert abs(getattr(r, k) - ex[k]) <= 2, (k, r, ex)


def test_fp16_detections_640(y):
    """configs[1] shape (batch of 640x640, fp16 tensor-core), synthetic weights: the prediction tensor stays
    within fp16 tolerance of the fp32 oracle and the strong detections survive.  (Random weights give
    heavily overlapping boxes whose near-threshold NMS decisions flip under fp16 noise, hence the
    loose survival bound; exact NMS behaviour is covered by the bit-exact NMS tests.)"""
    m = oracle_model("v8", "detect", "n")
    x = synth_image(4, 640, 640)
    with torch.no_grad():
        ref = m(x)[0]["boxes"]
    net = y.Yolov8(80, yoloSize="n", dtype=torch.float16, max_batch=4)
    net.load_state_dict(m.state_dict())
    pred = net.forward(x.half().cuda())[0]["boxes"]
    err = (pred.cpu() - ref).abs()
    assert float(err[:, :4].max()) < 4.0 and float(err[:, 4:].max()) < 0.05
    out, keep = y.Ops.non_max_suppression(pred, 0.25, 0.45)
    oout, okeep = oops.non_max_suppression(pred.cpu(), 0.25, 0.45)  # same input -> must be identical
    for i in range(4):
        assert torch.equal(keep[i].cpu(), okeep[i]) and torch.equal(out[i].cpu(), oout[i])
    oref, _ = oops.non_max_suppression(ref, 0.25, 0.45)
    ratios = []
    for i in range(4):
        strong = oref[i][oref[i][:, 4] > 0.35]
        ratios.append(match_detections(strong, out[i].cpu(), iou_thr=0.85))
    assert min(ratios) > 0.65 and sum(ratios) / 4 > 0.85, ratios


def test_batch_independence_full_size(y):
    """Size-independent property at BASELINE configs[1] size (32x3x640x640): image i of a batch gives
    exactly the bits it gives alone (no cross-image leakage through tiles, halos or the arena)."""
    m = oracle_model("v8", "detect", "n")
    e = make_engine(y, m, "f16", 32, 640, 640)
    x = synth_image(32, 640, 640, dtype=torch.float16).cuda()
    full = e.forward(x).clone()
    assert torch.isfinite(full).all()
    for i in (0, 13, 31):
        single = e.forward(x[i:i + 1].contiguous()).clone()
        assert torch.equal(single[0], full[i]), i
    # uint8 input path == float path on the same pixels (within fp16 rounding of x/255)
    u8 = synth_image(2, 640, 640, dtype=torch.uint8)
    a = e.forward(u8.cuda()).clone()
    b = e.forward((u8.float() / 255).half().cuda()).clone()
    assert float((a - b).abs()[:, 4:].max()) < 0.02


def test_predict_u8_end_to_end(y):
    m = oracle_model("v8", "detect", "n")
    e = make_engine(y, m, "f32", 2, 320, 320)
    u8 = synth_image(2, 320, 320, dtype=torch.uint8)
    dets, counts = e.predict_u8(u8.pin_memory(), 0.25, 0.45, 300)
    with torch.no_grad():
        ref = m(u8.float() / 255.0)[0]["boxes"]
    oout, _ = oops.non_max_suppression(ref, 0.25, 0.45)
    for i in range(2):
        assert counts[i].item() == oout[i].shape[0]
        np.testing.assert_allclose(dets[i, :counts[i]].numpy(), oout[i].numpy(), rtol=1e-3, atol=1e-3)
        assert torch.equal(dets[i, :counts[i], 5], oout[i][:, 5])


def test_predict_u8_submit_wait_pipelined(y):
    """Two-slot pipelined predict (yb_predict_u8_submit / _wait) returns the same detections as the
    synchronous call, for interleaved submissions of different batches."""
    m = oracle_model("v8", "detect", "n")
    e = make_engine(y, m, "f16", 4, 320, 320)
    imgs = [synth_image(4, 320, 320, seed=40 + i, dtype=torch.uint8).pin_memory() for i in range(3)]
    ref = [tuple(t.clone() for t in e.predict_u8(im, 0.25, 0.45, 300)) for im in imgs]
    dh = [torch.empty((4, 300, 6), dtype=torch.float32).pin_memory() for _ in range(2)]
    ch = [torch.empty((4,), dtype=torch.int32).pin_memory() for _ in range(2)]
    for rep in range(3):
        e.predict_u8_submit(0, imgs[0], dh[0], ch[0], 0.25, 0.45, 300)
        e.predict_u8_submit(1, imgs[1], dh[1], ch[1], 0.25, 0.45, 300)
        e.predict_u8_wait(0)
        assert torch.equal(ch[0], ref[0][1]) and torch.equal(dh[0], ref[0][0])
        e.predict_u8_submit(0, imgs[2], dh[0], ch[0], 0.25, 0.45, 300)
        e.predict_u8_wait(1)
        assert torch.equal(ch[1], ref[1][1]) and torch.equal(dh[1], ref[1][0])
        e.predict_u8_wait(0)
        assert torch.equal(ch[0], ref[2][1]) and torch.equal(dh[0], ref[2][0])
    with pytest.raises(y.YbError):
        e.predict_u8_wait(5)


def test_missing_weight_is_an_error(y):
    m = oracle_model("v8", "detect", "n")
    sd = dict(m.state_dict())
    del sd["model.4.cv2.bn.running_var"]
    e = y.Engine("v8", "n", "detect", 80, "f32", 0, 1, 64, 64)
    e.load_state_dict(sd)
    with pytest.raises(y.YbError) as ei:
        e.finalize()
    assert "model.4.cv2.bn.running_var" in str(ei.value)


# ------------------------------------------------------------------ YOLOv11 (C3k2 / C2PSA / DW head)
@pytest.mark.parametrize("prec,flags,tol,ptol", [("f32", 0, 1e-4, (1e-3, 1e-3)), ("f16", 0, 3e-2, (4.0, 0.05))])
def test_v11n_layers_and_pred(y, prec, flags, tol, ptol):
    m = oracle_model("v11", "detect", "n")
    x = synth_image(2, 256, 320)
    e = make_engine(y, m, prec, 2, 256, 320, flags=flags, arch="v11")
    pred, ref, worst = check_layers(e, m, x, tol, 2, min_ops=80)
    if prec == "f32":
        np.testing.assert_allclose(pred.numpy(), ref.numpy(), rtol=ptol[0], atol=ptol[1])
    else:
        err = (pred - ref).abs()
        assert float(err[:, :4].max()) < ptol[0] and float(err[:, 4:].max()) < ptol[1]


@pytest.mark.parametrize("prec,tol", [("f32", 1e-4), ("f16", 3e-2)])
def test_v11n_layers_704_general_attention(y, prec, tol):
    """At 704 x 704 the C2PSA attention (model.10) runs on 22 x 22 = 484 tokens, more than the register-blocked kernel
    takes (424), so this covers the general attention kernel of the engine."""
    m = oracle_model("v11", "detect", "n")
    x = synth_image(1, 704, 704)
    e = make_engine(y, m, prec, 1, 704, 704, arch="v11")
    check_layers(e, m, x, tol, 1, min_ops=80)


def test_v11s_fp32_pred(y):
    """configs[3] architecture (YOLOv11s; forward only - the train step is not built yet)."""
    m = oracle_model("v11", "detect", "s")
    x = synth_image(1, 128, 160)
    e = make_engine(y, m, "f32", 1, 128, 160, size="s", arch="v11")
    with torch.no_grad():
        ref = m(x)[0]["boxes"]
    np.testing.assert_allclose(e.forward(x.cuda()).cpu().numpy(), ref.numpy(), rtol=1e-3, atol=1e-3)


# ------------------------------------------------------------------ segmentation (Segment head, Proto, masks)
@pytest.mark.parametrize("prec,size", [("f32", "n"), ("f16", "n"), ("f32", "s")])
def test_v8_seg_pred_proto_masks(y, prec, size):
    m = oracle_model("v8", "segment", size)
    B, H, W = 2, 160, 192
    x = synth_image(B, H, W)
    e = make_engine(y, m, prec, B, H, W, size=size, task="segment")
    with torch.no_grad():
        inf, _ = m(x)
    pred, proto = e.forward(x.cuda())
    assert tuple(pred.shape) == tuple(inf["boxes"].shape) and tuple(proto.shape) == tuple(inf["proto"].shape)
    if prec == "f32":
        np.testing.assert_allclose(pred.cpu().numpy(), inf["boxes"].numpy(), rtol=1e-3, atol=1e-3)
        np.testing.assert_allclose(proto.cpu().numpy(), inf["proto"].numpy(), rtol=1e-3, atol=1e-3)
    else:
        assert rel_err(proto.cpu(), inf["proto"]) < 3e-2
        assert float((pred.cpu() - inf["boxes"]).abs()[:, 4:84].max()) < 0.05
    # NMS with 32 extra columns + masks, both computed from the ENGINE's pred/proto on each side
    dets, counts, keep = y.nms(pred, 0.25, 0.45, 300, 80)
    out, keepi = oops.non_max_suppression(pred.cpu(), 0.25, 0.45, nc=80)
    masks = y.masks(proto, dets, counts, H, W).cpu()
    for i in range(B):
        n = counts[i].item()
        assert n == out[i].shape[0] and torch.equal(keep[i, :n].cpu().long(), keepi[i])
        assert torch.equal(dets[i, :n].cpu(), out[i])
        if n == 0:
            continue
        ref_masks = oops.process_mask(proto[i].cpu(), out[i][:, 6:], out[i][:, :4], (H, W), upsample=True)
        agree = (masks[i, :n].bool() == ref_masks.bool()).float().mean().item()
        assert agree > 0.999, agree


# ------------------------------------------------------------------ training path: detection loss + gradients
def _loss_case(B=3, H=160, W=192, seed=0):
    from oracle import loss as oloss
    m = oracle_model("v8", "detect", "n").train()
    x = synth_image(B, H, W, seed=seed)
    with torch.no_grad():
        _, preds = m(x)
    g = torch.Generator().manual_seed(seed + 7)
    n = 11
    bidx = torch.randint(0, B, (n,), generator=g).sort().values  # the reference's collate keeps targets grouped by image
    bidx[0] = 0
    cls = torch.randint(0, 80, (n,), generator=g)
    xy = torch.rand(n, 2, generator=g) * 0.6 + 0.2
    wh = torch.rand(n, 2, generator=g) * 0.45 + 0.02
    wh[1] = torch.tensor([0.03, 0.025])  # smaller than the smallest stride: widened by select_candidates_in_gts
    batch = {"batch_idx": bidx.float(), "cls": cls.float(), "bboxes": torch.cat((xy, wh), 1)}
    return oloss, preds, batch, H, W


@pytest.mark.parametrize("seed", [0, 1])
def test_detection_loss_and_gradients_vs_oracle(y, seed):
    """yb_detection_loss vs autograd through the oracle restatement of v8DetectionLoss: loss items, assignment
    (target scores), d(loss * batch)/d(boxes, scores).  fp32 on both sides; tolerance 1e-3 relative."""
    oloss, preds, batch, H, W = _loss_case(seed=seed)
    crit = oloss.V8DetectionLoss(80)
    boxes = preds["boxes"].clone().requires_grad_(True)
    scores = preds["scores"].clone().requires_grad_(True)
    p = {"boxes": boxes, "scores": scores, "feats": preds["feats"]}
    loss, items = crit(p, batch)
    gb, gs = torch.autograd.grad(loss.sum(), (boxes, scores))
    fg, gt_idx, tbox, tscore = crit.assign(p, batch)
    tgt = torch.cat((batch["batch_idx"].view(-1, 1), batch["cls"].view(-1, 1), batch["bboxes"]), 1)
    out = y.detection_loss(preds["boxes"].cuda().contiguous(), preds["scores"].cuda().contiguous(), tgt, H, W)
    torch.cuda.synchronize()
    np.testing.assert_allclose(out["items"].cpu().numpy(), items.numpy(), rtol=1e-3, atol=1e-5)
    ts_ref = tscore.sum(-1)
    np.testing.assert_allclose(out["target_score"].cpu().numpy(), ts_ref.numpy(), rtol=1e-3, atol=1e-6)
    pos = ts_ref > 0
    assert int(pos.sum()) >= 20
    assert torch.equal(out["fg"].cpu().bool()[pos], fg[pos])
    assert torch.equal(out["gt_idx"].cpu().long()[pos], gt_idx[pos])
    for got, ref, name in ((out["grad_scores"], gs, "scores"), (out["grad_boxes"], gb, "boxes")):
        got = got.cpu()
        scale = float(ref.abs().max())
        assert scale > 0
        err = float((got - ref).abs().max())
        assert err < 2e-3 * scale, (name, err, scale)


def test_detection_loss_without_targets(y):
    oloss, preds, batch, H, W = _loss_case(B=2, H=96, W=96)
    crit = oloss.V8DetectionLoss(80)
    empty = {"batch_idx": torch.zeros(0), "cls": torch.zeros(0), "bboxes": torch.zeros(0, 4)}
    _, items = crit(preds, empty)
    out = y.detection_loss(preds["boxes"].cuda().contiguous(), preds["scores"].cuda().contiguous(), torch.zeros(0, 6), H, W)
    np.testing.assert_allclose(out["items"].cpu().numpy(), items.numpy(), rtol=1e-3, atol=1e-6)
    assert float(out["grad_boxes"].abs().max()) == 0.0 and int(out["fg"].sum()) == 0
    with pytest.raises(y.YbError):
        y.detection_loss(preds["boxes"].cuda().contiguous(), preds["scores"].cuda().contiguous(),
                         torch.tensor([[5.0, 1, 0.5, 0.5, 0.1, 0.1]]), H, W)


# ------------------------------------------------------------------ training path: BatchNorm(train)+SiLU, AdamW
@pytest.mark.parametrize("shape,act", [((4, 40, 52, 32), True), ((2, 20, 20, 256), True), ((3, 7, 9, 80), False)])
def test_bn_silu_train_forward_backward_vs_torch(y, shape, act):
    """Train-mode BatchNorm2d(eps 1e-3, momentum 0.03) + SiLU of the Conv block (Convs.cs:36-56) against
    torch.nn.functional.batch_norm(training=True) + autograd, NHWC storage."""
    g = torch.Generator().manual_seed(sum(shape))
    Cc = shape[-1]
    z = (torch.randn(shape, generator=g) * 1.7 + torch.randn(Cc, generator=g) * 3).contiguous()
    gamma, beta = torch.rand(Cc, generator=g) + 0.5, torch.randn(Cc, generator=g) * 0.3
    rm, rv = torch.randn(Cc, generator=g) * 0.1, torch.rand(Cc, generator=g) + 0.5
    dy = torch.randn(shape, generator=g)
    zt = z.permute(0, 3, 1, 2).clone().requires_grad_(True)
    gt, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    rm_ref, rv_ref = rm.clone(), rv.clone()
    u = torch.nn.functional.batch_norm(zt, rm_ref, rv_ref, gt, bt, training=True, momentum=0.03, eps=1e-3)
    yt = torch.nn.functional.silu(u) if act else u
    yt.backward(dy.permute(0, 3, 1, 2))
    rm_d, rv_d = rm.cuda(), rv.cuda()
    out, mean, invstd = y.bn_silu_train_forward(z.cuda(), gamma.cuda(), beta.cuda(), rm_d, rv_d, act=act)
    np.testing.assert_allclose(out.cpu().numpy(), yt.detach().permute(0, 2, 3, 1).numpy(), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(rm_d.cpu().numpy(), rm_ref.numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(rv_d.cpu().numpy(), rv_ref.numpy(), rtol=1e-4, atol=1e-6)
    dz, dg, db = y.bn_silu_backward(z.cuda(), dy.cuda().contiguous(), gamma.cuda(), beta.cuda(), mean, invstd, act=act)
    np.testing.assert_allclose(dz.cpu().numpy(), zt.grad.permute(0, 2, 3, 1).numpy(), rtol=1e-3, atol=2e-4)
    np.testing.assert_allclose(dg.cpu().numpy(), gt.grad.numpy(), rtol=1e-3, atol=1e-3)
    np.testing.assert_allclose(db.cpu().numpy(), bt.grad.numpy(), rtol=1e-3, atol=1e-3)


def test_adamw_step_vs_torch(y):
    g = torch.Generator().manual_seed(5)
    p0 = torch.randn(10007, generator=g)
    p_ref = p0.clone().requires_grad_(True)
    opt = torch.optim.AdamW([p_ref], lr=1.19e-4, weight_decay=5e-4)
    p, m, v = p0.cuda(), torch.zeros(10007, device="cuda"), torch.zeros(10007, device="cuda")
    for step in range(1, 4):
        grad = torch.randn(10007, generator=g) * 0.1
        p_ref.grad = grad.clone()
        opt.step()
        y.adamw_step(p, grad.cuda(), m, v, step, 1.19e-4)
        np.testing.assert_allclose(p.cpu().numpy(), p_ref.detach().numpy(), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("cin,cout,k,stride,hw", [(16, 32, 3, 2, (18, 22)), (32, 32, 3, 1, (12, 10)), (48, 24, 1, 1, (9, 7)), (3, 16, 3, 2, (20, 20))])
def test_conv_backward_vs_autograd(y, cin, cout, k, stride, hw):
    """fp32 parity kernels for the Conv2d backward (dgrad / wgrad) against torch autograd."""
    g = torch.Generator().manual_seed(cin * 100 + cout)
    x = torch.randn(2, cin, *hw, generator=g, requires_grad=True)
    w = (torch.randn(cout, cin, k, k, generator=g) * 0.2).requires_grad_(True)
    z = torch.nn.functional.conv2d(x, w, stride=stride, padding=k // 2)
    dz = torch.randn(z.shape, generator=g)
    z.backward(dz)
    dx, dw = y.conv_backward(x.detach().permute(0, 2, 3, 1).contiguous().cuda(), dz.permute(0, 2, 3, 1).contiguous().cuda(),
                             w.detach().cuda(), stride=stride)
    np.testing.assert_allclose(dx.cpu().permute(0, 3, 1, 2).numpy(), x.grad.numpy(), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(dw.cpu().numpy(), w.grad.numpy(), rtol=1e-4, atol=1e-4)


def test_conv_block_train_step_chain(y):
    """conv -> BN(train) -> SiLU forward through the parity kernels' pieces, then the full backward chain
    (BN/SiLU backward -> conv dgrad / wgrad) and one AdamW step, against the oracle Conv module under autograd."""
    from oracle.modules import Conv
    torch.manual_seed(3)
    blk = Conv(16, 32, 3, 2).train()
    with torch.no_grad():
        blk.bn.weight.uniform_(0.5, 1.5)
        blk.bn.bias.normal_(0, 0.2)
    x = torch.randn(2, 16, 24, 20, requires_grad=True)
    out = blk(x)
    dy = torch.randn_like(out)
    w0 = blk.conv.weight.detach().clone()
    opt = torch.optim.AdamW([blk.conv.weight], lr=1e-3, weight_decay=5e-4)
    out.backward(dy)
    opt.step()
    # ours: z from the reference conv (forward conv kernels are tested elsewhere), everything after it on our kernels
    z = torch.nn.functional.conv2d(x.detach(), w0, stride=2, padding=1).permute(0, 2, 3, 1).contiguous().cuda()
    gmm, bta = blk.bn.weight.detach().cuda(), blk.bn.bias.detach().cuda()
    yo, mean, invstd = y.bn_silu_train_forward(z, gmm, bta)
    np.testing.assert_allclose(yo.cpu().permute(0, 3, 1, 2).numpy(), out.detach().numpy(), rtol=1e-4, atol=1e-4)
    dzz, dgam, dbet = y.bn_silu_backward(z, dy.permute(0, 2, 3, 1).contiguous().cuda(), gmm, bta, mean, invstd)
    dx, dw = y.conv_backward(x.detach().permute(0, 2, 3, 1).contiguous().cuda(), dzz, w0.cuda(), stride=2)
    np.testing.assert_allclose(dx.cpu().permute(0, 3, 1, 2).numpy(), x.grad.numpy(), rtol=1e-3, atol=1e-4)
    np.testing.assert_allclose(dgam.cpu().numpy(), blk.bn.weight.grad.numpy(), rtol=1e-3, atol=1e-3)
    wq = w0.cuda().clone().reshape(-1)
    m, v = torch.zeros_like(wq), torch.zeros_like(wq)
    y.adamw_step(wq, dw.reshape(-1), m, v, 1, 1e-3)
    np.testing.assert_allclose(wq.cpu().numpy(), blk.conv.weight.detach().reshape(-1).numpy(), rtol=1e-4, atol=1e-6)
