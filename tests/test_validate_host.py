"""The validation pass without a GPU: the oracle restatement of `Detector.Val` (tests/val_oracle.py) on hand-built
predictions, and the trainer's validation entry points refusing calls out of order."""
import ctypes as C

import pytest
import torch

from tests.val_oracle import detector_val

H = W = 64
A = (H // 8) * (W // 8) + (H // 16) * (W // 16) + (H // 32) * (W // 32)
NC = 3


def _pred(rows):
    """(1, 4 + NC, A) decoded prediction with one anchor per (cx, cy, w, h, cls, prob) row, every other anchor empty"""
    p = torch.zeros(1, 4 + NC, A)
    for a, (cx, cy, w, h, c, s) in enumerate(rows):
        p[0, :4, a] = torch.tensor([cx, cy, w, h])
        p[0, 4 + c, a] = s
    return p


def _raw():
    g = torch.Generator().manual_seed(0)
    return torch.randn(1, 64, A, generator=g), torch.randn(1, NC, A, generator=g)


def test_perfect_predictions():
    """every label found with its exact box: P = R = 1, and both mAPs are the reference's AP of a perfect class - 0.99, not
    1: its `interp` returns `left = 0` at recall 0, so the first of the 101 trapezoid points counts zero precision"""
    labels = torch.tensor([[0, 1, 0.25, 0.25, 0.125, 0.125], [0, 2, 0.625, 0.5, 0.25, 0.375]])
    pred = _pred([(16, 16, 8, 8, 1, 0.9), (40, 32, 16, 24, 2, 0.8)])
    items, metrics, counts = detector_val([(pred, *_raw(), labels, H, W)], NC)
    assert counts == (1, 2, 2)
    assert torch.isfinite(items).all() and (items >= 0).all()
    p, r, map50, map5095 = metrics.tolist()
    assert p == 1.0 and r == 1.0
    assert abs(map50 - 0.99) < 1e-6 and abs(map5095 - 0.99) < 1e-6, metrics


def test_map50_95_leaves_out_the_050_column():
    """one detection at IoU 0.57 with its label: a true positive at 0.50 and 0.55 only.  mAP50-95 is the mean of the
    nine columns 0.55 .. 0.95 (the reference's ap[:, 1:]), i.e. AP(0.55) / 9 - not the ten-column mean AP * 2 / 10"""
    labels = torch.tensor([[0, 0, 0.3125, 0.3125, 0.15625, 0.15625]])  # box (15, 15) - (25, 25) px
    pred = _pred([(20, 15 + 5.7 / 2, 10, 5.7, 0, 0.9)])  # (15, 15) - (25, 20.7): IoU 57 / 100
    _, metrics, _ = detector_val([(pred, *_raw(), labels, H, W)], NC)
    ap = float(metrics[2])  # the 0.50 column equals the 0.55 one here
    assert abs(ap - 0.99) < 1e-6
    assert abs(float(metrics[3]) - ap / 9) < 1e-6 and abs(float(metrics[3]) - ap * 2 / 10) > 0.05, metrics


def test_target_less_batches_and_unlabelled_images():
    """a batch without targets changes nothing (:91-94); an image without labels in a labelled batch adds its detections
    as false positives; labels without any detection give n = 0 rows and zero metrics"""
    labels = torch.tensor([[0, 1, 0.25, 0.25, 0.125, 0.125]])
    pred = _pred([(16, 16, 8, 8, 1, 0.9)])
    one = detector_val([(pred, *_raw(), labels, H, W)], NC)
    two = detector_val([(pred, *_raw(), torch.zeros(0, 6), H, W), (pred, *_raw(), labels, H, W)], NC)
    assert torch.equal(one[0], two[0]) and torch.equal(one[1], two[1]) and one[2] == two[2]
    both = torch.cat([pred, pred])
    raw = [torch.cat([t, t]) for t in _raw()]
    _, m2, c2 = detector_val([(both, *raw, labels, H, W)], NC)
    assert c2 == (2, 1, 2) and float(m2[0]) < 1.0  # image 1's detection has no label: precision drops
    _, m0, c0 = detector_val([(torch.zeros(1, 4 + NC, A), *_raw(), labels, H, W)], NC)
    assert c0 == (1, 1, 0) and m0.tolist() == [0.0, 0.0, 0.0, 0.0]


def test_val_entry_points_refuse_calls_out_of_order():
    """without yb_trainer_val_begin every validation call is YB_ERR_STATE (a layout-only trainer cannot begin one)"""
    from yolosharp_b200 import _lib as L
    from yolosharp_b200.train_native import NativeTrainer
    tr = NativeTrainer(None, "v8", "n", 80, device="cpu", max_batch=2, height=64, width=64)
    lib, h = L.lib(), tr._h
    img = (C.c_uint8 * 16)()
    tg = (C.c_float * 6)(0, 1, 0.5, 0.5, 0.1, 0.1)
    out = (C.c_float * 8)()
    cnt = (C.c_int32 * 4)()
    assert lib.yb_trainer_val_batch(h, C.cast(img, C.c_void_p), L.YB_U8, 1, C.cast(tg, C.c_void_p), 1, None) == -4
    assert b"val_begin" in lib.yb_last_error()
    assert lib.yb_trainer_val_end(h, C.cast(out, C.c_void_p), C.cast(out, C.c_void_p), C.cast(cnt, C.c_void_p), None) == -4
    assert lib.yb_trainer_val_append(h, None, None, None, 0, None, 0, None) == -4
    assert lib.yb_trainer_val_rows(h, None, None, None, None, C.cast(cnt, C.c_void_p), 0, None) == -4
    assert lib.yb_trainer_val_begin(h, 4, 8, None) == -4  # no device buffers
    with pytest.raises(Exception):
        tr.validate([])
    tr.close()
