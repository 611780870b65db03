"""Oracle restatement of `Detector.Val` (Models/Detector.cs:73-160), test infrastructure only.

It composes the existing oracle pieces - v8DetectionLoss (oracle/loss.py), non_max_suppression and xywh2xyxy
(oracle/ops.py), box_iou, match_predictions and ap_per_class (oracle/val.py) - and is driven by caller-supplied per-batch
raw outputs, so the GPU tests can run it on the library's own eval outputs as well as on the oracle model's."""
import torch

from oracle import loss as oloss
from oracle import ops as oops
from oracle import val as oval


def detector_val(batches, nc):
    """batches: iterable of (pred (B, 4+nc, A) decoded, boxes (B, 64, A) and scores (B, nc, A) raw head outputs,
    targets (n, 6) rows [image, cls, x, y, w, h] normalised, H, W).
    -> (loss_items (3,) summed over the executed batches, metrics (4,) P, R, mAP50, mAP50-95, (images, labels, rows))."""
    crit = oloss.V8DetectionLoss(nc)
    loss_items, count = None, 0
    tp, conf, pcls, tcls = [], [], [], []
    for pred, boxes, scores, targets, H, W in batches:
        targets = torch.as_tensor(targets, dtype=torch.float32).reshape(-1, 6)
        if targets.shape[0] < 1:  # :91-94
            continue
        B = pred.shape[0]
        feats = [torch.zeros(B, 1, H // s, W // s) for s in (8, 16, 32)]  # the loss reads only their shapes (anchor grid)
        _, loss_detach = crit({"boxes": boxes.float(), "scores": scores.float(), "feats": feats},
                              {"batch_idx": targets[:, 0], "cls": targets[:, 1], "bboxes": targets[:, 2:]})  # :96
        out, _ = oops.non_max_suppression(pred.float(), 0.1, 0.7, max_det=300, nc=nc)  # :98
        scale = torch.tensor([W, H, W, H], dtype=torch.float32)  # :99-101
        for i, det in enumerate(out):  # :102-121
            sel = targets[:, 0] == i
            true_classes = targets[sel, 1]
            batch_bbox = oops.xywh2xyxy(targets[sel, 2:] * scale)
            iou = oval.box_iou(batch_bbox, det[:, :4])
            tp.append(oval.match_predictions(det[:, 5], true_classes, iou))
            conf.append(det[:, 4])
            pcls.append(det[:, 5])
            tcls.append(true_classes)
        loss_items = torch.zeros_like(loss_detach) if loss_items is None else loss_items  # :123-127
        loss_items = loss_items + loss_detach
        count += B
    tp, conf, pcls, tcls = torch.cat(tp), torch.cat(conf), torch.cat(pcls), torch.cat(tcls)  # :131-134 (throws when empty)
    res = oval.ap_per_class(tp, conf, pcls, tcls)
    p, r, ap = res["p"], res["r"], res["ap"]
    # :137-140 - mAP50-95 is ap[:, 1:].mean(): the reference's Slice(1) leaves the 0.50 column out
    metrics = torch.stack([p.mean(), r.mean(), ap[:, 0].mean(), ap[:, 1:].mean()])
    return loss_items, metrics, (count, tcls.shape[0], tp.shape[0])
