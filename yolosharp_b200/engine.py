"""Thin object wrapper over the C ABI (include/yolob200.h).  PyTorch is used only for device
memory and streams; every computation is a kernel of libyolob200.so."""
import ctypes as C

import numpy as np
import torch

from . import _lib as L


def _stream_ptr(stream=None):
    s = stream if stream is not None else torch.cuda.current_stream()
    return C.c_void_p(s.cuda_stream)


class Engine:
    def __init__(self, arch="v8", size="n", task="detect", nc=80, precision="f16", device=0, max_batch=1,
                 height=640, width=640, flags=0):
        self._h = C.c_void_p()
        lib = L.lib()
        cfg = L.yb_config(arch={"v8": L.YB_ARCH_V8, "v11": L.YB_ARCH_V11}[arch], size=L.SIZES[size],
                          task={"detect": L.YB_TASK_DETECT, "segment": L.YB_TASK_SEGMENT}[task], nc=nc, reg_max=16,
                          precision={"f32": L.YB_PREC_F32, "f16": L.YB_PREC_F16}[precision], device=device,
                          max_batch=max_batch, height=height, width=width, flags=flags)
        L.check(lib.yb_create(C.byref(cfg), C.byref(self._h)))
        self.cfg = cfg
        self.device = torch.device("cuda", device) if not flags & L.YB_FLAG_DRY_RUN else None
        self.nc, self.height, self.width, self.max_batch = nc, height, width, max_batch
        self.task = task
        self.anchors = lib.yb_num_anchors(self._h)
        self.pred_channels = lib.yb_pred_channels(self._h)
        self.finalized = False

    def close(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value and L is not None and getattr(L, "_lib", None) is not None:
            L._lib.yb_destroy(h)
            self._h = C.c_void_p()

    __del__ = close

    # ---- weights ----
    def expected_tensors(self):
        lib = L.lib()
        return [lib.yb_expected_tensor_name(self._h, i).decode() for i in range(lib.yb_num_expected_tensors(self._h))]

    def load_tensor_raw(self, name, dtype_code, shape, data_bytes):
        shp = (C.c_int64 * len(shape))(*shape)
        buf = C.create_string_buffer(data_bytes, len(data_bytes)) if data_bytes else None
        L.check(L.lib().yb_load_tensor(self._h, name.encode(), dtype_code, len(shape), shp,
                                       C.cast(buf, C.c_void_p) if buf else None))

    def load_state_dict(self, state_dict):
        """state_dict: reference names -> torch tensors / numpy arrays (fp16 / fp32 / bf16)."""
        want = set(self.expected_tensors())
        for name, t in state_dict.items():
            if name not in want:
                continue
            if isinstance(t, np.ndarray):
                t = torch.from_numpy(t)
            t = t.detach().cpu().contiguous()
            code = {torch.float16: L.YB_F16, torch.float32: L.YB_F32, torch.bfloat16: L.YB_BF16}.get(t.dtype)
            if code is None:
                t, code = t.float(), L.YB_F32
            shp = (C.c_int64 * t.dim())(*t.shape)
            L.check(L.lib().yb_load_tensor(self._h, name.encode(), code, t.dim(), shp, C.c_void_p(t.data_ptr())))

    def load_checkpoint(self, path):
        """yb_load_checkpoint: native .bin / .safetensors reader -> (tensors loaded, expected tensors missing)."""
        n, miss = C.c_int32(), C.c_int32()
        L.check(L.lib().yb_load_checkpoint(self._h, str(path).encode(), C.byref(n), C.byref(miss)))
        return n.value, miss.value

    def finalize(self):
        L.check(L.lib().yb_finalize_weights(self._h))
        self.finalized = True

    # ---- compute ----
    def forward(self, x, out_pred=None, out_proto=None, stream=None):
        """x: CUDA (B,3,H,W) uint8 / float16 / float32 -> pred float32 (B, C, A) [, proto]."""
        assert x.is_cuda and x.is_contiguous() and x.dim() == 4 and x.shape[1] == 3
        assert x.shape[2] <= self.height and x.shape[3] <= self.width, "engine was planned for a smaller input size"
        code = {torch.uint8: L.YB_U8, torch.float16: L.YB_F16, torch.float32: L.YB_F32}[x.dtype]
        B = x.shape[0]
        if out_pred is None:
            out_pred = torch.empty((B, self.pred_channels, self.anchors), dtype=torch.float32, device=x.device)
        proto_ptr = None
        if self.task == "segment":
            if out_proto is None:
                out_proto = torch.empty((B, 32, self.height // 4, self.width // 4), dtype=torch.float32, device=x.device)
            proto_ptr = C.c_void_p(out_proto.data_ptr())
        # smaller images are padded right / bottom with 114 inside the first kernel (Detector.cs:35-41)
        L.check(L.lib().yb_forward_padded(self._h, C.c_void_p(x.data_ptr()), code, B, x.shape[2], x.shape[3],
                                          C.c_void_p(out_pred.data_ptr()), proto_ptr, _stream_ptr(stream)))
        return (out_pred, out_proto) if self.task == "segment" else out_pred

    def predict_u8(self, images_host, conf_thres=0.25, iou_thres=0.45, max_det=300, dets_host=None, counts_host=None,
                   stream=None):
        """HOST uint8 (B,3,H,W) -> HOST (dets (B,max_det,6), counts (B,)); H2D + forward + NMS + D2H."""
        assert not images_host.is_cuda and images_host.dtype == torch.uint8 and images_host.is_contiguous()
        B = images_host.shape[0]
        row_w = 6 + self.pred_channels - 4 - self.nc
        if dets_host is None:
            dets_host = torch.empty((B, max_det, row_w), dtype=torch.float32).pin_memory()
            counts_host = torch.empty((B,), dtype=torch.int32).pin_memory()
        L.check(L.lib().yb_predict_u8(self._h, C.c_void_p(images_host.data_ptr()), B, conf_thres, iou_thres, max_det,
                                      C.c_void_p(dets_host.data_ptr()), C.c_void_p(counts_host.data_ptr()),
                                      _stream_ptr(stream)))
        return dets_host, counts_host

    def predict_u8_submit(self, slot, images_host, dets_host, counts_host, conf_thres=0.25, iou_thres=0.45, max_det=300):
        """Pipelined predict: enqueue H2D + forward + NMS + D2H on the engine's slot stream (slot 0/1)."""
        assert not images_host.is_cuda and images_host.dtype == torch.uint8 and images_host.is_contiguous()
        L.check(L.lib().yb_predict_u8_submit(self._h, slot, C.c_void_p(images_host.data_ptr()), images_host.shape[0],
                                             conf_thres, iou_thres, max_det, C.c_void_p(dets_host.data_ptr()),
                                             C.c_void_p(counts_host.data_ptr())))

    def predict_u8_submit_gather(self, comm, slot, images_host, all_dets_host, all_counts_host, conf_thres=0.25,
                                 iou_thres=0.45, max_det=300):
        """yb_predict_u8_submit_gather: as predict_u8_submit, the host buffers receive the detections of ALL ranks."""
        assert not images_host.is_cuda and images_host.dtype == torch.uint8 and images_host.is_contiguous()
        L.check(L.lib().yb_predict_u8_submit_gather(self._h, comm._h, slot, C.c_void_p(images_host.data_ptr()),
                                                    images_host.shape[0], conf_thres, iou_thres, max_det,
                                                    C.c_void_p(all_dets_host.data_ptr()), C.c_void_p(all_counts_host.data_ptr())))

    def predict_seg_u8_submit(self, slot, images_host, dets_host, counts_host, masks_host, conf_thres=0.25, iou_thres=0.45,
                              max_det=300):
        """yb_predict_seg_u8_submit: segment engines; masks_host uint8 (B, mask_cap, H, W) pinned."""
        assert not images_host.is_cuda and images_host.dtype == torch.uint8 and images_host.is_contiguous()
        assert masks_host.dtype == torch.uint8 and masks_host.is_contiguous() and masks_host.dim() == 4
        L.check(L.lib().yb_predict_seg_u8_submit(self._h, slot, C.c_void_p(images_host.data_ptr()), images_host.shape[0],
                                                 conf_thres, iou_thres, max_det, masks_host.shape[1],
                                                 C.c_void_p(dets_host.data_ptr()), C.c_void_p(counts_host.data_ptr()),
                                                 C.c_void_p(masks_host.data_ptr())))

    def predict_u8_wait(self, slot):
        L.check(L.lib().yb_predict_u8_wait(self._h, slot))

    # ---- debug ----
    def op_names(self):
        lib = L.lib()
        return [lib.yb_op_name(self._h, i).decode() for i in range(lib.yb_num_ops(self._h))]

    def read_activation(self, op_index, batch):
        """NCHW float32 copy of what op `op_index` wrote during the last forward."""
        chw = (C.c_int32 * 3)()
        cap = batch * 1024 * 640 * 640 // 16
        buf = np.empty(cap, dtype=np.float32)
        L.check(L.lib().yb_debug_read_activation(self._h, op_index, batch, buf.ctypes.data_as(C.c_void_p), cap,
                                                 C.byref(chw)))
        c, h, w = chw
        return torch.from_numpy(buf[:batch * c * h * w].reshape(batch, c, h, w).copy())

    def profile(self, x, out_pred=None, stream=None):
        """Per-op device times (ms) of one eager forward + per-op algorithmic flops/bytes/kind."""
        lib = L.lib()
        n = lib.yb_num_ops(self._h)
        B = x.shape[0]
        code = {torch.uint8: L.YB_U8, torch.float16: L.YB_F16, torch.float32: L.YB_F32}[x.dtype]
        if out_pred is None:
            out_pred = torch.empty((B, self.pred_channels, self.anchors), dtype=torch.float32, device=x.device)
        proto = torch.empty((B, 32, self.height // 4, self.width // 4), dtype=torch.float32, device=x.device) \
            if self.task == "segment" else None
        ms = (C.c_float * n)()
        L.check(lib.yb_profile_forward(self._h, C.c_void_p(x.data_ptr()), code, B, C.c_void_p(out_pred.data_ptr()),
                                       C.c_void_p(proto.data_ptr()) if proto is not None else None, ms, n,
                                       _stream_ptr(stream)))
        rows = []
        for i in range(n):
            fl, by = C.c_double(), C.c_double()
            L.check(lib.yb_op_cost(self._h, i, B, C.byref(fl), C.byref(by)))
            rows.append(dict(index=i, name=lib.yb_op_name(self._h, i).decode(), kind=lib.yb_op_kind(self._h, i),
                             ms=float(ms[i]), flops=fl.value, bytes=by.value))
        return rows

    def time_op(self, op_index, x, out_pred, out_proto=None, reps=20, stream=None):
        """yb_time_op: ms per launch of one op, `reps` launches back to back."""
        code = {torch.uint8: L.YB_U8, torch.float16: L.YB_F16, torch.float32: L.YB_F32}[x.dtype]
        ms = C.c_float()
        L.check(L.lib().yb_time_op(self._h, op_index, C.c_void_p(x.data_ptr()), code, x.shape[0],
                                   C.c_void_p(out_pred.data_ptr()),
                                   C.c_void_p(out_proto.data_ptr()) if out_proto is not None else None, reps,
                                   C.byref(ms), _stream_ptr(stream)))
        return float(ms.value)

    def launches_per_forward(self):
        return L.lib().yb_launches_per_forward(self._h)


def nms(pred, conf_thres=0.25, iou_thres=0.45, max_det=300, nc=0, max_nms=30000, max_wh=7680, stream=None,
        out=None):
    """Raw batched call of yb_nms.  pred: CUDA float32 (B,C,A).  -> dets (B,max_det,6+extra), counts, keep_idx."""
    assert pred.is_cuda and pred.dtype == torch.float32 and pred.is_contiguous() and pred.dim() == 3
    B, Cc, A = pred.shape
    ncc = nc or Cc - 4
    extra = Cc - 4 - ncc
    if out is None:
        dets = torch.empty((B, max_det, 6 + extra), dtype=torch.float32, device=pred.device)
        counts = torch.empty((B,), dtype=torch.int32, device=pred.device)
        keep = torch.empty((B, max_det), dtype=torch.int32, device=pred.device)
    else:
        dets, counts, keep = out
    L.check(L.lib().yb_nms(C.c_void_p(pred.data_ptr()), B, Cc, A, ncc, conf_thres, iou_thres, max_det, max_nms, max_wh,
                           C.c_void_p(dets.data_ptr()), C.c_void_p(counts.data_ptr()), C.c_void_p(keep.data_ptr()),
                           _stream_ptr(stream)))
    return dets, counts, keep


def topk_postprocess(pred, max_det=300, nc=0, agnostic=False, stream=None):
    """yb_topk_postprocess (end2end heads, Head.cs:117-127, 175-196): pred CUDA float32 (B, 4+nc, A) ->
    rows (B, k, 6) [x, y, w, h, score, class] sorted by score, anchor index of every row (B, k)."""
    assert pred.is_cuda and pred.dtype == torch.float32 and pred.is_contiguous() and pred.dim() == 3
    B, Cc, A = pred.shape
    ncc = nc or Cc - 4
    k = min(max_det, A)
    out = torch.empty((B, k, 6), dtype=torch.float32, device=pred.device)
    idx = torch.empty((B, k), dtype=torch.int32, device=pred.device)
    L.check(L.lib().yb_topk_postprocess(C.c_void_p(pred.data_ptr()), B, Cc, A, ncc, max_det, 1 if agnostic else 0,
                                        C.c_void_p(out.data_ptr()), C.c_void_p(idx.data_ptr()), _stream_ptr(stream)))
    return out, idx


def _f32c(t):
    assert t.is_cuda and t.dtype == torch.float32
    return t.contiguous()


def obb_decode(box_logits, cls_logits, angle_logits, anchors, strides, reg_max=16, stream=None):
    """yb_obb_decode: (B,4*reg_max,A), (B,nc,A), (B,1,A), anchors (2,A), strides (A) -> (B, 4+nc+1, A)."""
    box_logits, cls_logits, angle_logits, anchors, strides = map(_f32c, (box_logits, cls_logits, angle_logits, anchors, strides))
    B, _, A = box_logits.shape
    nc = cls_logits.shape[1]
    out = torch.empty((B, 4 + nc + 1, A), dtype=torch.float32, device=box_logits.device)
    L.check(L.lib().yb_obb_decode(C.c_void_p(box_logits.data_ptr()), C.c_void_p(cls_logits.data_ptr()), C.c_void_p(angle_logits.data_ptr()),
                                  C.c_void_p(anchors.data_ptr()), C.c_void_p(strides.data_ptr()), B, A, nc, reg_max,
                                  C.c_void_p(out.data_ptr()), _stream_ptr(stream)))
    return out


def pose_decode(kpts, anchors, strides, keypoint_dim=3, stream=None):
    """yb_pose_decode: kpts (B, nk, A) -> decoded (B, nk, A)."""
    kpts, anchors, strides = map(_f32c, (kpts, anchors, strides))
    B, nk, A = kpts.shape
    out = torch.empty_like(kpts)
    L.check(L.lib().yb_pose_decode(C.c_void_p(kpts.data_ptr()), C.c_void_p(anchors.data_ptr()), C.c_void_p(strides.data_ptr()), B, A, nk,
                                   keypoint_dim, C.c_void_p(out.data_ptr()), _stream_ptr(stream)))
    return out


def probiou(obb1, obb2, eps=1e-7, stream=None):
    """yb_probiou: xywhr (n,5) x (m,5) -> (n,m)."""
    obb1, obb2 = _f32c(obb1), _f32c(obb2)
    out = torch.empty((obb1.shape[0], obb2.shape[0]), dtype=torch.float32, device=obb1.device)
    L.check(L.lib().yb_probiou(C.c_void_p(obb1.data_ptr()), obb1.shape[0], C.c_void_p(obb2.data_ptr()), obb2.shape[0], eps,
                               C.c_void_p(out.data_ptr()), _stream_ptr(stream)))
    return out


def nms_rotated(boxes, scores, threshold=0.45, stream=None):
    """yb_nms_rotated: boxes (n,5) xywhr, scores (n) -> kept original indices in score order (int64)."""
    boxes, scores = _f32c(boxes), _f32c(scores)
    n = boxes.shape[0]
    keep = torch.empty((max(n, 1),), dtype=torch.int32, device=boxes.device)
    count = torch.zeros((1,), dtype=torch.int32, device=boxes.device)
    L.check(L.lib().yb_nms_rotated(C.c_void_p(boxes.data_ptr()), C.c_void_p(scores.data_ptr()), n, threshold,
                                   C.c_void_p(keep.data_ptr()), C.c_void_p(count.data_ptr()), _stream_ptr(stream)))
    return keep[:int(count.item())].long()


def masks(proto, dets, counts, height, width, stream=None, out=None):
    """yb_masks: proto (B,32,mh,mw) f32, dets (B,max_det,38), counts -> uint8 (B,max_det,H,W)."""
    B, nm, mh, mw = proto.shape
    max_det = dets.shape[1]
    if out is None:
        out = torch.zeros((B, max_det, height, width), dtype=torch.uint8, device=proto.device)
    L.check(L.lib().yb_masks(C.c_void_p(proto.data_ptr()), C.c_void_p(dets.data_ptr()), C.c_void_p(counts.data_ptr()), B,
                             max_det, nm, mh, mw, height, width, C.c_void_p(out.data_ptr()), _stream_ptr(stream)))
    return out


def box_iou(box1, box2, eps=1e-7, stream=None):
    """yb_box_iou: (n,4), (m,4) xyxy CUDA float32 -> (n,m)."""
    assert box1.is_cuda and box2.is_cuda and box1.dtype == torch.float32 and box2.dtype == torch.float32
    box1, box2 = box1.contiguous(), box2.contiguous()
    out = torch.empty((box1.shape[0], box2.shape[0]), dtype=torch.float32, device=box1.device)
    L.check(L.lib().yb_box_iou(C.c_void_p(box1.data_ptr()), box1.shape[0], C.c_void_p(box2.data_ptr()), box2.shape[0], eps,
                               C.c_void_p(out.data_ptr()), _stream_ptr(stream)))
    return out


def match_predictions(dets, counts, labels, iouv=None, stream=None):
    """yb_match_predictions: dets (B,max_det,W) / counts (B) from nms(), labels (M,6) [image, cls, x1,y1,x2,y2]
    -> uint8 (B, max_det, 10) true-positive matrix (rows >= counts[b] are 0)."""
    assert dets.is_cuda and dets.dtype == torch.float32 and dets.is_contiguous() and counts.dtype == torch.int32
    B, max_det, W = dets.shape
    if iouv is None:
        iouv = torch.linspace(0.5, 0.95, 10, dtype=torch.float32)
    iouv = iouv.float().cpu().contiguous()
    labels = torch.as_tensor(labels, dtype=torch.float32).reshape(-1, 6).to(dets.device).contiguous()
    correct = torch.empty((B, max_det, iouv.numel()), dtype=torch.uint8, device=dets.device)
    L.check(L.lib().yb_match_predictions(C.c_void_p(dets.data_ptr()), C.c_void_p(counts.data_ptr()), B, max_det, W,
                                         C.c_void_p(labels.data_ptr()) if labels.numel() else None, labels.shape[0],
                                         C.c_void_p(iouv.data_ptr()), iouv.numel(), C.c_void_p(correct.data_ptr()), _stream_ptr(stream)))
    return correct


def mask_iou(mask1, mask2, eps=1e-7, stream=None):
    """yb_mask_iou (Utils/Metrics.cs:120-125): mask1 (N, n), mask2 (M, n) float32 CUDA tensors -> (N, M) IoU."""
    assert mask1.is_cuda and mask2.is_cuda and mask1.dim() == 2 and mask2.dim() == 2 and mask1.shape[1] == mask2.shape[1]
    a, b = mask1.float().contiguous(), mask2.float().contiguous()
    out = torch.empty((a.shape[0], b.shape[0]), dtype=torch.float32, device=a.device)
    L.check(L.lib().yb_mask_iou(C.c_void_p(a.data_ptr()) if a.numel() else None, a.shape[0], C.c_void_p(b.data_ptr()) if b.numel() else None,
                                b.shape[0], a.shape[1], float(eps), C.c_void_p(out.data_ptr()) if out.numel() else None, _stream_ptr(stream)))
    return out


def ap_per_class(tp, conf, pred_cls, target_cls, max_classes=80, stream=None):
    """yb_ap_per_class (Utils/Metrics.cs:308-384): tp (n, T) uint8 / bool, conf (n,), pred_cls (n,), target_cls (m,) on the
    device -> dict with the reference's outputs (tp, fp, p, r, f1, ap, unique_classes, p_curve, r_curve, f1_curve, x,
    prec_values) plus `best`, the index of the smoothed-F1 maximum."""
    dev = conf.device
    assert conf.is_cuda
    n, T = tp.shape[0], tp.shape[1]
    tp8 = tp.to(torch.uint8).contiguous()
    conf = conf.float().contiguous()
    pc = pred_cls.to(torch.int32).contiguous()
    tc = target_cls.to(device=dev, dtype=torch.int32).contiguous()
    f = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)
    uniq = torch.empty(max_classes, dtype=torch.int32, device=dev)
    counts = torch.zeros(3, dtype=torch.int32)
    ap, pcv, rcv, f1c, pv = f(max_classes, T), f(max_classes, 1000), f(max_classes, 1000), f(max_classes, 1000), f(max_classes, 1000)
    p, r, f1, tpo, fpo = (f(max_classes) for _ in range(5))
    ptr = lambda t: C.c_void_p(t.data_ptr()) if t.numel() else None
    L.check(L.lib().yb_ap_per_class(ptr(tp8), ptr(conf), ptr(pc), n, T, ptr(tc), tc.numel(), max_classes, ptr(uniq), C.c_void_p(counts.data_ptr()),
                                    ptr(ap), ptr(pcv), ptr(rcv), ptr(f1c), ptr(pv), ptr(p), ptr(r), ptr(f1), ptr(tpo), ptr(fpo),
                                    _stream_ptr(stream)))
    nc, n_prec, best = (int(v) for v in counts)
    x = torch.empty(1000, dtype=torch.float32)
    L.check(L.lib().yb_linspace01(1000, C.c_void_p(x.data_ptr())))
    prec_values = pv[:n_prec] if n_prec else torch.zeros((1, 1000), dtype=torch.float32, device=dev)
    return {"tp": tpo[:nc], "fp": fpo[:nc], "p": p[:nc], "r": r[:nc], "f1": f1[:nc], "ap": ap[:nc], "unique_classes": uniq[:nc],
            "p_curve": pcv[:nc], "r_curve": rcv[:nc], "f1_curve": f1c[:nc], "x": x, "prec_values": prec_values, "best": best}


def segmentation_loss(fg, gt_idx, target_bboxes, masks, proto, mask_coefficient, height, width, hyp_box=7.5, stream=None):
    """yb_segmentation_loss: the instance-mask term of v8SegmentationLoss (Utils/Loss.cs:688-865) and its gradients.
    fg (B, A) uint8 / bool, gt_idx (B, A), target_bboxes (B, A, 4) px, masks (B, mh, mw) instance index + 1, proto
    (B, nm, mh, mw), mask_coefficient (B, nm, A): CUDA tensors -> dict(item, grad_proto, grad_coefficient)."""
    assert proto.is_cuda and proto.dtype == torch.float32 and proto.is_contiguous() and mask_coefficient.is_contiguous()
    B, nm, mh, mw = proto.shape
    A = mask_coefficient.shape[2]
    dev = proto.device
    fg8 = fg.to(device=dev, dtype=torch.uint8).contiguous()
    gi = gt_idx.to(device=dev, dtype=torch.int32).contiguous()
    tb = target_bboxes.to(device=dev, dtype=torch.float32).contiguous()
    mk = masks.to(device=dev, dtype=torch.float32).contiguous()
    assert fg8.shape == (B, A) and gi.shape == (B, A) and tb.shape == (B, A, 4) and mk.shape == (B, mh, mw)
    item = torch.empty(1, dtype=torch.float32, device=dev)
    gp, gc = torch.empty_like(proto), torch.empty_like(mask_coefficient)
    p = lambda t: C.c_void_p(t.data_ptr())
    L.check(L.lib().yb_segmentation_loss(p(fg8), p(gi), p(tb), p(mk), p(proto), p(mask_coefficient), B, A, nm, mh, mw, float(height), float(width),
                                         float(hyp_box), p(item), p(gp), p(gc), _stream_ptr(stream)))
    return {"item": item, "grad_proto": gp, "grad_coefficient": gc}


def detection_loss(boxes, scores, targets, height, width, reg_max=16, topk=10, hyp_box=7.5, hyp_cls=0.5, hyp_dfl=1.5,
                   want_grad=True, stream=None):
    """yb_detection_loss: v8DetectionLoss (Utils/Loss.cs:328-485) on the raw train-mode head outputs.
    boxes (B, 4*reg_max, A), scores (B, nc, A): CUDA float32;  targets: (n, 6) rows [image, cls, x, y, w, h]
    (normalised xywh), any device / dtype (copied to host float32).
    -> dict(items (3,), grad_boxes, grad_scores, fg (B, A) uint8, gt_idx (B, A) int32, target_score (B, A))."""
    assert boxes.is_cuda and scores.is_cuda and boxes.dtype == torch.float32 and scores.dtype == torch.float32
    assert boxes.is_contiguous() and scores.is_contiguous()
    B, c4, A = boxes.shape
    nc = scores.shape[1]
    assert c4 == 4 * reg_max and scores.shape[0] == B and scores.shape[2] == A
    t = torch.as_tensor(targets, dtype=torch.float32).reshape(-1, 6).cpu().contiguous()
    items = torch.empty(3, dtype=torch.float32, device=boxes.device)
    gb = torch.empty_like(boxes) if want_grad else None
    gs = torch.empty_like(scores) if want_grad else None
    fg = torch.empty((B, A), dtype=torch.uint8, device=boxes.device)
    gi = torch.empty((B, A), dtype=torch.int32, device=boxes.device)
    ts = torch.empty((B, A), dtype=torch.float32, device=boxes.device)
    L.check(L.lib().yb_detection_loss(
        C.c_void_p(boxes.data_ptr()), C.c_void_p(scores.data_ptr()), B, nc, reg_max, height, width,
        C.c_void_p(t.data_ptr()) if t.numel() else None, t.shape[0], topk, hyp_box, hyp_cls, hyp_dfl,
        C.c_void_p(items.data_ptr()), C.c_void_p(gb.data_ptr()) if want_grad else None,
        C.c_void_p(gs.data_ptr()) if want_grad else None, C.c_void_p(fg.data_ptr()), C.c_void_p(gi.data_ptr()),
        C.c_void_p(ts.data_ptr()), _stream_ptr(stream)))
    return {"items": items, "grad_boxes": gb, "grad_scores": gs, "fg": fg, "gt_idx": gi, "target_score": ts}


def bn_silu_train_forward(z, gamma, beta, running_mean=None, running_var=None, eps=1e-3, momentum=0.03, act=True, stream=None):
    """yb_bn_silu_train_forward on an NHWC tensor z (..., C) float32 (any leading dims, contiguous).
    -> (y, save_mean, save_invstd); running stats are updated in place when given."""
    assert z.is_cuda and z.dtype == torch.float32 and z.is_contiguous()
    Cc = z.shape[-1]
    M = z.numel() // Cc
    y = torch.empty_like(z)
    mean = torch.empty(Cc, dtype=torch.float32, device=z.device)
    invstd = torch.empty_like(mean)
    L.check(L.lib().yb_bn_silu_train_forward(
        C.c_void_p(z.data_ptr()), M, Cc, Cc, C.c_void_p(gamma.data_ptr()), C.c_void_p(beta.data_ptr()), eps, momentum, int(act),
        C.c_void_p(running_mean.data_ptr()) if running_mean is not None else None,
        C.c_void_p(running_var.data_ptr()) if running_var is not None else None, C.c_void_p(y.data_ptr()), Cc,
        C.c_void_p(mean.data_ptr()), C.c_void_p(invstd.data_ptr()), _stream_ptr(stream)))
    return y, mean, invstd


def bn_silu_backward(z, dy, gamma, beta, save_mean, save_invstd, act=True, stream=None):
    """yb_bn_silu_backward -> (dz, dgamma, dbeta)."""
    assert z.is_cuda and dy.is_cuda and z.is_contiguous() and dy.is_contiguous() and z.shape == dy.shape
    Cc = z.shape[-1]
    M = z.numel() // Cc
    dz = torch.empty_like(z)
    dg = torch.empty(Cc, dtype=torch.float32, device=z.device)
    db = torch.empty_like(dg)
    L.check(L.lib().yb_bn_silu_backward(
        C.c_void_p(z.data_ptr()), C.c_void_p(dy.data_ptr()), M, Cc, Cc, Cc, C.c_void_p(gamma.data_ptr()), C.c_void_p(beta.data_ptr()),
        C.c_void_p(save_mean.data_ptr()), C.c_void_p(save_invstd.data_ptr()), int(act), C.c_void_p(dz.data_ptr()), Cc,
        C.c_void_p(dg.data_ptr()), C.c_void_p(db.data_ptr()), _stream_ptr(stream)))
    return dz, dg, db


def adamw_step(p, g, m, v, step, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=5e-4, stream=None):
    """yb_adamw_step on flat float32 CUDA tensors (in place on p, m, v)."""
    for t in (p, g, m, v):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.numel() == p.numel()
    L.check(L.lib().yb_adamw_step(C.c_void_p(p.data_ptr()), C.c_void_p(g.data_ptr()), C.c_void_p(m.data_ptr()),
                                  C.c_void_p(v.data_ptr()), p.numel(), step, lr, beta1, beta2, eps, weight_decay, _stream_ptr(stream)))


def conv_backward(x, dz, w, stride=1, pad=None, stream=None):
    """yb_conv_backward_data / _weight: x (N,H,W,Cin), dz (N,Ho,Wo,Cout) NHWC float32, w (Cout,Cin,k,k) -> (dx, dw)."""
    for t in (x, dz, w):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
    N, H, W, Cin = x.shape
    Cout, _, k, _ = w.shape
    pad = k // 2 if pad is None else pad
    dx, dw = torch.empty_like(x), torch.empty_like(w)
    L.check(L.lib().yb_conv_backward_data(C.c_void_p(dz.data_ptr()), C.c_void_p(w.data_ptr()), N, H, W, Cin, Cout, k, stride, pad,
                                          C.c_void_p(dx.data_ptr()), _stream_ptr(stream)))
    L.check(L.lib().yb_conv_backward_weight(C.c_void_p(x.data_ptr()), C.c_void_p(dz.data_ptr()), N, H, W, Cin, Cout, k, stride, pad,
                                            C.c_void_p(dw.data_ptr()), _stream_ptr(stream)))
    return dx, dw


def conv_tc_supported(cin, cout, k, stride, pad, H=0, W=0):
    """Shapes the TF32 tensor-core training convolutions take (everything else: the fp32 kernels)."""
    return cin % 8 == 0 and cout % 8 == 0 and k in (1, 3) and stride in (1, 2) and pad == k // 2 and \
        (stride == 1 or (H % 2 == 0 and W % 2 == 0))


class ConvWorkspace:
    """Device scratch shared by the yb_conv_*_tc calls of one stream (re-packed weights / split-K partials); grows on
    demand, so a step allocates it once."""

    def __init__(self, device):
        self.device, self.buf = device, None

    def get(self, N, H, W, Cin, Cout, k, stride):
        need = int(L.lib().yb_conv_tc_workspace_bytes(N, H, W, Cin, Cout, k, stride))
        if self.buf is None or self.buf.numel() < need:
            self.buf = torch.empty(max(need, 1 << 20), dtype=torch.uint8, device=self.device)
        return self.buf


def conv_forward_tc(x, w, bias=None, stride=1, pad=None, ws=None, stream=None):
    """yb_conv_forward_tc: x (N,H,W,Cin) NHWC float32, w (Cout,Cin,k,k) -> z (N,Ho,Wo,Cout); TF32 tensor-core MMAs."""
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and w.is_cuda and w.dtype == torch.float32 and w.is_contiguous()
    N, H, W, Cin = x.shape
    Cout, _, k, _ = w.shape
    pad = k // 2 if pad is None else pad
    ws = ws or ConvWorkspace(x.device)
    buf = ws.get(N, H, W, Cin, Cout, k, stride)
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    z = torch.empty((N, Ho, Wo, Cout), dtype=torch.float32, device=x.device)
    L.check(L.lib().yb_conv_forward_tc(C.c_void_p(x.data_ptr()), C.c_void_p(w.data_ptr()),
                                       C.c_void_p(bias.data_ptr()) if bias is not None else None, N, H, W, Cin, Cout, k, stride, pad,
                                       C.c_void_p(z.data_ptr()), C.c_void_p(buf.data_ptr()), buf.numel(), _stream_ptr(stream)))
    return z


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _f16_nhwc(t):
    assert t.is_cuda and t.dtype == torch.float16 and t.is_contiguous() and t.dim() == 4
    return t


def debug_conv_f16(x, w, bias, out=None, stride=1, act=1, x_coff=0, out_coff=0, res=None, res_coff=0, plan_batch=None,
                   run_batch=None, share_sms=False, tile_counter=True, decode=None, pred=None):
    """yb_debug_conv_f16: one launch of the fp16 tensor-core conv on caller buffers -> the plan description.
    x (B, H, W, pitch) fp16 with the input at channels [x_coff, x_coff + Cin); w (Cout, k, k, Cin) fp16; bias (Cout) fp32;
    out / res (B, Ho, Wo, pitch) fp16 written / read at [out_coff, ..) / [res_coff, ..); plan_batch defaults to B, run_batch
    to plan_batch.  decode = dict(mode, A, Ctot, a0, ch0, Wl, HW, stride) writes pred (run_batch, Ctot, A) fp32 instead."""
    _f16_nhwc(x)
    assert w.is_cuda and w.dtype == torch.float16 and w.is_contiguous() and w.dim() == 4 and w.shape[1] == w.shape[2]
    assert bias.is_cuda and bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == w.shape[0]
    for t in (out, res):
        if t is not None:
            _f16_nhwc(t)
    B, H, W, pitch = x.shape
    Cout, k, _, Cin = w.shape
    plan_batch = plan_batch or B
    run_batch = run_batch or plan_batch
    d = decode or {}
    if decode is not None:
        assert pred is not None and pred.is_cuda and pred.dtype == torch.float32 and pred.is_contiguous()
    desc = C.create_string_buffer(256)
    L.check(L.lib().yb_debug_conv_f16(
        _ptr(x), plan_batch, run_batch, H, W, pitch, x_coff, Cin, _ptr(w), _ptr(bias), Cout, k, stride, int(act),
        _ptr(res), res.shape[3] if res is not None else 0, res_coff, _ptr(out), out.shape[3] if out is not None else 0, out_coff,
        int(share_sms), int(tile_counter), d.get("mode", 0), d.get("A", 0), d.get("Ctot", 0), d.get("a0", 0), d.get("ch0", 0),
        d.get("Wl", 0), d.get("HW", 0), float(d.get("stride", 0.0)), _ptr(pred), desc, len(desc)))
    return desc.value.decode()


def debug_bneck_f16(x, w_a, bias_a, w_b, bias_b, out, shortcut=True, x_coff=0, out_coff=0):
    """yb_debug_bneck_f16: one launch of the fused Bottleneck kernel -> the fused plan's description.
    x (B, H, W, pitch) fp16 with the block input at [x_coff, x_coff + cin); w_a (cmid, 3, 3, cin), w_b (cout, 3, 3, cmid) fp16;
    biases fp32; out (B, H, W, pitch) fp16 written at [out_coff, out_coff + cout)."""
    _f16_nhwc(x)
    _f16_nhwc(out)
    for w, b in ((w_a, bias_a), (w_b, bias_b)):
        assert w.is_cuda and w.dtype == torch.float16 and w.is_contiguous() and tuple(w.shape[1:3]) == (3, 3)
        assert b.is_cuda and b.dtype == torch.float32 and b.is_contiguous() and b.numel() == w.shape[0]
    B, H, W, pitch = x.shape
    desc = C.create_string_buffer(256)
    L.check(L.lib().yb_debug_bneck_f16(_ptr(x), B, H, W, pitch, x_coff, w_a.shape[3], _ptr(w_a), _ptr(bias_a), w_a.shape[0],
                                       _ptr(w_b), _ptr(bias_b), w_b.shape[0], int(shortcut), _ptr(out), out.shape[3], out_coff,
                                       desc, len(desc)))
    return desc.value.decode()


def debug_conv_tf32(pass_, out, w=None, x=None, dz=None, bias=None, stride=1, workspace=None):
    """yb_debug_conv_tf32: one pass of the TF32 training conv on caller buffers -> the launch descriptions (one per line).
    pass_ 0: out (N, Ho, Wo, Cout) = conv(x, w) + bias; 1: out (N, H, W, Cin) = dx from dz; 2: out (Cout, Cin, k, k) = dw.
    x (N, H, W, Cin) fp32 NHWC, dense or a channel slice x = buf[..., c0:c0 + Cin] of a wider buffer (passed pitched);
    w (Cout, Cin, k, k), dz (N, Ho, Wo, Cout), bias (Cout) fp32; workspace a uint8 CUDA tensor (default: allocated)."""
    for t in (out, w, dz, bias):
        assert t is None or (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous())
    x_pitch = 0
    if x is not None:
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.stride(3) == 1
        if not x.is_contiguous():
            N_, H_, W_, _ = x.shape
            x_pitch = x.stride(2)
            assert x.stride(1) == W_ * x_pitch and x.stride(0) == H_ * W_ * x_pitch, "x must be a channel slice of an NHWC buffer"
    if pass_ == 0:
        (N, H, W, Cin), Cout, k = x.shape, w.shape[0], w.shape[2]
    elif pass_ == 1:
        (N, H, W, Cin), Cout, k = out.shape, w.shape[0], w.shape[2]
    else:
        (N, H, W, Cin), (Cout, _, k, _) = x.shape, out.shape
    if workspace is None:
        need = int(L.lib().yb_conv_tc_workspace_bytes(N, H, W, Cin, Cout, k, stride))
        workspace = torch.empty(max(need, 256), dtype=torch.uint8, device=out.device)
    desc = C.create_string_buffer(2048)
    L.check(L.lib().yb_debug_conv_tf32(pass_, _ptr(x), x_pitch, _ptr(dz), _ptr(w), _ptr(bias), N, H, W, Cin, Cout, k, stride,
                                       _ptr(out), _ptr(workspace), workspace.numel(), desc, len(desc)))
    return desc.value.decode()


def conv_backward_tc(x, dz, w, stride=1, pad=None, ws=None, stream=None, need_dx=True):
    """yb_conv_backward_data_tc / _weight_tc -> (dx, dw); same tensors as conv_backward."""
    for t in (x, dz, w):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
    N, H, W, Cin = x.shape
    Cout, _, k, _ = w.shape
    pad = k // 2 if pad is None else pad
    ws = ws or ConvWorkspace(x.device)
    buf = ws.get(N, H, W, Cin, Cout, k, stride)
    dx, dw = (torch.empty_like(x) if need_dx else None), torch.empty_like(w)
    if need_dx:
        L.check(L.lib().yb_conv_backward_data_tc(C.c_void_p(dz.data_ptr()), C.c_void_p(w.data_ptr()), N, H, W, Cin, Cout, k, stride, pad,
                                                 C.c_void_p(dx.data_ptr()), C.c_void_p(buf.data_ptr()), buf.numel(), _stream_ptr(stream)))
    L.check(L.lib().yb_conv_backward_weight_tc(C.c_void_p(x.data_ptr()), C.c_void_p(dz.data_ptr()), N, H, W, Cin, Cout, k, stride, pad,
                                               C.c_void_p(dw.data_ptr()), C.c_void_p(buf.data_ptr()), buf.numel(), _stream_ptr(stream)))
    return dx, dw


def stem_conv_supported(w, stride, pad, H, W):
    return tuple(w.shape[1:]) == (3, 3, 3) and stride == 2 and pad == 1 and w.shape[0] % 8 == 0 and w.shape[0] <= 128 and H % 2 == 0 and W % 2 == 0


def stem_conv_forward(x, w, stream=None):
    """yb_stem_conv_forward_f32: x (N,H,W,>=3) NHWC float32, w (C,3,3,3) -> z (N,H/2,W/2,C)."""
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and w.is_cuda and w.is_contiguous()
    N, H, W, xc = x.shape
    Cout = w.shape[0]
    z = torch.empty((N, H // 2, W // 2, Cout), dtype=torch.float32, device=x.device)
    L.check(L.lib().yb_stem_conv_forward_f32(C.c_void_p(x.data_ptr()), xc, C.c_void_p(w.data_ptr()), N, H, W, Cout, C.c_void_p(z.data_ptr()),
                                             _stream_ptr(stream)))
    return z


def stem_conv_backward_weight(x, dz, w_shape, ws=None, stream=None):
    """yb_stem_conv_backward_weight_f32 -> dw (C,3,3,3)."""
    assert x.is_cuda and dz.is_cuda and x.is_contiguous() and dz.is_contiguous()
    N, H, W, xc = x.shape
    Cout = dz.shape[-1]
    ws = ws or ConvWorkspace(x.device)
    buf = ws.get(N, H, W, 8, Cout, 3, 2)
    dw = torch.empty(tuple(w_shape), dtype=torch.float32, device=x.device)
    L.check(L.lib().yb_stem_conv_backward_weight_f32(C.c_void_p(x.data_ptr()), xc, C.c_void_p(dz.data_ptr()), N, H, W, Cout,
                                                     C.c_void_p(dw.data_ptr()), C.c_void_p(buf.data_ptr()), buf.numel(), _stream_ptr(stream)))
    return dw


def dwconv3x3_forward(x, w, stream=None):
    """yb_dwconv3x3_forward_f32: x (N,H,W,C) NHWC float32, w (C,1,3,3) -> z (N,H,W,C) (stride 1, pad 1)."""
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and w.is_cuda and w.is_contiguous()
    N, H, W, Cc = x.shape
    assert tuple(w.shape) == (Cc, 1, 3, 3), "depthwise 3x3 only (groups == channels)"
    z = torch.empty_like(x)
    L.check(L.lib().yb_dwconv3x3_forward_f32(C.c_void_p(x.data_ptr()), C.c_void_p(w.data_ptr()), N, H, W, Cc,
                                             C.c_void_p(z.data_ptr()), _stream_ptr(stream)))
    return z


def dwconv3x3_backward(x, dz, w, stream=None):
    """yb_dwconv3x3_backward_f32 -> (dx like x, dw like w)."""
    for t in (x, dz, w):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
    N, H, W, Cc = x.shape
    assert tuple(w.shape) == (Cc, 1, 3, 3) and dz.shape == x.shape
    dx, dw = torch.empty_like(x), torch.empty_like(w)
    L.check(L.lib().yb_dwconv3x3_backward_f32(C.c_void_p(x.data_ptr()), C.c_void_p(dz.data_ptr()), C.c_void_p(w.data_ptr()), N, H, W,
                                              Cc, C.c_void_p(dx.data_ptr()), C.c_void_p(dw.data_ptr()), _stream_ptr(stream)))
    return dx, dw


def attention_forward(q, k, v, scale, stream=None):
    """yb_attention_forward_f32: q, k (B,N,nh,kd), v (B,N,nh,hd) float32 contiguous -> out (B,N,nh,hd)."""
    for t in (q, k, v):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
    B, N, nh, kd = q.shape
    hd = v.shape[-1]
    out = torch.empty_like(v)
    L.check(L.lib().yb_attention_forward_f32(C.c_void_p(q.data_ptr()), C.c_void_p(k.data_ptr()), C.c_void_p(v.data_ptr()), B, N, nh, kd,
                                             hd, float(scale), C.c_void_p(out.data_ptr()), _stream_ptr(stream)))
    return out


def attention_backward(q, k, v, scale, dout, stream=None):
    """yb_attention_backward_f32 -> (dq, dk, dv)."""
    for t in (q, k, v, dout):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
    B, N, nh, kd = q.shape
    hd = v.shape[-1]
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    L.check(L.lib().yb_attention_backward_f32(C.c_void_p(q.data_ptr()), C.c_void_p(k.data_ptr()), C.c_void_p(v.data_ptr()),
                                              C.c_void_p(dout.data_ptr()), B, N, nh, kd, hd, float(scale), C.c_void_p(dq.data_ptr()),
                                              C.c_void_p(dk.data_ptr()), C.c_void_p(dv.data_ptr()), _stream_ptr(stream)))
    return dq, dk, dv


def conv_forward(x, w, bias=None, stride=1, pad=None, stream=None):
    """yb_conv_forward_f32: x (N,H,W,Cin) NHWC float32, w (Cout,Cin,k,k) -> z (N,Ho,Wo,Cout) (no BN, no activation)."""
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and w.is_cuda and w.dtype == torch.float32
    N, H, W, Cin = x.shape
    Cout, _, k, _ = w.shape
    pad = k // 2 if pad is None else pad
    wp = w.permute(2, 3, 1, 0).contiguous()
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    z = torch.empty((N, Ho, Wo, Cout), dtype=torch.float32, device=x.device)
    L.check(L.lib().yb_conv_forward_f32(C.c_void_p(x.data_ptr()), C.c_void_p(wp.data_ptr()),
                                        C.c_void_p(bias.data_ptr()) if bias is not None else None, N, H, W, Cin, Cout, k, stride, pad,
                                        C.c_void_p(z.data_ptr()), _stream_ptr(stream)))
    return z


class Comm:
    """yb_comm (csrc/comm.cu): exchange of fixed-size payloads between the GPUs of one node over peer memory.
    `exchange(handle_bytes) -> list of every rank's handle bytes` is the host channel used once at connect time
    (torch.distributed all-gather by default)."""

    def __init__(self, rank, world, device, bytes_per_rank, slots=2, exchange=None):
        lib = L.lib()
        self._h = C.c_void_p()
        L.check(lib.yb_comm_create(rank, world, device, bytes_per_rank, slots, C.byref(self._h)))
        self.rank, self.world, self.bytes, self.slots = rank, world, bytes_per_rank, slots
        self.device = torch.device("cuda", device)
        hb = lib.yb_comm_handle_bytes()
        mine = C.create_string_buffer(hb)
        L.check(lib.yb_comm_local_handle(self._h, mine))
        if exchange is None:
            exchange = self._exchange_torch
        handles = exchange(bytes(mine.raw))
        assert len(handles) == world and all(len(h) == hb for h in handles)
        L.check(lib.yb_comm_connect(self._h, C.create_string_buffer(b"".join(handles), hb * world)))

    def _exchange_torch(self, mine):
        import torch.distributed as dist
        cuda = dist.get_backend() == "nccl"
        t = torch.frombuffer(bytearray(mine), dtype=torch.uint8)
        t = t.to(self.device) if cuda else t
        out = torch.empty(self.world * t.numel(), dtype=torch.uint8, device=t.device)
        dist.all_gather_into_tensor(out, t)
        raw = out.cpu().numpy().tobytes()
        return [raw[i * len(mine):(i + 1) * len(mine)] for i in range(self.world)]

    def _view(self, ptr, nbytes):
        """uint8 CUDA tensor over library-owned memory (no copy, not owned by torch)."""
        class _Arr:
            pass
        a = _Arr()
        a.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "version": 2,
                                      "data": (int(ptr), False)}
        return torch.as_tensor(a, device=self.device)

    def send_buffer(self, slot):
        return self._view(L.lib().yb_comm_send_buffer(self._h, slot), self.bytes)

    def window(self, slot):
        return self._view(L.lib().yb_comm_window(self._h, slot), self.bytes * self.world).view(self.world, self.bytes)

    def allgather(self, slot, stream=None):
        L.check(L.lib().yb_comm_allgather(self._h, slot, _stream_ptr(stream)))

    def release(self, slot, stream=None):
        L.check(L.lib().yb_comm_release(self._h, slot, _stream_ptr(stream)))

    def close(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value and getattr(L, "_lib", None) is not None:
            L._lib.yb_comm_destroy(h)
            self._h = C.c_void_p()

    __del__ = close


def detection_payload_bytes(batch, max_det, row_width):
    return int(L.lib().yb_comm_detection_payload_bytes(batch, max_det, row_width))


_TORCH_OF_CODE = {0: torch.uint8, 1: torch.int8, 2: torch.int16, 3: torch.int32, 4: torch.int64, 5: torch.float16, 6: torch.float32,
                  7: torch.float64, 11: torch.bool, 15: torch.bfloat16}
_CODE_OF_TORCH = {v: k for k, v in _TORCH_OF_CODE.items()}


def read_checkpoint(path):
    """yb_ckpt_*: native reader of TorchSharp .bin, .safetensors and torch.save (.pt / .pth) files -> ordered dict name -> torch
    tensor (file dtype)."""
    lib = L.lib()
    h = C.c_void_p()
    L.check(lib.yb_ckpt_open(str(path).encode(), C.byref(h)))
    out = {}
    try:
        for i in range(lib.yb_ckpt_count(h)):
            name, dt, nd, shp, data, nb = C.c_char_p(), C.c_int32(), C.c_int32(), C.POINTER(C.c_int64)(), C.c_void_p(), C.c_int64()
            L.check(lib.yb_ckpt_tensor(h, i, C.byref(name), C.byref(dt), C.byref(nd), C.byref(shp), C.byref(data), C.byref(nb)))
            shape = [shp[k] for k in range(nd.value)]
            td = _TORCH_OF_CODE[dt.value]
            if nb.value:
                t = torch.frombuffer(bytearray(C.string_at(data.value, nb.value)), dtype=td).reshape(shape)
            else:
                t = torch.empty(shape, dtype=td)
            out[name.value.decode("utf-8", errors="replace")] = t
    finally:
        lib.yb_ckpt_close(h)
    return out


def write_checkpoint_bin(path, state_dict):
    """yb_ckpt_write_bin: the reference's SaveWeight format (YoloBaseTaskModel.cs:470-490)."""
    items = [(k, v.detach().cpu().contiguous()) for k, v in state_dict.items()]
    n = len(items)
    names = (C.c_char_p * n)(*[k.encode() for k, _ in items])
    dts = (C.c_int32 * n)(*[_CODE_OF_TORCH[v.dtype] for _, v in items])
    nds = (C.c_int32 * n)(*[v.dim() for _, v in items])
    shape_arrs = [(C.c_int64 * max(v.dim(), 1))(*v.shape) for _, v in items]
    shapes = (C.POINTER(C.c_int64) * n)(*[C.cast(a, C.POINTER(C.c_int64)) for a in shape_arrs])
    datas = (C.c_void_p * n)(*[v.data_ptr() if v.numel() else None for _, v in items])
    L.check(L.lib().yb_ckpt_write_bin(str(path).encode(), n, names, dts, nds, shapes, datas))
