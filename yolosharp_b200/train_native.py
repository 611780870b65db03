"""Host side of the native training step (csrc/train_step.cu, yb_trainer_* / yb_train_*): the reference's
`AMPWrapper.TrainStep` (Utils/Amp.cs:260-286) as ONE C-ABI call per step.

The library owns the graph walk and the activation arena; this class owns what a TorchSharp host would own - the flat
fp32 buffers for parameters, gradients, Adam moments and BatchNorm running statistics, as torch tensors with named views -
so that checkpoints load into them, `torch.distributed.all_reduce` runs on the gradient buffer between
`yb_train_backward` and `yb_train_apply`, and tests read every gradient.  Same interface as train.py's TrainStepV8."""
import ctypes as C

import torch

from . import _lib as L


def nc_skip_list(state_dict, nc):
    """The `skipList` of `LoadModel(path, skipNcNotEqualLayers: true)` for a Detect head (Models/YoloBaseTaskModel.cs:82-92):
    the head is the last `model.<i>` of the checkpoint; the class count of the checkpoint is the row count of the LAST key matching
    `model\\.<i>\\.cv3.+bias`; when it differs from `nc`, every key matching `model\\.<i>\\.cv3` is skipped."""
    import re
    idx = [int(m.group(1)) for m in (re.match(r"model\.(\d+)\.", k) for k in state_dict) if m]
    if not idx:
        return []
    pat = rf"model\.{max(idx)}\.cv3"
    bias_keys = [k for k in state_dict if re.search(pat + r".+bias", k)]
    if not bias_keys or int(state_dict[bias_keys[-1]].shape[0]) == nc:
        return []
    return [k for k in state_dict if re.search(pat, k)]


class NativeTrainer:
    def __init__(self, state_dict, arch="v8", size="n", nc=80, device="cuda", max_batch=16, height=640, width=640, lr=None,
                 weight_decay=5e-4):
        self.device = torch.device(device)
        dev_index = self.device.index if self.device.index is not None else 0
        cfg = L.yb_config(arch=11 if str(arch) in ("v11", "11") else 8, size=L.SIZES[size], task=L.YB_TASK_DETECT, nc=nc, reg_max=16,
                          precision=L.YB_PREC_F32, device=dev_index, max_batch=max_batch, height=height, width=width,
                          flags=0 if self.device.type == "cuda" else L.YB_FLAG_DRY_RUN)
        self._h = C.c_void_p()
        L.check(L.lib().yb_trainer_create(C.byref(cfg), C.byref(self._h)))
        self.nc, self.step_count, self.group = nc, 0, None
        self.max_batch, self.height, self.width = max_batch, height, width
        self.lr = lr if lr is not None else round(0.002 * 5 / (4 + nc), 6)  # YoloBaseTaskModel.cs:142
        self.wd = weight_decay
        self.params, self.stats = self._layout(0), self._layout(1)
        lib = L.lib()
        n_p, n_s, self.n_bias = (int(lib.yb_trainer_flat_size(self._h, k)) for k in (0, 1, 2))
        if self.device.type != "cuda":
            return
        self.flat = torch.zeros(n_p, dtype=torch.float32, device=self.device)
        self.grad, self.m, self.v = torch.zeros_like(self.flat), torch.zeros_like(self.flat), torch.zeros_like(self.flat)
        self.running = torch.zeros(n_s, dtype=torch.float32, device=self.device)
        L.check(lib.yb_trainer_bind(self._h, *(C.c_void_p(t.data_ptr()) for t in (self.flat, self.grad, self.m, self.v, self.running))))
        if state_dict is not None:
            self.load_state_dict(state_dict)

    def _layout(self, kind):
        lib, out = L.lib(), {}
        for i in range(lib.yb_trainer_num_tensors(self._h, kind)):
            name, off, cnt, nd, shp = C.c_char_p(), C.c_int64(), C.c_int64(), C.c_int32(), C.POINTER(C.c_int64)()
            L.check(lib.yb_trainer_tensor_info(self._h, kind, i, C.byref(name), C.byref(off), C.byref(cnt), C.byref(nd), C.byref(shp)))
            out[name.value.decode()] = (off.value, cnt.value, tuple(shp[j] for j in range(nd.value)))
        return out

    def load_state_dict(self, sd, skipNcNotEqualLayers=False):
        """`yolo.load_state_dict(state_dict, skip: skipList, strict: false)` as `LoadModel` calls it
        (Models/YoloBaseTaskModel.cs:27-114).  skipNcNotEqualLayers: when the checkpoint's class count (rows of the last cv3
        bias of the Detect head) differs from this trainer's, every `model.<head>.cv3...` tensor is left as it is in the
        buffers (:82-92: the reference keeps the freshly constructed head there) - load a randomly initialised state_dict of
        the target class count first, then the checkpoint with this flag.  -> list of skipped keys."""
        skip = nc_skip_list(sd, self.nc) if skipNcNotEqualLayers else []
        missing = [k for k in list(self.params) + list(self.stats) if k not in sd and k not in skip]
        if missing:
            raise KeyError(f"state_dict lacks {len(missing)} tensors of the model, e.g. {missing[:3]}")
        for table, buf in ((self.params, self.flat), (self.stats, self.running)):
            for k, (o, c, shp) in table.items():
                if k in skip:
                    continue
                if tuple(sd[k].shape) != shp:
                    raise ValueError(f"{k}: shape {tuple(sd[k].shape)} != {shp}")
                buf[o:o + c].copy_(sd[k].detach().reshape(-1).to(device=self.device, dtype=torch.float32))
        return skip

    def p(self, k):
        table, buf = (self.params, self.flat) if k in self.params else (self.stats, self.running)
        o, c, shp = table[k]
        return buf[o:o + c].view(shp)

    def g(self, k):
        o, c, shp = self.params[k]
        return self.grad[o:o + c].view(shp)

    def step(self, images_nchw, targets, lrs=None, stream=None):
        """images (B,3,H,W) uint8 or float32 in [0,1] on the device; targets (n,6) rows [image, cls, x, y, w, h];
        lrs = (lr of the "bias" group, lr of the rest).  -> loss items (3,) on the host."""
        assert images_nchw.is_cuda and images_nchw.is_contiguous() and images_nchw.dtype in (torch.uint8, torch.float32)
        B = images_nchw.shape[0]
        t = torch.as_tensor(targets, dtype=torch.float32).reshape(-1, 6).cpu().contiguous()
        items = torch.empty(3, dtype=torch.float32)
        sp = C.c_void_p(stream.cuda_stream) if stream is not None else C.c_void_p(torch.cuda.current_stream().cuda_stream)
        L.check(L.lib().yb_train_backward(self._h, C.c_void_p(images_nchw.data_ptr()),
                                          L.YB_U8 if images_nchw.dtype == torch.uint8 else L.YB_F32, B,
                                          C.c_void_p(t.data_ptr()) if t.numel() else None, t.shape[0], C.c_void_p(items.data_ptr()), sp))
        if self.group is not False and torch.distributed.is_available() and torch.distributed.is_initialized() and \
                torch.distributed.get_world_size(self.group) > 1:
            torch.distributed.all_reduce(self.grad, group=self.group)  # summed, as train.py (Loss.cs:473 scales by the local batch)
        lr_bias, lr_other = lrs if lrs is not None else (self.lr, self.lr)
        L.check(L.lib().yb_train_apply(self._h, lr_bias, lr_other, self.wd, sp))
        self.step_count += 1
        return items

    def evaluate(self, images_nchw, stream=None):
        """`AMPWrapper.Evaluate` (Utils/Amp.cs:387-395): the model being trained in `eval()` - BatchNorm on the running
        statistics, TF32 tensor-core convolutions, fp32 storage - on images (B,3,H,W) uint8 or float32 in [0,1] on the device,
        B <= max_batch at the trainer's H x W.  Changes no parameter, running statistic, gradient or Adam moment.
        -> (pred (B, 4+nc, A) decoded xywh + class probabilities, boxes (B, 64, A), scores (B, nc, A) raw head outputs),
        device tensors written on `stream` (default: the current stream)."""
        self._check_images(images_nchw, "evaluate")
        B, _, H, W = images_nchw.shape
        A = sum((H // s) * (W // s) for s in (8, 16, 32))
        pred = torch.empty(B, 4 + self.nc, A, dtype=torch.float32, device=self.device)
        boxes = torch.empty(B, 64, A, dtype=torch.float32, device=self.device)
        scores = torch.empty(B, self.nc, A, dtype=torch.float32, device=self.device)
        sp = C.c_void_p(stream.cuda_stream) if stream is not None else C.c_void_p(torch.cuda.current_stream().cuda_stream)
        L.check(L.lib().yb_trainer_evaluate(self._h, C.c_void_p(images_nchw.data_ptr()),
                                            L.YB_U8 if images_nchw.dtype == torch.uint8 else L.YB_F32, B,
                                            *(C.c_void_p(t.data_ptr()) for t in (pred, boxes, scores)), sp))
        return pred, boxes, scores

    def _check_images(self, images_nchw, who):
        if not (torch.is_tensor(images_nchw) and images_nchw.dim() == 4 and images_nchw.shape[1] == 3 and
                images_nchw.dtype in (torch.uint8, torch.float32)):
            raise ValueError(f"{who}: images must be a (B, 3, H, W) uint8 or float32 tensor")
        B, _, H, W = images_nchw.shape
        if B < 1 or B > self.max_batch or (H, W) != (self.height, self.width):
            raise ValueError(f"{who}: batch {B} x {H} x {W}, the trainer takes 1..{self.max_batch} x {self.height} x {self.width}")
        if self.device.type != "cuda":
            raise RuntimeError(f"{who}: this trainer was created without a device (layout only)")
        assert images_nchw.is_cuda and images_nchw.is_contiguous()

    def validate(self, batches, group=None):
        """`Detector.Val` (Models/Detector.cs:73-160) over `batches`, a re-iterable of (images, targets) as `step` takes them,
        on the current stream: yb_trainer_val_begin, yb_trainer_val_batch per batch (a batch without targets is skipped),
        yb_trainer_val_end.  -> (loss_items (3,), metrics (4,)) host float32: the SUM of the executed batches' loss items
        and P, R, mAP50, mAP50-95 (mAP50-95 = ap[:, 1:].mean(), the reference's Slice(1)).  `last_val_counts` keeps
        (images, labels, detection rows).
        Data-parallel (an initialised torch.distributed `group` - default: this trainer's - of world > 1): every rank
        validates its own shard, then gathers all ranks' detection rows and labels and rebuilds its accumulators in rank
        order (rank 0's rows, then rank 1's, ...), so that every rank runs ap_per_class on the same rows in the same order
        (it breaks confidence ties by input order) and reports the same metrics as one device validating the rank-order
        concatenation of the shards.  The loss items and the image count stay per rank: `train.fit` all-reduces the
        fitness itself."""
        group = self.group if group is None else group
        lib, dev = L.lib(), self.device
        batches = [(x, torch.as_tensor(t, dtype=torch.float32).reshape(-1, 6).cpu().contiguous()) for x, t in batches]
        for x, _ in batches:
            self._check_images(x, "validate")
        dp = group is not False and torch.distributed.is_available() and torch.distributed.is_initialized() and \
            torch.distributed.get_world_size(group) > 1
        size = torch.tensor([sum(int(x.shape[0]) for x, t in batches if len(t)), sum(len(t) for _, t in batches)], dtype=torch.int64)
        if dp:  # the merged accumulators hold every rank's rows
            size = size.to(dev)
            torch.distributed.all_reduce(size, group=group)
            size = size.cpu()
        sp = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        L.check(lib.yb_trainer_val_begin(self._h, max(int(size[0]), 1), max(int(size[1]), 1), sp))
        for x, t in batches:
            L.check(lib.yb_trainer_val_batch(self._h, C.c_void_p(x.data_ptr()), L.YB_U8 if x.dtype == torch.uint8 else L.YB_F32,
                                              x.shape[0], C.c_void_p(t.data_ptr()) if len(t) else None, len(t), sp))
        if dp:
            self._merge_val_rows(group, sp)
        items, metrics, counts = torch.empty(3), torch.empty(4), torch.zeros(3, dtype=torch.int32)
        L.check(lib.yb_trainer_val_end(self._h, *(C.c_void_p(v.data_ptr()) for v in (items, metrics, counts)), sp))
        self.last_val_counts = tuple(int(v) for v in counts)
        return items, metrics

    def _merge_val_rows(self, group, sp):
        """Replace this rank's accumulated rows by all ranks' rows in rank order (the loss sums and image count stay)."""
        lib, dev, dist = L.lib(), self.device, torch.distributed
        nm = torch.zeros(2, dtype=torch.int32)
        L.check(lib.yb_trainer_val_rows(self._h, None, None, None, None, C.c_void_p(nm.data_ptr()), 0, sp))
        world = dist.get_world_size(group)
        sizes = [torch.zeros(2, dtype=torch.int32, device=dev) for _ in range(world)]
        dist.all_gather(sizes, nm.to(dev), group=group)
        sizes = [tuple(int(v) for v in s.cpu()) for s in sizes]
        N, M = max(max(s[0] for s in sizes), 1), max(max(s[1] for s in sizes), 1)
        mine = (torch.zeros((N, 10), dtype=torch.uint8, device=dev), torch.zeros(N, device=dev),
                torch.zeros(N, dtype=torch.int32, device=dev), torch.zeros(M, dtype=torch.int32, device=dev))
        L.check(lib.yb_trainer_val_rows(self._h, *(C.c_void_p(v.data_ptr()) for v in mine), C.c_void_p(nm.data_ptr()), 1, sp))
        gathered = []
        for t in mine:
            parts = [torch.empty_like(t) for _ in range(world)]
            dist.all_gather(parts, t, group=group)
            gathered.append(parts)
        for r, (n, m) in enumerate(sizes):
            tp, conf, cls, tcls = (g[r] for g in gathered)
            L.check(lib.yb_trainer_val_append(self._h, C.c_void_p(tp.data_ptr()), C.c_void_p(conf.data_ptr()), C.c_void_p(cls.data_ptr()),
                                              n, C.c_void_p(tcls.data_ptr()), m, sp))

    def validator(self, batches, group=None):
        """The `validate(epoch)` callback of `train.fit`: runs `validate(batches, group)` and returns its loss items
        (fit's fitness is -sum of them, YoloBaseTaskModel.cs:186); the metrics of the last pass are kept in `val_metrics`."""
        def run(epoch):
            items, self.val_metrics = self.validate(batches, group)
            return items
        return run

    def state_dict(self, dtype=torch.float32):
        """Reference-named tensors as `yolo.state_dict()` holds them (cf. TrainStepV8.state_dict)."""
        out = {k: self.p(k).detach().to(dtype).cpu() for k in self.params}
        for k in self.stats:
            out[k] = self.p(k).detach().to(dtype).cpu()
            if k.endswith(".running_mean"):
                out[k[:-len("running_mean")] + "num_batches_tracked"] = torch.tensor(self.step_count, dtype=torch.int64)
        head = next(k for k in self.params if ".cv2.0.0." in k).split(".cv2.")[0]
        out[head + ".dfl.conv.weight"] = torch.arange(16, dtype=torch.float32).view(1, 16, 1, 1)
        out[head + ".anchors"] = torch.empty(0, dtype=dtype)
        out[head + ".strides"] = torch.empty(0, dtype=dtype)
        return out

    def close(self):
        if getattr(self, "_h", None):
            L.lib().yb_trainer_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
