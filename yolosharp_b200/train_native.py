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
        if not (torch.is_tensor(images_nchw) and images_nchw.dim() == 4 and images_nchw.shape[1] == 3 and
                images_nchw.dtype in (torch.uint8, torch.float32)):
            raise ValueError("evaluate: images must be a (B, 3, H, W) uint8 or float32 tensor")
        B, _, H, W = images_nchw.shape
        if B < 1 or B > self.max_batch or (H, W) != (self.height, self.width):
            raise ValueError(f"evaluate: batch {B} x {H} x {W}, the trainer takes 1..{self.max_batch} x {self.height} x {self.width}")
        if self.device.type != "cuda":
            raise RuntimeError("evaluate: this trainer was created without a device (layout only)")
        assert images_nchw.is_cuda and images_nchw.is_contiguous()
        A = sum((H // s) * (W // s) for s in (8, 16, 32))
        pred = torch.empty(B, 4 + self.nc, A, dtype=torch.float32, device=self.device)
        boxes = torch.empty(B, 64, A, dtype=torch.float32, device=self.device)
        scores = torch.empty(B, self.nc, A, dtype=torch.float32, device=self.device)
        sp = C.c_void_p(stream.cuda_stream) if stream is not None else C.c_void_p(torch.cuda.current_stream().cuda_stream)
        L.check(L.lib().yb_trainer_evaluate(self._h, C.c_void_p(images_nchw.data_ptr()),
                                            L.YB_U8 if images_nchw.dtype == torch.uint8 else L.YB_F32, B,
                                            *(C.c_void_p(t.data_ptr()) for t in (pred, boxes, scores)), sp))
        return pred, boxes, scores

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
