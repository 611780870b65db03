"""Training step of the reference's YOLOv8 detect model on the fp32 parity kernels (SURVEY.md section 8 rows a14-a18).

One `TrainStepV8.step(images, targets)` = `yolo.train()` forward (Conv2d -> BatchNorm2d with batch statistics ->
SiLU, Modules/Convs.cs:36-56) -> `v8DetectionLoss` (Utils/Loss.cs:328-485) -> backward -> `AdamW.step()`
(YoloBaseTaskModel.cs:142-160, Utils/Amp.cs:260-286), i.e. what `AMPWrapper.TrainStep` does in its fp32 branch.
Every arithmetic op is a kernel of libyolob200.so reached through `ops` (conv forward / dgrad / wgrad, BN+SiLU
forward / backward, detection loss + gradient, AdamW); PyTorch only holds the NHWC tensors and does the data movement
of the graph (channel concat / chunk views, nearest 2x upsampling and its sum-reduction backward, the 5x5 max-pool of
SPPF and its index backward - the last two are the remaining library calls on this path).

This is the PARITY path of the training side: correct first (it matches autograd through the oracle restatement
parameter by parameter), CUDA-core fp32 kernels; the tensor-core dgrad / wgrad kernels and a captured train-mode graph
replace it next.  Parameter names are the reference's state_dict keys (`model.{i}.conv.weight`, ...).
"""
import math

import torch
import torch.nn.functional as F

V8_SIZES = {  # Models/Yolo.cs:45-49 (depth_multiple, width_multiple, max_channels)
    "n": (0.34, 0.25, 1024), "s": (0.34, 0.5, 1024), "m": (0.67, 0.75, 576), "l": (1.0, 1.0, 512), "x": (1.0, 1.25, 640),
}


def lr_lambda_linear(epoch, lrf=0.01, epochs=100):
    """LrLambda(1.0, Lrf, Epochs), YoloBaseTaskModel.cs:504-512."""
    return max(1 - epoch / epochs, 0) * (1.0 - lrf) + lrf


def lr_lambda_onecycle(epoch, lrf=0.01, epochs=100):
    """OneCycle(1.0, Lrf, Epochs), YoloBaseTaskModel.cs:492-502 (UseCosLR)."""
    return max((1 - math.cos(epoch * math.pi / epochs)) / 2, 0) * (lrf - 1.0) + 1.0


def interp(x, xp, fp):
    """YoloBaseTaskModel.cs:514-536 (two-point use: clamp outside, linear inside)."""
    if x <= xp[0]:
        return fp[0]
    if x >= xp[-1]:
        return fp[-1]
    for i in range(1, len(xp)):
        if x == xp[i]:
            return fp[i]
        if x < xp[i]:
            t = (x - xp[i - 1]) / (xp[i] - xp[i - 1])
            return fp[i - 1] + t * (fp[i] - fp[i - 1])


def warmup_lrs(ni, nw, initial_lr, lam, warmup_bias_lr=0.1):
    """Per-group learning rates during warm-up (YoloBaseTaskModel.cs:307-319): the FIRST parameter group (names
    containing "bias") ramps from WarmUpBiasLr, the others from 0, to initial_lr * lambda(epoch); None after warm-up."""
    if ni > nw:
        return None
    d = initial_lr * lam
    return interp(ni, [0, nw], [warmup_bias_lr, d]), interp(ni, [0, nw], [0.0, d])


class KernelOps:
    """The C-ABI kernels (no fallback: importing this on a machine without the CUDA library fails loudly)."""

    def __init__(self, tensor_cores=True):
        """tensor_cores: dense convolutions (forward, dgrad, wgrad) on the TF32 tensor-core kernels (csrc/conv_tf32.cu) where
        their shape rule holds (channels % 8, k in {1, 3}); False = the fp32 CUDA-core parity kernels everywhere."""
        from . import engine as E
        self.E = E
        self.tc = bool(tensor_cores)
        self.ws = None

    def _tc_ok(self, x, w, stride, pad):
        Cout, Cin, k, _ = w.shape
        return self.tc and self.E.conv_tc_supported((Cin + 7) // 8 * 8, Cout, k, stride, pad, x.shape[1], x.shape[2])

    @staticmethod
    def _pad8(x, w):
        """The 3-channel stem (Yolo.cs:53): input channels zero-padded to 8 so that it also runs on the tensor cores
        (zero channels contribute exact zeros; the padded gradient columns are dropped)."""
        Cin = w.shape[1]
        cp = (Cin + 7) // 8 * 8
        if cp == Cin:
            return x.contiguous(), w.contiguous(), Cin
        return torch.nn.functional.pad(x, (0, cp - Cin)), torch.nn.functional.pad(w, (0, 0, 0, 0, 0, cp - Cin)), Cin

    def _ws(self, x):
        if self.ws is None:
            self.ws = self.E.ConvWorkspace(x.device)
        return self.ws

    def conv_forward(self, x, w, bias, stride, pad):
        if self.tc and bias is None and self.E.stem_conv_supported(w, stride, pad, x.shape[1], x.shape[2]):
            return self.E.stem_conv_forward(x.contiguous(), w.contiguous())  # the 3-channel stem: fp32 CUDA cores
        if self._tc_ok(x, w, stride, pad):
            xp, wp, _ = self._pad8(x, w)
            return self.E.conv_forward_tc(xp, wp, bias, stride, pad, ws=self._ws(x))
        return self.E.conv_forward(x, w, bias, stride, pad)

    def conv_backward(self, x, dz, w, stride, pad, need_dx=True):
        """-> (dx or None when the caller does not need it (the network input), dw)."""
        if self.tc and not need_dx and self.E.stem_conv_supported(w, stride, pad, x.shape[1], x.shape[2]):
            return None, self.E.stem_conv_backward_weight(x.contiguous(), dz.contiguous(), w.shape, ws=self._ws(x))
        if self._tc_ok(x, w, stride, pad):
            xp, wp, Cin = self._pad8(x, w)
            dx, dw = self.E.conv_backward_tc(xp, dz.contiguous(), wp, stride, pad, ws=self._ws(x), need_dx=need_dx)
            if wp.shape[1] != Cin:
                dw = dw[:, :Cin].contiguous()
                dx = dx[..., :Cin].contiguous() if dx is not None else None
            return dx, dw
        return self.E.conv_backward(x, dz.contiguous(), w, stride, pad)

    def bn_silu_forward(self, z, gamma, beta, rm, rv, act):
        return self.E.bn_silu_train_forward(z, gamma, beta, rm, rv, act=act)

    def bn_silu_backward(self, z, dy, gamma, beta, mean, invstd, act):
        return self.E.bn_silu_backward(z, dy.contiguous(), gamma, beta, mean, invstd, act=act)

    def detection_loss(self, boxes, scores, targets, H, W):
        o = self.E.detection_loss(boxes.contiguous(), scores.contiguous(), targets, H, W)
        return o["items"], o["grad_boxes"], o["grad_scores"]

    def adamw(self, p, g, m, v, step, lr, wd):
        self.E.adamw_step(p, g, m, v, step, lr, weight_decay=wd)


class _Params:
    """Flat parameter / gradient / Adam-moment buffers with named views (one optimizer launch, one all-reduce)."""

    def __init__(self, state_dict, device):
        names = [k for k, v in state_dict.items() if v.dtype.is_floating_point and v.numel() > 0 and
                 not k.endswith(("running_mean", "running_var")) and ".dfl." not in k]
        # the reference's optimizer groups by name substring (YoloBaseTaskModel.cs:144-153): group 0 = "bias", then
        # "weight"; the flat buffers keep each group contiguous so a group is one optimizer launch with its own lr.
        # (BatchNorm parameters also match the third filter "bn"; whether TorchSharp then steps them twice cannot be
        # verified here - they are stepped once.)
        self.names = [k for k in names if "bias" in k] + [k for k in names if "bias" not in k]
        self.n_bias = sum(int(state_dict[k].numel()) for k in names if "bias" in k)
        self.shapes = {k: tuple(state_dict[k].shape) for k in self.names}
        n = sum(int(torch.Size(self.shapes[k]).numel()) for k in self.names)
        self.flat = torch.zeros(n, dtype=torch.float32, device=device)
        self.grad = torch.zeros_like(self.flat)
        self.m = torch.zeros_like(self.flat)
        self.v = torch.zeros_like(self.flat)
        self.off, o = {}, 0
        for k in self.names:
            c = int(torch.Size(self.shapes[k]).numel())
            self.off[k] = (o, c)
            self.flat[o:o + c].copy_(state_dict[k].detach().reshape(-1).to(device=device, dtype=torch.float32))
            o += c
        self.buffers = {k: v.detach().clone().to(device=device, dtype=torch.float32) for k, v in state_dict.items()
                        if k.endswith(("running_mean", "running_var"))}

    def p(self, k):
        o, c = self.off[k]
        return self.flat[o:o + c].view(self.shapes[k])

    def g(self, k):
        o, c = self.off[k]
        return self.grad[o:o + c].view(self.shapes[k])


class _Conv:
    """Conv block: Conv2d(bias=False) -> BatchNorm2d(train) -> SiLU / identity (Convs.cs:36-56)."""

    def __init__(self, net, name, k=1, s=1, act=True):
        self.net, self.name, self.k, self.s, self.act = net, name, k, s, act
        self.need_dx = True  # False for the first layer: nothing consumes the gradient of the images

    def forward(self, x):
        P, ops = self.net.P, self.net.ops
        self.x = x
        self.z = ops.conv_forward(x, P.p(self.name + ".conv.weight"), None, self.s, self.k // 2)
        y, self.mean, self.invstd = ops.bn_silu_forward(self.z, P.p(self.name + ".bn.weight"), P.p(self.name + ".bn.bias"),
                                                        P.buffers[self.name + ".bn.running_mean"],
                                                        P.buffers[self.name + ".bn.running_var"], self.act)
        return y

    def backward(self, dy):
        P, ops = self.net.P, self.net.ops
        dz, dg, db = ops.bn_silu_backward(self.z, dy, P.p(self.name + ".bn.weight"), P.p(self.name + ".bn.bias"), self.mean,
                                          self.invstd, self.act)
        dx, dw = ops.conv_backward(self.x, dz, P.p(self.name + ".conv.weight"), self.s, self.k // 2, need_dx=self.need_dx)
        P.g(self.name + ".conv.weight").copy_(dw)
        P.g(self.name + ".bn.weight").copy_(dg)
        P.g(self.name + ".bn.bias").copy_(db)
        return dx


class _Conv2dBias:
    """Plain Conv2d(k=1, bias=True): the last layer of every Detect branch (Head.cs:41-52)."""

    def __init__(self, net, name):
        self.net, self.name = net, name

    def forward(self, x):
        self.x = x
        return self.net.ops.conv_forward(x, self.net.P.p(self.name + ".weight"), self.net.P.p(self.name + ".bias"), 1, 0)

    def backward(self, dz):
        dx, dw = self.net.ops.conv_backward(self.x, dz, self.net.P.p(self.name + ".weight"), 1, 0)
        self.net.P.g(self.name + ".weight").copy_(dw)
        self.net.P.g(self.name + ".bias").copy_(dz.sum((0, 1, 2)))
        return dx


class _Bottleneck:
    """Block.cs:572-607, k = (3, 3), e = 1.0 inside C2f."""

    def __init__(self, net, name, shortcut):
        self.cv1, self.cv2, self.add = _Conv(net, name + ".cv1", 3), _Conv(net, name + ".cv2", 3), shortcut

    def forward(self, x):
        y = self.cv2.forward(self.cv1.forward(x))
        return x + y if self.add else y

    def backward(self, dy):
        dx = self.cv1.backward(self.cv2.backward(dy))
        return dx + dy if self.add else dx


class _C2f:
    """Block.cs:371-398."""

    def __init__(self, net, name, c2, n, shortcut):
        self.c = c2 // 2
        self.cv1, self.cv2 = _Conv(net, name + ".cv1", 1), _Conv(net, name + ".cv2", 1)
        self.m = [_Bottleneck(net, f"{name}.m.{i}", shortcut) for i in range(n)]

    def forward(self, x):
        y = self.cv1.forward(x)
        ys = [y[..., :self.c], y[..., self.c:]]
        for m in self.m:
            ys.append(m.forward(ys[-1].contiguous()))
        return self.cv2.forward(torch.cat(ys, -1))

    def backward(self, dy):
        d = list(self.cv2.backward(dy).split(self.c, -1))
        for i in range(len(self.m) - 1, -1, -1):
            d[i + 1] = d[i + 1] + self.m[i].backward(d[i + 2].contiguous())
        return self.cv1.backward(torch.cat((d[0], d[1]), -1))


def _pool(x):  # MaxPool2d(5, 1, 2) on NHWC (library call, see module docstring)
    y, idx = F.max_pool2d(x.permute(0, 3, 1, 2), 5, 1, 2, return_indices=True)
    return y.permute(0, 2, 3, 1).contiguous(), idx


def _pool_backward(dy, x, idx):
    d = torch.ops.aten.max_pool2d_with_indices_backward(dy.permute(0, 3, 1, 2).contiguous(), x.permute(0, 3, 1, 2).contiguous(),
                                                       [5, 5], [1, 1], [2, 2], [1, 1], False, idx)
    return d.permute(0, 2, 3, 1)


class _SPPF:
    """Block.cs:236-282: cv1 has NO activation in the reference (:257)."""

    def __init__(self, net, name):
        self.cv1, self.cv2 = _Conv(net, name + ".cv1", 1, act=False), _Conv(net, name + ".cv2", 1)

    def forward(self, x):
        self.t = [self.cv1.forward(x)]
        self.idx = []
        for _ in range(3):
            y, i = _pool(self.t[-1])
            self.t.append(y)
            self.idx.append(i)
        return self.cv2.forward(torch.cat(self.t, -1))

    def backward(self, dy):
        c = self.t[0].shape[-1]
        d = list(self.cv2.backward(dy).split(c, -1))
        for i in (2, 1, 0):
            d[i] = d[i] + _pool_backward(d[i + 1], self.t[i], self.idx[i])
        return self.cv1.backward(d[0].contiguous())


class _Detect:
    """Detect.forward_head (Head.cs:35-53, 71-87), legacy (v8) class branch."""

    def __init__(self, net, name, nc, ch, reg_max=16):
        self.nc, self.reg_max = nc, reg_max
        self.cv2 = [[_Conv(net, f"{name}.cv2.{i}.0", 3), _Conv(net, f"{name}.cv2.{i}.1", 3), _Conv2dBias(net, f"{name}.cv2.{i}.2")]
                    for i in range(len(ch))]
        self.cv3 = [[_Conv(net, f"{name}.cv3.{i}.0", 3), _Conv(net, f"{name}.cv3.{i}.1", 3), _Conv2dBias(net, f"{name}.cv3.{i}.2")]
                    for i in range(len(ch))]

    @staticmethod
    def _seq(layers, x):
        for layer in layers:
            x = layer.forward(x)
        return x

    def forward(self, feats):
        self.shapes = [f.shape for f in feats]
        b = [self._seq(self.cv2[i], f) for i, f in enumerate(feats)]
        s = [self._seq(self.cv3[i], f) for i, f in enumerate(feats)]
        B = feats[0].shape[0]
        boxes = torch.cat([t.permute(0, 3, 1, 2).reshape(B, 4 * self.reg_max, -1) for t in b], -1)
        scores = torch.cat([t.permute(0, 3, 1, 2).reshape(B, self.nc, -1) for t in s], -1)
        return boxes, scores

    def backward(self, gboxes, gscores):
        out, a0 = [], 0
        for i, shp in enumerate(self.shapes):
            B, h, w, _ = shp
            gb = gboxes[:, :, a0:a0 + h * w].reshape(B, 4 * self.reg_max, h, w).permute(0, 2, 3, 1).contiguous()
            gs = gscores[:, :, a0:a0 + h * w].reshape(B, self.nc, h, w).permute(0, 2, 3, 1).contiguous()
            a0 += h * w
            d = None
            for layers, g in ((self.cv2[i], gb), (self.cv3[i], gs)):
                for layer in reversed(layers):
                    g = layer.backward(g)
                d = g if d is None else d + g
            out.append(d)
        return out


class TrainStepV8:
    """YOLOv8 detect training step.  `state_dict`: the reference's names -> tensors (as loaded from a .bin)."""

    def __init__(self, state_dict, size="n", nc=80, device="cuda", ops=None, lr=None, weight_decay=5e-4):
        self.ops = ops if ops is not None else KernelOps()
        self.P = _Params(state_dict, device)
        d, wm, mc = V8_SIZES[size]
        w = [min(int(x * wm), mc) for x in (64, 128, 256, 512, 1024)]
        dp = [int(x * d) for x in (3, 6, 9)]
        self.nc, self.step_count = nc, 0
        self.group = None  # process group of the gradient all-reduce (None = default group, False = never reduce)
        self.lr = lr if lr is not None else round(0.002 * 5 / (4 + nc), 6)  # YoloBaseTaskModel.cs:142
        self.wd = weight_decay
        N = self
        self.layers = [  # Yolo.cs:53-89
            _Conv(N, "model.0", 3, 2), _Conv(N, "model.1", 3, 2), _C2f(N, "model.2", w[1], dp[0], True),
            _Conv(N, "model.3", 3, 2), _C2f(N, "model.4", w[2], dp[1], True), _Conv(N, "model.5", 3, 2),
            _C2f(N, "model.6", w[3], dp[1], True), _Conv(N, "model.7", 3, 2), _C2f(N, "model.8", w[4], dp[0], True),
            _SPPF(N, "model.9"), "up", "cat", _C2f(N, "model.12", w[3], dp[0], False), "up", "cat",
            _C2f(N, "model.15", w[2], dp[0], False), _Conv(N, "model.16", 3, 2), "cat", _C2f(N, "model.18", w[3], dp[0], False),
            _Conv(N, "model.19", 3, 2), "cat", _C2f(N, "model.21", w[4], dp[0], False),
        ]
        self.layers[0].need_dx = False
        self.detect = _Detect(N, "model.22", nc, (w[2], w[3], w[4]))
        self.output_indexs = (4, 6, 9, 12, 15, 18, 21)  # Yolo.cs:13
        self.concat_index = (1, 0, 3, 2)                 # Yolo.cs:14

    # ---- forward / backward of the graph wiring (Yolo.cs:92-134) ----
    def forward(self, images_nchw):
        x = images_nchw.permute(0, 2, 3, 1).contiguous()
        outputs, cat_count, self.cat_split = [], 0, []
        for i, m in enumerate(self.layers):
            if m == "up":
                x = x.repeat_interleave(2, 1).repeat_interleave(2, 2)
            elif m == "cat":
                other = outputs[self.concat_index[cat_count]]
                self.cat_split.append((x.shape[-1], self.concat_index[cat_count]))
                x = torch.cat((x, other), -1)
                cat_count += 1
            else:
                x = m.forward(x.contiguous())
            if i in self.output_indexs:
                outputs.append(x)
        self.n_out = len(outputs)
        return self.detect.forward([outputs[-3], outputs[-2], outputs[-1]])

    def backward(self, gboxes, gscores):
        dfeat = self.detect.backward(gboxes, gscores)
        dout = [None] * self.n_out  # gradient arriving at each saved output from its later consumers
        for k, d in zip((-3, -2, -1), dfeat):
            dout[self.n_out + k] = d
        out_pos = {idx: j for j, idx in enumerate(self.output_indexs)}
        cat_count = len(self.cat_split)
        dx = None
        for i in range(len(self.layers) - 1, -1, -1):
            if i in out_pos and dout[out_pos[i]] is not None:
                dx = dout[out_pos[i]] if dx is None else dx + dout[out_pos[i]]
            m = self.layers[i]
            if m == "up":
                B, H, W, C = dx.shape
                dx = dx.reshape(B, H // 2, 2, W // 2, 2, C).sum((2, 4))
            elif m == "cat":
                cat_count -= 1
                cx, src = self.cat_split[cat_count]
                d_other = dx[..., cx:]
                dout[src] = d_other if dout[src] is None else dout[src] + d_other
                dx = dx[..., :cx]
            else:
                dx = m.backward(dx.contiguous())
        return dx

    def state_dict(self, dtype=torch.float32):
        """Reference-named tensors of the trained model (what `yolo.state_dict()` holds, YoloBaseTaskModel.cs:470-490):
        parameters, BatchNorm running statistics, `num_batches_tracked` (= steps taken, int64), the fp32 DFL weight
        arange(16) (Block.cs:29-30; it never receives a gradient) and the head's empty `anchors` / `strides` buffers."""
        out = {}
        bn = sorted({k[:-len(".running_mean")] for k in self.P.buffers if k.endswith(".running_mean")})
        for k in self.P.names:
            out[k] = self.P.p(k).detach().to(dtype).cpu()
        for b in bn:
            out[b + ".running_mean"] = self.P.buffers[b + ".running_mean"].detach().to(dtype).cpu()
            out[b + ".running_var"] = self.P.buffers[b + ".running_var"].detach().to(dtype).cpu()
            out[b + ".num_batches_tracked"] = torch.tensor(self.step_count, dtype=torch.int64)
        head = next(k for k in self.P.names if ".cv2.0.0." in k).split(".cv2.")[0]
        out[head + ".dfl.conv.weight"] = torch.arange(16, dtype=torch.float32).view(1, 16, 1, 1)
        out[head + ".anchors"] = torch.empty(0, dtype=dtype)
        out[head + ".strides"] = torch.empty(0, dtype=dtype)
        return out

    def save(self, path, dtype=torch.float32):
        """SaveWeight (YoloBaseTaskModel.cs:470-490): the reference's `.bin` through the library's native writer."""
        from .engine import write_checkpoint_bin
        write_checkpoint_bin(path, self.state_dict(dtype))

    def step(self, images_nchw, targets, lrs=None):
        """images (B,3,H,W) float32 in [0,1] on the device; targets (n,6) rows [image, cls, x, y, w, h];
        lrs = (lr of the "bias" group, lr of the other parameters) for this iteration (warm-up / schedule), default
        the constant initial lr.  -> loss items (3,) (= the reference's `loss.detach()`)."""
        B, _, H, W = images_nchw.shape
        boxes, scores = self.forward(images_nchw)
        items, gb, gs = self.ops.detection_loss(boxes, scores, targets, H, W)
        self.P.grad.zero_()
        self.backward(gb, gs)
        # data-parallel: ONE all-reduce of the flat gradient buffer (NCCL on GPUs, gloo in the CPU tests); ranks are
        # summed, not averaged - the reference scales the loss by the local batch size (Loss.cs:473).  BatchNorm
        # statistics stay per rank, as in the reference (no SyncBN).
        if self.group is not False and torch.distributed.is_available() and torch.distributed.is_initialized() and \
                torch.distributed.get_world_size(self.group) > 1:
            torch.distributed.all_reduce(self.P.grad, group=self.group)
        self.step_count += 1
        lr_bias, lr_other = lrs if lrs is not None else (self.lr, self.lr)
        nb = self.P.n_bias
        for lo, hi, lr in ((0, nb, lr_bias), (nb, self.P.flat.numel(), lr_other)):
            if hi > lo:
                self.ops.adamw(self.P.flat[lo:hi], self.P.grad[lo:hi], self.P.m[lo:hi], self.P.v[lo:hi], self.step_count, lr, self.wd)
        return items


class EarlyStopping:
    """Utils/EarlyStopping.cs:3-40, restated.  `fitness` is whatever Train() feeds it: -sum(validation loss items)
    (YoloBaseTaskModel.cs:186), i.e. negative - the first epoch always becomes the best one because best_fitness starts at 0
    and `best_fitness == 0` counts as "no best yet" (:21)."""

    def __init__(self, patience=50):
        self.best_fitness, self.best_epoch, self.patience, self.possible_stop = 0.0, 0, float(patience), False

    def ShouldStop(self, fitness, epoch):
        if fitness > self.best_fitness or self.best_fitness == 0:
            self.best_epoch, self.best_fitness = epoch, fitness
        delta = epoch - self.best_epoch
        self.possible_stop = delta >= (self.patience - 1)
        return delta >= self.patience


def fit(step, batches, epochs, lrf=0.01, warmup_epochs=3, warmup_bias_lr=0.1, cos_lr=False, on_iteration=None, group=None,
        validate=None, patience=50, on_best=None, on_epoch_end=None):
    """The reference's epoch loop around the training step, restated index for index
    (YoloBaseTaskModel.cs:167-170 Train, :291-356 TrainEpoch):
      * epochs run 1 .. Epochs; inside an epoch `i` counts the EXECUTED batches only (the `continue` of a target-less
        batch skips the `i++`, :321-324 / :353), ni = i + nb * epoch - so warm-up starts at ni = nb, not 0;
      * while ni <= nw = max(WarmUpEpoches * nb, 100) both parameter groups are set to
        interp(ni, [0, nw], [WarmUpBiasLr | 0, InitialLR * lambda(epoch)]) (:307-319);
      * LambdaLR is stepped once AFTER each epoch (:182): past warm-up the rate during epoch e is
        InitialLR * lambda(e - 1); when warm-up ends in the middle of an epoch the groups keep the last interpolated
        value until that step (the reference never resets them).
    Data parallelism (net-new, the reference is single-device): `step.step` all-reduces gradients, so a rank must not
    skip it alone - a batch is skipped only when EVERY rank of `group` has no targets (one all-reduce of a flag per
    iteration); a rank with an empty shard calls step() with zero targets (the loss kernels handle n_targets = 0).
    `batches` is a re-iterable of (images (B,3,H,W) float32 on the device, targets (n,6)) - data loading and
    augmentation are outside this library.  Returns the per-epoch mean of the loss items.
    The tail of the reference's epoch (YoloBaseTaskModel.cs:184-207) is available through callbacks: `validate(epoch)` ->
    validation loss items; fitness = -sum(items) (:186); `on_best(epoch)` when it beats the best so far (best.bin, :188-194,
    best_fitness starts at float.MinValue, :118); EarlyStopping(patience).ShouldStop(fitness, epoch) ends the run BEFORE
    `on_epoch_end(epoch)` (last.bin, :205) of that epoch, as the reference's `break` does (:198-203)."""
    lam = lr_lambda_onecycle if cos_lr else lr_lambda_linear
    nb = len(batches)
    nw = max(warmup_epochs * nb, 100)
    dp = group is not False and torch.distributed.is_available() and torch.distributed.is_initialized() and \
        torch.distributed.get_world_size(group) > 1
    history = []
    stopper, best_fitness = EarlyStopping(patience), float("-inf")
    lrs = (step.lr * lam(0, lrf, epochs),) * 2  # LambdaLR construction: InitialLR * lambda(0)
    for epoch in range(1, epochs + 1):
        total, count, i = None, 0, 0
        for images, targets in batches:
            ni = i + nb * epoch
            w = warmup_lrs(ni, nw, step.lr, lam(epoch, lrf, epochs), warmup_bias_lr)
            if w is not None:
                lrs = w
            has = len(targets) >= 1
            if dp:
                flag = torch.tensor([1.0 if has else 0.0],
                                    device=step.P.grad.device if hasattr(step, "P") else getattr(step, "device", "cpu"))
                torch.distributed.all_reduce(flag, op=torch.distributed.ReduceOp.MAX, group=group)
                has = bool(flag.item() > 0)
            if not has:
                continue
            items = step.step(images, targets, lrs=lrs)
            if on_iteration is not None:
                on_iteration(epoch, i, lrs, items)
            total = items.detach().clone() if total is None else total + items.detach()
            count += 1
            i += 1
        lrs = (step.lr * lam(epoch, lrf, epochs),) * 2  # lr_scheduler.step() after the epoch
        history.append(total / max(count, 1) if total is not None else None)
        if validate is not None:
            fitness = -float(sum(float(v) for v in validate(epoch)))
            if dp:  # every rank validated its own shard: the decision to stop (and what counts as best) must be collective
                f = torch.tensor([fitness], dtype=torch.float64,
                                 device=step.P.grad.device if hasattr(step, "P") else getattr(step, "device", "cpu"))
                torch.distributed.all_reduce(f, group=group)
                fitness = float(f.item())
            if fitness > best_fitness:
                best_fitness = fitness
                if on_best is not None:
                    on_best(epoch)
            if stopper.ShouldStop(fitness, epoch):
                break
        if on_epoch_end is not None:
            on_epoch_end(epoch)
    return history
