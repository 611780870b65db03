"""Graph logic of the YOLOv11 detect training step (BASELINE configs[3]: YOLOv11s), on the same `ops` interface as
`train.py`: the wiring, the forward/backward of C3k2 / C3k / C2PSA / PSABlock / Attention and the v11 Detect head,
pinned against autograd through the oracle on the CPU (PyTorch stand-in of the kernel interface) and on the GPU with
the library's kernels (tests/test_train_step.py): csrc/train_v11.cu adds the depthwise 3x3 convolution (forward,
dgrad, wgrad) and csrc/attention.cu the attention core softmax(q^T k) v with its backward to the fp32 parity kernels
of the v8 step.

Reference: Models/Yolo.cs:200-258 (Yolov11 wiring, outputIndexs {4,6,10,13,16,19,22}), Modules/Block.cs:404-441 (C3),
:611-661 (C3k, C3k2), :664-810 (C2PSA, PSABlock, Attention), Modules/Convs.cs:108-114 (DWConv), Modules/Head.cs:35-53
(non-legacy class branch).  Quirks kept: Attention's qkv / proj / pe convs and ffn[1] keep the SiLU (Block.cs:708,
744-746).
"""
import math

import torch

from .train import KernelOps, TrainStepV8, _C2f, _Conv, _Conv2dBias, _Params, _SPPF  # noqa: F401

V11_SIZES = {  # Models/Yolo.cs:213-217 (depth, width, max_channels, c3k)
    "n": (0.5, 0.25, 1024, False), "s": (0.5, 0.5, 1024, False), "m": (0.5, 1.0, 512, True),
    "l": (1.0, 1.0, 512, True), "x": (1.0, 1.5, 768, True),
}


class KernelOpsV11(KernelOps):
    """+ the depthwise 3x3 (csrc/train_v11.cu) and attention (csrc/attention.cu) kernels.  Every grouped conv of Yolov11 is depthwise
    3x3 stride 1 (DWConv(c, c, 3) in the head, Attention.pe); anything else is refused, not emulated."""

    @staticmethod
    def _check_dw(x, w, stride, pad, groups):
        if not (groups == x.shape[-1] == w.shape[0] and w.shape[1] == 1 and tuple(w.shape[2:]) == (3, 3) and stride == 1 and pad == 1):
            raise NotImplementedError("only depthwise 3x3 stride-1 grouped convolutions have training kernels")

    def gconv_forward(self, x, w, stride, pad, groups):
        self._check_dw(x, w, stride, pad, groups)
        return self.E.dwconv3x3_forward(x.contiguous(), w.contiguous())

    def gconv_backward(self, x, dz, w, stride, pad, groups):
        self._check_dw(x, w, stride, pad, groups)
        return self.E.dwconv3x3_backward(x.contiguous(), dz.contiguous(), w.contiguous())

    def attention_forward(self, q, k, v, scale):
        return self.E.attention_forward(q.contiguous(), k.contiguous(), v.contiguous(), scale)

    def attention_backward(self, q, k, v, scale, dout):
        return self.E.attention_backward(q.contiguous(), k.contiguous(), v.contiguous(), scale, dout.contiguous())


class _GConv(_Conv):
    """Conv block with groups (DWConv: g = gcd(c1, c2), Convs.cs:108-114; Attention.pe: g = dim)."""

    def __init__(self, net, name, k, s, groups, act=True):
        super().__init__(net, name, k, s, act)
        self.groups = groups

    def forward(self, x):
        P, ops = self.net.P, self.net.ops
        self.x = x
        self.z = ops.gconv_forward(x, P.p(self.name + ".conv.weight"), self.s, self.k // 2, self.groups)
        y, self.mean, self.invstd = ops.bn_silu_forward(self.z, P.p(self.name + ".bn.weight"), P.p(self.name + ".bn.bias"),
                                                        P.buffers[self.name + ".bn.running_mean"],
                                                        P.buffers[self.name + ".bn.running_var"], self.act)
        return y

    def backward(self, dy):
        P, ops = self.net.P, self.net.ops
        dz, dg, db = ops.bn_silu_backward(self.z, dy, P.p(self.name + ".bn.weight"), P.p(self.name + ".bn.bias"), self.mean,
                                          self.invstd, self.act)
        dx, dw = ops.gconv_backward(self.x, dz, P.p(self.name + ".conv.weight"), self.s, self.k // 2, self.groups)
        P.g(self.name + ".conv.weight").copy_(dw)
        P.g(self.name + ".bn.weight").copy_(dg)
        P.g(self.name + ".bn.bias").copy_(db)
        return dx


class _BottleneckE:
    """Bottleneck(c1, c2, shortcut, k=(3,3), e): Block.cs:572-607."""

    def __init__(self, net, name, shortcut):
        self.cv1, self.cv2, self.add = _Conv(net, name + ".cv1", 3), _Conv(net, name + ".cv2", 3), shortcut

    def forward(self, x):
        y = self.cv2.forward(self.cv1.forward(x))
        return x + y if self.add else y

    def backward(self, dy):
        dx = self.cv1.backward(self.cv2.backward(dy.contiguous()))
        return dx + dy if self.add else dx


class _C3k:
    """C3k(c, c, n=2, shortcut): cv3(cat(m(cv1 x), cv2 x)), Block.cs:404-441, 611-620."""

    def __init__(self, net, name, n, shortcut):
        self.cv1, self.cv2, self.cv3 = _Conv(net, name + ".cv1", 1), _Conv(net, name + ".cv2", 1), _Conv(net, name + ".cv3", 1)
        self.m = [_BottleneckE(net, f"{name}.m.{i}", shortcut) for i in range(n)]

    def forward(self, x):
        a = self.cv1.forward(x)
        for m in self.m:
            a = m.forward(a)
        b = self.cv2.forward(x)
        self.ca = a.shape[-1]
        return self.cv3.forward(torch.cat((a, b), -1))

    def backward(self, dy):
        d = self.cv3.backward(dy)
        da, db = d[..., :self.ca].contiguous(), d[..., self.ca:].contiguous()
        for m in reversed(self.m):
            da = m.backward(da)
        return self.cv1.backward(da.contiguous()) + self.cv2.backward(db)


class _C3k2:
    """Block.cs:623-661."""

    def __init__(self, net, name, c2, n, c3k, e=0.5, shortcut=True):
        self.c = int(c2 * e)
        self.cv1, self.cv2 = _Conv(net, name + ".cv1", 1), _Conv(net, name + ".cv2", 1)
        self.m = [(_C3k(net, f"{name}.m.{i}", 2, shortcut) if c3k else _BottleneckE(net, f"{name}.m.{i}", shortcut)) for i in range(n)]

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


class _Attention:
    """Block.cs:752-809.  NHWC: qkv (B, H, W, nh*(2kd+hd)) viewed per head as [q (kd) | k (kd) | v (hd)]."""

    def __init__(self, net, name, dim, num_heads):
        self.nh, self.hd = num_heads, dim // num_heads
        self.kd = int(self.hd * 0.5)
        self.scale = float(self.kd ** -0.5)
        self.qkv, self.proj = _Conv(net, name + ".qkv", 1), _Conv(net, name + ".proj", 1)
        self.pe = _GConv(net, name + ".pe", 3, 1, dim)
        self.net = net

    def forward(self, x):
        B, H, W, C = x.shape
        self.shape = (B, H, W, C)
        qkv = self.qkv.forward(x).view(B, H * W, self.nh, 2 * self.kd + self.hd)
        q, k, v = qkv.split([self.kd, self.kd, self.hd], -1)  # (B, N, nh, .)
        self.q, self.k, self.v = q.contiguous(), k.contiguous(), v.contiguous()
        o = self.net.ops.attention_forward(self.q, self.k, self.v, self.scale)  # (B, N, nh, hd)
        y = o.reshape(B, H, W, C) + self.pe.forward(self.v.reshape(B, H, W, C))
        return self.proj.forward(y.contiguous())

    def backward(self, dy):
        B, H, W, C = self.shape
        d = self.proj.backward(dy)
        dv_pe = self.pe.backward(d.contiguous()).reshape(B, H * W, self.nh, self.hd)
        dq, dk, dv = self.net.ops.attention_backward(self.q, self.k, self.v, self.scale, d.reshape(B, H * W, self.nh, self.hd).contiguous())
        dqkv = torch.cat((dq, dk, dv + dv_pe), -1).reshape(B, H, W, -1)
        return self.qkv.backward(dqkv.contiguous())


class _PSABlock:
    """Block.cs:697-722 (shortcut = True)."""

    def __init__(self, net, name, c):
        self.attn = _Attention(net, name + ".attn", c, c // 64)
        self.ffn = [_Conv(net, name + ".ffn.0", 1), _Conv(net, name + ".ffn.1", 1)]

    def forward(self, x):
        x = x + self.attn.forward(x)
        return x + self.ffn[1].forward(self.ffn[0].forward(x.contiguous()))

    def backward(self, dy):
        d = dy + self.ffn[0].backward(self.ffn[1].backward(dy.contiguous()))
        return d + self.attn.backward(d.contiguous())


class _C2PSA:
    """Block.cs:664-695."""

    def __init__(self, net, name, c1, n):
        self.c = int(c1 * 0.5)
        self.cv1, self.cv2 = _Conv(net, name + ".cv1", 1), _Conv(net, name + ".cv2", 1)
        self.m = [_PSABlock(net, f"{name}.m.{i}", self.c) for i in range(n)]

    def forward(self, x):
        y = self.cv1.forward(x)
        a, b = y[..., :self.c], y[..., self.c:].contiguous()
        for m in self.m:
            b = m.forward(b)
        return self.cv2.forward(torch.cat((a, b), -1))

    def backward(self, dy):
        d = self.cv2.backward(dy)
        da, db = d[..., :self.c], d[..., self.c:].contiguous()
        for m in reversed(self.m):
            db = m.backward(db)
        return self.cv1.backward(torch.cat((da, db), -1))


class _Seq:
    def __init__(self, layers):
        self.layers = layers

    def forward(self, x):
        for layer in self.layers:
            x = layer.forward(x)
        return x

    def backward(self, d):
        for layer in reversed(self.layers):
            d = layer.backward(d.contiguous())
        return d


class _DetectV11:
    """Detect with the non-legacy class branch (Head.cs:35-53): cv3[i] = Seq(Seq(DWConv(x,x,3), Conv(x,c3,1)),
    Seq(DWConv(c3,c3,3), Conv(c3,c3,1)), Conv2d(c3,nc,1))."""

    def __init__(self, net, name, nc, ch, reg_max=16):
        self.nc, self.reg_max = nc, reg_max
        c3 = max(ch[0], min(nc, 100))
        self.cv2 = [_Seq([_Conv(net, f"{name}.cv2.{i}.0", 3), _Conv(net, f"{name}.cv2.{i}.1", 3), _Conv2dBias(net, f"{name}.cv2.{i}.2")])
                    for i in range(len(ch))]
        self.cv3 = [_Seq([_GConv(net, f"{name}.cv3.{i}.0.0", 3, 1, x), _Conv(net, f"{name}.cv3.{i}.0.1", 1),
                          _GConv(net, f"{name}.cv3.{i}.1.0", 3, 1, c3), _Conv(net, f"{name}.cv3.{i}.1.1", 1),
                          _Conv2dBias(net, f"{name}.cv3.{i}.2")]) for i, x in enumerate(ch)]

    def forward(self, feats):
        self.shapes = [f.shape for f in feats]
        B = feats[0].shape[0]
        b = [self.cv2[i].forward(f) for i, f in enumerate(feats)]
        s = [self.cv3[i].forward(f) for i, f in enumerate(feats)]
        boxes = torch.cat([t.permute(0, 3, 1, 2).reshape(B, 4 * self.reg_max, -1) for t in b], -1)
        scores = torch.cat([t.permute(0, 3, 1, 2).reshape(B, self.nc, -1) for t in s], -1)
        return boxes, scores

    def backward(self, gboxes, gscores):
        out, a0 = [], 0
        for i, (B, h, w, _) in enumerate(self.shapes):
            gb = gboxes[:, :, a0:a0 + h * w].reshape(B, 4 * self.reg_max, h, w).permute(0, 2, 3, 1).contiguous()
            gs = gscores[:, :, a0:a0 + h * w].reshape(B, self.nc, h, w).permute(0, 2, 3, 1).contiguous()
            a0 += h * w
            out.append(self.cv2[i].backward(gb) + self.cv3[i].backward(gs))
        return out


class TrainStepV11(TrainStepV8):
    """YOLOv11 detect training step (wiring: Yolo.cs:209-257)."""

    def __init__(self, state_dict, size="s", nc=80, device="cuda", ops=None, lr=None, weight_decay=5e-4):
        self.ops = ops if ops is not None else KernelOpsV11()
        self.P = _Params(state_dict, device)
        d, wm, mc, c3k = V11_SIZES[size]
        w = [min(int(x * wm), mc) for x in (64, 128, 256, 512, 1024)]
        n = int(2 * d)
        self.nc, self.step_count = nc, 0
        self.group = None
        self.lr = lr if lr is not None else round(0.002 * 5 / (4 + nc), 6)
        self.wd = weight_decay
        N = self
        self.layers = [
            _Conv(N, "model.0", 3, 2), _Conv(N, "model.1", 3, 2), _C3k2(N, "model.2", w[2], n, c3k, 0.25),
            _Conv(N, "model.3", 3, 2), _C3k2(N, "model.4", w[3], n, c3k, 0.25), _Conv(N, "model.5", 3, 2),
            _C3k2(N, "model.6", w[3], n, True), _Conv(N, "model.7", 3, 2), _C3k2(N, "model.8", w[4], n, True),
            _SPPF(N, "model.9"), _C2PSA(N, "model.10", w[4], n), "up", "cat", _C3k2(N, "model.13", w[3], n, c3k), "up", "cat",
            _C3k2(N, "model.16", w[2], n, c3k), _Conv(N, "model.17", 3, 2), "cat", _C3k2(N, "model.19", w[3], n, c3k),
            _Conv(N, "model.20", 3, 2), "cat", _C3k2(N, "model.22", w[4], n, True),
        ]
        self.layers[0].need_dx = False
        self.detect = _DetectV11(N, "model.23", nc, (w[2], w[3], w[4]))
        self.output_indexs = (4, 6, 10, 13, 16, 19, 22)  # Yolo.cs:202
        self.concat_index = (1, 0, 3, 2)


assert math  # (kept for symmetry with train.py's helpers)
