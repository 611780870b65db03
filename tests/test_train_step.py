"""Whole training step of YOLOv8n (yolosharp_b200/train.py) against autograd through the oracle model + oracle loss
+ torch.optim.AdamW.  On CPU the step runs on a PyTorch stand-in of the kernel interface (tests/torch_train_ops.py):
this pins the graph logic; the -m gpu test runs the same comparison with the real kernels."""
import numpy as np
import pytest
import torch

from oracle import loss as oloss
from tests.util import oracle_model, synth_image


def _targets(B, seed=0):
    g = torch.Generator().manual_seed(seed)
    n = 7
    bidx = torch.randint(0, B, (n,), generator=g).sort().values.float()
    cls = torch.randint(0, 80, (n,), generator=g).float()
    xy = torch.rand(n, 2, generator=g) * 0.6 + 0.2
    wh = torch.rand(n, 2, generator=g) * 0.4 + 0.05
    return torch.cat((bidx.view(-1, 1), cls.view(-1, 1), xy, wh), 1)


def _reference_step(m, x, targets, lr, wd):
    """oracle: train-mode forward, v8DetectionLoss, backward, AdamW on every trained parameter."""
    m.train()
    params = [(k, p) for k, p in m.named_parameters() if ".dfl." not in k]
    opt = torch.optim.AdamW([p for _, p in params], lr=lr, weight_decay=wd)
    _, preds = m(x)
    crit = oloss.V8DetectionLoss(80)
    batch = {"batch_idx": targets[:, 0], "cls": targets[:, 1], "bboxes": targets[:, 2:]}
    loss, items = crit(preds, batch)
    opt.zero_grad()
    loss.sum().backward()
    grads = {k: p.grad.detach().clone() for k, p in params}
    opt.step()
    return items, grads


def _compare(step_cls, ops, device, tol, arch="v8"):
    torch.manual_seed(0)
    m = oracle_model(arch, "detect", "n")
    sd0 = {k: v.detach().clone() for k, v in m.state_dict().items()}
    B, H, W = 2, 64, 96
    if arch == "v11":
        H, W = 64, 64
    x = synth_image(B, H, W)
    targets = _targets(B)
    lr, wd = 1e-3, 5e-4
    items_ref, grads_ref = _reference_step(m, x, targets, lr, wd)
    ts = step_cls(sd0, "n", 80, device=device, ops=ops, lr=lr, weight_decay=wd)
    items = ts.step(x.to(device), targets)
    np.testing.assert_allclose(items.detach().cpu().numpy(), items_ref.numpy(), rtol=tol, atol=1e-5)
    worst = ("", 0.0)
    gmax = max(float(g.abs().max()) for g in grads_ref.values())
    for k, g in grads_ref.items():
        got = ts.P.g(k).detach().cpu()
        # gradients that are mathematically ~0 (e.g. the BN bias of SPPF.cv1: the BatchNorm of cv2 cancels a per-channel
        # shift of its input, only the max-pool paths leak) are rounding noise on both sides: compare them absolutely
        scale = max(float(g.abs().max()), 1e-4 * gmax)
        err = float((got - g).abs().max()) / scale
        worst = max(worst, (k, err), key=lambda t: t[1])
    print(f"worst parameter gradient: {worst[0]} {worst[1]:.3e} of its tensor's largest entry")
    assert worst[1] < tol * 20, worst
    new = m.state_dict()
    # Adam's first step moves every weight by lr * g / (|g| + eps'): where the gradient is rounding noise its SIGN is
    # noise too, so a handful of weights may differ by up to 2 * lr; everything else must agree closely
    for k in grads_ref:
        d = (ts.P.p(k).detach().cpu() - new[k].detach()).abs()
        bad = d > (tol + tol * 10 * new[k].detach().abs())
        # single entries whose gradient is ~0 relative to their own tensor flip sign the same way (e.g. one BatchNorm bias of
        # a 64-channel layer): they do not count as disagreement of the step
        bad &= grads_ref[k].abs() >= 1e-3 * grads_ref[k].abs().max()
        noise_only = float(grads_ref[k].abs().max()) < 1e-4 * gmax  # the whole gradient is rounding noise (see above)
        assert float(d.max()) <= 2.1 * lr and (noise_only or float(bad.float().mean()) < 2e-3), (k, float(d.max()), int(bad.sum()))
    for k, v in ts.P.buffers.items():  # BatchNorm running statistics after one train-mode forward
        np.testing.assert_allclose(v.cpu().numpy(), new[k].numpy(), rtol=1e-3, atol=1e-4)
    assert len(grads_ref) == len(ts.P.names)


def test_train_step_graph_logic_cpu():
    from tests.torch_train_ops import TorchOps
    from yolosharp_b200.train import TrainStepV8
    _compare(TrainStepV8, TorchOps(), "cpu", 2e-4)


@pytest.mark.gpu
def test_train_step_kernels_gpu():
    import yolosharp_b200  # noqa: F401  (fails loudly without the CUDA library)
    from yolosharp_b200.train import KernelOps, TrainStepV8
    _compare(TrainStepV8, KernelOps(tensor_cores=False), "cuda", 1e-3)


def _compare_tc(step_cls, ops_cls, arch, head_tol):
    """TF32 tensor-core step against the SAME step on the fp32 parity kernels.

    What is pinned where: every tensor-core kernel is checked in isolation in tests/test_gpu_conv_tc.py (1e-2 of the
    output rms per element, bit-exact on TF32-representable inputs).  Through the whole network the TF32 operand
    truncation (10 mantissa bits; the tensor core drops the low 13 bits of each fp32 operand, as cuDNN's TF32 path does)
    compounds smoothly with depth - tools/dbg_train_tc.py: 4e-4 rms after the first conv, 1e-2 at the ~57th, no jump
    at any layer - and batch-statistics BatchNorm over the few positions of the deep levels amplifies it.  The
    task-aligned assigner is discrete (top-k per target), so a 1e-2 perturbation of the head outputs can move an
    assignment and the loss by percents, which says nothing about the kernels.  The comparison is therefore split at
    the loss: (1) train-mode head outputs of both paths on the same batch (rms relative error), (2) both backward
    passes driven by the SAME loss gradient (the fp32 path's): relative L2 error and cosine of the whole flat gradient
    vector - what the optimizer consumes, (3) the whole step end to end with a loose bound on the loss items."""
    torch.manual_seed(0)
    m = oracle_model(arch, "detect", "n")
    sd0 = {k: v.detach().clone() for k, v in m.state_dict().items()}
    # 4 x 320 x 320: the deepest level still has 400 positions per channel for the batch statistics (at 64 x 64 it has 8,
    # and BatchNorm's backward - a difference of nearly equal sums - amplifies any perturbation by orders of magnitude)
    B, H, W = 4, 320, 320
    x = synth_image(B, H, W).cuda()
    targets = _targets(B)
    a = step_cls(sd0, "n", 80, device="cuda", ops=ops_cls(tensor_cores=False), lr=1e-3)
    b = step_cls(sd0, "n", 80, device="cuda", ops=ops_cls(tensor_cores=True), lr=1e-3)
    ba, sa = a.forward(x)
    bb, sb = b.forward(x)

    def rel(u, v):
        return float((u - v).pow(2).mean().sqrt() / v.pow(2).mean().sqrt())
    e_box, e_cls = rel(bb, ba), rel(sb, sa)
    items, gb, gs = a.ops.detection_loss(ba, sa, targets, H, W)
    a.P.grad.zero_()
    b.P.grad.zero_()
    a.backward(gb, gs)
    b.backward(gb, gs)
    ga, gt = a.P.grad.double(), b.P.grad.double()
    l2 = float((gt - ga).norm() / ga.norm())
    cos = float((gt * ga).sum() / (gt.norm() * ga.norm()))
    print(f"{arch}: head outputs rms rel box {e_box:.2e} cls {e_cls:.2e}; flat gradient rel L2 {l2:.2e} cosine {cos:.6f}")
    assert e_box < head_tol and e_cls < head_tol
    # PyTorch's own cuDNN TF32 convolutions against its fp32 ones on the same model and batch differ by the same order
    # (tools/exp_torch_tf32.py)
    assert l2 < 0.4 and cos > 0.93  # a chaotic quantity: one last-bit reordering anywhere moves it by a few percent
    c = step_cls(sd0, "n", 80, device="cuda", ops=ops_cls(tensor_cores=True), lr=1e-3)
    it_tc = c.step(x, targets).cpu()
    np.testing.assert_allclose(it_tc.numpy(), items.cpu().numpy(), rtol=0.15)


@pytest.mark.gpu
def test_train_step_tensor_cores_gpu():
    """Every dense convolution (forward, dgrad, wgrad) on the TF32 tensor-core kernels - the default of KernelOps, the
    arithmetic class of libtorch's own CUDA convolutions."""
    import yolosharp_b200  # noqa: F401
    from yolosharp_b200.train import KernelOps, TrainStepV8
    _compare_tc(TrainStepV8, KernelOps, "v8", 3e-2)


def test_lr_schedule_and_warmup():
    """LrLambda / OneCycle / Interp / warm-up restated from YoloBaseTaskModel.cs:307-319, 492-536."""
    from yolosharp_b200.train import interp, lr_lambda_linear, lr_lambda_onecycle, warmup_lrs
    assert lr_lambda_linear(0, 0.01, 100) == 1.0 and abs(lr_lambda_linear(100, 0.01, 100) - 0.01) < 1e-12
    assert abs(lr_lambda_linear(50, 0.01, 100) - 0.505) < 1e-12 and lr_lambda_linear(150, 0.01, 100) == 0.01
    assert lr_lambda_onecycle(0, 0.01, 100) == 1.0 and abs(lr_lambda_onecycle(100, 0.01, 100) - 0.01) < 1e-12
    assert abs(lr_lambda_onecycle(50, 0.01, 100) - 0.505) < 1e-12
    assert interp(-1, [0, 10], [3, 5]) == 3 and interp(11, [0, 10], [3, 5]) == 5 and interp(5, [0, 10], [3, 5]) == 4
    lr0 = round(0.002 * 5 / (4 + 80), 6)
    assert lr0 == 0.000119
    b, o = warmup_lrs(0, 300, lr0, 1.0)
    assert b == 0.1 and o == 0.0                       # bias group starts at WarmUpBiasLr, the others at 0
    b, o = warmup_lrs(150, 300, lr0, 1.0)
    assert abs(b - (0.1 + lr0) / 2) < 1e-12 and abs(o - lr0 / 2) < 1e-12
    assert warmup_lrs(301, 300, lr0, 1.0) is None


def test_train_step_param_groups_cpu():
    """Two steps with different learning rates for the "bias" group and the rest (warm-up) against
    torch.optim.AdamW with the same two parameter groups."""
    from tests.torch_train_ops import TorchOps
    from yolosharp_b200.train import TrainStepV8
    torch.manual_seed(0)
    m = oracle_model("v8", "detect", "n")
    sd0 = {k: v.detach().clone() for k, v in m.state_dict().items()}
    B, H, W = 2, 64, 64
    x, targets = synth_image(B, H, W), _targets(B, seed=3)
    m.train()
    named = [(k, p) for k, p in m.named_parameters() if ".dfl." not in k]
    groups = [{"params": [p for k, p in named if "bias" in k]}, {"params": [p for k, p in named if "bias" not in k]}]
    opt = torch.optim.AdamW(groups, lr=1e-3, weight_decay=5e-4)
    crit = oloss.V8DetectionLoss(80)
    batch = {"batch_idx": targets[:, 0], "cls": targets[:, 1], "bboxes": targets[:, 2:]}
    ts = TrainStepV8(sd0, "n", 80, device="cpu", ops=TorchOps(), lr=1e-3)
    for lrs in ((0.05, 1e-4), (0.02, 3e-4)):
        opt.param_groups[0]["lr"], opt.param_groups[1]["lr"] = lrs
        _, preds = m(x)
        loss, _ = crit(preds, batch)
        opt.zero_grad()
        loss.sum().backward()
        opt.step()
        ts.step(x, targets, lrs=lrs)
    new = m.state_dict()
    bad = 0
    for k, _ in named:
        d = (ts.P.p(k).detach() - new[k].detach()).abs()
        assert float(d.max()) <= 2.1 * 2 * 0.05, k      # sign-of-noise elements move by at most lr per step
        bad += int((d > 1e-4 + 1e-3 * new[k].detach().abs()).sum())
    assert bad < 0.01 * ts.P.flat.numel(), bad


def test_train_step_v11_graph_logic_cpu():
    """YOLOv11 (C3k2 / C3k / C2PSA attention / depthwise convs / non-legacy head): graph logic of train_v11.py against
    autograd through the oracle, with the PyTorch stand-in of the kernel interface."""
    from tests.torch_train_ops import TorchOps
    from yolosharp_b200.train_v11 import TrainStepV11
    _compare(TrainStepV11, TorchOps(), "cpu", 2e-4, arch="v11")
    from yolosharp_b200.train_v11 import KernelOpsV11
    with pytest.raises(NotImplementedError):  # only depthwise 3x3 stride-1 grouped convs have kernels: refused, not emulated
        KernelOpsV11._check_dw(torch.zeros(1, 4, 4, 8), torch.zeros(8, 2, 3, 3), 1, 1, 4)


def test_fit_loop_learning_rates():
    """Epoch loop: warm-up per iteration, lambda per epoch, target-less batches skipped (YoloBaseTaskModel.cs:289-345)."""
    from yolosharp_b200.train import fit, lr_lambda_linear

    class FakeStep:
        lr = 1e-3

        def __init__(self):
            self.calls = []

        def step(self, images, targets, lrs=None):
            self.calls.append(lrs)
            return torch.tensor([1.0, 2.0, 3.0])
    batches = [(None, torch.zeros(2, 6)), (None, torch.zeros(0, 6)), (None, torch.zeros(1, 6))] * 20  # nb = 60
    st = FakeStep()
    hist = fit(st, batches, epochs=3, lrf=0.01, warmup_epochs=1)
    assert len(st.calls) == 3 * 40 and len(hist) == 3 and torch.equal(hist[0], torch.tensor([1.0, 2.0, 3.0]))
    nw = 100                                            # max(1 * 60, 100)
    # the reference's epochs are 1-based and `i` counts executed batches only: the first call has ni = 0 + 60 * 1
    d1 = 1e-3 * lr_lambda_linear(1, 0.01, 3)
    b0, o0 = st.calls[0]
    assert abs(o0 - 60 / nw * d1) < 1e-12 and abs(b0 - (0.1 + 60 / nw * (d1 - 0.1))) < 1e-12
    # executed call 40 of epoch 1 has i = 39 -> ni = 99 <= nw: still warming up
    b, o = st.calls[39]
    assert abs(o - 99 / nw * d1) < 1e-12
    # epoch 2 starts at ni = 120 > nw: LambdaLR was stepped once after epoch 1 -> InitialLR * lambda(1)
    assert st.calls[40] == (d1,) * 2
    assert st.calls[-1] == (1e-3 * lr_lambda_linear(2, 0.01, 3),) * 2   # epoch 3: lambda(2)
    # warm-up that ends in the middle of an epoch leaves the last interpolated value in place (never reset)
    st2 = FakeStep()
    fit(st2, [(None, torch.zeros(1, 6))] * 70, epochs=1, lrf=0.01, warmup_epochs=1)   # nb = 70, nw = 100, ni = 70 .. 139
    d = 1e-3 * lr_lambda_linear(1, 0.01, 1)
    assert abs(st2.calls[30][1] - d) < 1e-15 and st2.calls[31] == st2.calls[30] == st2.calls[-1]   # ni = 100 is the last update


def test_early_stopping_and_epoch_tail():
    """Utils/EarlyStopping.cs and the tail of the reference's epoch (YoloBaseTaskModel.cs:184-207): fitness = -sum(val loss),
    best.bin when it improves, stop after `patience` epochs without improvement, no last.bin for the stopping epoch."""
    from yolosharp_b200.train import EarlyStopping, fit
    es = EarlyStopping(patience=2)
    # negative fitness: the first epoch becomes the best although best_fitness starts at 0 (the `== 0` clause)
    assert [es.ShouldStop(f, e) for e, f in enumerate([-5.0, -4.0, -4.5, -4.2, -4.1], start=1)] == [False, False, False, True, True]
    assert es.best_epoch == 2 and es.best_fitness == -4.0
    es0 = EarlyStopping(patience=0)
    assert es0.ShouldStop(-1.0, 1) is True  # delta 0 >= patience 0: the reference's literal behaviour for patience = 0

    class FakeStep:
        lr = 1e-3

        def step(self, images, targets, lrs=None):
            return torch.tensor([1.0, 1.0, 1.0])
    val = {1: [3.0, 1.0, 1.0], 2: [2.0, 1.0, 1.0], 3: [2.5, 1.0, 1.0], 4: [2.6, 1.0, 1.0], 5: [1.0, 1.0, 1.0]}
    best, ends = [], []
    hist = fit(FakeStep(), [(None, torch.zeros(1, 6))] * 3, epochs=5, validate=lambda e: val[e], patience=2, on_best=best.append,
               on_epoch_end=ends.append)
    assert best == [1, 2] and ends == [1, 2, 3] and len(hist) == 4  # epoch 4: two epochs without improvement -> stop before last.bin


@pytest.mark.gpu
def test_train_step_v11_kernels_gpu():
    """The same comparison with the library's kernels (csrc/train_v11.cu, csrc/attention.cu: depthwise conv + attention forward / backward,
    plus the fp32 parity kernels of the v8 step): BASELINE configs[3] architecture (n size), one full step."""
    import yolosharp_b200  # noqa: F401
    from yolosharp_b200.train_v11 import KernelOpsV11, TrainStepV11
    _compare(TrainStepV11, KernelOpsV11(tensor_cores=False), "cuda", 1e-3, arch="v11")


@pytest.mark.gpu
def test_train_step_v11_tensor_cores_gpu():
    """YOLOv11n step with the dense convolutions on the TF32 tensor-core kernels (depthwise conv / attention stay fp32)."""
    import yolosharp_b200  # noqa: F401
    from yolosharp_b200.train_v11 import KernelOpsV11, TrainStepV11
    _compare_tc(TrainStepV11, KernelOpsV11, "v11", 1e-1)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(2, 20, 20, 256), (3, 9, 7, 48), (1, 40, 40, 128),
                                   (2, 9, 11, 30),      # C % 4 != 0: the scalar forward, dgrad and wgrad partial
                                   (1, 5, 6, 1368)])    # C % 4 == 0 but the row kernel's weight tile (9 C floats) > 48 KiB
def test_dwconv3x3_forward_backward_vs_autograd(shape):
    import yolosharp_b200 as y
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn(shape, generator=g)
    w = (torch.randn(shape[-1], 1, 3, 3, generator=g) * 0.3)
    dz = torch.randn(shape, generator=g)
    xt, wt = x.permute(0, 3, 1, 2).clone().requires_grad_(True), w.clone().requires_grad_(True)
    zt = torch.nn.functional.conv2d(xt, wt, None, 1, 1, 1, shape[-1])
    zt.backward(dz.permute(0, 3, 1, 2))
    z = y.engine.dwconv3x3_forward(x.cuda(), w.cuda())
    np.testing.assert_allclose(z.cpu().permute(0, 3, 1, 2).numpy(), zt.detach().numpy(), rtol=1e-5, atol=1e-5)
    dx, dw = y.engine.dwconv3x3_backward(x.cuda(), dz.cuda(), w.cuda())
    np.testing.assert_allclose(dx.cpu().permute(0, 3, 1, 2).numpy(), xt.grad.numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(dw.cpu().numpy(), wt.grad.numpy(), rtol=1e-4, atol=1e-4)


@pytest.mark.gpu
# kd = 32 / hd = 64 runs the register-blocked forward up to N = 424 tokens and the register-blocked backward up to 448;
# every other shape runs the general kernels
@pytest.mark.parametrize("B,N,nh,kd,hd", [(2, 400, 2, 32, 64), (3, 49, 4, 16, 32), (1, 130, 1, 32, 64),
                                          (2, 440, 2, 32, 64),   # general forward, register-blocked backward
                                          (1, 600, 2, 32, 64)])  # general forward and backward
def test_attention_forward_backward_vs_autograd(B, N, nh, kd, hd):
    import yolosharp_b200 as y
    from tests.torch_train_ops import TorchOps
    g = torch.Generator().manual_seed(N + nh)
    q, k = torch.randn(B, N, nh, kd, generator=g), torch.randn(B, N, nh, kd, generator=g)
    v, do = torch.randn(B, N, nh, hd, generator=g), torch.randn(B, N, nh, hd, generator=g)
    scale = kd ** -0.5
    ref = TorchOps._attn(q, k, v, scale)
    rq, rk, rv = TorchOps().attention_backward(q, k, v, scale, do)
    out = y.engine.attention_forward(q.cuda(), k.cuda(), v.cuda(), scale)
    np.testing.assert_allclose(out.cpu().numpy(), ref.numpy(), rtol=1e-4, atol=1e-5)
    dq, dk, dv = y.engine.attention_backward(q.cuda(), k.cuda(), v.cuda(), scale, do.cuda())
    for got, exp in ((dq, rq), (dk, rk), (dv, rv)):
        np.testing.assert_allclose(got.cpu().numpy(), exp.numpy(), rtol=1e-3, atol=2e-5)


@pytest.mark.gpu
def test_attention_shape_limits():
    """key_dim <= 64, head_dim <= 128 and 8 N + 32 (key_dim + 1) + 32 head_dim floats <= 200 KiB (N <= 6 012 at 32 / 64),
    for the forward and the backward alike; beyond them YB_ERR_SHAPE with the limit in the message."""
    import yolosharp_b200 as y
    from tests.torch_train_ops import TorchOps
    g = torch.Generator().manual_seed(7)

    def qkvo(N, kd, hd):
        return [torch.randn(1, N, 1, d, generator=g).cuda() for d in (kd, kd, hd, hd)]

    for N, kd, hd, what in ((16, 96, 64, "key_dim <= 64"), (16, 32, 160, "head_dim <= 128"), (6013, 32, 64, "limit of 6012")):
        q, k, v, do = qkvo(N, kd, hd)
        for call in (lambda: y.engine.attention_forward(q, k, v, kd ** -0.5),
                     lambda: y.engine.attention_backward(q, k, v, kd ** -0.5, do)):
            with pytest.raises(y.YbError) as ei:
                call()
            assert ei.value.status == -6 and what in str(ei.value), str(ei.value)
    q, k, v, do = qkvo(6012, 32, 64)
    out = y.engine.attention_forward(q, k, v, 32 ** -0.5)
    ref = TorchOps._attn(q.cpu(), k.cpu(), v.cpu(), 32 ** -0.5)
    np.testing.assert_allclose(out.cpu().numpy(), ref.numpy(), rtol=1e-4, atol=1e-5)
