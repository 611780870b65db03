"""TF32 tensor-core training convolutions (csrc/conv_tf32.cu: yb_conv_forward_tc / _backward_data_tc / _backward_weight_tc)
against the library's own fp32 CUDA-core kernels (yb_conv_forward_f32 / yb_conv_backward_*) and against
torch.nn.functional.conv2d + autograd in fp32 (TF32 disabled) on the same inputs.

Tolerance: TF32 keeps 10 mantissa bits of every operand (products exact in fp32, fp32 accumulation), so an output that
sums K products of O(1) terms carries an absolute error of about 2^-11 * sqrt(K) * rms; the tests bound the error by
1e-2 of the output's rms scale (max over all elements; observed 2e-3 .. 6e-3) (observed values are printed) - the tolerance class libtorch's own TF32 convolutions
have against fp32.  Element-wise bounds, integer bit-exactness and the stem are in test_gpu_conv_tf32_ops.py."""
import pytest
import torch

gpu = pytest.mark.gpu

# (N, H, W, Cin, Cout, k, stride): the layer classes of YOLOv8n / YOLOv11s plus ragged edges
SHAPES = [
    (2, 32, 32, 16, 32, 3, 2),     # stride-2 3x3, smallest channel slabs (BK = 16)
    (2, 24, 40, 32, 32, 1, 1),     # 1x1, flattened batch
    (2, 24, 40, 16, 16, 3, 1),     # 3x3 s1, 64-byte rows
    (3, 20, 20, 64, 64, 3, 1),     # 20x20 images: rectangle tiles with padding waste
    (2, 20, 20, 128, 256, 3, 2),   # wide N tile (256), odd output size 10x10
    (2, 16, 16, 48, 80, 3, 1),     # ragged K slab (48 = 32 + 16) and N = 80
    (2, 16, 24, 384, 128, 1, 1),   # long K for 1x1 (concat inputs)
    (1, 8, 8, 8, 8, 1, 1),         # minimum channels (32-byte rows)
    (2, 16, 16, 24, 40, 1, 2),     # 1x1 stride 2 (not in the nets; the dgrad parity-zero path)
    (2, 12, 20, 320, 328, 3, 1),   # two N tiles (328 > 256) and K = 2880
]


def _mk(shape, seed=0):
    N, H, W, Cin, Cout, k, s = shape
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, H, W, Cin, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
    dz = torch.randn(N, Ho, Wo, Cout, generator=g)
    b = torch.randn(Cout, generator=g)
    return x, w, dz, b


def _rel(a, ref):
    return float((a - ref).abs().max() / ref.pow(2).mean().sqrt().clamp_min(1e-12))


@gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_conv_tc_forward_dgrad_wgrad(shape):
    import yolosharp_b200.engine as E
    N, H, W, Cin, Cout, k, s = shape
    x, w, dz, b = (t.cuda() for t in _mk(shape))
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        xt = x.permute(0, 3, 1, 2).contiguous().requires_grad_(True)
        wt = w.clone().requires_grad_(True)
        zt = torch.nn.functional.conv2d(xt, wt, b, stride=s, padding=k // 2)
        zt.backward(dz.permute(0, 3, 1, 2).contiguous())
        z_ref = zt.detach().permute(0, 2, 3, 1).contiguous()
        dx_ref = xt.grad.permute(0, 2, 3, 1).contiguous()
        dw_ref = wt.grad
    finally:
        torch.backends.cudnn.allow_tf32 = old
    ws = E.ConvWorkspace(x.device)
    z = E.conv_forward_tc(x, w, b, s, k // 2, ws=ws)
    dx, dw = E.conv_backward_tc(x, dz, w, s, k // 2, ws=ws)
    torch.cuda.synchronize()
    ez, edx, edw = _rel(z, z_ref), _rel(dx, dx_ref), _rel(dw, dw_ref)
    print(f"{shape}: forward {ez:.2e} dgrad {edx:.2e} wgrad {edw:.2e} (max abs error / rms of the fp32 result)")
    assert z.shape == z_ref.shape and ez < 1e-2
    assert edx < 1e-2
    assert edw < 1e-2
    # the library's fp32 CUDA-core twins see the same inputs
    z32 = E.conv_forward(x, w, b, s, k // 2)
    dx32, dw32 = E.conv_backward(x, dz, w, s, k // 2)
    assert _rel(z, z32) < 1e-2 and _rel(dx, dx32) < 1e-2 and _rel(dw, dw32) < 1e-2


@gpu
def test_conv_tc_rejects_unsupported_shapes():
    import yolosharp_b200.engine as E
    from yolosharp_b200._lib import YbError
    x = torch.randn(1, 8, 8, 3, device="cuda")
    w = torch.randn(16, 3, 3, 3, device="cuda")
    assert not E.conv_tc_supported(3, 16, 3, 2, 1, 8, 8)
    with pytest.raises(YbError):
        E.conv_forward_tc(x, w, None, 2, 1)


def test_conv_tc_symbols_and_shape_rule():
    """CPU: the entry points are exported and the shape rule matches the header's statement."""
    import yolosharp_b200.engine as E
    from yolosharp_b200 import _lib
    l = _lib.lib()
    for name in ("yb_conv_tc_workspace_bytes", "yb_conv_forward_tc", "yb_conv_backward_data_tc", "yb_conv_backward_weight_tc"):
        assert hasattr(l, name)
    assert E.conv_tc_supported(16, 32, 3, 2, 1, 640, 640)
    assert not E.conv_tc_supported(16, 32, 3, 2, 1, 641, 640)
    assert not E.conv_tc_supported(3, 16, 3, 2, 1, 640, 640)
    assert not E.conv_tc_supported(16, 32, 5, 1, 2)
