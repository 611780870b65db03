"""Eval-mode forward of the native trainer (`AMPWrapper.Evaluate`, Utils/Amp.cs:387-395), on the H100.

Op level: `yb_debug_conv_tf32_eval` makes one fold launch and one eval-mode `tf_conv_kernel` launch.  The folded weights
and bias it returns must equal the float64 fold rounded to fp32 bit for bit; its output is held per element to a bound
against float64 computed from those returned operands, truncated to TF32 as the tensor core reads them:
    pre-activation   n_k 2^-23 S            (the bound of test_gpu_conv_tf32_ops.py, S = sum |x| |w| + |bias|)
    SiLU             1.1 x that (|silu'| <= 1.0998) + 2^-20 |silu(u)| for expf, the add and the division of silu_f
    residual add     + 2^-24 |out| (one rounding)
Graph level: `NativeTrainer.evaluate` on the shipped v8n / v11n weights against the fp32 oracle in `eval()`."""
import ctypes as C
import math
import os
import re
import zlib

import numpy as np
import pytest
import torch

from tests.test_gpu_conv_tf32_ops import (CASES, GUARD, F32_NAN, Guarded, _bits, _vp, conv_nk, fwd_ref, operands, out_hw, tf32)
from tests.util import GOLDEN

gpu = pytest.mark.gpu

EVAL_RE = re.compile(r"tf_conv_kernel_eval BK (\d+) chunks (\d+) n_tile (\d+) x(\d+) BW (\d+) BH (\d+) in_stride (\d+) flat (\d+) "
                     r"ntaps (\d+) occ (\d+) stages (\d+) grid (\d+)$")
EVAL_KEYS = ("BK", "chunks", "n_tile", "n_tiles", "BW", "BH", "in_stride", "flat", "ntaps", "occ", "stages", "grid")
# (name, out view (extra pitch, channel offset) or None = dense, act, residual)
VARIANTS = [("dense", None, 0, False), ("view_silu", (16, 8), 1, False), ("view_silu_res", (16, 8), 1, True),
            ("view_res", (24, 16), 0, True)]


def fold64(w, g, b, rm, rv):
    """float64 fold rounded to fp32 once: (folded [tap][cout][cin], folded bias)"""
    s = g.double() / torch.sqrt(rv.double() + 1e-3)
    wf = (w.double() * s.view(-1, 1, 1, 1)).float()
    bf = (b.double() - rm.double() * s).float()
    k = w.shape[2]
    return wf.permute(2, 3, 0, 1).reshape(k * k, w.shape[0], w.shape[1]).contiguous(), bf


def bn_operands(c, data):
    g = torch.Generator().manual_seed(zlib.crc32((c["name"] + data + "bn").encode()))
    cout = c["cout"]
    if data == "integer":  # scale gamma / sqrt(rv + 1e-3) within 2^-27 of a power of two, bias = beta: the fold is exact
        j = torch.randint(-1, 2, (cout,), generator=g).float()
        return torch.exp2(j), torch.randint(-8, 9, (cout,), generator=g).float(), torch.zeros(cout), \
            torch.full((cout,), 1.0 - 1e-3, dtype=torch.float32)
    return (torch.rand(cout, generator=g) * 1.5 + 0.25, torch.randn(cout, generator=g), torch.randn(cout, generator=g) * 0.5,
            torch.rand(cout, generator=g) * 2.0 + 0.05)


def run_eval(c, data, variant):
    """One case x variant: fold bit-exactness, per-element bound (or exactness), NaN fills, repeats -> description line"""
    from yolosharp_b200 import _lib as L
    vname, view, act, with_res = variant
    N, H, W, cin, cout, k, s = (c[n] for n in ("N", "H", "W", "cin", "cout", "k", "s"))
    Ho, Wo = out_hw(H, W, k, s)
    x, w, _, _ = operands(c, data, seed_extra="eval")
    gam, bet, rm, rv = bn_operands(c, data)
    gr = torch.Generator().manual_seed(zlib.crc32((c["name"] + data + "res").encode()))
    r = (torch.randint(-4, 5, (N, Ho, Wo, cout), generator=gr).float() if data == "integer" else
         torch.randn(N, Ho, Wo, cout, generator=gr))
    xpitch, xc0 = c["view"] or (cin, 0)
    xg = Guarded((N, H, W, xpitch))
    xg.t[..., xc0:xc0 + cin] = x.cuda()
    xv = xg.t[..., xc0:]
    ins = [Guarded(t.shape, t.cuda()) for t in (w, gam, bet, rm, rv)]
    rg = Guarded((N, Ho, Wo, cout + 8))  # the residual as channels [4, 4 + cout) of a wider buffer
    rg.t[..., 4:4 + cout] = r.cuda()
    extra, coff = view or (0, 0)
    opitch = cout + extra
    out = Guarded((N, Ho, Wo, opitch))
    fw, fb = Guarded((k * k, cout, cin)), Guarded((cout,))
    desc = C.create_string_buffer(512)
    lib = L.lib()

    def call():
        out.reset(); fw.reset(); fb.reset()
        L.check(lib.yb_debug_conv_tf32_eval(_vp(xv), xpitch, *(_vp(g.t) for g in ins), N, H, W, cin, cout, k, s, act,
                                            _vp(rg.t[..., 4:]) if with_res else None, cout + 8 if with_res else 0,
                                            _vp(out.t), opitch, coff, _vp(fw.t), _vp(fb.t), desc, 512))
        return out.t.clone(), fw.t.clone(), fb.t.clone()

    first = call()
    second = call()
    for a, b in zip(first, second):
        assert torch.equal(_bits(a), _bits(b)), f"{c['name']} {vname}: a repeated call is not bitwise identical"
    got_full, got_w, got_b = (t.cpu() for t in first)
    assert all(g.guards_intact() for g in [out, fw, fb, xg, rg] + ins), "stores outside a buffer"
    # the fold: bit for bit the float64 fold rounded to fp32
    ref_w, ref_b = fold64(w, gam, bet, rm, rv)
    assert torch.equal(_bits(got_w), _bits(ref_w)), f"folded weights differ in {int((got_w != ref_w).sum())} elements"
    assert torch.equal(_bits(got_b), _bits(ref_b)), f"folded bias differs in {int((got_b != ref_b).sum())} elements"
    # channels around the output view keep their NaN fill
    ob = _bits(got_full)
    assert (ob[..., :coff] == F32_NAN).all() and (ob[..., coff + cout:] == F32_NAN).all(), "stores outside the output view"
    got = got_full[..., coff:coff + cout]
    assert not torch.isnan(got).any(), "output view not fully written"
    # float64 reference on the returned operands, truncated to TF32
    w_ck = tf32(got_w).view(k, k, cout, cin).permute(2, 3, 0, 1).double()
    u, S = fwd_ref(x.double(), w_ck, got_b.double(), s)
    line = desc.value.decode()
    m = EVAL_RE.match(line)
    assert m, line
    plan = dict(zip(EVAL_KEYS, map(int, m.groups())))
    bound = conv_nk(plan) * 2.0 ** -23 * S
    y = u
    if act:
        y = u * torch.sigmoid(u)
        bound = 1.1 * bound + 2.0 ** -20 * y.abs()
    if with_res:
        y = r.double() + y
        bound = bound + 2.0 ** -24 * y.abs()
    if data == "integer":
        assert not act
        assert torch.equal(got.double(), y), f"not exact on integer operands: {int((got.double() != y).sum())} elements differ"
    else:
        err = (got.double() - y).abs()
        ratio = float((err / bound.clamp_min(1e-300)).max())
        print(f"{c['name']} {vname}: {line}: max err/bound {ratio:.3f}")
        assert ratio <= 1.0, f"{c['name']} {vname}: err/bound {ratio:.3f}"
    return plan


@gpu
@pytest.mark.parametrize("variant", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_eval_conv_sweep(variant):
    """Every forward shape case of the training-convolution sweep, per output / epilogue variant; the sweep reaches one and
    two CTAs per SM, several N tiles, flat and tiled 1x1."""
    plans = [(c, run_eval(c, "random", variant)) for c in CASES]
    occ = {p["occ"] for _, p in plans}
    assert occ == {1, 2}, occ
    assert max(p["n_tiles"] for _, p in plans) >= 2
    one = [p["flat"] for c, p in plans if c["k"] == 1]
    assert set(one) == {0, 1}, one


@gpu
@pytest.mark.parametrize("variant", [v for v in VARIANTS if not v[2]], ids=[v[0] for v in VARIANTS if not v[2]])
@pytest.mark.parametrize("name", ["bk32_ragged_20x20", "flat_c32_2x24x40", "s2_c128_n256", "view_halo"])
def test_eval_conv_exact_on_integer_operands(name, variant):
    """Integer activations and weights, power-of-two BatchNorm scales, integer bias and residual: every partial sum is exact
    in fp32, so the output must equal float64 exactly."""
    run_eval(next(c for c in CASES if c["name"] == name), "integer", variant)


# ------------------------------------------------------------------ graph level
def shipped_oracle(arch):
    from oracle import yolo as oyolo
    z = np.load(os.path.join(GOLDEN, "yolov8n_f16.npz" if arch == "v8" else "yolov11n_f16.npz"))
    m = oyolo.build(arch, "detect", "n").eval()
    own = m.state_dict()
    m.load_state_dict({k: torch.from_numpy(z[k].astype(np.float32)).reshape(own[k].shape) for k in z.files if k in own}, strict=False)
    return m


def _detect(m):
    from oracle import modules as om
    return next(mod for mod in m.modules() if isinstance(mod, om.Detect))


def rms_rel(a, b):
    return float(((a.double() - b.double()) ** 2).mean().sqrt() / (b.double() ** 2).mean().sqrt())


RAW_TOL = 1e-2  # rms relative error of the raw head outputs; train mode allows 3e-2 (v8) / 1e-1 (v11): measured values in DESIGN.md §4.3


@gpu
@pytest.mark.parametrize("arch", ["v8", "v11"])
@pytest.mark.parametrize("B,HW", [(4, 320), (2, 640)])
def test_evaluate_matches_oracle(arch, B, HW):
    from tests.util import synth_image
    from yolosharp_b200.train_native import NativeTrainer
    m = shipped_oracle(arch)
    x = synth_image(B, HW, HW, seed=3)
    with torch.no_grad():
        inf, preds = m(x)
    tr = NativeTrainer(m.state_dict(), arch, "n", 80, device="cuda", max_batch=B, height=HW, width=HW)
    pred, boxes, scores = tr.evaluate(x.cuda())
    torch.cuda.synchronize()
    eb, es = rms_rel(boxes.cpu(), preds["boxes"]), rms_rel(scores.cpu(), preds["scores"])
    print(f"{arch} {B}x{HW}^2: rms rel err boxes {eb:.3e} scores {es:.3e}")
    assert eb < RAW_TOL and es < RAW_TOL, (eb, es)
    # the decode of the library's own raw outputs, as the oracle's Detect._inference does it
    with torch.no_grad():
        ref = _detect(m)._inference({"feats": preds["feats"], "boxes": boxes.cpu(), "scores": scores.cpu()})
    d = (pred.cpu().double() - ref.double()).abs()
    # class probabilities: relative to the value itself (a probability that underflows to 0 in one of the two must be below
    # 1e-30 in the other); box coordinates (pixels): relative, with one pixel as the floor of the scale - a coordinate near
    # the image origin is a difference of two anchor-sized terms, so its rounding is relative to those, not to itself
    rel_cls = float((d[:, 4:] / ref[:, 4:].double().abs().clamp_min(1e-30)).max())
    rel_box = float((d[:, :4] / ref[:, :4].double().abs().clamp_min(1.0)).max())
    print(f"{arch} {B}x{HW}^2: pred vs decode of the raw outputs: class rel {rel_cls:.2e}, box rel {rel_box:.2e}")
    assert rel_cls < 1e-5 and rel_box < 1e-5, (rel_cls, rel_box)
    tr.close()


def _trainer(m, B=2, HW=128):
    from yolosharp_b200.train_native import NativeTrainer
    return NativeTrainer(m.state_dict(), "v8", "n", 80, device="cuda", max_batch=B, height=HW, width=HW, lr=1e-3)


@gpu
def test_evaluate_has_no_side_effects():
    """evaluate changes no parameter, running statistic, gradient or Adam moment; step, evaluate, step leaves the same trainer
    state as step, step, bit for bit; two evaluate calls are bitwise identical."""
    from tests.test_train_step import _targets
    from tests.util import synth_image
    m = shipped_oracle("v8")
    x, tg = synth_image(2, 128, 128, seed=5).cuda(), _targets(2)
    a, b = _trainer(m), _trainer(m)
    a.step(x, tg)
    b.step(x, tg)
    state = [t.clone() for t in (a.flat, a.grad, a.m, a.v, a.running)]
    p1 = a.evaluate(x)
    p2 = a.evaluate(x)
    torch.cuda.synchronize()
    for t1, t2 in zip(p1, p2):
        assert torch.equal(_bits(t1), _bits(t2)), "two evaluate calls differ"
    for before, after in zip(state, (a.flat, a.grad, a.m, a.v, a.running)):
        assert torch.equal(_bits(before), _bits(after)), "evaluate changed trainer state"
    ia, ib = a.step(x, tg), b.step(x, tg)
    # the loss items are per-block partials summed with float atomics (csrc/loss.cu), so only their last bits may differ
    assert torch.allclose(ia, ib, rtol=1e-6, atol=0), (ia, ib)
    for ta, tb in zip((a.flat, a.grad, a.m, a.v, a.running), (b.flat, b.grad, b.m, b.v, b.running)):
        assert torch.equal(_bits(ta), _bits(tb)), "a step after evaluate differs from a step without it"
    a.close(), b.close()


@gpu
def test_evaluate_refuses_bad_arguments():
    from yolosharp_b200 import _lib as L
    m = shipped_oracle("v8")
    tr = _trainer(m)
    img = torch.zeros(3, 3, 128, 128, dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):
        tr.evaluate(img)
    rc = L.lib().yb_trainer_evaluate(tr._h, C.c_void_p(img.data_ptr()), L.YB_U8, 3, None, None, None, None)
    assert rc == -1 and "max_batch" in L.lib().yb_last_error().decode()
    pred, _, _ = tr.evaluate(img[:2].contiguous())  # still usable
    torch.cuda.synchronize()
    assert torch.isfinite(pred).all()
    tr.close()
