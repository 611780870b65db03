"""Op-level tests of the fp16 tensor-core inference kernels of csrc/conv_tc.cu against a float64 reference of the same
operation: conv_tc_kernel through yb_debug_conv_f16, bneck_tc_kernel through yb_debug_bneck_f16, and stem_tc_kernel as op 0
of an f16 engine (yb_debug_read_activation).

The reference is computed in float64 from the kernel's exact fp16 operands: z = sum w x + b, y = act(z) (+ r).  Every
output element must satisfy

    |got - y| <= ulp16(y) + [act] 2^-11 |z| + n_k 2^-23 S + 2^-24

  ulp16(y)    the fp16 store (round to nearest: half an ulp, the other half absorbs a binade crossing)
  2^-11 |z|   silu_tanh = h + h tanh.approx(h), h = z / 2: tanh.approx has a relative error below 2^-11, so the SiLU error
              is below 2^-12 |z|
  S           sum |w x| + |b|, a float64 convolution of |x| with |w|
  n_k         k^2 * chunks * BK / 16 k16 MMA steps; each rounds the fp32 accumulator (|partial sum| <= S) once: 2^-24 S,
              doubled to cover the SiLU slope (<= 1.1) the accumulator error passes through
The decode epilogues get the same accumulator term pushed through their own arithmetic (see decode_ref).

Three more checks per case: with integer operands (act none, x and w in -2..2, integer bias and residual) every partial sum
is an integer below 2^24, exact in fp32, so the kernel must equal half(exact) bit for bit - a layout, swizzle or indexing
error cannot hide in rounding; nothing outside the output view (other channels, images >= the launched batch, other
anchors / channels of pred) changes from its NaN fill; a second launch is bitwise identical (every output has one owner CTA
and a fixed summation order).  Input channels outside the input view are NaN as well, so a load from them poisons the
result.  The largest err / bound of each case is printed; the sweep's plan descriptions must reach every planner branch
listed in test_conv_plan_coverage."""
import ctypes as C
import re
import types
import zlib

import pytest
import torch
import torch.nn.functional as F

gpu = pytest.mark.gpu

F16_NAN = 0x7E00
F32_NAN = 0x7FC00000
EPI_STORE, EPI_DFL_BOX, EPI_SIGMOID, EPI_RAW = 0, 1, 2, 3


# ------------------------------------------------------------------ float64 reference
def ulp16(v):
    """spacing of fp16 numbers at |v| (subnormal spacing 2^-24 below 2^-14)"""
    a = v.abs().clamp_min(2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 10)


def view(buf, coff, c):
    """channels [coff, coff + c) of an NHWC buffer as float64"""
    return buf[..., coff:coff + c].double()


def conv_ref(x, w, b, stride, act=0, r=None):
    """x (B, H, W, Cin), w (Cout, k, k, Cin), b (Cout), r (B, Ho, Wo, Cout) or None, all float64 NHWC; pad k // 2.
    A sum over taps of shifted matrix products, independent of torch's convolution -> z, y = act(z) (+ r), S."""
    B, H, W, _ = x.shape
    cout, k = w.shape[0], w.shape[1]
    p = k // 2
    Ho, Wo = (H + 2 * p - k) // stride + 1, (W + 2 * p - k) // stride + 1
    xp = F.pad(x, (0, 0, p, p, p, p))
    z = b.view(1, 1, 1, cout).expand(B, Ho, Wo, cout).clone()
    S = b.abs().view(1, 1, 1, cout).expand(B, Ho, Wo, cout).clone()
    for kh in range(k):
        for kw in range(k):
            tap = xp[:, kh:kh + stride * (Ho - 1) + 1:stride, kw:kw + stride * (Wo - 1) + 1:stride, :]
            z = z + tap @ w[:, kh, kw, :].T
            S = S + tap.abs() @ w[:, kh, kw, :].abs().T
    y = F.silu(z) if act else z
    if r is not None:
        y = y + r
    return z, y, S


def conv_bound(y, z, S, n_k, act):
    return ulp16(y) + (2.0 ** -11 * z.abs() if act else 0.0) + n_k * 2.0 ** -23 * S + 2.0 ** -24


def decode_ref(z, S, mode, n_k, stride, Wl):
    """Fused Detect tail on a flattened 1x1 conv, z / S (B, HW, Cout) -> (values (B, rows, HW), bound) where rows are the
    pred channels written: DFL box -> 4 (xywh * stride, csrc/conv_tc.cu tc_epilogue), sigmoid / raw -> Cout."""
    acc = n_k * 2.0 ** -23 * S + 2.0 ** -23 * z.abs() + 2.0 ** -24  # MMA steps + the fp32 bias add
    if mode == EPI_RAW:
        return z.transpose(1, 2), acc.transpose(1, 2)
    if mode == EPI_SIGMOID:  # sigmoid' <= 1/4; __expf / __fdividef: a few fp32 ulps of the result
        v = torch.sigmoid(z)
        return v.transpose(1, 2), (0.25 * acc + 2.0 ** -20 * v + 2.0 ** -24).transpose(1, 2)
    B, HW, _ = z.shape
    zz = z.view(B, HW, 4, 16)
    d = (torch.softmax(zz, -1) * torch.arange(16, dtype=z.dtype, device=z.device)).sum(-1)
    # |d(expectation) / d(logit j)| summed over the bins <= 15; __expf / __fdividef and the fp32 sums: <= 16 * 2^-18
    ed = 15 * acc.view(B, HW, 4, 16).amax(-1) + 16 * 2.0 ** -18
    i = torch.arange(HW, device=z.device, dtype=z.dtype)
    ax, ay = (i % Wl + 0.5).view(1, HW), (torch.div(i, Wl, rounding_mode="floor") + 0.5).view(1, HW)
    x1, y1, x2, y2 = ax - d[..., 0], ay - d[..., 1], ax + d[..., 2], ay + d[..., 3]
    v = torch.stack([(x1 + x2) / 2 * stride, (y1 + y2) / 2 * stride, (x2 - x1) * stride, (y2 - y1) * stride], 1)
    e = torch.stack([(ed[..., 0] + ed[..., 2]) / 2, (ed[..., 1] + ed[..., 3]) / 2, ed[..., 0] + ed[..., 2],
                     ed[..., 1] + ed[..., 3]], 1) * stride
    return v, e + 2.0 ** -21 * v.abs() + 2.0 ** -24


def parse_conv_desc(desc):
    m = re.match(r"mode (\d+) BK (\d+) chunks (\d+) n_tile (\d+) x(\d+) stages a/b (\d+)/(\d+) resident (\d+) occ (\d+) "
                 r"threads \d+ smem \d+ KiB grid (\d+)", desc)
    assert m, desc
    keys = ("mode", "BK", "chunks", "n_tile", "n_tiles", "stages_a", "stages_b", "resident", "occ", "grid")
    return dict(zip(keys, map(int, m.groups())))


def parse_bneck_desc(desc):
    m = re.match(r"fused bottleneck (\d+)->(\d+) BK (\d+)/(\d+) chunks (\d+)/(\d+) shortcut (\d) stages (\d+) occ (\d+)", desc)
    assert m, desc
    return dict(zip(("cmid", "cout", "BK1", "BK2", "chunks1", "chunks2", "shortcut", "stages", "occ"), map(int, m.groups())))


# ------------------------------------------------------------------ conv cases
def case(name, B, H, W, cin, cout, k=3, s=1, **kw):
    c = dict(name=name, B=B, H=H, W=W, cin=cin, cout=cout, k=k, s=s, act=1, x_pitch=None, x_coff=0, res=None, out_pitch=None,
             out_coff=0, res_coff=0, run_batch=None, share_sms=False, tile_counter=True, decode=None)
    c.update(kw)
    return c


CONV_CASES = [
    # TC_HALO (3x3 s1): BK 16 / 32 / 64, ragged last slabs, chunks > 1; tiles ending mid-image at every edge; N tiles of
    # 48 .. 256 columns and 16 x 17, 112 x 3, 144 x 7, 256 x 4
    case("halo_c16_1x1", 2, 1, 1, 16, 32),
    case("halo_c32_3x5", 2, 3, 5, 32, 48),
    case("halo_c48_17x9", 2, 17, 9, 48, 80),
    case("halo_c64_40x24_res", 1, 40, 24, 64, 64, res="own"),
    case("halo_c80_17x9_view", 2, 17, 9, 80, 112, x_pitch=112, x_coff=16, out_pitch=128, out_coff=8),
    case("halo_c96_40x24", 1, 40, 24, 96, 144),
    case("halo_c144_17x9", 1, 17, 9, 144, 160),
    case("halo_c400_3x5_n272", 2, 3, 5, 400, 272),
    case("halo_c64_80x80_n336", 1, 80, 80, 64, 336),
    case("halo_c32_17x9_n1008", 1, 17, 9, 32, 1008),
    case("halo_c16_40x24_n1024", 1, 40, 24, 16, 1024, act=0),
    # TC_S2P (3x3 s2 over a whole buffer, Cin <= 32, even W): odd H, odd W / 2
    case("s2p_c16_17x30", 2, 17, 30, 16, 32, s=2),
    case("s2p_c32_33x46", 1, 33, 46, 32, 64, s=2),
    # TC_TAP: 3x3 s2 with Cin > 32; an input channel offset or an odd W forces it at Cin <= 32; outputs narrower than 16
    case("tap_c64_s2_40x24", 2, 40, 24, 64, 128, s=2),
    case("tap_c48_s2_coff", 2, 18, 26, 48, 48, s=2, x_pitch=80, x_coff=16),
    case("tap_c16_s2_oddw", 2, 20, 15, 16, 32, s=2),
    case("tap_c32_s2_9x13", 1, 9, 13, 32, 96, s=2),
    case("tap_c32_s2_coff", 1, 64, 64, 32, 32, s=2, x_pitch=64, x_coff=32),
    case("tap_c144_s2_40x40", 1, 40, 40, 144, 256, s=2),
    # flattened 1x1: B*H*W not a multiple of 128, long K, and a C2f-style residual / output in two slices of one buffer
    case("flat_c384_3x7x11", 3, 7, 11, 384, 64, k=1),
    case("flat_c512_slices", 2, 9, 13, 512, 128, k=1, x_pitch=640, x_coff=64, res="shared", out_pitch=256, res_coff=0,
         out_coff=128),
    case("flat_c16_5x5", 1, 5, 5, 16, 16, k=1),
    case("flat_c32_act0", 2, 6, 7, 32, 48, k=1, act=0),
    # plans made for 4 images, launched with fewer
    case("batch_halo_4to1", 4, 17, 9, 32, 32, run_batch=1),
    case("batch_flat_4to3", 4, 7, 9, 64, 80, k=1, run_batch=3),
    case("batch_tap_4to3", 4, 20, 14, 64, 64, s=2, run_batch=3),
    # grid and scheduling: several tiles per atomic draw, grid trimming for a shared GPU, static round-robin order
    case("sched_tile_batch", 8, 320, 320, 32, 32),
    case("sched_share_sms", 1, 40, 24, 64, 64, share_sms=True),
    case("sched_round_robin", 2, 80, 80, 32, 64, tile_counter=False),
    case("sched_round_robin_flat", 3, 20, 20, 64, 64, k=1, tile_counter=False),
    # fused Detect epilogues on a flattened 1x1 conv: anchors a0.. of a level, two images
    case("dec_dfl", 3, 5, 7, 64, 64, k=1, run_batch=2, decode=dict(mode=EPI_DFL_BOX, a0=13, extra=20, Ctot=84, ch0=0, stride=8.0)),
    case("dec_sigmoid", 2, 9, 15, 64, 80, k=1, decode=dict(mode=EPI_SIGMOID, a0=40, extra=3, Ctot=84, ch0=4, stride=16.0)),
    case("dec_raw", 2, 6, 22, 32, 32, k=1, decode=dict(mode=EPI_RAW, a0=7, extra=9, Ctot=116, ch0=84, stride=32.0)),
]
CASE_BY_NAME = {c["name"]: c for c in CONV_CASES}
DESCS = {}   # case name -> plan description (filled by the sweep, read by the coverage test)
WORST = {}   # kernel -> (largest err / bound, case)


def _note(kernel, ratio, name):
    if ratio > WORST.get(kernel, (-1.0, ""))[0]:
        WORST[kernel] = (ratio, name)


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for kernel, (ratio, name) in sorted(WORST.items()):
        print(f"worst err/bound of {kernel}: {ratio:.3f} ({name})")


def _f16(t):
    return t.to(torch.float16)


def _nan_buf(shape, dtype=torch.float16):
    bits = F16_NAN if dtype == torch.float16 else F32_NAN
    itype = torch.int16 if dtype == torch.float16 else torch.int32
    return torch.full(shape, bits, dtype=itype, device="cuda").view(dtype)


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def run_conv(c, data):
    """Launches case `c` twice on seeded operands ('random' or 'integer') and checks it; returns the plan description."""
    import yolosharp_b200.engine as E
    g = torch.Generator().manual_seed(zlib.crc32((c["name"] + data).encode()))
    integer = data == "integer"
    B, H, W, cin, cout, k, s = (c[n] for n in ("B", "H", "W", "cin", "cout", "k", "s"))
    rb = c["run_batch"] or B
    act = 0 if integer else c["act"]
    dec = c["decode"]
    p = k // 2
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1

    def values(*shape, scale=1.0):
        if integer:
            return torch.randint(-2, 3, shape, generator=g).float()
        return torch.randn(*shape, generator=g) * scale

    xp, xc = c["x_pitch"] or cin, c["x_coff"]
    x = _nan_buf((B, H, W, xp))
    x[..., xc:xc + cin] = _f16(values(B, H, W, cin)).cuda()
    w = values(cout, k, k, cin, scale=1.0 / (cin * k * k) ** 0.5)
    if not integer:  # low-magnitude output channels next to large ones: the bound is per element, not per layer range
        w = w * torch.exp2(torch.randint(-6, 2, (cout, 1, 1, 1), generator=g).float())
    w = _f16(w).cuda()
    b = (torch.randint(-8, 9, (cout,), generator=g).float() if integer else torch.randn(cout, generator=g) * 0.5).cuda()
    r_vals = _f16(torch.randint(-8, 9, (B, Ho, Wo, cout), generator=g).float() if integer
                  else torch.randn(B, Ho, Wo, cout, generator=g)).float() if c["res"] else None
    out = res = pred = None
    op, oc, rc = c["out_pitch"] or cout, c["out_coff"], c["res_coff"]
    if dec is None:
        out = _nan_buf((B, Ho, Wo, op))
        if c["res"] == "shared":
            out[..., rc:rc + cout] = _f16(r_vals).cuda()
            res = out
        elif c["res"] == "own":
            res = _f16(r_vals).cuda().contiguous()
    decode = None
    if dec is not None:
        A = dec["a0"] + H * W + dec["extra"]
        pred = _nan_buf((B, dec["Ctot"], A), torch.float32)
        decode = dict(mode=dec["mode"], A=A, Ctot=dec["Ctot"], a0=dec["a0"], ch0=dec["ch0"], Wl=W, HW=H * W, stride=dec["stride"])
    dst = out if dec is None else pred
    before = dst.clone()

    def launch():
        return E.debug_conv_f16(x, w, b, out, stride=s, act=act, x_coff=xc, out_coff=oc, res=res, res_coff=rc, plan_batch=B,
                                run_batch=rb, share_sms=c["share_sms"], tile_counter=c["tile_counter"], decode=decode, pred=pred)

    desc = launch()
    first = dst.clone()
    assert launch() == desc
    assert torch.equal(_bits(dst), _bits(first)), "a repeated launch is not bitwise identical"
    info = parse_conv_desc(desc)
    n_k = k * k * info["chunks"] * info["BK"] // 16

    # nothing outside the written region changes
    region = torch.zeros(dst.shape, dtype=torch.bool, device="cuda")
    if dec is None:
        region[:rb, ..., oc:oc + cout] = True
    else:
        a0, rows = dec["a0"], (range(4) if dec["mode"] == EPI_DFL_BOX else range(dec["ch0"], dec["ch0"] + cout))
        region[:rb, rows.start:rows.stop, a0:a0 + H * W] = True
    changed = _bits(first) != _bits(before)
    assert not (changed & ~region).any(), "stores outside the output view: %d elements" % int((changed & ~region).sum())

    xr = view(x[:rb], xc, cin)
    z, yv, S = conv_ref(xr, w.double(), b.double(), s, act, r_vals[:rb].double().cuda() if r_vals is not None else None)
    if dec is None:
        got = view(first[:rb], oc, cout)
        bound = conv_bound(yv, z, S, n_k, act)
        exact = yv.half() if integer else None
    else:
        got = first[:rb, rows.start:rows.stop, dec["a0"]:dec["a0"] + H * W].double()
        yv, bound = decode_ref(z.reshape(rb, H * W, cout), S.reshape(rb, H * W, cout), dec["mode"], n_k, dec["stride"], W)
        exact = yv.float() if integer and dec["mode"] == EPI_RAW else None
    assert not torch.isnan(got).any(), "output view not fully written"
    ratio = float(((got - yv).abs() / bound).max())
    kernel = "conv_tc_kernel" + (" (decode %d)" % dec["mode"] if dec else "")
    print(f"{c['name']} [{data}] {desc}: max err/bound {ratio:.3f}")
    if integer and exact is not None:
        assert torch.equal(got.to(exact.dtype), exact), \
            f"not bit-exact on integer operands: {int((got.to(exact.dtype) != exact).sum())} elements differ"
    else:
        _note(kernel, ratio, f"{c['name']} [{data}]")
    assert ratio <= 1.0, f"err/bound {ratio:.3f}"
    DESCS[c["name"]] = desc
    return desc


@gpu
@pytest.mark.parametrize("data", ["random", "integer"])
@pytest.mark.parametrize("name", list(CASE_BY_NAME))
def test_conv_f16_op(name, data):
    c = CASE_BY_NAME[name]
    desc = run_conv(c, data)
    if name == "sched_tile_batch":  # tc_conv_launch draws max(1, min(8, tiles / (4 grid))) tiles per atomic
        info = parse_conv_desc(desc)
        tiles = c["B"] * ((c["W"] + 7) // 8) * ((c["H"] + 15) // 16) * info["n_tiles"]
        assert info["mode"] == 1 and tiles // (4 * info["grid"]) >= 2, desc


@gpu
def test_conv_plan_coverage():
    """The sweep reaches every planner branch it is meant to pin: a planner change that moves the cases off one fails here
    instead of silently shrinking the coverage."""
    for name, c in CASE_BY_NAME.items():
        if name not in DESCS:
            run_conv(c, "integer")
    plans = {n: parse_conv_desc(d) for n, d in DESCS.items()}
    seen = lambda key: {p[key] for p in plans.values()}
    assert seen("mode") >= {0, 1, 2}, seen("mode")
    for mode in (0, 1):  # TC_TAP, TC_HALO
        bks = {p["BK"] for p in plans.values() if p["mode"] == mode}
        assert bks >= {16, 32, 64}, (mode, bks)
    assert max(seen("n_tiles")) >= 2
    assert seen("n_tile") >= {48, 80, 112, 144, 160}, seen("n_tile")
    assert seen("resident") == {0, 1}
    assert seen("occ") == {1, 2}


# ------------------------------------------------------------------ fused Bottleneck
BNECK_CASES = [(cin, cmid, cout, sc) for cin, cmid, cout, sc in
               [(16, 16, 16, 1), (16, 16, 16, 0), (32, 32, 32, 1), (32, 32, 32, 0), (48, 48, 48, 1), (64, 64, 64, 1),
                (32, 16, 32, 1), (64, 32, 64, 1), (32, 16, 16, 0)]]
BNECK_SHAPES = [(1, 5, 7), (3, 21, 13)]  # smaller than one 16 x 8 tile; tiles ending mid-image at both edges


@gpu
@pytest.mark.parametrize("B,H,W", BNECK_SHAPES)
@pytest.mark.parametrize("cin,cmid,cout,shortcut", BNECK_CASES)
def test_bneck_f16_op(cin, cmid, cout, shortcut, B, H, W):
    """t = fp16(SiLU(conv_a(x) + b_a)) and out = SiLU(conv_b(t) + b_b) [+ x].  The reference rounds t to fp16 where the
    kernel does; where the kernel's t differs from the reference's (the stage-1 error of the bound above, then one fp16 ulp
    of rounding), that difference reaches the output through |w_b| and the SiLU slope (<= 1.1)."""
    import yolosharp_b200.engine as E
    g = torch.Generator().manual_seed(1000 * cin + 10 * cmid + cout + shortcut + B)
    xc = 8 if B > 1 else 0
    x = _nan_buf((B, H, W, cin + 2 * xc))
    x[..., xc:xc + cin] = _f16(torch.randn(B, H, W, cin, generator=g)).cuda()
    wa = _f16(torch.randn(cmid, 3, 3, cin, generator=g) / (9 * cin) ** 0.5 *
              torch.exp2(torch.randint(-4, 2, (cmid, 1, 1, 1), generator=g).float())).cuda()
    wb = _f16(torch.randn(cout, 3, 3, cmid, generator=g) / (9 * cmid) ** 0.5 *
              torch.exp2(torch.randint(-4, 2, (cout, 1, 1, 1), generator=g).float())).cuda()
    ba, bb = (torch.randn(cmid, generator=g) * 0.5).cuda(), (torch.randn(cout, generator=g) * 0.5).cuda()
    oc = 16
    out = _nan_buf((B, H, W, cout + 24))
    before = out.clone()
    desc = E.debug_bneck_f16(x, wa, ba, wb, bb, out, shortcut=bool(shortcut), x_coff=xc, out_coff=oc)
    first = out.clone()
    assert E.debug_bneck_f16(x, wa, ba, wb, bb, out, shortcut=bool(shortcut), x_coff=xc, out_coff=oc) == desc
    assert torch.equal(_bits(out), _bits(first)), "a repeated launch is not bitwise identical"
    info = parse_bneck_desc(desc)
    assert (info["cmid"], info["cout"], info["shortcut"]) == (cmid, cout, shortcut), desc
    region = torch.zeros(out.shape, dtype=torch.bool, device="cuda")
    region[..., oc:oc + cout] = True
    changed = _bits(first) != _bits(before)
    assert not (changed & ~region).any(), "stores outside the output view"

    xr = view(x, xc, cin)
    za, ya, Sa = conv_ref(xr, wa.double(), ba.double(), 1, 1)
    t = ya.half().double()
    n1 = 9 * info["chunks1"] * info["BK1"] // 16
    n2 = 9 * info["chunks2"] * info["BK2"] // 16
    dt = conv_bound(t, za, Sa, n1, 1)  # stage-1 error before the rounding, plus one ulp of t
    zb, yb, Sb = conv_ref(t, wb.double(), bb.double(), 1, 1, xr if shortcut else None)
    _, prop, _ = conv_ref(dt, wb.double().abs(), torch.zeros_like(bb).double(), 1, 0)
    bound = conv_bound(yb, zb, Sb, n2, 1) + 1.1 * prop
    got = view(first, oc, cout)
    assert not torch.isnan(got).any()
    ratio = float(((got - yb).abs() / bound).max())
    print(f"bneck {cin}->{cmid}->{cout} shortcut {shortcut} {B}x{H}x{W}: {desc}: max err/bound {ratio:.3f}")
    _note("bneck_tc_kernel", ratio, f"{cin}->{cmid}->{cout} sc {shortcut} {B}x{H}x{W}")
    assert ratio <= 1.0, f"err/bound {ratio:.3f}"


@gpu
@pytest.mark.parametrize("cin,cmid,cout,shortcut,reason", [
    (128, 128, 128, 1, "not a fusable 3x3 / 3x3 pair"),
    (64, 64, 64, 0, "one CTA per SM and no shortcut"),
    (48, 48, 48, 0, "one CTA per SM and no shortcut"),
    (64, 32, 32, 1, "shortcut is not the block input"),
])
def test_bneck_f16_refusals(cin, cmid, cout, shortcut, reason):
    import yolosharp_b200.engine as E
    from yolosharp_b200._lib import YbError
    x = torch.zeros(1, 20, 12, cin, dtype=torch.float16, device="cuda")
    wa = torch.zeros(cmid, 3, 3, cin, dtype=torch.float16, device="cuda")
    wb = torch.zeros(cout, 3, 3, cmid, dtype=torch.float16, device="cuda")
    out = _nan_buf((1, 20, 12, cout))
    with pytest.raises(YbError) as ei:
        E.debug_bneck_f16(x, wa, torch.zeros(cmid, device="cuda"), wb, torch.zeros(cout, device="cuda"), out, shortcut=bool(shortcut))
    assert ei.value.status == -6 and reason in str(ei.value), str(ei.value)
    assert (_bits(out) == F16_NAN).all()


# ------------------------------------------------------------------ stem (op 0 of an f16 engine)
STEM_H, STEM_W, STEM_B = 64, 96, 2


@pytest.fixture(scope="module")
def stem_engines():
    """f16 engines of YOLOv8n (stem Cout 16: one short pass) and YOLOv8x (Cout 80: a 64-column pass and a 16-column one)
    with a random stem conv and random BatchNorm statistics."""
    import yolosharp_b200 as y
    from oracle import emul16
    from tests.util import oracle_model
    engines = {}
    for size in ("n", "x"):
        sd = oracle_model("v8", "detect", size).state_dict()
        g = torch.Generator().manual_seed(77)
        cout = sd["model.0.conv.weight"].shape[0]
        sd["model.0.conv.weight"] = torch.randn(cout, 3, 3, 3, generator=g) * 0.4
        sd["model.0.bn.weight"] = torch.rand(cout, generator=g) + 0.5
        sd["model.0.bn.bias"] = torch.randn(cout, generator=g) * 0.5
        sd["model.0.bn.running_mean"] = torch.randn(cout, generator=g) * 0.3
        sd["model.0.bn.running_var"] = torch.rand(cout, generator=g) * 2 + 0.2
        conv = types.SimpleNamespace(weight=sd["model.0.conv.weight"])
        bn = types.SimpleNamespace(weight=sd["model.0.bn.weight"], bias=sd["model.0.bn.bias"],
                                   running_mean=sd["model.0.bn.running_mean"], running_var=sd["model.0.bn.running_var"])
        w, b = emul16.fold_bn(conv, bn)
        e = y.Engine("v8", size, "detect", 80, "f16", 0, STEM_B, STEM_H, STEM_W)
        e.load_state_dict(sd)
        e.finalize()
        engines[size] = (e, w, b)
    yield engines
    for e, _, _ in engines.values():
        e.close()


@gpu
@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("dtype", ["u8", "f16", "f32"])
@pytest.mark.parametrize("size", ["n", "x"])
def test_stem_f16_op(stem_engines, size, dtype, padded):
    """stem_tc_kernel: NCHW u8 / f16 / f32 input, 3x3 s2 conv + folded BN + SiLU -> fp16 NHWC, against float64 on the input
    rounded as stem_load4 / stem_load1 round it.  padded: a (50, 73) image inside the planned 64 x 96 - odd rows take
    stem_load4_ragged, and the right / bottom padding is the value 114 (/ 255) produced in the kernel."""
    from oracle import emul16
    e, w, b = stem_engines[size]
    sh, sw = (50, 73) if padded else (STEM_H, STEM_W)
    g = torch.Generator().manual_seed(5 + padded)
    u8 = torch.randint(0, 256, (STEM_B, 3, sh, sw), dtype=torch.uint8, generator=g)
    pad = (0, STEM_W - sw, 0, STEM_H - sh)
    if dtype == "u8":
        src = u8
        xr = emul16.input_u8(F.pad(u8, pad, value=114))
    else:
        xf = torch.rand(STEM_B, 3, sh, sw, generator=g)
        src = xf.half() if dtype == "f16" else xf
        xr = emul16.r16(F.pad(src.float(), pad, value=114.0 / 255.0))
    e.forward(src.cuda().contiguous())
    torch.cuda.synchronize()
    got = e.read_activation(0, STEM_B).double().permute(0, 2, 3, 1).cuda()
    e.forward(src.cuda().contiguous())
    torch.cuda.synchronize()
    assert torch.equal(e.read_activation(0, STEM_B).double().permute(0, 2, 3, 1).cuda(), got), "repeat differs"
    z, yv, S = conv_ref(xr.double().permute(0, 2, 3, 1).cuda(), w.double().permute(0, 2, 3, 1).cuda(), b.double().cuda(), 2, 1)
    assert got.shape == yv.shape
    ratio = float(((got - yv).abs() / conv_bound(yv, z, S, 3, 1)).max())  # K = 36 padded to 48: three k16 steps per pass
    print(f"stem v8{size} {dtype} padded {padded}: max err/bound {ratio:.3f}")
    _note("stem_tc_kernel", ratio, f"v8{size} {dtype} padded {padded}")
    assert ratio <= 1.0, f"err/bound {ratio:.3f}"


# ------------------------------------------------------------------ CPU
@pytest.mark.parametrize("k,s,act,res", [(3, 1, 1, False), (3, 2, 0, True), (1, 1, 1, True)])
def test_reference_matches_torch_conv2d(k, s, act, res):
    """conv_ref on channel-slice views (pitch, coff) of NHWC buffers equals torch's float64 conv2d on the dense NCHW slice,
    and the ulp16 helper returns the fp16 spacing."""
    g = torch.Generator().manual_seed(3)
    B, H, W, cin, cout, pitch, coff = 2, 9, 7, 24, 8, 40, 8
    buf = torch.randn(B, H, W, pitch, generator=g, dtype=torch.float64)
    w = torch.randn(cout, k, k, cin, generator=g, dtype=torch.float64)
    b = torch.randn(cout, generator=g, dtype=torch.float64)
    Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
    rbuf = torch.randn(B, Ho, Wo, 3 * cout, generator=g, dtype=torch.float64)
    r = view(rbuf, cout, cout) if res else None
    z, yv, S = conv_ref(view(buf, coff, cin), w, b, s, act, r)
    zt = F.conv2d(buf[..., coff:coff + cin].permute(0, 3, 1, 2), w.permute(0, 3, 1, 2), b, s, k // 2).permute(0, 2, 3, 1)
    torch.testing.assert_close(z, zt, rtol=1e-12, atol=1e-12)
    yt = (F.silu(zt) if act else zt) + (rbuf[..., cout:2 * cout] if res else 0)
    torch.testing.assert_close(yv, yt, rtol=1e-12, atol=1e-12)
    St = F.conv2d(buf[..., coff:coff + cin].abs().permute(0, 3, 1, 2), w.abs().permute(0, 3, 1, 2), b.abs(), s, k // 2)
    torch.testing.assert_close(S, St.permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
    v = torch.tensor([1.0, 1.5, 2.0, -3.0, 65504.0, 1e-6, 0.0], dtype=torch.float64)
    assert ulp16(v).tolist() == [2.0 ** -10, 2.0 ** -10, 2.0 ** -9, 2.0 ** -9, 32.0, 2.0 ** -24, 2.0 ** -24]


def test_decode_reference_plain():
    """decode_ref's DFL box decode against a per-anchor restatement of the DFL expectation and dist2bbox."""
    g = torch.Generator().manual_seed(4)
    B, Hl, Wl = 2, 3, 5
    z = torch.randn(B, Hl * Wl, 64, generator=g, dtype=torch.float64) * 3
    v, e = decode_ref(z, z.abs(), EPI_DFL_BOX, 4, 8.0, Wl)
    for n in range(B):
        for i in range(Hl * Wl):
            d = [sum(j * p for j, p in enumerate(torch.softmax(z[n, i, 16 * sd:16 * sd + 16], 0).tolist())) for sd in range(4)]
            ax, ay = i % Wl + 0.5, i // Wl + 0.5
            want = [(ax + (d[2] - d[0]) / 2) * 8, (ay + (d[3] - d[1]) / 2) * 8, (d[0] + d[2]) * 8, (d[1] + d[3]) * 8]
            assert torch.allclose(v[n, :, i], torch.tensor(want, dtype=torch.float64), rtol=1e-12, atol=1e-12)
    assert (e > 0).all()
    vs, _ = decode_ref(z[..., :8], z[..., :8].abs(), EPI_SIGMOID, 4, 8.0, Wl)
    torch.testing.assert_close(vs, torch.sigmoid(z[..., :8]).transpose(1, 2))


def _args_conv(lib, **over):
    """yb_debug_conv_f16 arguments of a valid 3x3 32 -> 32 conv on non-null (never dereferenced) pointers"""
    fake = C.c_void_p(256)
    a = dict(inp=fake, plan_batch=2, run_batch=2, H=8, W=8, in_pitch=32, in_coff=0, cin=32, w=fake, bias=fake, cout=32, k=3,
             s=1, act=1, res=None, res_pitch=0, res_coff=0, out=fake, out_pitch=32, out_coff=0, share=0, ctr=1, mode=0, A=0,
             Ctot=0, a0=0, ch0=0, Wl=0, HW=0, stride=0.0, pred=None, desc=None, cap=0)
    a.update(over)
    return lib.yb_debug_conv_f16(*a.values())


def _args_bneck(lib, **over):
    fake = C.c_void_p(256)
    a = dict(x=fake, B=1, H=8, W=8, pitch=32, coff=0, cin=32, wa=fake, ba=fake, cmid=32, wb=fake, bb=fake, cout=32, sc=1,
             out=fake, out_pitch=32, out_coff=0, desc=None, cap=0)
    a.update(over)
    return lib.yb_debug_bneck_f16(*a.values())


def test_debug_entry_points_refuse_bad_arguments(built_lib):
    """Both entry points validate before they touch the device: an error code and a message, never a crash."""
    from yolosharp_b200 import _lib as L
    lib = L.lib()
    for over in (dict(inp=None), dict(w=None), dict(bias=None), dict(out=None), dict(mode=EPI_RAW, pred=None),
                 dict(run_batch=3), dict(run_batch=0), dict(in_pitch=16), dict(k=5), dict(act=2), dict(mode=4),
                 dict(out_coff=8), dict(res=C.c_void_p(256), res_pitch=16)):
        assert _args_conv(lib, **over) == -1, over
        assert b"yb_debug_conv_f16" in lib.yb_last_error()
    for over in (dict(cin=24, in_pitch=24), dict(cout=40, out_pitch=40), dict(in_coff=4, in_pitch=40), dict(s=3), dict(k=1, s=2)):
        assert _args_conv(lib, **over) == -6, over
        assert b"not supported" in lib.yb_last_error()
    for over in (dict(x=None), dict(wa=None), dict(bb=None), dict(out=None), dict(B=0), dict(pitch=16), dict(out_coff=8)):
        assert _args_bneck(lib, **over) == -1, over
    for over in (dict(cin=24, pitch=24), dict(cmid=40), dict(coff=4, pitch=40)):
        assert _args_bneck(lib, **over) == -6, over
    if not torch.cuda.is_available():
        assert _args_conv(lib) == -7 and b"no CUDA device" in lib.yb_last_error()
        assert _args_bneck(lib) == -7 and b"no CUDA device" in lib.yb_last_error()
