"""Op-level tests of the TF32 training convolutions of csrc/conv_tf32.cu against a float64 reference of the same operation:
tf_conv_kernel (forward, stride-1 and stride-2 data gradient) and tf_wgrad_kernel + tf_wgrad_fold_kernel (weight gradient)
through yb_debug_conv_tf32, their fp32 CUDA-core twins (yb_conv_forward_f32, yb_conv_backward_data / _weight) and the fp32
stem (yb_stem_conv_forward_f32 / _backward_weight_f32).

Operands are TF32-representable (the low 13 mantissa bits cleared), so the tensor core's operand conversion is the
identity whether it truncates or rounds, and every product is exact in fp32 and float64.  Their magnitudes are spread
over 2^-8 .. 2^8 per channel and per pixel, so an error confined to a small channel stands out against its own elements.
The reference is a float64 sum over taps of shifted matrix products (not torch's convolution); S is the same sum over
absolute values (+ |b|).  Every output element must satisfy

    |got - y| <= n_k 2^-23 S

  forward / dgrad   n_k = ntaps * chunks * BK / 8 k8 MMA steps of the launch that wrote the element, + 1 for the fp32 bias
                    add.  Each step rounds the fp32 accumulator (|partial sum| <= S) once: 2^-24 S, doubled for the tensor
                    core's internal alignment of the products.
  wgrad             n_k = 8 ceil(pix_tiles / splits) k8 steps of one split + splits for the fp32 fold of the partials.
  fp32 twins, stem  n 2^-24 S, n the longest fp32 FMA / add chain of the kernel (see the *_chain helpers).
The plan values come from the launch descriptions the entry returns (the split count depends on the SM count).

Per case, besides the bound: integer operands make every partial sum an integer below 2^24, so every pass must equal the
float64 result exactly; NaN sentinels - input channels outside a pitched view, guard regions around every buffer, NaN
prefilled outputs (every element must be written; the odd parities of a 1x1 stride-2 dgrad must be exactly 0) and a NaN
prefilled workspace (padded partial rows must never reach dw); a second call is bitwise identical (the wgrad fold too).
The largest err / bound of each kernel and pass is printed; test_conv_tf32_plan_coverage asserts that the sweep reaches
every planner branch it is meant to pin."""
import ctypes as C
import math
import re
import zlib

import pytest
import torch
import torch.nn.functional as F

gpu = pytest.mark.gpu

F32_NAN = 0x7FC00000
GUARD = 256          # NaN elements before and after every device buffer of a case
ERR_INVALID_ARG, ERR_SHAPE, ERR_NO_DEVICE = -1, -6, -7


# ------------------------------------------------------------------ float64 reference
def tf32(t):
    """float32 t with the low 13 mantissa bits cleared: TF32-representable, truncated toward zero"""
    return (t.float().contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def tf32_rne(t):
    """float32 t rounded to the nearest TF32 value, ties to even (finite inputs)"""
    b = t.float().contiguous().view(torch.int32)
    return ((b + 0xFFF + ((b >> 13) & 1)) & ~0x1FFF).view(torch.float32)


def _taps(k, s, Ho, Wo):
    for kh in range(k):
        for kw in range(k):
            yield kh, kw, (slice(None), slice(kh, kh + s * (Ho - 1) + 1, s), slice(kw, kw + s * (Wo - 1) + 1, s))


def out_hw(H, W, k, s):
    p = k // 2
    return (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1


def fwd_ref(x, w, b, s):
    """x (N, H, W, Cin), w (Cout, Cin, k, k), b (Cout) or None, float64; pad k // 2 -> z (N, Ho, Wo, Cout), S"""
    N, H, W, _ = x.shape
    cout, _, k, _ = w.shape
    p = k // 2
    Ho, Wo = out_hw(H, W, k, s)
    xp = F.pad(x, (0, 0, p, p, p, p))
    z = x.new_zeros(N, Ho, Wo, cout)
    S = x.new_zeros(N, Ho, Wo, cout)
    if b is not None:
        z += b
        S += b.abs()
    for kh, kw, sl in _taps(k, s, Ho, Wo):
        tap, wt = xp[sl], w[:, :, kh, kw]
        z += tap @ wt.T
        S += tap.abs() @ wt.abs().T
    return z, S


def dgrad_ref(dz, w, H, W, s):
    """dz (N, Ho, Wo, Cout), w (Cout, Cin, k, k) -> dx (N, H, W, Cin), S: each tap scatters dz @ W[kh][kw] back onto the
    input positions it read"""
    N, Ho, Wo, _ = dz.shape
    _, cin, k, _ = w.shape
    p = k // 2
    dxp = dz.new_zeros(N, H + 2 * p, W + 2 * p, cin)
    Sp = torch.zeros_like(dxp)
    for kh, kw, sl in _taps(k, s, Ho, Wo):
        wt = w[:, :, kh, kw]
        dxp[sl] += dz @ wt
        Sp[sl] += dz.abs() @ wt.abs()
    return dxp[:, p:p + H, p:p + W], Sp[:, p:p + H, p:p + W]


def wgrad_ref(x, dz, k, s):
    """x (N, H, W, Cin), dz (N, Ho, Wo, Cout) -> dw (Cout, Cin, k, k), S"""
    cin, cout = x.shape[3], dz.shape[3]
    Ho, Wo = dz.shape[1:3]
    p = k // 2
    xp = F.pad(x, (0, 0, p, p, p, p))
    d2 = dz.reshape(-1, cout)
    dw = x.new_zeros(cout, cin, k, k)
    S = torch.zeros_like(dw)
    for kh, kw, sl in _taps(k, s, Ho, Wo):
        tap = xp[sl].reshape(-1, cin)
        dw[:, :, kh, kw] = d2.T @ tap
        S[:, :, kh, kw] = d2.abs().T @ tap.abs()
    return dw, S


def err_ratio(got, ref, bound):
    """largest |got - ref| / bound; where the bound is 0 (every product 0) the result must be exact"""
    err = (got.double() - ref).abs()
    zero = bound == 0
    assert not (err[zero] > 0).any(), f"{int((err[zero] > 0).sum())} elements with S = 0 are not exactly 0"
    return float((err[~zero] / bound[~zero]).max()) if (~zero).any() else 0.0


# ------------------------------------------------------------------ plan descriptions
CONV_RE = re.compile(r"tf_conv_kernel BK (\d+) chunks (\d+) n_tile (\d+) x(\d+) BW (\d+) BH (\d+) in_stride (\d+) flat (\d+) "
                     r"ntaps (\d+) occ (\d+) stages (\d+) grid (\d+)$")
CONV_KEYS = ("BK", "chunks", "n_tile", "n_tiles", "BW", "BH", "in_stride", "flat", "ntaps", "occ", "stages", "grid")
WG_RE = re.compile(r"tf_wgrad_kernel halo (\d+) tpc (\d+) nb (\d+) co_tiles (\d+) ci_tiles (\d+) co_blocks (\d+) splits (\d+) "
                   r"pix_tiles (\d+) b_stages (\d+) grid (\d+)$")
WG_KEYS = ("halo", "tpc", "nb", "co_tiles", "ci_tiles", "co_blocks", "splits", "pix_tiles", "b_stages", "grid")


def parse_desc(desc):
    lines = []
    for line in desc.split("\n"):
        m, keys = (CONV_RE.match(line), CONV_KEYS) if line.startswith("tf_conv") else (WG_RE.match(line), WG_KEYS)
        assert m, line
        lines.append(dict(zip(keys, map(int, m.groups()))))
    return lines


def conv_nk(line):
    return line["ntaps"] * line["chunks"] * line["BK"] // 8 + 1


def dgrad_nk(lines, H, W, k, s):
    """k8 steps + 1 per element of dx: stride 2 writes each output parity (py, px) with its own launch, in this order"""
    if s == 1:
        assert len(lines) == 1
        return torch.full((1, H, W, 1), float(conv_nk(lines[0])), dtype=torch.float64)
    parities = [(0, 0), (0, 1), (1, 0), (1, 1)] if k == 3 else [(0, 0)]  # 1x1: the other parities receive no tap
    assert len(lines) == len(parities), lines
    nk = torch.zeros(1, H, W, 1, dtype=torch.float64)
    for (py, px), line in zip(parities, lines):
        nk[:, py::2, px::2] = conv_nk(line)
    return nk


def wgrad_nk(line):
    return 8 * -(-line["pix_tiles"] // line["splits"]) + line["splits"]


# ------------------------------------------------------------------ fp32 twins: chain lengths
def twin_wgrad_chain(N, Ho, Wo, cin, cout, k):
    """conv_backward_weight (csrc/bn_train.cu): a serial FMA chain over one slab of output rows, then the fold of the slabs"""
    dw_size = cout * cin * k * k
    slabs = max(1, min(64, N * Ho * Wo // 2048))
    slabs = max(1, min(slabs, (16 << 20) // dw_size))
    slabs = min(slabs, N * Ho)
    rows = -(-N * Ho // slabs)
    slabs = -(-N * Ho // rows)
    return rows * Wo + slabs


def stem_wgrad_chain(N, Ho, Wo):
    """stem3_wgrad_partial_kernel: per thread ceil(npx / 8) FMAs of each of its block's tiles (ST_WG_BLOCKS = 592 blocks
    stride over the N * Ho * ceil(Wo / 128) row segments), then the fold of the 8 warps and of the 592 block partials"""
    tiles = N * Ho * -(-Wo // 128)
    return -(-tiles // 592) * -(-min(Wo, 128) // 8) + 8 + 592


# ------------------------------------------------------------------ device buffers with NaN guards
def _nan(n):
    return torch.full((n,), F32_NAN, dtype=torch.int32, device="cuda").view(torch.float32)


def _bits(t):
    return t.contiguous().view(torch.int32)


class Guarded:
    """A float32 tensor of `shape` inside a NaN-filled buffer with GUARD NaN elements before and after it."""

    def __init__(self, shape, values=None):
        self.n = math.prod(shape)
        self.buf = _nan(self.n + 2 * GUARD)
        self.t = self.buf[GUARD:GUARD + self.n].view(shape)
        if values is not None:
            self.t.copy_(values)

    def reset(self):
        _bits(self.buf).fill_(F32_NAN)

    def guards_intact(self):
        b = _bits(self.buf)
        return bool((b[:GUARD] == F32_NAN).all()) and bool((b[GUARD + self.n:] == F32_NAN).all())


def _vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


# ------------------------------------------------------------------ cases
def case(name, N, H, W, cin, cout, k, s, view=None):
    """view = (pitch, c0): x is channels [c0, c0 + cin) of an NHWC buffer `pitch` channels wide"""
    return dict(name=name, N=N, H=H, W=W, cin=cin, cout=cout, k=k, s=s, view=view)


CASES = [
    case("bk8_9x13", 2, 9, 13, 8, 8, 3, 1),                  # BK 8, n_tile 16 with 8 stored columns, partial 8x8 pixel tiles
    case("bk16_ragged", 2, 16, 24, 24, 40, 3, 1),            # BK 16, second chunk 8 of 16; n_tile 48
    case("bk32_ragged_20x20", 2, 20, 20, 48, 80, 3, 1),      # BK 32 ragged (32 + 16), rectangle tiles on 20 x 20
    case("chunks3_40x24", 1, 40, 24, 96, 144, 3, 1),         # 3 chunks; wgrad ci_tiles 3, co_tiles 2 (second tile 16 wide)
    case("ntiles2_k2880", 2, 12, 20, 320, 328, 3, 1),        # two N tiles forward and dgrad
    case("ntile256_splits1", 1, 8, 8, 64, 256, 3, 1),        # n_tile 256; one pixel tile: splits = 1
    case("s2_c128_n256", 2, 20, 20, 128, 256, 3, 2),         # stride 2: dgrad parities with 1 / 2 / 2 / 4 taps
    case("s2_c16_18x30", 2, 18, 30, 16, 24, 3, 2),           # stride 2, non-halo wgrad, BK 16 / 8
    case("s2_odd_17x31", 2, 17, 31, 16, 24, 3, 2),           # odd extents: forward and wgrad; the dgrad refusal
    case("flat_c32_2x24x40", 2, 24, 40, 32, 32, 1, 1),       # flat 1x1, B*H*W a multiple of 128
    case("flat_c384_3x7x11", 3, 7, 11, 384, 64, 1, 1),       # flat 1x1, B*H*W not one; wgrad nb 4 x ci_tiles 3
    case("s2_1x1", 2, 16, 16, 24, 40, 1, 2),                 # 1x1 stride 2: non-flat forward, one dgrad launch
    case("nb2_n136", 2, 9, 13, 64, 136, 1, 1),               # wgrad nb 2; co_tiles 2 with 8 channels in the second
    case("nb3_c96", 2, 9, 13, 96, 64, 1, 1),                 # wgrad nb 3
    case("nb4_c160", 2, 9, 13, 160, 40, 1, 1),               # wgrad nb 4 + a ragged second ci tile
    case("one_pixel", 1, 1, 1, 32, 32, 3, 1),                # every tap but the centre is padding
    case("wide_row_200", 1, 3, 200, 32, 48, 3, 1),           # Wo > 128: several tiles across one row
    case("occ2_96x96", 8, 96, 96, 32, 32, 3, 1),             # two CTAs per SM
    case("v8n_80x80", 4, 80, 80, 64, 64, 3, 1),              # a YOLOv8n layer at 320^2: wgrad over 25 600 pixels
    case("view_halo", 2, 18, 26, 48, 64, 3, 1, view=(80, 16)),
    case("view_flat_c2f", 2, 9, 13, 64, 32, 1, 1, view=(128, 64)),
    case("view_s2", 2, 20, 20, 32, 64, 3, 2, view=(96, 32)),
]
# the three layouts on which the TF32 kernels were first pinned bit-exact (against the fp32 twins, on small integers)
INTEGER_LAYOUT_CASES = [
    case("int_20x20_c32", 2, 20, 20, 32, 48, 3, 1),
    case("int_s2_16x16", 2, 16, 16, 16, 24, 3, 2),
    case("int_1x1_12x12", 1, 12, 12, 64, 64, 1, 1),
]
CASE_BY_NAME = {c["name"]: c for c in CASES + INTEGER_LAYOUT_CASES}
PLANS = {}   # (case, pass) -> list of launch descriptions (filled by the sweep, read by the coverage test)
WORST = {}   # kernel / pass -> (largest err / bound, case)


def _note(kernel, ratio, name):
    if ratio > WORST.get(kernel, (-1.0, ""))[0]:
        WORST[kernel] = (ratio, name)


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for kernel, (ratio, name) in sorted(WORST.items()):
        print(f"worst err/bound of {kernel}: {ratio:.3f} ({name})")


def operands(c, data, seed_extra=""):
    """x (N, H, W, Cin), w (Cout, Cin, k, k), dz (N, Ho, Wo, Cout), b (Cout): float32 on the CPU.  'integer': small integers;
    'random' / 'raw': normal values scaled by 2^-4 .. 2^4 per channel and per pixel, TF32-rounded for 'random' only."""
    g = torch.Generator().manual_seed(zlib.crc32((c["name"] + data + seed_extra).encode()))
    N, H, W, cin, cout, k, s = (c[n] for n in ("N", "H", "W", "cin", "cout", "k", "s"))
    Ho, Wo = out_hw(H, W, k, s)
    if data == "integer":
        ri = lambda lo, hi, *shape: torch.randint(lo, hi + 1, shape, generator=g).float()
        return ri(-4, 4, N, H, W, cin), ri(-3, 3, cout, cin, k, k), ri(-2, 2, N, Ho, Wo, cout), ri(-8, 8, cout)
    spread = lambda *shape: torch.exp2(torch.randint(-4, 5, shape, generator=g).float())
    x = torch.randn(N, H, W, cin, generator=g) * spread(1, 1, 1, cin) * spread(N, H, W, 1)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5 * spread(cout, 1, 1, 1)
    dz = torch.randn(N, Ho, Wo, cout, generator=g) * spread(1, 1, 1, cout) * spread(N, Ho, Wo, 1)
    b = torch.randn(cout, generator=g) * spread(cout)
    if data == "raw":
        return x, w, dz, b
    return tf32(x), tf32(w), tf32(dz), b


class Bufs:
    """The operands of a case on the device: x (pitched inside NaN channels for a view case), w, dz, b, each guarded."""

    def __init__(self, c, x, w, dz, b):
        pitch, c0 = c["view"] or (c["cin"], 0)
        self.xg = Guarded((c["N"], c["H"], c["W"], pitch))
        self.xg.t[..., c0:c0 + c["cin"]] = x.cuda()
        self.x = self.xg.t[..., c0:c0 + c["cin"]] if c["view"] else self.xg.t
        self.wg, self.dzg, self.bg = Guarded(w.shape, w.cuda()), Guarded(dz.shape, dz.cuda()), Guarded(b.shape, b.cuda())
        self.w, self.dz, self.b = self.wg.t, self.dzg.t, self.bg.t

    def intact(self):
        return all(g.guards_intact() for g in (self.xg, self.wg, self.dzg, self.bg))


def out_shape(c, pss):
    N, H, W, cin, cout, k, s = (c[n] for n in ("N", "H", "W", "cin", "cout", "k", "s"))
    return [(N, *out_hw(H, W, k, s), cout), (N, H, W, cin), (cout, cin, k, k)][pss]


def dgrad_supported(c):
    return c["s"] == 1 or not ((c["H"] | c["W"]) & 1)


def run_tf32_pass(c, d, pss, ws):
    """Runs one pass twice on NaN-prefilled out and workspace; checks the guards, full coverage, repeatability; -> (out, desc)"""
    import yolosharp_b200.engine as E
    out = Guarded(out_shape(c, pss))
    kw = dict(w=d.w if pss != 2 else None, x=d.x if pss != 1 else None, dz=d.dz if pss != 0 else None,
              bias=d.b if pss == 0 else None, stride=c["s"], workspace=ws)

    def call():
        ws.fill_(255)  # every 4-byte word a NaN
        out.reset()
        return E.debug_conv_tf32(pss, out.t, **kw)

    desc = call()
    first = out.t.clone()
    assert call() == desc
    assert torch.equal(_bits(out.t), _bits(first)), "a repeated call is not bitwise identical"
    assert out.guards_intact(), "stores outside the output"
    assert not torch.isnan(first).any(), f"{int(torch.isnan(first).sum())} output elements not written (or NaN read)"
    return first.cpu(), desc


PASS_NAMES = ("forward", "dgrad", "wgrad")


def check_case(c, data):
    """All three TF32 passes (or the refusal of a stride-2 dgrad on odd extents) and the three fp32 twins of case c."""
    import yolosharp_b200.engine as E
    from yolosharp_b200._lib import YbError
    N, H, W, cin, cout, k, s = (c[n] for n in ("N", "H", "W", "cin", "cout", "k", "s"))
    integer = data == "integer"
    x, w, dz, b = operands(c, data)
    d = Bufs(c, x, w, dz, b)
    ws = torch.empty(max(int(E.L.lib().yb_conv_tc_workspace_bytes(N, H, W, cin, cout, k, s)), 256), dtype=torch.uint8,
                     device="cuda")
    x64, w64, dz64, b64 = x.double(), w.double(), dz.double(), b.double()
    refs = [fwd_ref(x64, w64, b64, s), dgrad_ref(dz64, w64, H, W, s) if dgrad_supported(c) else None, wgrad_ref(x64, dz64, k, s)]
    for pss in range(3):
        if refs[pss] is None:
            out = Guarded(out_shape(c, 1))
            with pytest.raises(YbError) as ei:
                E.debug_conv_tf32(1, out.t, w=d.w, dz=d.dz, stride=s, workspace=ws)
            assert ei.value.status == ERR_SHAPE and "even extents" in str(ei.value), str(ei.value)
            assert (_bits(out.buf) == F32_NAN).all()
            continue
        got, desc = run_tf32_pass(c, d, pss, ws)
        lines = parse_desc(desc)
        PLANS[(c["name"], pss)] = lines
        y, S = refs[pss]
        if pss == 0:
            assert len(lines) == 1
            nk = conv_nk(lines[0])
        elif pss == 1:
            nk = dgrad_nk(lines, H, W, k, s)
            if k == 1 and s == 2:
                assert (got[:, 1::2] == 0).all() and (got[:, :, 1::2] == 0).all(), "odd parities of a 1x1 s2 dgrad not zeroed"
        else:
            assert len(lines) == 1
            nk = wgrad_nk(lines[0])
        ratio = err_ratio(got, y, nk * 2.0 ** -23 * S)
        print(f"{c['name']} [{data}] {PASS_NAMES[pss]}: {desc.replace(chr(10), ' | ')}: max err/bound {ratio:.3f}")
        if integer:
            assert torch.equal(got.double(), y), \
                f"{PASS_NAMES[pss]} not exact on integer operands: {int((got.double() != y).sum())} elements differ"
        else:
            _note(f"tf32 {PASS_NAMES[pss]}", ratio, c["name"])
        assert ratio <= 1.0, f"{PASS_NAMES[pss]}: err/bound {ratio:.3f}"
    assert d.intact(), "an input buffer's guard region changed"
    check_twins(c, data, d, refs)


def check_twins(c, data, d, refs):
    """yb_conv_forward_f32 / yb_conv_backward_data / yb_conv_backward_weight on the same operands (x dense), bound n 2^-24 S"""
    from yolosharp_b200 import _lib as L
    N, H, W, cin, cout, k, s = (c[n] for n in ("N", "H", "W", "cin", "cout", "k", "s"))
    Ho, Wo = out_hw(H, W, k, s)
    lib = L.lib()
    x = Guarded((N, H, W, cin), d.x)
    wp = Guarded((k, k, cin, cout), d.w.permute(2, 3, 1, 0))  # the generic kernel's [tap][Cin][Cout]
    outs = [Guarded(out_shape(c, p)) for p in range(3)]
    L.check(lib.yb_conv_forward_f32(_vp(x.t), _vp(wp.t), _vp(d.b), N, H, W, cin, cout, k, s, k // 2, _vp(outs[0].t), None))
    L.check(lib.yb_conv_backward_data(_vp(d.dz), _vp(d.w), N, H, W, cin, cout, k, s, k // 2, _vp(outs[1].t), None))
    L.check(lib.yb_conv_backward_weight(_vp(x.t), _vp(d.dz), N, H, W, cin, cout, k, s, k // 2, _vp(outs[2].t), None))
    torch.cuda.synchronize()
    chains = [k * k * cin + 1, k * k * cout, twin_wgrad_chain(N, Ho, Wo, cin, cout, k)]
    names = ("conv_generic_kernel", "conv_dgrad_kernel", "conv_wgrad_kernel")
    if not dgrad_supported(c):  # the fp32 dgrad takes odd stride-2 extents
        refs = [refs[0], dgrad_ref(d.dz.double().cpu(), d.w.double().cpu(), H, W, s), refs[2]]
    for p in range(3):
        assert outs[p].guards_intact(), f"{names[p]}: stores outside the output"
        got = outs[p].t.cpu()
        assert not torch.isnan(got).any(), f"{names[p]}: output not fully written"
        y, S = refs[p]
        ratio = err_ratio(got, y, chains[p] * 2.0 ** -24 * S)
        print(f"{c['name']} [{data}] {names[p]}: chain {chains[p]}: max err/bound {ratio:.3f}")
        if data == "integer":
            assert torch.equal(got.double(), y), f"{names[p]} not exact on integer operands"
        else:
            _note(names[p], ratio, c["name"])
        assert ratio <= 1.0, f"{names[p]}: err/bound {ratio:.3f}"


@gpu
@pytest.mark.parametrize("data", ["random", "integer"])
@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_conv_tf32_op(name, data):
    check_case(CASE_BY_NAME[name], data)


@gpu
def test_conv_tf32_exact_on_integer_operands():
    """On small-integer operands every partial sum is exact in fp32, so all three TF32 passes and the fp32 twins must equal
    float64 exactly: layout, swizzle or indexing errors cannot hide in rounding.  The random operands of the same cases
    are held to the per-element bound."""
    for c in INTEGER_LAYOUT_CASES:
        for data in ("integer", "random"):
            check_case(c, data)


@gpu
def test_conv_tf32_plan_coverage():
    """The sweep reaches every planner branch it is meant to pin: a planner change that moves the cases off one fails here
    instead of silently shrinking the coverage.  Split counts are not hard-coded: they follow the SM count."""
    for name, c in CASE_BY_NAME.items():
        if not any(key[0] == name for key in PLANS):
            check_case(c, "integer")
    conv, wg = [], []  # (case, pass, line)
    for (name, pss), lines in PLANS.items():
        for line in lines:
            (wg if pss == 2 else conv).append((CASE_BY_NAME[name], pss, line))
    seen = lambda rows, key: {line[key] for _, _, line in rows}
    assert seen(conv, "BK") >= {8, 16, 32}, seen(conv, "BK")
    kc = lambda c, pss: c["cin"] if pss == 0 else c["cout"]
    assert any(line["chunks"] * line["BK"] > kc(c, pss) for c, pss, line in conv), "no ragged last chunk"
    assert max(seen(conv, "n_tiles")) >= 2 and 256 in seen(conv, "n_tile")
    assert seen(conv, "flat") == {0, 1}
    assert any(pss == 0 and not line["flat"] and line["BW"] < out_hw(c["H"], c["W"], c["k"], c["s"])[1] and
               out_hw(c["H"], c["W"], c["k"], c["s"])[1] > 128 for c, pss, line in conv), "no row wider than one tile"
    assert 2 in seen(conv, "in_stride")
    assert seen(conv, "occ") == {1, 2}, seen(conv, "occ")
    dgrads = {name: [l["ntaps"] for l in lines] for (name, pss), lines in PLANS.items() if pss == 1}
    assert any(sorted(t) == [1, 2, 2, 4] for t in dgrads.values()), "no four-launch stride-2 dgrad"
    assert any(CASE_BY_NAME[n]["k"] == 1 and CASE_BY_NAME[n]["s"] == 2 and t == [1] for n, t in dgrads.items())
    assert seen(wg, "halo") == {0, 1} and seen(wg, "tpc") == {1, 3}
    assert seen(wg, "nb") >= {1, 2, 3, 4}, seen(wg, "nb")
    assert max(seen(wg, "ci_tiles")) >= 2 and max(seen(wg, "co_tiles")) >= 2
    assert min(seen(wg, "co_blocks")) < 4
    splits = seen(wg, "splits")
    assert 1 in splits and max(splits) > 1, splits
    assert any(h % 8 or w % 8 for h, w in (out_hw(c["H"], c["W"], c["k"], c["s"]) for c, _, _ in wg))
    assert any(c["view"] for c, pss, _ in conv if pss == 0) and any(c["view"] for c, _, _ in wg), "no pitched input"


@gpu
def test_tf32_operand_truncation():
    """DESIGN 4.3: the tensor core drops the low 13 mantissa bits of each fp32 operand.  With raw fp32 operands the forward
    and dgrad (wgmma) and wgrad (mma.sync) results must meet the bound against float64 on operands truncated toward zero
    to 10 mantissa bits; the ratio against operands rounded to nearest is printed next to it."""
    import yolosharp_b200.engine as E
    c = case("raw_16x24", 2, 16, 24, 48, 40, 3, 1)
    x, w, dz, b = operands(c, "raw")
    d = Bufs(c, x, w, dz, b)
    ws = torch.empty(int(E.L.lib().yb_conv_tc_workspace_bytes(2, 16, 24, 48, 40, 3, 1)), dtype=torch.uint8, device="cuda")
    results = []
    for pss in range(3):
        got, desc = run_tf32_pass(c, d, pss, ws)
        line = parse_desc(desc)
        ratios = {}
        for mode, rnd in (("truncated", tf32), ("rounded", tf32_rne)):
            xr, wr, dzr = (rnd(t).double() for t in (x, w, dz))
            if pss == 0:
                (y, S), nk = fwd_ref(xr, wr, b.double(), 1), conv_nk(line[0])
            elif pss == 1:
                (y, S), nk = dgrad_ref(dzr, wr, 16, 24, 1), conv_nk(line[0])
            else:
                (y, S), nk = wgrad_ref(xr, dzr, 3, 1), wgrad_nk(line[0])
            ratios[mode] = err_ratio(got, y, nk * 2.0 ** -23 * S)
        print(f"raw fp32 operands, {PASS_NAMES[pss]}: err/bound against truncated operands {ratios['truncated']:.3f}, "
              f"against rounded operands {ratios['rounded']:.3f}")
        results.append((PASS_NAMES[pss], ratios))
    for pname, ratios in results:
        assert ratios["truncated"] <= 1.0, f"{pname}: the tensor core does not truncate its operands: {ratios}"


@gpu
@pytest.mark.parametrize("name", ["bk32_ragged_20x20", "s2_c128_n256"])
def test_public_entry_points_match_debug_entry(name):
    """yb_conv_forward_tc / _backward_data_tc / _backward_weight_tc run the same launches as the debug entry: bit-identical."""
    import yolosharp_b200.engine as E
    c = CASE_BY_NAME[name]
    x, w, dz, b = (t.cuda() for t in operands(c, "random", "public"))
    ws = E.ConvWorkspace(x.device)
    z = E.conv_forward_tc(x, w, b, c["s"], ws=ws)
    dx, dw = E.conv_backward_tc(x, dz, w, c["s"], ws=ws)
    torch.cuda.synchronize()
    outs = [torch.empty_like(z), torch.empty_like(dx), torch.empty_like(dw)]
    E.debug_conv_tf32(0, outs[0], w=w, x=x, bias=b, stride=c["s"])
    E.debug_conv_tf32(1, outs[1], w=w, dz=dz, stride=c["s"])
    E.debug_conv_tf32(2, outs[2], x=x, dz=dz, stride=c["s"])
    for got, want in zip(outs, (z, dx, dw)):
        assert torch.equal(_bits(got), _bits(want))


# ------------------------------------------------------------------ the fp32 stem
STEM_CASES = [  # (N, H, W, C, x_channels)
    (2, 64, 96, 16, 3), (1, 32, 32, 32, 8), (2, 40, 24, 80, 8), (1, 640, 640, 32, 8),
    (2, 18, 22, 8, 3),        # C = 8: one 32-channel group, 24 idle lanes
    (1, 32, 300, 48, 8),      # C = 48 (CG 2); Wo = 150: a 128-pixel row segment and a 22-pixel one
    (2, 20, 270, 96, 3),      # C = 96 (CG 3); Wo = 135
    (1, 10, 260, 128, 8),     # C = 128 (CG 4); Wo = 130
]


@gpu
@pytest.mark.parametrize("data", ["random", "integer"])
@pytest.mark.parametrize("N,H,W,Cc,xc", STEM_CASES)
def test_stem_f32_op(N, H, W, Cc, xc, data):
    """stem3_forward (27-FMA chain per output) and stem3_backward_weight (stem_wgrad_chain) against float64; channels 3 ..
    xc - 1 of the input are NaN and must never be used."""
    from yolosharp_b200 import _lib as L
    lib = L.lib()
    c = case(f"stem_{N}x{H}x{W}_c{Cc}_x{xc}", N, H, W, 3, Cc, 3, 2)
    x, w, dz, _ = operands(c, data)
    xg = Guarded((N, H, W, xc))
    xg.t[..., :3] = x.cuda()
    wg, dzg = Guarded(w.shape, w.cuda()), Guarded(dz.shape, dz.cuda())
    Ho, Wo = H // 2, W // 2
    z, dw = Guarded((N, Ho, Wo, Cc)), Guarded((Cc, 3, 3, 3))
    ws = torch.empty(592 * 27 * Cc * 4, dtype=torch.uint8, device="cuda")

    def call():
        z.reset()
        dw.reset()
        ws.fill_(255)
        L.check(lib.yb_stem_conv_forward_f32(_vp(xg.t), xc, _vp(wg.t), N, H, W, Cc, _vp(z.t), None))
        L.check(lib.yb_stem_conv_backward_weight_f32(_vp(xg.t), xc, _vp(dzg.t), N, H, W, Cc, _vp(dw.t), _vp(ws), ws.numel(), None))
        torch.cuda.synchronize()
        return z.t.clone(), dw.t.clone()

    z1, dw1 = call()
    z2, dw2 = call()
    assert torch.equal(_bits(z1), _bits(z2)) and torch.equal(_bits(dw1), _bits(dw2)), "a repeated call is not bitwise identical"
    assert all(g.guards_intact() for g in (xg, wg, dzg, z, dw))
    (y, S), (dy, dS) = fwd_ref(x.double(), w.double(), None, 2), wgrad_ref(x.double(), dz.double(), 3, 2)
    for kname, got, ref, Sx, n in (("stem3_forward", z1, y, S, 27), ("stem3_backward_weight", dw1, dy, dS, stem_wgrad_chain(N, Ho, Wo))):
        got = got.cpu()
        assert not torch.isnan(got).any(), f"{kname}: output not fully written (or a NaN channel read)"
        ratio = err_ratio(got, ref, n * 2.0 ** -24 * Sx)
        print(f"{c['name']} [{data}] {kname}: chain {n}: max err/bound {ratio:.3f}")
        if data == "integer":
            assert torch.equal(got.double(), ref), f"{kname} not exact on integer operands"
        else:
            _note(kname, ratio, c["name"])
        assert ratio <= 1.0, f"{kname}: err/bound {ratio:.3f}"


# ------------------------------------------------------------------ CPU
@pytest.mark.parametrize("k,s,H,W,view", [(3, 1, 9, 7, None), (3, 2, 9, 7, (40, 8)), (3, 2, 10, 6, None), (1, 2, 8, 6, None),
                                          (1, 1, 5, 7, (48, 24))])
def test_reference_matches_torch_autograd(k, s, H, W, view):
    """fwd_ref / dgrad_ref / wgrad_ref (and their S) equal torch's float64 conv2d and its autograd gradients, also on a
    channel slice of a wider NHWC buffer."""
    g = torch.Generator().manual_seed(11)
    N, cin, cout = 2, 8, 12
    pitch, c0 = view or (cin, 0)
    buf = torch.randn(N, H, W, pitch, generator=g, dtype=torch.float64)
    x = buf[..., c0:c0 + cin]
    w = torch.randn(cout, cin, k, k, generator=g, dtype=torch.float64)
    b = torch.randn(cout, generator=g, dtype=torch.float64)
    Ho, Wo = out_hw(H, W, k, s)
    dz = torch.randn(N, Ho, Wo, cout, generator=g, dtype=torch.float64)

    def torch_conv(xv, wv, bv, gv):
        xt = xv.permute(0, 3, 1, 2).contiguous().requires_grad_(True)
        wt = wv.clone().requires_grad_(True)
        zt = F.conv2d(xt, wt, bv, s, k // 2)
        zt.backward(gv.permute(0, 3, 1, 2).contiguous())
        return zt.detach().permute(0, 2, 3, 1), xt.grad.permute(0, 2, 3, 1), wt.grad

    zt, dxt, dwt = torch_conv(x, w, b, dz)
    Szt, _, _ = torch_conv(x.abs(), w.abs(), b.abs(), dz.abs())
    _, Sdx, _ = torch_conv(x, w.abs(), None, dz.abs())
    _, _, Sdw = torch_conv(x.abs(), w, None, dz.abs())
    close = lambda a, e: torch.testing.assert_close(a, e, rtol=1e-12, atol=1e-12)
    z, S = fwd_ref(x, w, b, s)
    close(z, zt), close(S, Szt)
    dx, S = dgrad_ref(dz, w, H, W, s)
    close(dx, dxt), close(S, Sdx)
    dw, S = wgrad_ref(x, dz, k, s)
    close(dw, dwt), close(S, Sdw)


def test_tf32_rounding_helpers():
    """tf32 clears the low 13 mantissa bits (truncation toward zero, both signs); tf32_rne rounds to nearest, ties to even."""
    v = torch.tensor([1.0, 1 + 2.0 ** -10, 1 + 2.0 ** -11, -(1 + 2.0 ** -10 + 2.0 ** -12), 1 + 3 * 2.0 ** -11, 0.0, -3.0])
    assert tf32(v).tolist() == [1.0, 1 + 2.0 ** -10, 1.0, -(1 + 2.0 ** -10), 1 + 2.0 ** -10, 0.0, -3.0]
    # 1 + 2^-11 and 1 + 3 * 2^-11 are ties: to the even neighbour
    assert tf32_rne(v).tolist() == [1.0, 1 + 2.0 ** -10, 1.0, -(1 + 2.0 ** -10), 1 + 2.0 ** -9, 0.0, -3.0]
    r = torch.randn(10000, generator=torch.Generator().manual_seed(2)) * 1e3
    for f in (tf32, tf32_rne):
        t = f(r)
        assert ((t.view(torch.int32) & 0x1FFF) == 0).all()
        assert ((t.double() - r.double()).abs() <= 2.0 ** -10 * r.double().abs()).all()
    assert (tf32(r).abs() <= r.abs()).all() and (tf32(r).double() * r.double() >= 0).all()
    assert ((tf32_rne(r).double() - r.double()).abs() <= 2.0 ** -11 * r.double().abs()).all()


def _args_tf32(lib, **over):
    """yb_debug_conv_tf32 arguments of a valid 3x3 32 -> 32 forward on non-null (never dereferenced) pointers"""
    fake = C.c_void_p(256)
    a = dict(pss=0, x=fake, x_pitch=0, dz=fake, w=fake, bias=None, n=2, H=8, W=8, cin=32, cout=32, k=3, s=1, out=fake, ws=fake,
             ws_bytes=1 << 20, desc=None, cap=0)
    a.update(over)
    return lib.yb_debug_conv_tf32(*a.values())


def test_debug_conv_tf32_refuses_bad_arguments(built_lib):
    """The entry validates before it touches the device: an error code and a message, never a crash."""
    from yolosharp_b200 import _lib as L
    lib = L.lib()
    for over in (dict(pss=3), dict(pss=-1), dict(x=None), dict(w=None), dict(out=None), dict(ws=None), dict(pss=1, dz=None),
                 dict(pss=2, x=None), dict(pss=2, dz=None), dict(n=0), dict(H=0), dict(W=-1), dict(cin=0), dict(cout=0),
                 dict(ws_bytes=0), dict(x_pitch=-4), dict(x_pitch=28), dict(x_pitch=34), dict(x_pitch=40, x=C.c_void_p(260)),
                 dict(pss=1, x_pitch=40)):
        assert _args_tf32(lib, **over) == ERR_INVALID_ARG, over
        assert b"yb_debug_conv_tf32" in lib.yb_last_error()
    for over in (dict(cin=12, x_pitch=0), dict(cout=20), dict(k=5), dict(k=2), dict(s=3), dict(pss=1, H=9, s=2),
                 dict(pss=1, W=7, s=2, k=1)):
        assert _args_tf32(lib, **over) == ERR_SHAPE, over
        assert b"not supported" in lib.yb_last_error()
    if not torch.cuda.is_available():
        for over in (dict(), dict(pss=1, x=None), dict(pss=2, w=None, x_pitch=40), dict(pss=0, H=9, s=2), dict(bias=C.c_void_p(256))):
            assert _args_tf32(lib, **over) == ERR_NO_DEVICE, over
            assert b"no CUDA device" in lib.yb_last_error()
