"""fp64 parity of the high-precision mode one kernel at a time (the GP_F16_PAIR layout of the per-kernel entry points).

The mode promises fp32-class results: every activation and weight is an fp16 (hi, lo) pair and every contraction runs
hi*hi + lo*hi + hi*lo with fp32 accumulation.  Each reference here is computed in fp64 on exactly the operands the kernel
sees: inputs hi + lo of the wrapper's split, weights hi + lo of split_hi_lo(w) (mode 3 sums its per-parity weights in fp32
before splitting, at most 4 * 2^-24 relative, so its reference takes the unsummed fp32 weights), fp32 bias as given.

Bounds are elementwise, in units of u = 2^-24:
  contractions   |err| <= C * u * (sqrt(K) * rss + |ref|) + u,  rss = sqrt(conv(x^2, w^2) + bias^2 + residual^2),
                 K the reduction length;
  normalisations |err| <= C * u * (|x| * rstd * |gamma| + |beta| + |ref|) + u  (GroupNorm, LayerNorm; the apply step's
                 fp32 floor is the first term).
Calibrated on an NVIDIA H100 80GB HBM3 (700 W power limit), over this whole file:
  - normalisations and the bilinear resize: worst |err| / bound = 1.30 at C = 4 (GroupNorm, HW = 63, mean/std = 1000), so
    C_NORM = 8;
  - contractions: worst 14.9 at C = 4, at the longest reduction (K = 9 x 1920); the ratio grows with K faster than the
    sqrt(K) of the bound, as fp32 accumulation that is not rounded to nearest would.  C_GEMM = 80 passes every case.
The bound can fail: the fp64 output with the lo*hi pass removed, and separately with the hi*lo pass removed, breaks it
DISCRIMINATION times over at small K (the CPU test below asserts that).  The GPU cases print the same ratios.  At C_GEMM
they stay above 10 only for K <= 576 and fall to 1.6 at K = 17280: at the engine's longest reductions the tensor cores'
accumulation error is as large as a missing correction pass, so the three-pass products cannot be told from two there
by the output alone.  The worst |err| / bound at the final constants was 0.75 (contractions) and 0.71 (the rest).
"""
import math

import pytest
import torch
import torch.nn.functional as F
from test_gpu_kernels import _check, _rand

U = 2.0 ** -24
C_GEMM = 80.0           # contractions (calibration above)
C_NORM = 8.0            # GroupNorm, LayerNorm, bilinear
DISCRIMINATION = 10.0


# ------------------------------------------------------------------------------------------------ references (fp64)
def _conv(x, w, b, mode):
    """F.conv2d in the engine's four modes (x NCHW, any float dtype)."""
    if mode == 0:
        return F.conv2d(x, w, b, padding=w.shape[-1] // 2)
    if mode == 1:
        return F.conv2d(x, w, b, stride=2, padding=1)
    if mode == 2:
        return F.conv2d(F.pad(x, (0, 1, 0, 1)), w, b, stride=2)
    return F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), w, b, padding=1)


def _split(t):
    from genpercept_b200.engine import split_hi_lo
    hi, lo = split_hi_lo(t)
    return hi.double(), lo.double()


def _pair_value(t):
    """The exact value the pair layout stores for fp32 t."""
    hi, lo = _split(t)
    return hi + lo


def _contraction(x, w, b, mode, res=None, relu=False):
    """fp64 reference, rss, and the two dropped-pass outputs' errors of conv(x, w) + b (+ res) (x fp32 NCHW, w fp32).
    Returns (ref, rss, drop_lohi, drop_hilo), all fp64 NCHW (the drops before any ReLU, as magnitudes)."""
    xh, xl = _split(x)
    wh, wl = _split(w)
    we = w.double() if mode == 3 else wh + wl
    bd = None if b is None else b.double()
    ref = _conv(xh + xl, we, bd, mode)
    sq = _conv((xh + xl) ** 2, we ** 2, None if b is None else bd ** 2, mode)
    if res is not None:
        r = _pair_value(res)
        ref = ref + r
        sq = sq + r ** 2
    if relu:
        ref = ref.relu()
    return ref, sq.sqrt(), _conv(xl, wh, None, mode).abs(), _conv(xh, wl, None, mode).abs()


def _contraction_bound(ref, rss, K):
    return C_GEMM * U * (math.sqrt(K) * rss + ref.abs()) + U


def _gn_ref(x, groups, gamma, beta, eps, silu):
    """fp64 GroupNorm(+SiLU) of NCHW x: (ref, the bound's magnitude |x| rstd |gamma| + |beta| + |ref|)."""
    N, Cc = x.shape[:2]
    xg = x.reshape(N, groups, -1)
    mu = xg.mean(-1, keepdim=True)
    rstd = 1.0 / ((xg - mu) ** 2).mean(-1, keepdim=True).add(eps).sqrt()
    g = gamma.double().to(x.device).view(1, Cc, 1, 1)
    b = beta.double().to(x.device).view(1, Cc, 1, 1)
    y = ((xg - mu) * rstd).reshape(x.shape) * g + b
    scale = (xg.abs() * rstd).reshape(x.shape) * g.abs()
    if silu:
        y = y * torch.sigmoid(y)
    return y, scale + b.abs() + y.abs()


def _report(name, err, bound, drops=(), discriminate=False):
    """Prints and asserts err <= bound elementwise, and prints how far each dropped-pass error breaks the bound
    (`discriminate`: asserts DISCRIMINATION times)."""
    ratio = (err / bound).max().item()
    disc = [(d / bound).max().item() for d in drops]
    print(f"{name}: max|err|/bound = {ratio:.3f}" + (f", dropped-pass ratios {', '.join(f'{v:.1f}' for v in disc)}"
                                                    if disc else ""))
    assert torch.isfinite(err).all(), name + ": non-finite output"
    assert ratio <= 1.0, f"{name}: |err| exceeds the bound {ratio:.3f}x"
    if discriminate:
        for v in disc:
            assert v >= DISCRIMINATION, f"{name}: a dropped pass stays within {DISCRIMINATION}x of the bound ({v:.2f})"


def _operands(N, H, W, Cin, Cout, ks, mag, gen, res_shape=None):
    """x ~ mag N(0, 1); weights scaled so the output is of order one (of order 5e3 at mag >= 1e4, below fp16's range)."""
    K = Cin * ks * ks
    out_scale = 0.5 * mag if mag > 1 else 1.0
    x = torch.randn((N, Cin, H, W), generator=gen) * mag
    w = torch.randn((Cout, Cin, ks, ks), generator=gen) * (out_scale / (mag * math.sqrt(K)))
    b = torch.randn((Cout,), generator=gen) * 0.1 * out_scale
    res = None if res_shape is None else torch.randn(res_shape, generator=gen) * out_scale
    return x, w, b, res


def _out_shape(N, H, W, Cout, mode):
    if mode == 1:
        return (N, Cout, (H + 1) // 2, (W + 1) // 2)
    if mode == 2:
        return (N, Cout, H // 2, W // 2)
    if mode == 3:
        return (N, Cout, 2 * H, 2 * W)
    return (N, Cout, H, W)


# ------------------------------------------------------------------------------------------------ the implicit-GEMM table
# (N, H, W, Cin, Cout, ks, mode, magnitude, residual, relu); the comment gives the planner's (BN, MT) tile and the epilogue.
# The staged (TMA store) epilogue takes Cout % 64 == 0, the direct one the rest.  Cin = 4 is the direct conv's (below).
IGEMM = {
    "c4":          (1, 32, 32, 320, 4, 3, 0, 1.0, False, False),       # BN 16, MT 1, direct epilogue
    "c32_tiny":    (1, 32, 32, 320, 32, 3, 0, 1e-3, False, False),     # BN 32, MT 1, direct; lo subnormal in fp16
    "c36_res":     (1, 32, 32, 320, 36, 3, 0, 1.0, True, False),       # BN 64, MT 1, direct: lo plane at Cout % 8 != 0
    "c36_b2":      (2, 9, 11, 8, 36, 3, 0, 1e4, False, True),          # BN 64, MT 1, direct, K padded (Cin 8), ReLU
    "c320_res":    (2, 24, 24, 320, 320, 3, 0, 1.0, True, True),       # BN 64, MT 1, staged, residual + ReLU, batch 2
    "c1280_big":   (1, 8, 8, 1280, 1280, 3, 0, 1e4, False, False),     # BN 64, MT 1, staged
    "k17280":      (1, 16, 16, 1920, 1280, 3, 0, 1.0, False, False),   # BN 64, MT 1, staged; the longest K (9 x 1920)
    "cin8":        (1, 64, 64, 8, 320, 3, 0, 1e-3, False, False),      # BN 128, MT 1, staged; K of 64 per tap, 8 used
    "mt2":         (1, 256, 256, 64, 64, 3, 0, 1.0, True, False),      # BN 64, MT 2, staged, residual
    "tok_mt2":     (1, 1, 34077, 1280, 64, 1, 0, 1.0, False, False),   # tokens mode, BN 64, MT 2, ragged last tile
    "tok1000":     (1, 1, 1000, 320, 320, 1, 0, 1e-3, True, False),    # tokens, BN 64, MT 1, staged, residual
    "tok77":       (1, 1, 77, 1280, 320, 1, 0, 1e4, False, True),      # tokens, BN 64, MT 1, 77 tokens, ReLU
    "s2_pad1":     (2, 33, 47, 320, 320, 3, 1, 1.0, False, False),     # stride 2, odd H / W, staged
    "s2_pad01":    (1, 33, 47, 128, 36, 3, 2, 1e4, True, False),       # stride 2 (0,1,0,1), odd H / W, direct, residual
    "up":          (1, 12, 12, 320, 320, 3, 3, 1.0, False, False),     # nearest 2x + 3x3 (four parity classes), staged
    "up_1x1":      (1, 1, 1, 1280, 1280, 3, 3, 1e-3, False, False),    # mode 3 at 1 x 1
    "up_c36":      (2, 7, 5, 64, 36, 3, 3, 1.0, True, True),           # mode 3, direct epilogue, residual + ReLU
}


def test_case_table_reaches_every_tile_shape():
    """The planner's (BN, MT) of the table's stride-1 cases covers every N tile and both M tilings."""
    from genpercept_b200 import engine as E
    bns, mts = set(), set()
    for (N, H, W, Cin, Cout, ks, mode, *_rest) in IGEMM.values():
        if mode != 0:
            continue
        bn, mt = E.tile_shape(Cout, Cin, ks, N, H, W, tokens_mode=(ks == 1))
        bns.add(bn)
        mts.add(mt)
    assert bns == {16, 32, 64, 128}, bns
    assert mts == {1, 2}, mts


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
@pytest.mark.parametrize("mag", [1.0, 1e-3, 1e4])
def test_bound_discriminates_dropped_passes(mode, mag):
    """CPU: on a small shape, the output with the lo*hi or the hi*lo pass removed breaks the bound by a wide margin, while
    the exact output's fp32 rounding stays inside it."""
    g = torch.Generator().manual_seed(mode * 10 + int(math.log10(mag)) + 3)
    N, H, W, Cin, Cout = 1, 7, 9, 2, 8
    x, w, b, res = _operands(N, H, W, Cin, Cout, 3, mag, g, _out_shape(N, H, W, Cout, mode))
    ref, rss, d1, d2 = _contraction(x, w, b, mode, res)
    bound = _contraction_bound(ref, rss, Cin * 9)
    _report(f"cpu mode{mode} mag{mag:g}", (ref.float().double() - ref).abs(), bound, (d1, d2), discriminate=True)


def _setup():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _run_conv(name, N, H, W, Cin, Cout, ks, mode, mag, residual, relu, direct=False):
    from genpercept_b200 import engine as E
    _setup()
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x, w, b, res = _operands(N, H, W, Cin, Cout, ks, mag, g, _out_shape(N, H, W, Cout, mode) if residual else None)
    xc = x.cuda()
    resc = None if res is None else res.cuda()
    ref, rss, d1, d2 = _contraction(xc, w.cuda(), b.cuda(), mode, resc, relu)
    y = E.conv2d(E._nhwc(xc), w, b, mode=mode, residual=None if resc is None else E._nhwc(resc), relu=relu, direct=direct)
    torch.cuda.synchronize()
    got = y.permute(0, 3, 1, 2)
    # the direct conv multiplies hi + lo by the fp32 weights: no weight split, so only the lo*hi pass can be dropped
    drops = (d1,) if direct else (d1, d2)
    K = Cin * (4 if mode == 3 and not direct else ks * ks)
    _report(f"{name} {'direct' if direct else 'igemm'}", (got - ref).abs(), _contraction_bound(ref, rss, K), drops)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(IGEMM))
def test_conv_pair(name):
    _run_conv(name, *IGEMM[name])


@pytest.mark.gpu
@pytest.mark.parametrize("case", [
    (2, 12, 12, 4, 24, 3, 0, 1.0, True, True),     # the VAE's conv_in width
    (1, 13, 9, 4, 8, 3, 1, 1e-3, False, False),
    (1, 13, 9, 4, 8, 3, 2, 1e4, True, False),
    (2, 6, 5, 8, 4, 3, 3, 1.0, False, True),
    (1, 8, 8, 36, 3, 1, 0, 1.0, True, False),      # odd channel counts on both sides
])
def test_direct_conv_pair(case):
    # the direct conv needs no weight split: reference and drop use the fp32 weights as the kernel does
    N, H, W, Cin, Cout, ks, mode, mag, residual, relu = case
    from genpercept_b200 import engine as E
    _setup()
    g = torch.Generator().manual_seed(Cin * 100 + Cout + mode)
    x, w, b, res = _operands(N, H, W, Cin, Cout, ks, mag, g, _out_shape(N, H, W, Cout, mode) if residual else None)
    xc, wc = x.cuda(), w.cuda().double()
    xh, xl = _split(xc)
    ref = _conv(xh + xl, wc, b.cuda().double(), mode)
    sq = _conv((xh + xl) ** 2, wc ** 2, b.cuda().double() ** 2, mode)
    resc = None
    if residual:
        resc = res.cuda()
        ref = ref + _pair_value(resc)
        sq = sq + _pair_value(resc) ** 2
    if relu:
        ref = ref.relu()
    y = E.conv2d(E._nhwc(xc), w, b, mode=mode, residual=None if resc is None else E._nhwc(resc), relu=relu, direct=True)
    torch.cuda.synchronize()
    _report(f"direct {case}", (y.permute(0, 3, 1, 2) - ref).abs(), _contraction_bound(ref, sq.sqrt(), Cin * ks * ks),
            (_conv(xl, wc, None, mode).abs(),))


# ------------------------------------------------------------------------------------------------ GroupNorm + conv
@pytest.mark.gpu
@pytest.mark.parametrize("case", [
    dict(N=1, H=16, W=16, Cin=320, Cout=320),                                 # GroupNorm pass + tap-streaming conv, BN 64
    dict(N=2, H=12, W=20, Cin=128, Cout=320, Csc=64, ratio=100.0),            # + 1x1 shortcut: A view 1 and its lo view 5
    dict(N=1, H=8, W=128, Cin=128, Cout=128, residual=True, silu=False),
    dict(N=1, H=16, W=24, Cin=128, Cout=3, out_f32=True, ratio=10.0),         # fp32 NCHW map: direct epilogue, no lo plane
])
def test_gn_conv3x3_pair(case):
    from genpercept_b200 import engine as E
    _setup()
    N, H, W, Cin, Cout = (case[k] for k in ("N", "H", "W", "Cin", "Cout"))
    Csc, silu, ratio = case.get("Csc"), case.get("silu", True), case.get("ratio", 0.0)
    g = torch.Generator().manual_seed(Cin + 7 * Cout)
    x = torch.randn((N, Cin, H, W), generator=g) + ratio + torch.randn((1, Cin, 1, 1), generator=g)
    gamma = 1 + 0.1 * torch.randn((Cin,), generator=g)
    beta = 0.1 * torch.randn((Cin,), generator=g)
    w = torch.randn((Cout, Cin, 3, 3), generator=g) / math.sqrt(9 * Cin)
    b = 0.1 * torch.randn((Cout,), generator=g)
    xc = x.cuda()
    a, amag = _gn_ref(_pair_value(xc), 32, gamma, beta, 1e-6, silu)
    wh, wl = _split(w.cuda())
    ref = _conv(a, wh + wl, b.cuda().double(), 0)
    # each normalised operand carries the GroupNorm bound's error: the contraction's rss is taken over that magnitude
    sq = _conv(amag ** 2, (wh + wl) ** 2, b.cuda().double() ** 2, 0)
    ah, al = _split(a.float())
    drops = [_conv(al, wh, None, 0).abs(), _conv(ah, wl, None, 0).abs()]
    K = 9 * Cin
    sc_x = sc_w = sc_b = res = None
    if Csc:
        sc = torch.randn((N, Csc, H, W), generator=g).cuda()
        sc_w = torch.randn((Cout, Csc, 1, 1), generator=g) / math.sqrt(Csc)
        sc_b = 0.1 * torch.randn((Cout,), generator=g)
        sh, sl = _split(sc_w.cuda())
        ref = ref + _conv(_pair_value(sc), sh + sl, sc_b.cuda().double(), 0)
        sq = sq + _conv(_pair_value(sc) ** 2, (sh + sl) ** 2, sc_b.cuda().double() ** 2, 0)
        K += Csc
        sc_x = E._nhwc(sc)
    if case.get("residual"):
        r = torch.randn((N, Cout, H, W), generator=g).cuda()
        ref = ref + _pair_value(r)
        sq = sq + _pair_value(r) ** 2
        res = E._nhwc(r)
    y = E.gn_conv3x3(E._nhwc(xc), 32, gamma, beta, 1e-6, silu, w, b, sc_x=sc_x, sc_w=sc_w, sc_b=sc_b, residual=res,
                     out_f32=case.get("out_f32", False))
    torch.cuda.synchronize()
    got = y.double() if case.get("out_f32") else y.permute(0, 3, 1, 2)
    _report(f"gn+conv pair {case}", (got - ref).abs(), _contraction_bound(ref, sq.sqrt(), K), drops)


# ------------------------------------------------------------------------------------------------ normalisations
def _offset_input(shape_nchw, ratio, varying, gen, sigma=0.7):
    """N(0, sigma^2) plus a per-channel offset of ratio * sigma: the same for all channels (`varying` False, so every group
    has mean / std = ratio) or ratio * sigma + N(0, sigma^2) per channel."""
    N, Cc = shape_nchw[:2]
    off = torch.full((1, Cc, 1, 1), ratio * sigma)
    if varying:
        off = off + sigma * torch.randn((1, Cc, 1, 1), generator=gen)
    return torch.randn(shape_nchw, generator=gen) * sigma + off


GN_SHAPES = [
    (2, 7, 9, 128),       # HW = 63: below one 64-pixel chunk
    (1, 33, 47, 320),     # HW = 1551: not a multiple of the chunk count (25)
    (1, 192, 192, 128),   # 256 chunks of 144 pixels
    (1, 16, 16, 1920),
    (1, 12, 20, 2560),    # from C >= 1032 gn_stats runs one pixel lane per block
]


@pytest.mark.gpu
@pytest.mark.parametrize("varying", [False, True])
@pytest.mark.parametrize("ratio", [0.0, 10.0, 100.0, 1000.0])
@pytest.mark.parametrize("shape", GN_SHAPES)
def test_groupnorm_pair(shape, ratio, varying):
    from genpercept_b200 import engine as E
    N, H, W, Cc = shape
    silu = (GN_SHAPES.index(shape) + int(varying)) % 2 == 0
    g = torch.Generator().manual_seed(Cc + H + int(ratio) + int(varying))
    x = _offset_input((N, Cc, H, W), ratio, varying, g).cuda()
    gamma = 1 + 0.1 * torch.randn((Cc,), generator=g)
    beta = 0.1 * torch.randn((Cc,), generator=g)
    ref, mag = _gn_ref(_pair_value(x), 32, gamma, beta, 1e-6, silu)
    y = E.groupnorm(E._nhwc(x), 32, gamma, beta, 1e-6, silu)
    torch.cuda.synchronize()
    _report(f"groupnorm pair {shape} ratio {ratio:g} varying={varying} silu={silu}", (y.permute(0, 3, 1, 2) - ref).abs(),
            C_NORM * U * mag + U)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,ratio,silu", [((1, 32, 32, 128), 100.0, True), ((1, 96, 96, 320), 300.0, False),
                                              ((2, 32, 32, 512), 1000.0, True)])
def test_groupnorm_16bit_large_offsets(shape, ratio, silu):
    """The 16-bit mode's GroupNorm with every group's mean at `ratio` standard deviations, against F.group_norm on the
    same fp16 input, with the per-kernel bound of test_gpu_kernels.py::test_groupnorm (input and parameters drawn the
    same way, the offset 0.3 there replaced by 1.5 * ratio).  Sums of x and x^2 lose the variance to cancellation here."""
    from genpercept_b200 import engine as E
    _setup()
    g = torch.Generator().manual_seed(1)
    N, H, W, Cc = shape
    x = (_rand((N, Cc, H, W), g).float() * 1.5 + 1.5 * ratio).half()
    gamma = 1 + 0.1 * torch.randn((Cc,), generator=g)
    beta = 0.1 * torch.randn((Cc,), generator=g)
    ref = F.group_norm(x.cuda().float(), 32, gamma.cuda(), beta.cuda(), 1e-6)
    if silu:
        ref = F.silu(ref)
    y = E.groupnorm(E._nhwc(x.cuda()), 32, gamma, beta, 1e-6, silu)
    _check(f"groupnorm 16-bit {shape} ratio {ratio:g} silu={silu}", y.permute(0, 3, 1, 2), ref)


@pytest.mark.gpu
@pytest.mark.parametrize("varying", [False, True])
@pytest.mark.parametrize("ratio", [0.0, 10.0, 100.0, 1000.0])
@pytest.mark.parametrize("tokens,Cc", [(100, 320), (64, 640), (33, 1280)])
def test_layernorm_pair(tokens, Cc, ratio, varying):
    from genpercept_b200 import engine as E
    g = torch.Generator().manual_seed(tokens + Cc + int(ratio))
    x = _offset_input((1, Cc, tokens, 1), ratio, varying, g)[0, :, :, 0].t().contiguous().cuda()   # [tokens, C]
    gamma = 1 + 0.1 * torch.randn((Cc,), generator=g)
    beta = 0.1 * torch.randn((Cc,), generator=g)
    xe = _pair_value(x)
    mu = xe.mean(-1, keepdim=True)
    rstd = 1.0 / ((xe - mu) ** 2).mean(-1, keepdim=True).add(1e-5).sqrt()
    gd, bd = gamma.double().cuda(), beta.double().cuda()
    ref = (xe - mu) * rstd * gd + bd
    y = E.layernorm(x, gamma, beta, 1e-5)
    torch.cuda.synchronize()
    _report(f"layernorm pair {tokens}x{Cc} ratio {ratio:g} varying={varying}", (y - ref).abs(),
            C_NORM * U * (xe.abs() * rstd * gd.abs() + bd.abs() + ref.abs()) + U)


@pytest.mark.gpu
def test_bilinear_up2x_pair():
    from genpercept_b200 import engine as E
    g = torch.Generator().manual_seed(4)
    x = (torch.randn((2, 64, 12, 20), generator=g) * 3 + 50).cuda()
    xe = _pair_value(x)
    ref = F.interpolate(xe, scale_factor=2, mode="bilinear", align_corners=True)
    mag = F.interpolate(xe.abs(), scale_factor=2, mode="bilinear", align_corners=True)   # sum of |w_i x_i|
    y = E.bilinear_up2x(E._nhwc(x))
    torch.cuda.synchronize()
    _report("bilinear pair", (y.permute(0, 3, 1, 2) - ref).abs(), C_NORM * U * (mag + ref.abs()) + U)


# ------------------------------------------------------------------------------------------------ conv -> GroupNorm
# Cout 320: in the 16-bit modes the statistics come out of the conv's staged epilogue; 640: from a gn_stats pass (the
# pair layout always takes gn_stats).  960 = 640 + 320 and 320 + 640 channels give 30 per group, so one group straddles
# the two sources.  Batch 2 flushes the epilogue's statistics per image.  `bias`: the per-channel offset, in units of the
# conv output's standard deviation (about 1).
CONV_GN = {
    "c320":             dict(N=2, H=16, W=16, Cin=320, Cout=320, Cskip=0, bias=100.0, silu=True),
    "c320_skip640":     dict(N=2, H=12, W=24, Cin=64, Cout=320, Cskip=640, bias=10.0, silu=False),
    "c640_skip320":     dict(N=2, H=16, W=16, Cin=320, Cout=640, Cskip=320, bias=1000.0, silu=True),
    "c640":             dict(N=1, H=24, W=24, Cin=128, Cout=640, Cskip=0, bias=0.0, silu=True),
    "c320_big":         dict(N=2, H=16, W=16, Cin=128, Cout=320, Cskip=0, bias=1000.0, silu=False),
}


def _conv_gn_operands(case, gen):
    N, H, W, Cin, Cout, Cskip = (case[k] for k in ("N", "H", "W", "Cin", "Cout", "Cskip"))
    x = torch.randn((N, Cin, H, W), generator=gen)
    w = torch.randn((Cout, Cin, 3, 3), generator=gen) / math.sqrt(9 * Cin)
    b = case["bias"] + torch.randn((Cout,), generator=gen)
    skip = case["bias"] + torch.randn((N, Cskip, H, W), generator=gen) if Cskip else None
    gamma = 1 + 0.1 * torch.randn((Cout + Cskip,), generator=gen)
    beta = 0.1 * torch.randn((Cout + Cskip,), generator=gen)
    return x, w, b, skip, gamma, beta


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CONV_GN))
def test_conv_groupnorm_pair(name):
    from genpercept_b200 import engine as E
    _setup()
    case = CONV_GN[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x, w, b, skip, gamma, beta = _conv_gn_operands(case, g)
    xc = x.cuda()
    skc = None if skip is None else skip.cuda()
    yc, y = E.conv_groupnorm(E._nhwc(xc), w, b, 32, gamma, beta, 1e-6, case["silu"], None if skc is None else E._nhwc(skc))
    torch.cuda.synchronize()
    ref, rss, d1, d2 = _contraction(xc, w.cuda(), b.cuda(), 0)
    _report(f"conv_groupnorm pair {name}: conv", (yc.permute(0, 3, 1, 2) - ref).abs(),
            _contraction_bound(ref, rss, 9 * case["Cin"]), (d1, d2))
    # the normalisation's reference reads the stored y_conv (exact in float64) and skip
    src = yc.permute(0, 3, 1, 2)
    if skc is not None:
        src = torch.cat([src, _pair_value(skc)], dim=1)
    gref, mag = _gn_ref(src, 32, gamma, beta, 1e-6, case["silu"])
    _report(f"conv_groupnorm pair {name}: groupnorm", (y.permute(0, 3, 1, 2) - gref).abs(), C_NORM * U * mag + U)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("name", list(CONV_GN))
def test_conv_groupnorm_16bit(name, dtype):
    """The 16-bit modes: y_conv against F.conv2d, y against F.group_norm of the stored y_conv, with the per-kernel bound of
    test_gpu_kernels.py (one 16-bit ulp of the output magnitude plus accumulation noise)."""
    from genpercept_b200 import engine as E
    _setup()
    case = CONV_GN[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)) + 1)
    x, w, b, skip, gamma, beta = _conv_gn_operands(case, g)
    xq = x.to(dtype).cuda()
    wq = w.to(dtype).float()
    skq = None if skip is None else skip.to(dtype).cuda()
    yc, y = E.conv_groupnorm(E._nhwc(xq), wq, b, 32, gamma, beta, 1e-6, case["silu"], None if skq is None else E._nhwc(skq))
    torch.cuda.synchronize()
    rel = 2e-3 if dtype == torch.float16 else 1.6e-2
    ref = F.conv2d(xq.float(), wq.cuda(), b.cuda(), padding=1)
    _check(f"conv_groupnorm {name} {dtype}: conv", yc.permute(0, 3, 1, 2), ref, rel)
    src = yc.permute(0, 3, 1, 2).float()
    if skq is not None:
        src = torch.cat([src, skq.float()], dim=1)
    gref = F.group_norm(src, 32, gamma.cuda(), beta.cuda(), 1e-6)
    if case["silu"]:
        gref = F.silu(gref)
    _check(f"conv_groupnorm {name} {dtype}: groupnorm", y.permute(0, 3, 1, 2), gref, rel)

