"""Per-kernel parity of the UNet's transformer and up-block ops: the GEGLU projection, the 2-token and the general
cross-attention, the ResnetBlock2D over [hidden | skip], and the nearest / bilinear resizes.  Each runs through its C-ABI
entry point (gp_geglu, gp_cross_attention, gp_resnet, gp_resize), which emits the engine's own ops, and is compared with a
plain torch reference on exactly the operands the kernel sees: 16-bit-rounded inputs (and, where the kernel packs them as
given, weights) in the 16-bit modes, hi + lo of split_hi_lo in the pair layout.  The cross-attention's weights are folded
on the host before the kernel sees them, so its reference takes the raw fp32 weights and the bound carries the fold.

Bounds, with u_s the storage unit (2^-11 fp16, 2^-8 bf16, 2^-22 for an fp16 (hi, lo) pair) and u = 2^-24:
  16-bit   |err| <= C16 * u_s * max|ref| + u_s: one output ulp of the magnitude plus accumulation noise.  The general
           cross-attention adds, per element, the effect of its 16-bit LN output, folded A, scores, P and folded B:
           score error delta_j = u_s (|s_j| + 2 sqrt(l^2 . A_j^2)); dP_j = P_j (delta_j - sum_k P_k delta_k) over the
           head's group moves the output by sum_j P_j delta_j (B_j - O_head); these add in quadrature, as do the
           roundings of P and B: the term C16 * (sqrt(sum_j (P_j delta_j)^2 (B_j - O_head)^2) + 2 u_s sqrt(P^2 . B^2)).
  pair     elementwise C * u * (...):
           GEGLU    C_GEGLU u (|gelu(g)| E_v + |v| |gelu'(g)| E_g + |ref| + |v| (|g| + 1)),  E = sqrt(K) rss + |h| for the
                    value / gate pre-activations h (the last term is the erf approximation's);
           2-token  C_XATTN2 u (|x| + |bo| + sum |B| + |ref| + sum_h |M_h| p_h (1 - p_h) Z_h),  Z_h = the magnitude of the
                    head's logit sum_c (|x_c - mean| + |mean|) rstd |U_hc| + |z_h| (the fp32 LayerNorm and dot products);
           general  C_XATTN_GEN (the 16-bit term above at u_s = 2^-22, plus u (|x| + |bo| + |ref|));
           ResNet   the contraction bound of test_gpu_high_precision_kernels (C_RES) on conv2, whose normalised operand
                    carries GroupNorm's bound plus conv1's error scaled by norm2's rstd;
           bilinear C_NORM (u (interp(|x|) + |ref|) + the fp32 source coordinates' rounding, 2 u (|f| + 1), times the
                    slope along each axis): the coordinates are those F.interpolate computes for an fp32 tensor.
  nearest  bit-identical to F.interpolate(size=..., mode="nearest"): it is a gather.

Calibrated on an NVIDIA H100 80GB HBM3 (700 W power limit), over this whole file.  Worst |err| / bound at the constants
below (fp16 / bf16 / pair): GEGLU 0.44 / 0.43 / 0.76 (T = 9253; C = 320 in 16 bit, 1280 in the pair layout);
2-token cross-attention 0.45 / 0.43 / 0.43 (C = 640); general cross-attention 0.32 / 0.33 / 0.64 (n = 77; at the
first run's C_XATTN_GEN = 16 the pair case C = 1280 stood at 2.6); ResNet 0.44 / 0.40 / 0.59 (the pair case
1280 + 1280); bilinear 0.26 / 0.26 / 0.22.  Every nearest case is bit-identical.

Discrimination (CPU, test_bounds_discriminate_*): fp64 outputs of plausible wrong kernels, built from the same operands,
break each bound at least DISCRIMINATION times.  The token count does not enter a token's bound, so the token-wise ops
are checked over the first 64 tokens of each GPU case; the ResNets at the GPU cases' channels and batch over at most
16 x 16 pixels.  Not asserted (the ratios are printed):
  - the tanh-approximate GELU in the 16-bit modes: it differs from the erf form by less than 2.5e-4 |v|, inside one
    output ulp (in the pair layout it breaks the bound about 100 times);
  - the per-token-offset cross-attention cases in bf16: the output carries the offset (|x| ~ 150), whose bf16 rounding
    is as large as a wrong kernel's change (1.4 - 15x the bound; 11 - 114x in fp16, where it is asserted);
  - per-source statistics for the straddling group in bf16: one group of 30 of 960 channels moves the output by 5x the
    bf16 bound (39 - 45x in fp16, 600x in the pair layout).
"""
import math

import pytest
import torch
import torch.nn.functional as F
from test_gpu_high_precision_kernels import C_NORM, DISCRIMINATION, U, _report, _split

C16 = 2.0           # 16-bit: rel = 2 u_s, one output ulp (1e-3 fp16, 7.8e-3 bf16)
C_GEGLU = 16.0      # pair GEGLU
C_XATTN2 = 4.0      # pair 2-token cross-attention
C_XATTN_GEN = 64.0  # pair general cross-attention
C_RES = 24.0        # pair ResNets

DTYPES = {"f16": torch.float16, "bf16": torch.bfloat16, "pair": torch.float32}
US = {"f16": 2.0 ** -11, "bf16": 2.0 ** -8, "pair": 2.0 ** -22}


def _setup():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _seen(t, dt):
    """fp32 t as the kernel sees it in layout dt: the 16-bit value, or hi + lo of the pair (fp64)."""
    if dt == "pair":
        hi, lo = _split(t)
        return hi + lo
    return t.to(DTYPES[dt]).double()


def _arg(t, dt):
    """fp32 t as the entry point's wrapper takes it (fp32 selects the pair layout)."""
    return t if dt == "pair" else t.to(DTYPES[dt])


def _bound16(ref, dt):
    us = US[dt]
    return torch.full_like(ref, C16 * us * ref.abs().max().item() + us)


# ------------------------------------------------------------------------------------------------ GEGLU
def _gelu(g, tanh=False):
    if tanh:
        return 0.5 * g * (1 + torch.tanh(math.sqrt(2 / math.pi) * (g + 0.044715 * g ** 3)))
    return 0.5 * g * (1 + torch.erf(g / math.sqrt(2)))


def _geglu_operands(T, C, gen):
    x = torch.randn((T, C), generator=gen)
    w = torch.randn((8 * C, C), generator=gen) * (1.5 / math.sqrt(C))
    b = torch.randn((8 * C,), generator=gen) * 0.5
    return x, w, b


def _geglu_ref(x, w, b, variant=None):
    """fp64 GEGLU of fp64 x [T,C], w [8C,C], b [8C]; variant: a wrong kernel ("swap", "no_gate_bias", "tanh")."""
    h = x @ w.t() + b
    c4 = w.shape[0] // 2
    v, g = h[:, :c4], h[:, c4:]
    if variant == "swap":
        v, g = g, v
    if variant == "no_gate_bias":
        g = g - b[c4:]
    return v * _gelu(g, tanh=variant == "tanh")


def _geglu_case(T, C, dt, gen, device, variants=()):
    x, w, b = _geglu_operands(T, C, gen)
    x, w, b = x.to(device), w.to(device), b.to(device)
    xs, ws, bd = _seen(x, dt), _seen(w, dt), b.double()
    ref = _geglu_ref(xs, ws, bd)
    if dt == "pair":
        h = xs @ ws.t() + bd
        rss = ((xs ** 2) @ (ws ** 2).t() + bd ** 2).sqrt()
        e = math.sqrt(C) * rss + h.abs()
        c4 = 4 * C
        v, g = h[:, :c4], h[:, c4:]
        dgelu = 0.5 * (1 + torch.erf(g / math.sqrt(2))) + g * torch.exp(-0.5 * g ** 2) / math.sqrt(2 * math.pi)
        bound = C_GEGLU * U * (_gelu(g).abs() * e[:, :c4] + v.abs() * dgelu.abs() * e[:, c4:] + ref.abs() +
                               v.abs() * (g.abs() + 1)) + U
    else:
        bound = _bound16(ref, dt)
    wrong = [(name, (_geglu_ref(xs, ws, bd, name) - ref).abs()) for name in variants]
    return x, w, b, ref, bound, wrong


GEGLU_CASES = [(T, C) for C in (320, 640, 1280) for T in (1, 77, 4096, 9216 + 37)] + [(1000, 200)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("T,C", GEGLU_CASES)
def test_geglu(T, C, dt):
    """ff.net.0.proj + GEGLU through the projection's epilogue.  8C a multiple of 128 takes the LEAN epilogue in the
    16-bit modes; C = 200 (8C = 1600) and the pair layout take the general one."""
    from genpercept_b200 import engine as E
    _setup()
    x, w, b, ref, bound, _ = _geglu_case(T, C, dt, torch.Generator().manual_seed(T + C), "cuda")
    y = E.geglu(_arg(x, dt), w, b)
    torch.cuda.synchronize()
    _report(f"geglu {dt} T{T} C{C}", (y.double() - ref).abs(), bound)


# ------------------------------------------------------------------------------------------------ cross-attention
E_CTX = 1024   # SD-2.1's text width


def _xattn_operands(C, heads, n, T, offset, gen):
    x = torch.randn((T, C), generator=gen)
    if offset:
        x = x + 50.0 * torch.randn((T, 1), generator=gen)        # a large per-token mean
    ctx = torch.randn((n, E_CTX), generator=gen)
    wq = torch.randn((C, C), generator=gen) * (0.5 / math.sqrt(C))
    wk = torch.randn((C, E_CTX), generator=gen) / math.sqrt(E_CTX)
    wv = torch.randn((C, E_CTX), generator=gen) * math.sqrt(n / E_CTX)   # P . V averages over n: keep it of order one
    wo = torch.randn((C, C), generator=gen) / math.sqrt(C)
    bo = 0.5 * torch.randn((C,), generator=gen)
    g = 2.0 + 0.3 * torch.randn((C,), generator=gen)             # LayerNorm affine far from the identity: the fold matters
    bt = 1.0 + 0.3 * torch.randn((C,), generator=gen)
    return x, ctx, (wq, wk, wv, wo, bo, g, bt)


def _xattn_ref(x, ctx, heads, wts, eps=1e-5, variant=None):
    """fp64 x + attn2(LN(x), ctx) and its intermediates.  variant: a wrong kernel ("swap_p": p and 1 - p exchanged (n = 2),
    "ln_unfolded": LN without its affine, "no_bias": to_out without bias, "softmax_all": one softmax over all Kp score
    columns, "groups_shifted": the head groups shifted by one column)."""
    wq, wk, wv, wo, bo, g, bt = (t.double() for t in wts)
    T, C = x.shape
    n, d = ctx.shape[0], C // heads
    hn = heads * n
    kp = (hn + 63) // 64 * 64
    mu = x.mean(-1, keepdim=True)
    rstd = 1.0 / ((x - mu) ** 2).mean(-1, keepdim=True).add(eps).sqrt()
    if variant == "ln_unfolded":
        g, bt = torch.ones_like(g), torch.zeros_like(bt)
    l = (x - mu) * rstd * g + bt
    K, V = ctx.double() @ wk.t(), ctx.double() @ wv.t()                                  # [n, C]
    A = torch.einsum("hdc,jhd->chj", wq.view(heads, d, C), K.view(n, heads, d)).reshape(C, hn) / math.sqrt(d)
    Bm = torch.einsum("ohd,jhd->hjo", wo.view(C, heads, d), V.view(n, heads, d)).reshape(hn, C)
    s = l @ A
    if variant == "softmax_all":
        P = torch.softmax(torch.cat([s, s.new_zeros(T, kp - hn)], 1), -1)[:, :hn]
    elif variant == "groups_shifted":
        sp = torch.cat([s, s.new_zeros(T, kp - hn)], 1)
        P = sp.clone()
        P[:, 1:hn + 1] = torch.softmax(sp[:, 1:hn + 1].view(T, heads, n), -1).reshape(T, hn)
        P = P[:, :hn]
    else:
        P = torch.softmax(s.view(T, heads, n), -1).reshape(T, hn)
        if variant == "swap_p":
            P = P.view(T, heads, n).flip(-1).reshape(T, hn)
    out = x + P @ Bm + (0 if variant == "no_bias" else bo)
    return out, dict(l=l, A=A, Bm=Bm, s=s, P=P, mu=mu, rstd=rstd, g=g, bo=bo)


def _xattn_general_term(it, heads, n, us):
    """The general path's score, P and B roundings carried to the output (see the module docstring)."""
    l, A, s, P, Bm = it["l"], it["A"], it["s"], it["P"], it["Bm"]
    T, C = s.shape[0], Bm.shape[1]
    # independent roundings of l and A add in quadrature, as in the contraction bound's rss
    delta = us * (s.abs() + 2 * ((l ** 2) @ (A ** 2)).sqrt())
    # dP_j = P_j (delta_j - sum_k P_k delta_k) moves the output by sum_j P_j delta_j (B_j - O_h), O_h the head's output:
    # no error at all in a group of one column.  Its square, expanded so that no [T, heads * n, C] tensor is formed:
    w = ((P * delta) ** 2).view(T, heads, n)
    Bh = Bm.view(heads, n, C)
    O = torch.einsum("thn,hnc->thc", P.view(T, heads, n), Bh)
    var = (w.reshape(T, -1) @ Bm ** 2 - 2 * (O * torch.einsum("thn,hnc->thc", w, Bh)).sum(1) +
           (O ** 2 * w.sum(-1, keepdim=True)).sum(1))
    return var.clamp(min=0).sqrt() + 2 * us * ((P ** 2) @ Bm ** 2).sqrt()   # + the roundings of P and B


def _xattn_bound(x, ref, it, heads, n, dt):
    us = US[dt]
    if dt != "pair":
        b = _bound16(ref, dt)
        return b if n == 2 else b + C16 * _xattn_general_term(it, heads, n, us)
    if n != 2:
        return C_XATTN_GEN * (_xattn_general_term(it, heads, n, us) + U * (x.abs() + it["bo"].abs() + ref.abs())) + U
    # the closed form: y = x + c0 + sum_h p_h M_h, p_h = sigmoid(z_h), in fp32 from the folded U, u0, M, c0
    T, C = x.shape
    A, Bm, P, g = it["A"], it["Bm"], it["P"], it["g"]
    Ud = (A[:, 0::2] - A[:, 1::2]) * g[:, None]                                           # [C, heads]
    M = (Bm[0::2] - Bm[1::2]).abs()                                                       # [heads, C]
    z = (it["s"][:, 0::2] - it["s"][:, 1::2]).abs()
    Z = (((x - it["mu"]).abs() + it["mu"].abs()) * it["rstd"]) @ Ud.abs() + z
    p = P[:, 0::2]
    mag = x.abs() + it["bo"].abs() + Bm.abs().sum(0) + ref.abs() + (p * (1 - p) * Z) @ M
    return C_XATTN2 * U * mag + U


XATTN_WIDTHS = [(320, 5), (640, 10), (1280, 20)]
XATTN_CASES = ([(C, h, 2, T, False) for C, h in XATTN_WIDTHS for T in (1, 3, 4096, 9216)] +
               [(C, h, n, 1031, False) for C, h in XATTN_WIDTHS for n in (1, 3, 77)] +
               [(640, 10, 2, 4096, True), (640, 10, 77, 1031, True)])


def _xattn_id(case):
    C, h, n, T, off = case
    return f"C{C}h{h}n{n}T{T}" + ("_offset" if off else "")


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("case", XATTN_CASES, ids=_xattn_id)
def test_cross_attention(case, dt):
    """n = 2: the closed-form kernel (1 token, a TOK = 2 tail at 3, 9216 tokens past one sweep of the persistent grid);
    n = 1, 3, 77: LN -> scores GEMM (heads * n columns padded to 64) -> per-head softmax -> output GEMM + residual."""
    from genpercept_b200 import engine as E
    _setup()
    C, heads, n, T, off = case
    x, ctx, wts = _xattn_operands(C, heads, n, T, off, torch.Generator().manual_seed(C + n + T))
    xc = x.cuda()
    xs = _seen(xc, dt)
    ref, it = _xattn_ref(xs, ctx.cuda(), heads, [t.cuda() for t in wts])
    y = E.cross_attention(_arg(xc, dt), ctx, heads, *wts)
    torch.cuda.synchronize()
    _report(f"cross_attention {dt} {_xattn_id(case)}", (y.double() - ref).abs(), _xattn_bound(xs, ref, it, heads, n, dt))


# ------------------------------------------------------------------------------------------------ ResNet
RESNET = {   # (N, H, W, Cx, Cskip, Cout, eps)
    "r320":        (2, 32, 32, 320, 0, 320, 1e-5),       # identity residual; conv1's epilogue statistics feed norm2
    "r640_320":    (2, 16, 24, 640, 320, 320, 1e-5),     # two-source shortcut; group 21 straddles the sources
    "r320_640":    (1, 16, 16, 320, 640, 640, 1e-5),     # group 10 straddles; Cout 640: a statistics pass for norm2
    "r1280_1280":  (1, 12, 12, 1280, 1280, 1280, 1e-5),  # Cout > 512: a statistics pass for norm2
    "vae128":      (1, 128, 256, 128, 0, 128, 1e-6),     # W % 128 == 0: the patch-resident convolutions with statistics
}


def _resnet_operands(N, H, W, Cx, Cskip, Cout, gen):
    cin = Cx + Cskip
    off = torch.tensor([0.0, 2.0])[:N].view(N, 1, 1, 1)                     # per-image offsets: per-image statistics
    x = torch.randn((N, Cx, H, W), generator=gen) + off + 0.3 * torch.randn((1, Cx, 1, 1), generator=gen)
    skip = None
    if Cskip:   # a different distribution from x: a group that straddles the two has statistics of neither alone
        skip = 3.0 * torch.randn((N, Cskip, H, W), generator=gen) + 4.0 + off
    p = dict(
        norm1=(1 + 0.2 * torch.randn((cin,), generator=gen), 0.2 * torch.randn((cin,), generator=gen)),
        conv1=(torch.randn((Cout, cin, 3, 3), generator=gen) / math.sqrt(9 * cin), 0.2 * torch.randn((Cout,), generator=gen)),
        norm2=(1 + 0.2 * torch.randn((Cout,), generator=gen), 0.2 * torch.randn((Cout,), generator=gen)),
        # x 2: the block's own contribution is of the residual's order
        conv2=(2 * torch.randn((Cout, Cout, 3, 3), generator=gen) / math.sqrt(9 * Cout),
               0.2 * torch.randn((Cout,), generator=gen)),
        shortcut=None)
    if cin != Cout:
        p["shortcut"] = (torch.randn((Cout, cin, 1, 1), generator=gen) / math.sqrt(cin),
                         0.2 * torch.randn((Cout,), generator=gen))
    return x, skip, p


def _gn(x, gamma, beta, eps, silu=True, merge_batch=False, split_at=None):
    """fp64 GroupNorm(32)(+SiLU) of NCHW x: (y, |x| rstd |gamma| + |beta| + |y|, rstd per channel).  merge_batch: one set
    of statistics over the whole batch; split_at: statistics per source for a group that straddles channel split_at."""
    N, C = x.shape[:2]
    G, cg = 32, C // 32
    xg = x.reshape(N, G, -1)
    if merge_batch:
        xg = xg.transpose(0, 1).reshape(1, G, -1)
    mu = xg.mean(-1, keepdim=True)
    var = ((xg - mu) ** 2).mean(-1, keepdim=True)

    def per_channel(t):   # [N or 1, G, 1] -> [N, C, 1, 1]
        return t.repeat_interleave(cg, dim=1).view(t.shape[0], C, 1, 1).expand(N, C, 1, 1)
    mu_c, rstd_c = per_channel(mu), per_channel(1.0 / (var + eps).sqrt())
    if split_at is not None and split_at % cg:
        g0 = split_at // cg
        for lo_c, hi_c in ((g0 * cg, split_at), (split_at, (g0 + 1) * cg)):
            part = x[:, lo_c:hi_c].reshape(N, -1)
            m = part.mean(-1)
            r = 1.0 / (((part - m[:, None]) ** 2).mean(-1) + eps).sqrt()
            mu_c = mu_c.clone()
            rstd_c = rstd_c.clone()
            mu_c[:, lo_c:hi_c] = m.view(N, 1, 1, 1)
            rstd_c[:, lo_c:hi_c] = r.view(N, 1, 1, 1)
    gd, bd = gamma.double().view(1, C, 1, 1), beta.double().view(1, C, 1, 1)
    y = (x - mu_c) * rstd_c * gd + bd
    mag = x.abs() * rstd_c * gd.abs() + bd.abs()
    if silu:
        y = y * torch.sigmoid(y)
    return y, mag + y.abs(), rstd_c * gd.abs()


def _resnet_ref(x, skip, p, eps, round_to=None, variant=None):
    """fp64 ResnetBlock2D of fp64 x / skip with fp64 weights p (round_to: the 16-bit storage of the normalised operands and
    of conv1's output, as the kernels store them).  Returns (out, the pair bound's magnitude but for |out|).  variant: a wrong kernel
    ("merged_batch", "per_source_stats", "shortcut_first_source", "no_silu")."""
    rnd = (lambda t: t.to(round_to).double()) if round_to is not None else (lambda t: t)
    src = x if skip is None else torch.cat([x, skip], 1)
    silu = variant != "no_silu"
    kw = dict(silu=silu, merge_batch=variant == "merged_batch")
    if variant == "per_source_stats" and skip is not None:
        kw["split_at"] = x.shape[1]
    a1, a1mag, _ = _gn(src, *p["norm1"], eps, **kw)
    w1, b1 = p["conv1"]
    h = rnd(F.conv2d(rnd(a1), w1, b1, padding=1))
    rss1 = (F.conv2d(a1mag ** 2, w1 ** 2, b1 ** 2, padding=1)).sqrt()
    a2, a2mag, scale2 = _gn(h, *p["norm2"], eps, silu=silu, merge_batch=kw["merge_batch"])
    w2, b2 = p["conv2"]
    out = F.conv2d(rnd(a2), w2, b2, padding=1)
    sq = F.conv2d(a2mag ** 2, w2 ** 2, b2 ** 2, padding=1)
    # conv1's error (its contraction bound, in units of C u) moves the normalised operand by rstd |gamma| times; conv2
    # carries these independent errors in quadrature
    prop = F.conv2d((scale2 * (math.sqrt(9 * src.shape[1]) * rss1 + h.abs())) ** 2, w2 ** 2, padding=1).sqrt()
    K = 9 * w2.shape[1]
    if p["shortcut"] is not None:
        ws, bs = p["shortcut"]
        scs = src
        if variant == "shortcut_first_source":
            scs = torch.cat([x, torch.zeros_like(skip)], 1)
        out = out + F.conv2d(scs, ws, bs)
        sq = sq + F.conv2d(src ** 2, ws ** 2, bs ** 2)
        K += src.shape[1]
    else:
        out = out + x
        sq = sq + x ** 2
    return out, math.sqrt(K) * sq.sqrt() + prop


def _resnet_case(name, dt, device, variants=(), max_hw=None):
    N, H, W, Cx, Cskip, Cout, eps = RESNET[name]
    if max_hw:
        H, W = min(H, max_hw), min(W, max_hw)
    x, skip, p = _resnet_operands(N, H, W, Cx, Cskip, Cout, torch.Generator().manual_seed(sum(map(ord, name))))
    x = x.to(device)
    skip = None if skip is None else skip.to(device)
    if dt != "pair":   # the kernels take the 16-bit weights as given: hand them over already rounded
        p = {k: None if v is None else (v[0].to(DTYPES[dt]).float(), v[1]) for k, v in p.items()}
    p = {k: None if v is None else tuple(t.to(device) for t in v) for k, v in p.items()}
    ps = {k: None if v is None else (_seen(v[0], dt) if dt == "pair" else v[0].double(), v[1].double())
          for k, v in p.items()}
    xs, sks = _seen(x, dt), None if skip is None else _seen(skip, dt)
    rt = None if dt == "pair" else DTYPES[dt]
    ref, mag = _resnet_ref(xs, sks, ps, eps, rt)
    bound = C_RES * U * (mag + ref.abs()) + U if dt == "pair" else _bound16(ref, dt)
    wrong = []
    for v in variants:
        if (v == "merged_batch" and N == 1 or v in ("per_source_stats", "shortcut_first_source") and skip is None or
                v == "per_source_stats" and Cx % ((Cx + Cskip) // 32) == 0):   # no group straddles the sources
            continue
        wrong.append((v, (_resnet_ref(xs, sks, ps, eps, rt, v)[0] - ref).abs()))
    return x, skip, p, eps, Cout, ref, bound, wrong


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("name", list(RESNET))
def test_resnet(name, dt):
    from genpercept_b200 import engine as E
    _setup()
    x, skip, p, eps, Cout, ref, bound, _ = _resnet_case(name, dt, "cuda")
    nh = lambda t: None if t is None else E._nhwc(_arg(t, dt))
    y = E.resnet(nh(x), nh(skip), Cout, eps, p["norm1"], p["conv1"], p["norm2"], p["conv2"], p["shortcut"])
    torch.cuda.synchronize()
    _report(f"resnet {dt} {name}", (y.double().permute(0, 3, 1, 2) - ref).abs(), bound)


# ------------------------------------------------------------------------------------------------ resizes
NEAREST = [(2, 15, 15, 320, 29, 29), (1, 8, 8, 1280, 15, 15), (1, 12, 15, 640, 12, 29)]   # the UNet's odd skip sizes
BILINEAR = [(1, 9, 13, 256, 18, 25), (2, 5, 7, 256, 9, 13), (1, 24, 24, 256, 47, 48)]    # the DPT fusion's mismatches


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("case", NEAREST)
def test_nearest_resize(case, dt):
    from genpercept_b200 import engine as E
    N, H, W, C, OH, OW = case
    x = (torch.randn((N, C, H, W), generator=torch.Generator().manual_seed(H * W + C)) * 3).cuda()
    xs = _seen(x, dt)
    ref = F.interpolate(xs, size=(OH, OW), mode="nearest")
    y = E.resize(E._nhwc(_arg(x, dt)), OH, OW, "nearest")
    torch.cuda.synchronize()
    got = y.double().permute(0, 3, 1, 2)
    print(f"nearest {dt} {case}: max|err| = {(got - ref).abs().max().item():.3e}")
    assert torch.equal(got, ref), f"nearest {dt} {case}: not the gather of F.interpolate"


def _bilinear_coordinate_term(x, OH, OW):
    """The output's change when each source coordinate f = (o + 0.5) in / out - 0.5 moves by 2 u (|f| + 1): the rounding of
    the fp32 coordinates that the kernel computes (as F.interpolate does for an fp32 tensor), times the slope there."""
    def axis(I, O):
        f = ((torch.arange(O, dtype=torch.float64, device=x.device) + 0.5) * (I / O) - 0.5).clamp(min=0)
        i0 = f.floor().long().clamp(max=I - 1)
        return i0, (i0 + 1).clamp(max=I - 1), f - i0, 2 * U * (f + 1)
    y0, y1, h1, ey = axis(x.shape[2], OH)
    x0, x1, w1, ex = axis(x.shape[3], OW)
    a00, a01 = x[:, :, y0][:, :, :, x0], x[:, :, y0][:, :, :, x1]
    a10, a11 = x[:, :, y1][:, :, :, x0], x[:, :, y1][:, :, :, x1]
    h1 = h1.view(-1, 1)
    dy = (1 - w1) * (a10 - a00) + w1 * (a11 - a01)
    dx = (1 - h1) * (a01 - a00) + h1 * (a11 - a10)
    return ey.view(-1, 1) * dy.abs() + ex * dx.abs()


def _bilinear_case(case, dt, device):
    N, H, W, C, OH, OW = case
    x = (torch.randn((N, C, H, W), generator=torch.Generator().manual_seed(H * W + C)) * 3 + 5).to(device)
    xs = _seen(x, dt)
    ref = F.interpolate(xs, size=(OH, OW), mode="bilinear", align_corners=False)
    if dt == "pair":
        mag = F.interpolate(xs.abs(), size=(OH, OW), mode="bilinear", align_corners=False)
        bound = C_NORM * (U * (mag + ref.abs()) + _bilinear_coordinate_term(xs, OH, OW)) + U
    else:
        bound = _bound16(ref, dt)
    wrong = (F.interpolate(xs, size=(OH, OW), mode="bilinear", align_corners=True) - ref).abs()
    return x, ref, bound, wrong


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("case", BILINEAR)
def test_bilinear_resize(case, dt):
    from genpercept_b200 import engine as E
    x, ref, bound, _ = _bilinear_case(case, dt, "cuda")
    y = E.resize(E._nhwc(_arg(x, dt)), case[4], case[5], "bilinear")
    torch.cuda.synchronize()
    _report(f"bilinear {dt} {case}", (y.double().permute(0, 3, 1, 2) - ref).abs(), bound)


# ------------------------------------------------------------------------------------------------ discrimination (CPU)
def _discriminates(name, bound, wrong, exempt=()):
    """Asserts each wrong output breaks the bound DISCRIMINATION times, but for the `exempt` variants (the docstring's
    list), whose ratios are printed only."""
    for v, d in wrong:
        r = (d / bound).max().item()
        print(f"{name}: {v} breaks the bound {r:.1f}x" + (" (not asserted)" if v in exempt else ""))
        assert v in exempt or r >= DISCRIMINATION, f"{name}: {v} stays within {DISCRIMINATION}x of the bound ({r:.2f})"


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("T,C", [(64, C) for C in sorted({c for _, c in GEGLU_CASES})])
def test_bounds_discriminate_geglu(T, C, dt):
    variants = ("swap", "no_gate_bias") + (("tanh",) if dt == "pair" else ())
    *_, bound, wrong = _geglu_case(T, C, dt, torch.Generator().manual_seed(T + C), "cpu", variants)
    _discriminates(f"geglu {dt} C{C}", bound, wrong)


def _xattn_discrimination_cases():
    seen, out = set(), []
    for C, h, n, _T, off in XATTN_CASES:
        if (C, h, n, off) not in seen:
            seen.add((C, h, n, off))
            out.append((C, h, n, 64, off))
    return out


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("case", _xattn_discrimination_cases(), ids=_xattn_id)
def test_bounds_discriminate_cross_attention(case, dt):
    C, heads, n, T, off = case
    x, ctx, wts = _xattn_operands(C, heads, n, T, off, torch.Generator().manual_seed(C + n + T))
    xs = _seen(x, dt)
    ref, it = _xattn_ref(xs, ctx, heads, wts)
    bound = _xattn_bound(xs, ref, it, heads, n, dt)
    variants = ("swap_p", "ln_unfolded", "no_bias") if n == 2 else ("softmax_all", "groups_shifted")
    wrong = [(v, (_xattn_ref(xs, ctx, heads, wts, variant=v)[0] - ref).abs()) for v in variants]
    # a bf16 output carries the offset's rounding, as large as these changes
    _discriminates(f"cross_attention {dt} {_xattn_id(case)}", bound, wrong, variants if off and dt == "bf16" else ())


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("name", list(RESNET))
def test_bounds_discriminate_resnet(name, dt):
    *_, bound, wrong = _resnet_case(name, dt, "cpu", ("merged_batch", "per_source_stats", "shortcut_first_source", "no_silu"),
                                    max_hw=16)
    _discriminates(f"resnet {dt} {name}", bound, wrong, ("per_source_stats",) if dt == "bf16" else ())


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("case", BILINEAR)
def test_bounds_discriminate_bilinear(case, dt):
    _, _, bound, wrong = _bilinear_case(case, dt, "cpu")
    _discriminates(f"bilinear {dt} {case}", bound, [("align_corners=True", wrong)])
