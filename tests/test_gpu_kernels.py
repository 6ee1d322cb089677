"""GPU parity of the individual CUDA kernels (through the C-ABI per-kernel entry points) against
plain fp32 PyTorch references of the same op on the same 16-bit-rounded inputs.

Tolerances: the kernels accumulate in fp32 and round once to fp16 on store, so the bound is one
fp16 ulp of the output magnitude plus accumulation-order noise: |err| <= 2e-3 * max|ref| + 1e-3.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _setup():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _rand(shape, gen, scale=1.0, dtype=torch.float16):
    return (torch.randn(shape, generator=gen) * scale).to(dtype)


def _check(name, got, ref, rel=2e-3, abs_=1e-3):
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs().max().item()
    bound = rel * ref.abs().max().item() + abs_
    print(f"{name}: max|err|={err:.3e} bound={bound:.3e} max|ref|={ref.abs().max().item():.3f}")
    assert torch.isfinite(got).all(), name + ": non-finite output"
    assert err <= bound, f"{name}: max|err| {err:.3e} > {bound:.3e}"


def _conv_ref(x_nchw, w, b, mode):
    x = x_nchw.float()
    if mode == 0:
        return F.conv2d(x, w, b, padding=w.shape[-1] // 2)
    if mode == 1:
        return F.conv2d(x, w, b, stride=2, padding=1)
    if mode == 2:
        return F.conv2d(F.pad(x, (0, 1, 0, 1)), w, b, stride=2)
    return F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), w, b, padding=1)


def _run_conv(N, H, W, Cin, Cout, ks, mode, direct, dtype=torch.float16, bias=True, residual=False, relu=False,
              seed=0):
    from genpercept_b200 import engine as E
    _setup()
    g = torch.Generator().manual_seed(seed)
    x = _rand((N, Cin, H, W), g, 1.0, dtype)
    w = _rand((Cout, Cin, ks, ks), g, 1.0 / (Cin * ks * ks) ** 0.5, dtype).float()
    b = torch.randn((Cout,), generator=g) * 0.1 if bias else None
    ref = _conv_ref(x.cuda(), w.cuda(), b.cuda() if bias else None, mode)
    res = None
    if residual:
        res = _rand(tuple(ref.shape), g, 1.0, dtype).cuda()
        ref = ref + res.float()
    if relu:
        ref = ref.relu()
    xn = E._nhwc(x.cuda())
    resn = E._nhwc(res) if residual else None
    y = E.conv2d(xn, w, b, mode=mode, residual=resn, relu=relu, direct=direct)
    torch.cuda.synchronize()
    rel = 2e-3 if dtype == torch.float16 else 1.6e-2
    if mode == 3 and not direct:
        rel *= 2   # the fused kernel rounds the parity-summed weights to 16 bit (SURVEY.md App. C.7)
    _check(f"conv N{N} {H}x{W} {Cin}->{Cout} k{ks} mode{mode} direct{int(direct)}", y.permute(0, 3, 1, 2), ref, rel)


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_direct_conv_matches_torch(mode):
    _run_conv(2, 12, 12, 8, 24, 3, mode, direct=True)


def test_direct_conv_1x1():
    _run_conv(1, 8, 8, 32, 1, 1, 0, direct=True)


@pytest.mark.parametrize("tokens,cin,cout", [(256, 64, 64), (1000, 320, 640), (4096, 1280, 320), (144, 640, 5120),
                                             (77, 32, 16)])
def test_igemm_linear(tokens, cin, cout):
    _run_conv(1, 1, tokens, cin, cout, 1, 0, direct=False)


def test_igemm_linear_bias_residual_relu():
    _run_conv(2, 16, 16, 320, 320, 1, 0, direct=False, residual=True, relu=True)


@pytest.mark.parametrize("shape", [(1, 16, 16, 64, 64), (2, 32, 32, 128, 128), (1, 24, 24, 320, 320),
                                   (1, 12, 12, 1280, 256), (2, 96, 96, 128, 256), (1, 8, 8, 512, 512),
                                   (1, 4, 4, 64, 32), (1, 2, 2, 64, 16), (1, 1, 1, 128, 64), (1, 48, 48, 1920, 640),
                                   (1, 128, 128, 128, 128), (1, 64, 64, 256, 8), (2, 32, 32, 8, 128), (1, 16, 16, 8, 320),
                                   # wide images with narrow N: the patch-resident main loop (halo reuse)
                                   (2, 256, 256, 128, 128), (1, 256, 256, 64, 64), (1, 256, 384, 256, 128)])
def test_igemm_conv3x3(shape):
    _run_conv(*shape, 3, 0, direct=False)


def test_igemm_conv3x3_residual():
    _run_conv(2, 32, 32, 256, 256, 3, 0, direct=False, residual=True)


def test_igemm_conv3x3_patch_mode_residual_relu():
    _run_conv(1, 256, 256, 128, 128, 3, 0, direct=False, residual=True, relu=True)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("shape", [(1, 16, 16, 64, 64), (2, 96, 96, 128, 128), (1, 8, 8, 320, 320), (1, 2, 2, 1280, 1280)])
def test_igemm_conv3x3_stride2(shape, mode):
    _run_conv(*shape, 3, mode, direct=False)


@pytest.mark.parametrize("shape", [(1, 16, 16, 64, 64), (2, 48, 48, 256, 256), (1, 12, 12, 1280, 1280), (1, 1, 1, 128, 128),
                                   (1, 96, 96, 128, 128)])
def test_igemm_conv3x3_upsample_fused(shape):
    _run_conv(*shape, 3, 3, direct=False)


def test_igemm_conv_bf16():
    _run_conv(1, 32, 32, 128, 128, 3, 0, direct=False, dtype=torch.bfloat16)


@pytest.mark.parametrize("shape,groups,silu", [((2, 32, 32, 128), 32, True), ((1, 24, 24, 320), 32, False),
                                               ((1, 8, 8, 1920), 32, True), ((2, 64, 64, 512), 32, True)])
def test_groupnorm(shape, groups, silu):
    from genpercept_b200 import engine as E
    _setup()
    g = torch.Generator().manual_seed(1)
    N, H, W, C = shape
    x = (_rand((N, C, H, W), g).float() * 1.5 + 0.3).half()
    gamma = 1 + 0.1 * torch.randn((C,), generator=g)
    beta = 0.1 * torch.randn((C,), generator=g)
    ref = F.group_norm(x.cuda().float(), groups, gamma.cuda(), beta.cuda(), 1e-6)
    if silu:
        ref = F.silu(ref)
    y = E.groupnorm(E._nhwc(x.cuda()), groups, gamma, beta, 1e-6, silu)
    _check(f"groupnorm {shape} silu={silu}", y.permute(0, 3, 1, 2), ref)


# Each case runs the GroupNorm pass, then the tap-streaming convolution: the patch-resident kernel also needs at least
# 128 output pixels per SM, more than any of these sizes has (test_igemm_conv3x3 runs it on wide images).
@pytest.mark.parametrize("case", [
    dict(N=1, H=64, W=128, Cin=128, Cout=128),
    dict(N=2, H=16, W=256, Cin=128, Cout=256),                     # two images: per-image statistics
    dict(N=1, H=8, W=128, Cin=64, Cout=512),                       # several N tiles over the same normalised source
    dict(N=1, H=5, W=128, Cin=64, Cout=64),                        # odd height
    dict(N=1, H=32, W=128, Cin=128, Cout=128, Csc=256),            # + 1x1 shortcut over the raw block input (extra K segment)
    dict(N=1, H=16, W=384, Cin=256, Cout=256, Csc=512),            # same with wider maps and channels
    dict(N=1, H=32, W=128, Cin=128, Cout=128, residual=True),      # + identity residual
    dict(N=2, H=32, W=256, Cin=128, Cout=1, out_f32=True),         # conv_norm_out -> conv_out (channel mean) -> fp32 map
    dict(N=1, H=32, W=128, Cin=128, Cout=3, out_f32=True),
    dict(N=1, H=24, W=96, Cin=128, Cout=128),                      # W % 128 != 0
    dict(N=1, H=16, W=128, Cin=128, Cout=128, silu=False),
])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_groupnorm_conv3x3(case, dtype):
    """GroupNorm(32)+SiLU as a GroupNorm pass followed by the convolution, against F.group_norm -> F.silu -> F.conv2d
    on the same 16-bit inputs and weights, with the normalised tensor rounded to the storage type in between."""
    from genpercept_b200 import engine as E
    _setup()
    N, H, W, Cin, Cout = (case[k] for k in ("N", "H", "W", "Cin", "Cout"))
    Csc, silu = case.get("Csc"), case.get("silu", True)
    g = torch.Generator().manual_seed(Cin * 7 + Cout)
    x = (_rand((N, Cin, H, W), g).float() * 1.5 + 0.3 * torch.randn((N, Cin, 1, 1), generator=g)).to(dtype)
    gamma = 1 + 0.1 * torch.randn((Cin,), generator=g)
    beta = 0.1 * torch.randn((Cin,), generator=g)
    w = _rand((Cout, Cin, 3, 3), g, 1.0 / (Cin * 9) ** 0.5, dtype).float()
    b = torch.randn((Cout,), generator=g) * 0.1
    a = F.group_norm(x.cuda().float(), 32, gamma.cuda(), beta.cuda(), 1e-6)
    if silu:
        a = F.silu(a)
    ref = F.conv2d(a.to(dtype).float(), w.cuda(), b.cuda(), padding=1)
    sc_x = sc_w = sc_b = res = None
    if Csc:
        sc = _rand((N, Csc, H, W), g, dtype=dtype)
        sc_w = _rand((Cout, Csc, 1, 1), g, 1.0 / Csc ** 0.5, dtype).float()
        sc_b = torch.randn((Cout,), generator=g) * 0.1
        ref = ref + F.conv2d(sc.cuda().float(), sc_w.cuda(), sc_b.cuda())
        sc_x = E._nhwc(sc.cuda())
    if case.get("residual"):
        r = _rand((N, Cout, H, W), g, dtype=dtype)
        ref = ref + r.cuda().float()
        res = E._nhwc(r.cuda())
    y = E.gn_conv3x3(E._nhwc(x.cuda()), 32, gamma, beta, 1e-6, silu, w, b, sc_x=sc_x, sc_w=sc_w, sc_b=sc_b, residual=res,
                     out_f32=case.get("out_f32", False))
    torch.cuda.synchronize()
    got = y if case.get("out_f32") else y.permute(0, 3, 1, 2)
    # the normalised operand is rounded to 16 bit before the MMA, as in the reference, but with tanh.approx inside
    # SiLU: 2^-11 relative on operands of magnitude ~1 over K = 9 Cin terms.  bf16 outputs carry 8 significant bits:
    # the bound of the other bf16 convolutions.
    rel = 3e-3 if dtype == torch.float16 else 1.6e-2
    _check(f"gn+conv {case} {dtype}", got, ref, rel=rel, abs_=2e-3)


@pytest.mark.parametrize("tokens,C", [(100, 320), (64, 640), (33, 1280)])
def test_layernorm(tokens, C):
    from genpercept_b200 import engine as E
    _setup()
    g = torch.Generator().manual_seed(2)
    x = _rand((tokens, C), g, 2.0)
    gamma = 1 + 0.1 * torch.randn((C,), generator=g)
    beta = 0.1 * torch.randn((C,), generator=g)
    ref = F.layer_norm(x.cuda().float(), (C,), gamma.cuda(), beta.cuda(), 1e-5)
    y = E.layernorm(x.cuda(), gamma, beta, 1e-5)
    _check(f"layernorm {tokens}x{C}", y, ref)


@pytest.mark.parametrize("B,T,heads,d", [(2, 256, 5, 64), (1, 144, 20, 64), (1, 1024, 1, 512), (1, 16, 20, 64),
                                         (2, 4, 20, 64), (1, 1, 20, 64), (1, 2304, 10, 64),
                                         # long d = 512 rows: the bulk-copy pipelined row softmax (3 / 6 vectors per thread)
                                         (1, 2304, 1, 512), (1, 9216, 1, 512), (1, 9600, 1, 512)])
def test_attention(B, T, heads, d):
    from genpercept_b200 import engine as E
    _setup()
    g = torch.Generator().manual_seed(3)
    C = heads * d
    q, k, v = (_rand((B, T, C), g) for _ in range(3))
    scale = d ** -0.5

    def sp(t):
        return t.cuda().float().view(B, T, heads, d).transpose(1, 2)
    # the engine rounds scale*q to 16 bit (scale is folded into Wq there); mirror that in the reference
    qs = (q.float() * scale).half()
    ref = F.scaled_dot_product_attention(sp(qs), sp(k), sp(v), scale=1.0).transpose(1, 2).reshape(B, T, C)
    o = E.attention(q.cuda(), k.cuda(), v.cuda(), heads, scale)
    # S and P are stored in fp16 by this (unfused) path: allow 1e-2 relative
    _check(f"attention B{B} T{T} h{heads} d{d}", o, ref, rel=1e-2, abs_=2e-3)


def test_bilinear_up2x_align_corners():
    from genpercept_b200 import engine as E
    _setup()
    g = torch.Generator().manual_seed(4)
    x = _rand((2, 256, 12, 20), g)
    ref = F.interpolate(x.cuda().float(), scale_factor=2, mode="bilinear", align_corners=True)
    y = E.bilinear_up2x(E._nhwc(x.cuda()))
    _check("bilinear", y.permute(0, 3, 1, 2), ref)
