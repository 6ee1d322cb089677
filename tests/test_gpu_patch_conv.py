"""GPU parity of the patch-resident implicit GEMM (igemm_patch.cu) at the shapes it now takes: 16 x 8 MT pixel tiles of 8 x 8
m64 blocks, the 1x1 shortcut as more K chunks, epilogue statistics, and both storage types.

Each case is compared with F.conv2d in fp32 on the same 16-bit operands and weights, at the bounds of test_igemm_conv3x3:
|err| <= rel * max|ref| + abs with rel = 2e-3 in fp16 and 1.6e-2 in bf16 (one output rounding plus accumulation-order
noise).  Every case first asserts, through the planner's own rule (gp_conv_tile), that the layer is planned onto the patch
kernel with the tile it is meant to exercise, and every size has at least as many tiles as an H100 has SMs.
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


def _rel(dtype):
    return 2e-3 if dtype == torch.float16 else 1.6e-2


def _check(name, got, ref, rel, abs_=1e-3):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs().max().item()
    bound = rel * ref.abs().max().item() + abs_
    print(f"{name}: max|err|={err:.3e} bound={bound:.3e} max|ref|={ref.abs().max().item():.3f}")
    assert torch.isfinite(got).all(), name + ": non-finite output"
    assert err <= bound, f"{name}: max|err| {err:.3e} > {bound:.3e}"


def _assert_patch(N, H, W, cin, cout, csc=0, mt=None):
    from genpercept_b200 import engine as E
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    plan = E.conv_tile(N, H, W, cin, cout, csc=csc, num_sms=sms)
    assert plan["patch"], f"{N}x{H}x{W} {cin}->{cout}: planned onto the tap-streaming kernel ({plan})"
    if mt is not None:
        assert plan["mt"] == mt, plan
    tiles = N * (W // plan["tw"]) * (H // plan["th"]) * -(-cout // plan["bn"])
    assert tiles >= sms, (plan, tiles)


@pytest.mark.parametrize("case", [
    dict(N=1, H=192, W=192, Cin=512, Cout=512),                    # the VAE's 192^2 level
    dict(N=1, H=96, W=96, Cin=512, Cout=512, residual=True),       # the VAE's 96^2 level, identity residual through TMA
    dict(N=4, H=96, W=96, Cin=320, Cout=320, mt=2),                # the UNet's 96^2 level: BN = 64, 16 x 16 tiles
    dict(N=2, H=48, W=48, Cin=640, Cout=640),                      # the UNet's 48^2 level
    dict(N=1, H=768, W=768, Cin=128, Cout=128),                    # the widest maps (formerly the one-row tiles)
    dict(N=1, H=64, W=272, Cin=128, Cout=128, relu=True),          # W % 128 != 0, tiles of a non-square map
    dict(N=1, H=192, W=192, Cin=256, Cout=512, dtype=torch.bfloat16),
], ids=lambda c: "_".join(f"{k}{v}" for k, v in c.items() if k != "dtype") + ("_bf16" if c.get("dtype") else ""))
def test_patch_conv3x3(case):
    from genpercept_b200 import engine as E
    _setup()
    N, H, W, Cin, Cout = (case[k] for k in ("N", "H", "W", "Cin", "Cout"))
    dtype = case.get("dtype", torch.float16)
    _assert_patch(N, H, W, Cin, Cout, mt=case.get("mt"))
    g = torch.Generator().manual_seed(Cin * 3 + Cout + H)
    x = _rand((N, Cin, H, W), g, 1.0, dtype)
    w = _rand((Cout, Cin, 3, 3), g, 1.0 / (Cin * 9) ** 0.5, dtype).float()
    b = torch.randn((Cout,), generator=g) * 0.1
    ref = F.conv2d(x.cuda().float(), w.cuda(), b.cuda(), padding=1)
    res = None
    if case.get("residual"):
        res = _rand(tuple(ref.shape), g, 1.0, dtype).cuda()
        ref = ref + res.float()
    if case.get("relu"):
        ref = ref.relu()
    y = E.conv2d(E._nhwc(x.cuda()), w, b, mode=0, residual=None if res is None else E._nhwc(res), relu=case.get("relu", False),
                 direct=False)
    torch.cuda.synchronize()
    _check(f"patch conv {case}", y.permute(0, 3, 1, 2), ref, _rel(dtype))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_patch_conv3x3_shortcut_one_source(dtype):
    """GroupNorm+SiLU -> 3x3 conv + 1x1 shortcut over the raw block input (the VAE's channel-changing ResNets), 96^2 x
    512 -> 256: the shortcut's chunks run through the patch slots after the nine taps."""
    from genpercept_b200 import engine as E
    _setup()
    N, H, W, Cin, Cout, Csc = 1, 96, 96, 512, 256, 512
    _assert_patch(N, H, W, Cin, Cout, csc=Csc)
    g = torch.Generator().manual_seed(11)
    x = (_rand((N, Cin, H, W), g).float() * 1.5 + 0.3 * torch.randn((N, Cin, 1, 1), generator=g)).to(dtype)
    gamma = 1 + 0.1 * torch.randn((Cin,), generator=g)
    beta = 0.1 * torch.randn((Cin,), generator=g)
    w = _rand((Cout, Cin, 3, 3), g, 1.0 / (Cin * 9) ** 0.5, dtype).float()
    b = torch.randn((Cout,), generator=g) * 0.1
    sc = _rand((N, Csc, H, W), g, dtype=dtype)
    sc_w = _rand((Cout, Csc, 1, 1), g, 1.0 / Csc ** 0.5, dtype).float()
    sc_b = torch.randn((Cout,), generator=g) * 0.1
    a = F.silu(F.group_norm(x.cuda().float(), 32, gamma.cuda(), beta.cuda(), 1e-6))
    ref = F.conv2d(a.to(dtype).float(), w.cuda(), b.cuda(), padding=1) + F.conv2d(sc.cuda().float(), sc_w.cuda(), sc_b.cuda())
    y = E.gn_conv3x3(E._nhwc(x.cuda()), 32, gamma, beta, 1e-6, True, w, b, sc_x=E._nhwc(sc.cuda()), sc_w=sc_w, sc_b=sc_b)
    torch.cuda.synchronize()
    # the normalised operand is rounded to 16 bit as in the reference, but SiLU runs with tanh.approx: the bound of
    # test_groupnorm_conv3x3
    _check(f"patch gn+conv+shortcut {dtype}", y.permute(0, 3, 1, 2), ref, 3e-3 if dtype == torch.float16 else 1.6e-2, 2e-3)


def test_patch_resnet_shortcut_two_sources():
    """ResnetBlock2D over concat(hidden, skip), 96^2 x (256 + 128) -> 512: conv2's 1x1 shortcut reads the two sources as two
    shortcut segments of the patch kernel (the planner takes a shortcut along when it is no wider than the main source).  Reference: fp32 torch on the same 16-bit operands, with
    the normalised operands and conv1's output rounded to fp16 as the kernels store them."""
    from genpercept_b200 import engine as E
    _setup()
    N, H, W, Cx, Cskip, Cout = 1, 96, 96, 256, 128, 512
    cin = Cx + Cskip
    _assert_patch(N, H, W, cin, Cout)              # conv1 (GroupNorm materialised: one source)
    _assert_patch(N, H, W, Cout, Cout, csc=cin)    # conv2 + the two-source shortcut
    g = torch.Generator().manual_seed(21)
    x = (torch.randn((N, Cx, H, W), generator=g) + 0.3 * torch.randn((1, Cx, 1, 1), generator=g)).half()
    skip = (2.0 * torch.randn((N, Cskip, H, W), generator=g) + 1.0).half()
    rw = lambda *s: (torch.randn(s, generator=g) / (s[1] * s[2] * s[3]) ** 0.5).half().float()
    norm1 = (1 + 0.2 * torch.randn((cin,), generator=g), 0.2 * torch.randn((cin,), generator=g))
    conv1 = (rw(Cout, cin, 3, 3), 0.2 * torch.randn((Cout,), generator=g))
    norm2 = (1 + 0.2 * torch.randn((Cout,), generator=g), 0.2 * torch.randn((Cout,), generator=g))
    conv2 = (rw(Cout, Cout, 3, 3), 0.2 * torch.randn((Cout,), generator=g))
    short = (rw(Cout, cin, 1, 1), 0.2 * torch.randn((Cout,), generator=g))
    cu = lambda t: t.cuda().float()
    src = torch.cat([cu(x), cu(skip)], 1)
    a1 = F.silu(F.group_norm(src, 32, cu(norm1[0]), cu(norm1[1]), 1e-5)).half().float()
    h = F.conv2d(a1, cu(conv1[0]), cu(conv1[1]), padding=1).half().float()
    a2 = F.silu(F.group_norm(h, 32, cu(norm2[0]), cu(norm2[1]), 1e-5)).half().float()
    ref = F.conv2d(a2, cu(conv2[0]), cu(conv2[1]), padding=1) + F.conv2d(src, cu(short[0]), cu(short[1]))
    y = E.resnet(E._nhwc(x.cuda()), E._nhwc(skip.cuda()), Cout, 1e-5, norm1, conv1, norm2, conv2, short)
    torch.cuda.synchronize()
    # two chained convolutions: a one-ulp difference in conv1's rounded output moves norm2's operand; the bound of the
    # GroupNorm convolutions
    _check("patch resnet 256+128->512", y.permute(0, 3, 1, 2), ref, 3e-3, 2e-3)


def test_patch_conv_groupnorm_statistics():
    """3x3 conv 96^2 x 512 -> 512 whose epilogue produces the GroupNorm partial sums, then GroupNorm+SiLU over the
    conv's output and a skip (gp_conv_groupnorm): the statistics are gathered over the 8 x 4-pixel store boxes."""
    from genpercept_b200 import engine as E
    _setup()
    N, H, W, Cin, Cout, Cskip = 2, 96, 96, 512, 512, 128
    _assert_patch(N, H, W, Cin, Cout)
    g = torch.Generator().manual_seed(31)
    x = _rand((N, Cin, H, W), g)
    w = _rand((Cout, Cin, 3, 3), g, 1.0 / (Cin * 9) ** 0.5).float()
    b = torch.randn((Cout,), generator=g) * 0.1
    skip = (_rand((N, Cskip, H, W), g).float() + 2.0).half()
    gamma = 1 + 0.1 * torch.randn((Cout + Cskip,), generator=g)
    beta = 0.1 * torch.randn((Cout + Cskip,), generator=g)
    yc_ref = F.conv2d(x.cuda().float(), w.cuda(), b.cuda(), padding=1)
    yc, y = E.conv_groupnorm(E._nhwc(x.cuda()), w, b, 32, gamma, beta, 1e-6, True, skip=E._nhwc(skip.cuda()))
    torch.cuda.synchronize()
    _check("patch conv (statistics)", yc.permute(0, 3, 1, 2), yc_ref, 2e-3)
    # GroupNorm of what the conv stored (its 16-bit output), as the kernel normalises it
    cat = torch.cat([yc.permute(0, 3, 1, 2).float(), skip.cuda().float()], 1)
    y_ref = F.silu(F.group_norm(cat, 32, gamma.cuda(), beta.cuda(), 1e-6))
    _check("patch conv -> groupnorm", y.permute(0, 3, 1, 2), y_ref, 3e-3, 2e-3)
