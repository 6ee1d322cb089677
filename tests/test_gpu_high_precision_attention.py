"""Memory-efficient attention in the high-precision mode (precision="high", what torch_dtype=float32 selects): with the
switch on, every head-dim-64 self-attention and head-dim-512 VAE mid-block attention runs through the fused
split-precision kernels (fattn.cu, fattn512.cu), so no T x T score matrix is stored.  With it off, the plans are the
ones the mode always had.

  * kernel parity of both paths against fp64 attention on the exact (hi + lo) inputs, and the fused kernel alone at
    T = 20000, where the unfused softmax cannot run;
  * the engine with the switch on against the oracle golden (64 x 64) and the CPU oracle at 512 x 512;
  * the plan's shape with the switch on, and no change at all with it off or in the 16-bit modes;
  * a clean, non-poisoning failure with the switch off where the unfused softmax cannot run;
  * GenPerceptPipeline(torch_dtype=float32) at native photo sizes after enable_xformers_memory_efficient_attention().
"""
import os
import re

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# test_gpu_fullsize.py's bounds for the high-precision engine (north_star: |delta| < 1e-3)
TOL_HIGH = {"rgb_latent": 2e-4, "z_rel": 4e-4, "out": 1e-3, "out_p999": 1e-3, "out_mean": 2e-4, "dpt": 1e-3}
SWITCH = re.compile(r"memory.efficient attention", re.I)


def _stats(name, got, ref):
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    err = np.abs(got - ref).reshape(-1)
    p999 = float(np.quantile(err, 0.999)) if err.size > 1000 else float(err.max())
    print(f"  {name:<28s} max {err.max():.3e}  p99.9 {p999:.3e}  mean {err.mean():.3e}  (max|ref| {np.abs(ref).max():.3f})")
    return float(err.max()), p999, float(err.mean())


def _rgb(B, H, W, seed):
    """Smooth synthetic images (bicubic-upsampled noise) plus pixel noise, as in test_gpu_fullsize.py."""
    g = torch.Generator().manual_seed(seed)
    base = torch.rand((B, 3, max(H // 48, 2), max(W // 48, 2)), generator=g)
    img = torch.nn.functional.interpolate(base, size=(H, W), mode="bicubic", align_corners=False)
    img = img + 0.05 * torch.randn((B, 3, H, W), generator=g)
    return (img.clamp(0, 1) * 255).to(torch.uint8)


def _engine(synth_state, text_embed, precision="high", readout="vae", mea=False):
    from genpercept_b200.engine import Engine
    torch.cuda.empty_cache()
    e = Engine(dtype=torch.float16, readout=readout, precision=precision, memory_efficient_attention=mea)
    e.load_state("unet", synth_state["unet"])
    e.load_state("vae", synth_state["vae"])
    if readout == "dpt":
        e.load_state("dpt", synth_state["dpt"])
    e.set_text_embed(text_embed)
    e.finalize()
    return e


def _inputs(B, T, heads, d, seed):
    g = torch.Generator().manual_seed(seed)
    C = heads * d
    # q scaled up so that each row's softmax is dominated by a few keys (the running maximum has to move)
    q = (3.0 * torch.randn((B, T, C), generator=g)).cuda()
    k = torch.randn((B, T, C), generator=g).cuda()
    v = torch.randn((B, T, C), generator=g).cuda()
    return q, k, v


def _exact(x):
    """the value the engine sees: hi + lo of x's split, in fp64"""
    from genpercept_b200.engine import split_hi_lo
    hi, lo = split_hi_lo(x)
    return hi.double() + lo.double()


def _attention_ref(q, k, v, heads, scale, rows=1024):
    """fp64 softmax(scale q k^T) v per head on the exact split values, a chunk of query rows at a time"""
    B, T, C = q.shape
    d = C // heads
    qs, kx, vx = _exact(q * scale), _exact(k), _exact(v)
    out = torch.empty((B, T, C), dtype=torch.float64, device=q.device)
    for b in range(B):
        for h in range(heads):
            cs = slice(h * d, (h + 1) * d)
            for r in range(0, T, rows):
                s = qs[b, r:r + rows, cs] @ kx[b, :, cs].T
                out[b, r:r + rows, cs] = torch.softmax(s, dim=-1) @ vx[b, :, cs]
    return out


# ragged T: not a multiple of 64 or 128
@pytest.mark.parametrize("heads,d", [(5, 64), (1, 512)])
@pytest.mark.parametrize("B,T", [(1, 3001), (2, 4100)])
def test_fused_split_attention_matches_fp64(B, T, heads, d):
    from genpercept_b200 import engine as E
    q, k, v = _inputs(B, T, heads, d, 64 * T + d + B)
    scale = d ** -0.5
    ref = _attention_ref(q, k, v, heads, scale)
    errs = {}
    for fused in (True, False):
        o = E.attention_high(q, k, v, heads, scale, fused)
        torch.cuda.synchronize()
        assert torch.isfinite(o).all()
        errs[fused] = (o.double() - ref).abs().max().item()
    print(f"split attention B{B} T{T} heads {heads} d {d}: max|err| fused {errs[True]:.3e}  unfused {errs[False]:.3e}  "
          f"(max|ref| {ref.abs().max().item():.3f})")
    assert errs[True] <= 2.0 * errs[False] + 1e-5


@pytest.mark.parametrize("heads,d", [(5, 64), (1, 512)])
def test_fused_split_attention_past_the_unfused_row_limit(heads, d):
    """T = 20000 is a multiple of 8 past the 16384 keys the unfused softmax takes: only the fused kernel runs."""
    from genpercept_b200 import engine as E
    B, T = 1, 20000
    q, k, v = _inputs(B, T, heads, d, 20000 + d)
    scale = d ** -0.5
    with pytest.raises(RuntimeError):
        E.attention_high(q, k, v, heads, scale, fused=False)
    o = E.attention_high(q, k, v, heads, scale, fused=True)
    ref = _attention_ref(q, k, v, heads, scale, rows=512)
    err = (o.double() - ref).abs().max().item()
    print(f"split attention T{T} heads {heads} d {d}: fused max|err| {err:.3e} (max|ref| {ref.abs().max().item():.3f})")
    assert torch.isfinite(o).all()
    # the ragged-T cases above measure 1e-5 relative to max|ref| at T ~ 4000 for both paths; the error grows with T
    assert err <= 1e-4 * ref.abs().max().item()


def test_engine_with_the_switch_matches_the_golden(synth_state, text_embed, golden_dir):
    """test_gpu_e2e.py::test_high_precision_mode_meets_the_stated_tolerance's bounds, with the switch on."""
    from oracle.pipeline import LATENT_SCALE, OraclePipeline
    g = np.load(os.path.join(golden_dir, "oracle_e2e_64.npz"))
    rgb = torch.from_numpy(g["rgb"]).cuda()
    z_ref = OraclePipeline(synth_state, text_embed).vae.post_quant_conv(
        -torch.from_numpy(g["unet_out"]) / LATENT_SCALE).detach().numpy()
    e = _engine(synth_state, text_embed, mea=True)
    try:
        depth = e.infer(rgb, out_channels=1).cpu().numpy()
        lat, z = e.read_tensor("rgb_latent"), e.read_tensor("z")
        normal = e.infer(rgb, out_channels=3).cpu().numpy()
    finally:
        e.close()
    assert _stats("rgb_latent", lat, g["rgb_latent"])[0] < 2e-4
    assert _stats("z", z, z_ref)[0] < 4e-4 * np.abs(z_ref).max()
    assert _stats("depth", depth, g["depth"])[0] < 1e-3
    assert _stats("normal", normal, g["normal"])[0] < 1e-3
    e = _engine(synth_state, text_embed, readout="dpt", mea=True)
    try:
        assert _stats("dpt", e.infer(rgb).cpu().numpy(), g["dpt"])[0] < 1e-3
    finally:
        e.close()


def test_plan_with_the_switch(synth_state, text_embed):
    """1024 x 1024 (T = 16384, the largest the unfused softmax takes): every attention fused, no score matrix, and a
    smaller arena than the same plan without the switch (5.4 GB of S at the UNet's first level)."""
    e = _engine(synth_state, text_embed)
    try:
        e.plan(1, 1024, 1024)
        arena_off = e.plan_info()["arena_bytes"]
        e.set_memory_efficient_attention(True)
        assert e.plan_count() == 0                     # a change of the switch drops the cached plans
        e.plan(1, 1024, 1024)
        arena_on = e.plan_info()["arena_bytes"]
        names = [op["name"] for op in e.profile_ops()]
    finally:
        e.close()
    print(f"1024x1024 high precision: arena {arena_off} bytes without the switch, {arena_on} with it")
    assert not any(n.endswith(".softmax") for n in names)
    assert sum(n.endswith(".fattn") for n in names) == 16
    fused512 = [n for n in names if n.endswith(".fattn512")]
    assert len(fused512) == 2 and all(".mid_block." in n for n in fused512)
    assert arena_on < arena_off


def test_engine_at_512_matches_the_oracle(synth_state, text_embed):
    """512 x 512 with the switch on, against the CPU oracle with test_gpu_fullsize.py's TOL_HIGH."""
    from oracle.pipeline import LATENT_SCALE, OraclePipeline
    H, W = 512, 512
    rgb = _rgb(1, H, W, 5121)
    e = _engine(synth_state, text_embed, mea=True)
    try:
        depth = e.infer(rgb.cuda(), out_channels=1).cpu().numpy()
        lat = e.read_tensor("rgb_latent")
        z = e.read_tensor("z")
        normal = e.infer(rgb.cuda(), out_channels=3).cpu().numpy()
    finally:
        e.close()
    n = torch.get_num_threads()
    torch.set_num_threads(min(32, max(n, 1)))
    try:
        p = OraclePipeline(synth_state, text_embed)
        ref_n, inter = p.single_infer(rgb.float() / 255.0 * 2.0 - 1.0, mode="normal", return_intermediates=True)
        z_ref = p.vae.post_quant_conv(inter["pred_latent"] / LATENT_SCALE).detach().numpy()
    finally:
        torch.set_num_threads(n)
    dec = inter["decoded"]
    ref_d = (torch.clip(dec.mean(dim=1, keepdim=True), -1.0, 1.0) + 1.0) / 2.0
    assert _stats("rgb_latent", lat, inter["rgb_latent"].numpy())[0] < TOL_HIGH["rgb_latent"]
    assert _stats("z (decoder input)", z, z_ref)[0] / np.abs(z_ref).max() < TOL_HIGH["z_rel"]
    for name, got, ref in (("depth", depth, ref_d.numpy()), ("normal", normal, ref_n.numpy())):
        mx, p999, mean = _stats(name, got, ref)
        assert mx < TOL_HIGH["out"] and p999 < TOL_HIGH["out_p999"] and mean < TOL_HIGH["out_mean"], name


def test_switch_toggled_off_changes_nothing(synth_state, text_embed):
    """768 x 768, high precision: an engine switched on and off again computes a fresh engine's maps bit for bit."""
    rgb = _rgb(1, 768, 768, 768).cuda()
    e = _engine(synth_state, text_embed)
    try:
        e.infer(rgb, out_channels=1)
        e.set_memory_efficient_attention(True)
        e.infer(rgb, out_channels=1)
        e.set_memory_efficient_attention(False)
        got = e.infer(rgb, out_channels=1).cpu().numpy()
    finally:
        e.close()
    f = _engine(synth_state, text_embed)
    try:
        ref = f.infer(rgb, out_channels=1).cpu().numpy()
    finally:
        f.close()
    assert np.array_equal(got, ref)


def test_switch_is_ignored_by_the_16bit_mode(synth_state, text_embed):
    rgb = _rgb(1, 768, 768, 769).cuda()
    res = {}
    for mea in (False, True):
        e = _engine(synth_state, text_embed, precision="default", mea=mea)
        try:
            out = e.infer(rgb, out_channels=1).cpu().numpy()
            res[mea] = (out, e.plan_info()["arena_bytes"], [op["name"] for op in e.profile_ops()])
        finally:
            e.close()
    assert res[True][1] == res[False][1]
    assert res[True][2] == res[False][2]
    assert np.array_equal(res[True][0], res[False][0])


def test_unfused_row_limit_fails_cleanly_without_the_switch(synth_state, text_embed):
    """1280 x 960 (T = 19200) without the switch: gp_plan refuses, names the switch, and the engine stays usable."""
    rgb = _rgb(1, 64, 64, 65)
    e = _engine(synth_state, text_embed)
    try:
        with pytest.raises(RuntimeError) as ei:
            e.plan(1, 960, 1280)
        print("plan without the switch:", ei.value)
        assert SWITCH.search(str(ei.value))
        got = e.infer(rgb.cuda(), out_channels=1).cpu().numpy()
    finally:
        e.close()
    f = _engine(synth_state, text_embed)
    try:
        ref = f.infer(rgb.cuda(), out_channels=1).cpu().numpy()
    finally:
        f.close()
    assert np.isfinite(got).all()
    assert np.array_equal(got, ref)


def test_native_photo_sizes_in_fp32(synth_state, text_embed):
    """GenPerceptPipeline(torch_dtype=float32) + enable_xformers_memory_efficient_attention(), processing_res=0."""
    import time

    from PIL import Image
    from genpercept_b200.pipeline import GenPerceptPipeline
    torch.cuda.empty_cache()
    pipe = GenPerceptPipeline(unet=synth_state["unet"], vae=synth_state["vae"], text_embed=text_embed,
                              torch_dtype=torch.float32)
    pipe.enable_xformers_memory_efficient_attention()
    arena = {}
    try:
        for (W, H) in ((2016, 1512), (4032, 3024), (2591, 3873)):
            img = _rgb(1, H, W, W + H)[0].permute(1, 2, 0).numpy()
            t0 = time.perf_counter()
            out = pipe(Image.fromarray(img), processing_res=0, mode="depth", color_map=None)
            dt = time.perf_counter() - t0
            arena[(W, H)] = pipe._engine.plan_info()["arena_bytes"]
            pred = out.pred_np
            print(f"{W}x{H}: arena {arena[(W, H)] / 2**30:.2f} GiB, first call {dt:.2f} s, "
                  f"pred range [{pred.min():.3f}, {pred.max():.3f}]")
            assert pred.shape == (H, W)
            assert np.isfinite(pred).all() and pred.min() >= 0.0 and pred.max() <= 1.0
    finally:
        pipe._engine.close()
    # 4x the pixels: linear growth gives ~4x the arena, a T^2 score matrix would give ~16x
    assert arena[(4032, 3024)] <= 5 * arena[(2016, 1512)]
