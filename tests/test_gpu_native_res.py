"""Native-resolution inputs in the 16-bit modes: the fused head-dim-512 attention of the VAE mid-block (fattn512.cu)
takes over once the unfused path's score matrix would pass 2 GiB, so the memory a plan needs grows with the pixel count
rather than its square.

  * kernel parity just past the threshold, ragged T, fp16 and bf16, against an fp32 reference;
  * the whole engine past the threshold against the CPU oracle on the seeded weights (test_gpu_fullsize.py's bounds);
  * GenPerceptPipeline at a 12 MP photo's own size (processing_res=0), and a portrait size that is not a multiple of 8;
  * a plan too large for the card raises without poisoning the engine.
"""
import re

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# test_gpu_fullsize.py's bounds for the fp16-storage engine
TOL16 = {"rgb_latent": 8e-3, "z_rel": 6e-3, "out": 2e-2, "out_p999": 9e-3, "out_mean": 1.5e-3}


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


def _engine(synth_state, text_embed, precision="default"):
    from genpercept_b200.engine import Engine
    torch.cuda.empty_cache()                      # the large plans here want the memory earlier tests left cached
    e = Engine(dtype=torch.float16, readout="vae", precision=precision)
    e.load_state("unet", synth_state["unet"])
    e.load_state("vae", synth_state["vae"])
    e.set_text_embed(text_embed)
    e.finalize()
    return e


def _attention_ref(qs, k, v, rows=2048):
    """softmax(qs k^T) v in fp32 on the GPU, a chunk of query rows at a time (the full S would not fit)."""
    out = torch.empty(qs.shape, dtype=torch.float32, device=qs.device)
    kf, vf = k.float(), v.float()
    for b in range(qs.shape[0]):
        for r in range(0, qs.shape[1], rows):
            s = qs[b, r:r + rows].float() @ kf[b].T
            out[b, r:r + rows] = torch.softmax(s, dim=-1) @ vf[b]
    return out


# S = B * T * Tp * 2 bytes: 2.59 GB and 2.30 GB, both past the 2 GiB at which the fused kernel takes over; and
# T = 20000 (0.8 GB), a multiple of 8 past the 16384-key rows the unfused path's softmax takes
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,T", [(1, 36001), (2, 24001), (1, 20000)])
def test_fused_d512_attention_matches_fp32(B, T, dtype):
    from genpercept_b200 import engine as E
    assert B * T * ((T + 7) // 8 * 8) * 2 > 2 << 30 or (T % 8 == 0 and T > 16384)
    g = torch.Generator().manual_seed(512 + T)
    d = 512
    scale = d ** -0.5
    # q scaled up so that each row's softmax is dominated by a few keys (the running maximum has to move)
    q = (3.0 * torch.randn((B, T, d), generator=g)).to(dtype).cuda()
    k = torch.randn((B, T, d), generator=g).to(dtype).cuda()
    v = torch.randn((B, T, d), generator=g).to(dtype).cuda()
    o = E.attention(q, k, v, 1, scale)
    # the engine rounds scale * q to 16 bit (the scale is folded into Wq there); mirror that in the reference
    qs = (q.float() * scale).to(dtype)
    ref = _attention_ref(qs, k, v)
    torch.cuda.synchronize()
    assert torch.isfinite(o).all()
    err = (o.float() - ref).abs()
    bound = 1e-2 * ref.abs().max().item() + 2e-3              # test_gpu_kernels.py::test_attention's bound
    print(f"fused d512 B{B} T{T} {dtype}: max|err| {err.max().item():.3e} mean {err.mean().item():.3e} "
          f"bound {bound:.3e} max|ref| {ref.abs().max().item():.3f}")
    assert err.max().item() <= bound


def test_engine_past_threshold_matches_oracle(synth_state, text_embed):
    """1544 x 1736: T = 193 * 217 = 41881 latent tokens, 3.5 GB of S on the unfused path."""
    from oracle.pipeline import LATENT_SCALE, OraclePipeline
    H, W = 1544, 1736
    rgb = _rgb(1, H, W, 1544)
    e = _engine(synth_state, text_embed)
    try:
        depth = e.infer(rgb.cuda(), out_channels=1).cpu().numpy()
        lat = e.read_tensor("rgb_latent")
        z = e.read_tensor("z")
        normal = e.infer(rgb.cuda(), out_channels=3).cpu().numpy()
        names = [op["name"] for op in e.profile_ops(out_channels=1)]
    finally:
        e.close()
    fused = [n for n in names if n.endswith(".fattn512")]
    print("fused d=512 attention ops:", fused)
    assert len(fused) == 2 and all(".mid_block." in n for n in fused)
    assert not any(n.endswith(".softmax") for n in names)

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
    assert _stats("rgb_latent", lat, inter["rgb_latent"].numpy())[0] < TOL16["rgb_latent"]
    assert _stats("z (decoder input)", z, z_ref)[0] / np.abs(z_ref).max() < TOL16["z_rel"]
    for name, got, ref in (("depth", depth, ref_d.numpy()), ("normal", normal, ref_n.numpy())):
        mx, p999, mean = _stats(name, got, ref)
        assert mx < TOL16["out"] and p999 < TOL16["out_p999"] and mean < TOL16["out_mean"], name


def test_native_photo_sizes(synth_state, text_embed):
    """pipe(photo, processing_res=0) at a 12 MP photo's own size and at a portrait size that is not a multiple of 8."""
    from PIL import Image
    from genpercept_b200.pipeline import GenPerceptPipeline
    torch.cuda.empty_cache()
    pipe = GenPerceptPipeline(unet=synth_state["unet"], vae=synth_state["vae"], text_embed=text_embed,
                              torch_dtype=torch.float16)
    arena = {}
    for (W, H) in ((2016, 1512), (4032, 3024), (2591, 3873)):
        img = _rgb(1, H, W, W + H)[0].permute(1, 2, 0).numpy()
        out = pipe(Image.fromarray(img), processing_res=0, mode="depth", color_map=None)
        arena[(W, H)] = pipe._engine.plan_info()["arena_bytes"]
        pred = out.pred_np
        print(f"{W}x{H}: arena {arena[(W, H)] / 2**30:.2f} GiB, pred range [{pred.min():.3f}, {pred.max():.3f}]")
        assert pred.shape == (H, W)
        assert np.isfinite(pred).all() and pred.min() >= 0.0 and pred.max() <= 1.0
    # 4x the pixels: linear growth gives ~4x the arena, a T^2 score matrix would give ~16x
    assert arena[(4032, 3024)] <= 5 * arena[(2016, 1512)]


def test_oversized_plan_raises_without_poisoning(synth_state, text_embed):
    """The high-precision mode still stores S for the attention layers; at 4032 x 3024 its arena cannot be allocated.
    The plan fails with the size it needs, and the same engine then runs a small image exactly as a fresh engine does."""
    rgb = _rgb(1, 64, 64, 64)
    e = _engine(synth_state, text_embed, precision="high")
    try:
        with pytest.raises(RuntimeError) as ei:
            e.plan(1, 3024, 4032)
        msg = str(ei.value)
        print("oversized plan:", msg)
        m = re.search(r"(\d+) bytes", msg)
        assert m and int(m.group(1)) > torch.cuda.get_device_properties(0).total_memory
        got = e.infer(rgb.cuda(), out_channels=1).cpu().numpy()
    finally:
        e.close()
    f = _engine(synth_state, text_embed, precision="high")
    try:
        ref = f.infer(rgb.cuda(), out_channels=1).cpu().numpy()
    finally:
        f.close()
    assert np.isfinite(got).all()
    assert np.array_equal(got, ref)
