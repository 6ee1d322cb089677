"""Oracle parity at the BASELINE.json shapes (768x768 depth / normal / DPT readout, plus the 512 and 1024 points of
the resolution sweep): the engine through the C-ABI against the CPU oracle on the same seeded weights and inputs,
with the error attributed per stage (rgb_latent -> z -> out).  The oracle needs ~20 s per 768x768 image on the GPU
box's host cores, so every test runs it once and compares everything it can against that one run.

Two precisions are checked:
  * the default fp16-storage engine against fixed bounds (TOL16, the class of the reference's own fp16 run);
  * the opt-in high-precision engine (precision="high": split-fp16 operands, fp32-class products) against the
    |delta| < 1e-3 that BASELINE.json's north_star states (TOL_HIGH).
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# fp16-storage engine at 768x768 x 2: the maximum is taken over 1.2 - 3.5 M pixels, so it is bounded together with the
# 99.9th percentile and the mean (the reference's own fp16 run deviates by the same amount, test_gpu_e2e.py).
TOL16 = {"rgb_latent": 8e-3, "z_rel": 6e-3, "out": 2e-2, "out_p999": 9e-3, "out_mean": 1.5e-3, "dpt": 8e-3}
TOL_HIGH = {"rgb_latent": 2e-4, "z_rel": 4e-4, "out": 1e-3, "out_p999": 1e-3, "out_mean": 2e-4, "dpt": 1e-3}   # north_star: |delta| < 1e-3


def _stats(name, got, ref):
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    err = np.abs(got - ref).reshape(-1)
    p999 = float(np.quantile(err, 0.999)) if err.size > 1000 else float(err.max())
    print(f"  {name:<28s} max {err.max():.3e}  p99.9 {p999:.3e}  mean {err.mean():.3e}  (max|ref| {np.abs(ref).max():.3f})")
    return _Err(float(err.max()), p999, float(err.mean()))


class _Err(float):
    """max |err| as a float, with the tail and mean attached"""
    def __new__(cls, mx, p999, mean):
        o = super().__new__(cls, mx)
        o.p999, o.mean = p999, mean
        return o


def _rgb(B, H, W, seed):
    """Smooth synthetic images (bicubic-upsampled noise) plus pixel noise: closer to photographs than white noise,
    which GroupNorm turns into a constant map."""
    g = torch.Generator().manual_seed(seed)
    base = torch.rand((B, 3, max(H // 48, 2), max(W // 48, 2)), generator=g)
    img = torch.nn.functional.interpolate(base, size=(H, W), mode="bicubic", align_corners=False)
    img = img + 0.05 * torch.randn((B, 3, H, W), generator=g)
    return (img.clamp(0, 1) * 255).to(torch.uint8)


def _engine(synth_state, text_embed, readout, precision):
    from genpercept_b200.engine import Engine
    e = Engine(dtype=torch.float16, readout=readout, precision=precision)
    e.load_state("unet", synth_state["unet"])
    e.load_state("vae", synth_state["vae"])
    if readout == "dpt":
        e.load_state("dpt", synth_state["dpt"])
    e.set_text_embed(text_embed)
    e.finalize()
    return e


@pytest.fixture(scope="module")
def oracle_threads():
    n = torch.get_num_threads()
    torch.set_num_threads(min(32, max(n, 1)))
    yield
    torch.set_num_threads(n)


def _precisions(want):
    """GP_TEST_PRECISIONS=default limits a run to the fp16-storage engine (bring-up aid)."""
    import os
    only = os.environ.get("GP_TEST_PRECISIONS")
    return tuple(p for p in want if p in only.split(",")) if only else tuple(want)


def _vae_case(synth_state, text_embed, B, R, seed, precisions=("default", "high")):
    from oracle.pipeline import LATENT_SCALE, OraclePipeline
    rgb = _rgb(B, R, R, seed)
    p = OraclePipeline(synth_state, text_embed)
    x = rgb.float() / 255.0 * 2.0 - 1.0
    ref_n, inter = p.single_infer(x, mode="normal", return_intermediates=True)
    dec = inter["decoded"]                                          # [B,3,R,R] before the clip
    ref_d = (torch.clip(dec.mean(dim=1, keepdim=True), -1.0, 1.0) + 1.0) / 2.0       # :523-525, :470-472
    z_ref = p.vae.post_quant_conv(inter["pred_latent"] / LATENT_SCALE).detach().numpy()
    worst = {}
    for prec in _precisions(precisions):
        tol = TOL16 if prec == "default" else TOL_HIGH
        e = _engine(synth_state, text_embed, "vae", prec)
        try:
            print(f"\n{R}x{R} batch {B}, precision={prec}")
            depth = e.infer(rgb.cuda(), out_channels=1).cpu().numpy()
            lat = e.read_tensor("rgb_latent")
            z = e.read_tensor("z")
            normal = e.infer(rgb.cuda(), out_channels=3).cpu().numpy()
        finally:
            e.close()
        w = {"rgb_latent": _stats("rgb_latent", lat, inter["rgb_latent"].numpy()),
             "z": _stats("z (decoder input)", z, z_ref) / np.abs(z_ref).max(),
             "depth": _stats("depth", depth, ref_d.numpy()),
             "normal": _stats("normal", normal, ref_n.numpy())}
        worst[prec] = w
        assert w["rgb_latent"] < tol["rgb_latent"]
        assert w["z"] < tol["z_rel"]
        for k in ("depth", "normal"):
            assert w[k] < tol["out"] and w[k].p999 < tol["out_p999"] and w[k].mean < tol["out_mean"], (k, prec)
    return worst


def test_depth_and_normal_768_batch2(synth_state, text_embed, oracle_threads):
    """BASELINE.json configs[1] / configs[2] shape (768x768; depth = channel mean, normal = 3 channels)."""
    _vae_case(synth_state, text_embed, 2, 768, 7681)


def test_depth_512_batch1(synth_state, text_embed, oracle_threads):
    """configs[0] / configs[4] point: one 512x512 image."""
    _vae_case(synth_state, text_embed, 1, 512, 5121)


def test_depth_1024_batch1(synth_state, text_embed, oracle_threads):
    """configs[4] point: 1024x1024 (T = 16384 self-attention keys, the largest tensors of the sweep)."""
    _vae_case(synth_state, text_embed, 1, 1024, 10241, precisions=("default",))


def test_dpt_readout_768(synth_state, text_embed, oracle_threads):
    """configs[3] shape: DPT-head readout at 768x768 (min-max normalised per image)."""
    from oracle.pipeline import OraclePipeline
    rgb = _rgb(1, 768, 768, 7683)
    ref, inter = OraclePipeline(synth_state, text_embed, use_dpt=True).single_infer(
        rgb.float() / 255.0 * 2.0 - 1.0, return_intermediates=True)
    for prec in _precisions(("default", "high")):
        tol = TOL16 if prec == "default" else TOL_HIGH
        e = _engine(synth_state, text_embed, "dpt", prec)
        try:
            print(f"\nDPT readout 768x768, precision={prec}")
            out = e.infer(rgb.cuda()).cpu().numpy()
            feats = [e.read_tensor(f"feat{i}") for i in range(4)]
        finally:
            e.close()
        for i, f in enumerate(feats):                     # engine keeps up-block order; the oracle list is reversed
            r = inter["feats"][3 - i].numpy()
            _stats(f"unet feat{i} (rel to max)", f / np.abs(r).max(), r / np.abs(r).max())
        assert _stats("dpt map", out, ref.numpy()) < tol["dpt"]
