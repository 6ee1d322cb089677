"""End-to-end GPU parity: the engine (through the C-ABI) against the CPU oracle on the same seeded
synthetic weights and inputs, stage by stage and for the whole single_infer path."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# fp16 storage / fp32 accumulate through ~110 GEMM-class layers: rgb_latent bounded absolutely (|ref| <= 0.87), z (unnormalised,
# std 5) relative to max|ref|, depth / normal maps absolutely.  The full-size cases and the high-precision mode
# (|delta| < 1e-3) are in tests/test_gpu_fullsize.py.
TOL = {"rgb_latent": 4e-3, "z_rel": 6e-3, "depth": 8e-3, "normal": 1.3e-2}


def _report(name, got, ref):
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    err = np.abs(got - ref)
    print(f"{name}: max|err|={err.max():.3e} mean|err|={err.mean():.3e} max|ref|={np.abs(ref).max():.3f} "
          f"std(ref)={ref.std():.3f}")
    return err.max()


@pytest.fixture(scope="module")
def engines(synth_state, text_embed):
    from genpercept_b200.engine import Engine
    out = {}
    for readout in ("vae", "dpt"):
        e = Engine(dtype=torch.float16, readout=readout)
        e.load_state("unet", synth_state["unet"])
        e.load_state("vae", synth_state["vae"])
        if readout == "dpt":
            e.load_state("dpt", synth_state["dpt"])
        e.set_text_embed(text_embed)
        e.finalize()
        out[readout] = e
    yield out
    for e in out.values():
        e.close()


def test_vae_readout_matches_golden_and_oracle(engines, synth_state, text_embed, golden_dir):
    g = np.load(os.path.join(golden_dir, "oracle_e2e_64.npz"))
    e = engines["vae"]
    rgb = torch.from_numpy(g["rgb"]).cuda()
    depth = e.infer(rgb, out_channels=1).cpu().numpy()
    lat = e.read_tensor("rgb_latent")
    z = e.read_tensor("z")
    normal = e.infer(rgb, out_channels=3).cpu().numpy()
    from oracle.pipeline import LATENT_SCALE, OraclePipeline
    p = OraclePipeline(synth_state, text_embed)
    z_ref = p.vae.post_quant_conv(-torch.from_numpy(g["unet_out"]) / LATENT_SCALE).detach().numpy()
    assert _report("rgb_latent", lat, g["rgb_latent"]) < TOL["rgb_latent"]
    assert _report("z (decoder input)", z, z_ref) < TOL["z_rel"] * np.abs(z_ref).max()
    assert _report("depth", depth, g["depth"]) < TOL["depth"]
    assert _report("normal", normal, g["normal"]) < TOL["normal"]
    assert depth.min() >= 0 and depth.max() <= 1


def test_stage_isolation_unet_and_decoder(engines, synth_state, text_embed, golden_dir):
    """Inject the oracle's latent / z so each stage is checked without upstream error."""
    from genpercept_b200 import engine as E
    from oracle.pipeline import LATENT_SCALE, OraclePipeline
    g = np.load(os.path.join(golden_dir, "oracle_e2e_64.npz"))
    e = engines["vae"]
    e.plan(2, 64, 64)
    p = OraclePipeline(synth_state, text_embed)
    e.write_tensor("rgb_latent", g["rgb_latent"])
    e.run_stage(E.STAGE_UNET)
    z_ref = p.vae.post_quant_conv(-torch.from_numpy(g["unet_out"]) / LATENT_SCALE).detach().numpy()
    assert _report("unet stage z", e.read_tensor("z"), z_ref) < TOL["z_rel"] * np.abs(z_ref).max()
    e.write_tensor("z", z_ref)
    e.run_stage(E.STAGE_READOUT, 1)
    out = e.read_tensor("out").reshape(-1)[:2 * 64 * 64].reshape(2, 1, 64, 64)   # packed [B,1,H,W]
    assert _report("decoder stage", out, g["depth"]) < TOL["depth"]


def test_dpt_readout_matches_golden(engines, golden_dir):
    g = np.load(os.path.join(golden_dir, "oracle_e2e_64.npz"))
    e = engines["dpt"]
    rgb = torch.from_numpy(g["rgb"]).cuda()
    out = e.infer(rgb).cpu().numpy()
    assert _report("dpt", out, g["dpt"]) < 8e-3          # measured 3.9e-3
    assert abs(out.min()) < 1e-6 and abs(out.max() - 1) < 1e-6     # per-image min-max


def test_determinism_host_io_and_batch_independence(engines, golden_dir):
    """(1) Run-to-run determinism: every reduction (GroupNorm partial sums included) runs in a fixed
    order with no atomics, so the same batch gives the same bits, and host-buffer I/O (the e2e path)
    equals device-buffer I/O bit for bit.  (2) Images are independent (SURVEY.md 8e): a batch of 3
    equals three batches of 1 up to the summation order of the GroupNorm partial sums (the per-CTA
    tile assignment depends on the batch shape), i.e. within the fp16 noise floor of the maps."""
    e = engines["vae"]
    gen = torch.Generator().manual_seed(11)
    rgb = torch.randint(0, 256, (3, 3, 64, 128), generator=gen, dtype=torch.uint8)
    full = e.infer(rgb.cuda(), out_channels=1).cpu()
    again = e.infer(rgb.cuda(), out_channels=1).cpu()
    host = e.infer(rgb, out_channels=1, out=torch.empty((3, 1, 64, 128), dtype=torch.float32))
    assert torch.equal(full, again)
    assert torch.equal(full, host)
    worst = 0.0
    for i in range(3):
        one = e.infer(rgb[i:i + 1].cuda(), out_channels=1).cpu()
        worst = max(worst, (one[0] - full[i]).abs().max().item())
    print(f"batch-of-3 vs 3x batch-of-1: max|delta| = {worst:.3e}")
    assert worst < 6e-3


def test_error_not_worse_than_the_reference_fp16_path(engines, synth_state, text_embed, golden_dir):
    """Tolerance calibration.  BASELINE.json asks for |delta| < 1e-3 "(fp16)" against the reference's
    diffusers path.  That path in fp16 (run.py --half_precision: every module and activation fp16,
    emulated here by the oracle in torch.float16 on CPU) itself deviates from fp32 by ~8e-3 max /
    ~8e-4 mean on these maps.  The engine (fp16 storage, fp32 accumulate and statistics) must be at
    least as close to the fp32 oracle as that reference-fp16 run is."""
    from oracle.pipeline import OraclePipeline
    g = np.load(os.path.join(golden_dir, "oracle_e2e_64.npz"))
    x = torch.from_numpy(g["rgb"]).float() / 255.0 * 2.0 - 1.0
    half = OraclePipeline(synth_state, text_embed, dtype=torch.float16)
    for mode, ch, key in (("depth", 1, "depth"), ("normal", 3, "normal")):
        ref16 = half.single_infer(x, mode=mode).float().numpy()
        ours = engines["vae"].infer(torch.from_numpy(g["rgb"]).cuda(), out_channels=ch).cpu().numpy()
        e_ref = np.abs(ref16 - g[key])
        e_ours = np.abs(ours - g[key])
        print(f"{mode}: reference-fp16 vs fp32 max {e_ref.max():.3e} mean {e_ref.mean():.3e} | "
              f"engine vs fp32 max {e_ours.max():.3e} mean {e_ours.mean():.3e}")
        assert e_ours.mean() <= 1.25 * e_ref.mean() + 1e-4
        assert e_ours.max() <= 1.25 * e_ref.max() + 1e-3


@pytest.mark.parametrize("hw", [(72, 88), (104, 64), (64, 120)])
def test_sizes_that_are_multiples_of_8_only(engines, synth_state, text_embed, hw):
    """H/8 or W/8 odd at some UNet level: diffusers' `upsample_size` path (resize to the skip's 2n-1 extent, then the
    plain 3x3 conv) — e.g. the 432x768 a 16:9 image becomes at the default processing resolution."""
    from oracle.pipeline import OraclePipeline
    H, W = hw
    g = torch.Generator().manual_seed(H * 1000 + W)
    rgb = torch.randint(0, 256, (2, 3, H, W), generator=g, dtype=torch.uint8)
    e = engines["vae"]
    depth = e.infer(rgb.cuda(), out_channels=1).cpu().numpy()
    normal = e.infer(rgb.cuda(), out_channels=3).cpu().numpy()
    p = OraclePipeline(synth_state, text_embed)
    x = rgb.float() / 255.0 * 2.0 - 1.0
    ref_d = p.single_infer(x, mode="depth").numpy()
    ref_n = p.single_infer(x, mode="normal").numpy()
    assert depth.shape == (2, 1, H, W) and normal.shape == (2, 3, H, W)
    assert _report(f"depth {H}x{W}", depth, ref_d) < TOL["depth"]
    assert _report(f"normal {H}x{W}", normal, ref_n) < TOL["normal"]
    # sizes that are not multiples of 8 / 64 run too (tests/test_gpu_boundary.py); the result extent follows the graph
    assert tuple(e.infer(torch.zeros((1, 3, 68, 64), dtype=torch.uint8, device="cuda")).shape) == (1, 1, 64, 64)
    assert tuple(engines["dpt"].infer(torch.zeros((1, 3, 72, 64), dtype=torch.uint8, device="cuda")).shape) == (1, 1, 96, 64)


@pytest.mark.parametrize("ntok", [1, 5, 13])
def test_general_context_length(synth_state, text_embed, ntok):
    """Non-empty prompts (SURVEY.md §8 f3): an n-token context takes the general cross-attention path (two 1x1 GEMMs
    around a per-head softmax) instead of the 2-token closed form; compared with the oracle's SDPA."""
    from genpercept_b200.engine import Engine
    from oracle.pipeline import OraclePipeline
    g = torch.Generator().manual_seed(100 + ntok)
    te = torch.randn((1, ntok, 1024), generator=g) * float(text_embed.float().std())
    e = Engine(dtype=torch.float16, readout="vae")
    try:
        e.load_state("unet", synth_state["unet"])
        e.load_state("vae", synth_state["vae"])
        e.set_text_embed(te)
        e.finalize()
        rgb = torch.randint(0, 256, (2, 3, 64, 64), generator=g, dtype=torch.uint8)
        depth = e.infer(rgb.cuda(), out_channels=1).cpu().numpy()
    finally:
        e.close()
    ref = OraclePipeline(synth_state, te).single_infer(rgb.float() / 255.0 * 2.0 - 1.0, mode="depth").numpy()
    assert _report(f"depth, {ntok}-token context", depth, ref) < TOL["depth"]
    # the context matters: the 2-token empty-prompt result is a different map
    ref2 = OraclePipeline(synth_state, text_embed).single_infer(rgb.float() / 255.0 * 2.0 - 1.0, mode="depth").numpy()
    print("   |oracle(n tokens) - oracle(empty prompt)| max", float(np.abs(ref - ref2).max()))


def test_high_precision_mode_meets_the_stated_tolerance(synth_state, text_embed, golden_dir):
    """precision="high" (what torch_dtype=float32, the reference's default, selects): every operand an fp16 (hi, lo)
    pair, hi*hi + lo*hi + hi*lo on the tensor cores, fp32 accumulate.  BASELINE.json's north_star asks |delta| < 1e-3
    against the reference path; stage by stage the error must be fp32-class."""
    from genpercept_b200.engine import Engine
    from oracle.pipeline import LATENT_SCALE, OraclePipeline
    g = np.load(os.path.join(golden_dir, "oracle_e2e_64.npz"))
    rgb = torch.from_numpy(g["rgb"]).cuda()
    p = OraclePipeline(synth_state, text_embed)
    z_ref = p.vae.post_quant_conv(-torch.from_numpy(g["unet_out"]) / LATENT_SCALE).detach().numpy()
    for readout in ("vae", "dpt"):
        e = Engine(dtype=torch.float16, readout=readout, precision="high")
        try:
            e.load_state("unet", synth_state["unet"])
            e.load_state("vae", synth_state["vae"])
            if readout == "dpt":
                e.load_state("dpt", synth_state["dpt"])
            e.set_text_embed(text_embed)
            e.finalize()
            if readout == "vae":
                depth = e.infer(rgb, out_channels=1).cpu().numpy()
                lat, z = e.read_tensor("rgb_latent"), e.read_tensor("z")
                normal = e.infer(rgb, out_channels=3).cpu().numpy()
                assert _report("high: rgb_latent", lat, g["rgb_latent"]) < 2e-4
                assert _report("high: z", z, z_ref) < 4e-4 * np.abs(z_ref).max()      # measured 1.3e-4
                assert _report("high: depth", depth, g["depth"]) < 1e-3
                assert _report("high: normal", normal, g["normal"]) < 1e-3
            else:
                assert _report("high: dpt", e.infer(rgb).cpu().numpy(), g["dpt"]) < 1e-3
        finally:
            e.close()


def test_mid_size_against_the_oracle(engines, synth_state, text_embed):
    """256x384, batch 2: the largest size the CPU oracle finishes in seconds; exercises the patch-resident conv
    loop (W % 128 == 0), multi-block attention (T = 1536) and the TMA residual path with full tiles."""
    from oracle.pipeline import OraclePipeline
    g = torch.Generator().manual_seed(256384)
    rgb = torch.randint(0, 256, (2, 3, 256, 384), generator=g, dtype=torch.uint8)
    depth = engines["vae"].infer(rgb.cuda(), out_channels=1).cpu().numpy()
    torch.set_num_threads(min(16, torch.get_num_threads()))
    ref = OraclePipeline(synth_state, text_embed).single_infer(rgb.float() / 255.0 * 2.0 - 1.0, mode="depth").numpy()
    assert _report("depth 256x384", depth, ref) < TOL["depth"]


def test_full_size_properties(engines):
    """BASELINE.json configs[1] shape (8 x 768 x 768), where the oracle would take minutes: size-independent
    properties of the path instead — run-to-run bits, host I/O == device I/O, batch permutation equivariance
    (images are independent, SURVEY.md 8e), output range, and the DPT readout's per-image min-max."""
    e = engines["vae"]
    g = torch.Generator().manual_seed(768)
    base = torch.rand((8, 3, 12, 12), generator=g)
    rgb = (torch.nn.functional.interpolate(base, size=(768, 768), mode="bicubic").clamp(0, 1) * 255).to(torch.uint8)
    a = e.infer(rgb.cuda(), out_channels=1).cpu()
    b = e.infer(rgb.cuda(), out_channels=1).cpu()
    assert torch.equal(a, b)
    host_out = torch.empty((8, 1, 768, 768), dtype=torch.float32).pin_memory()
    assert torch.equal(e.infer(rgb.pin_memory(), out_channels=1, out=host_out), a)
    assert a.min() >= 0 and a.max() <= 1 and a.std() > 1e-3
    perm = torch.tensor([3, 0, 7, 1, 6, 2, 5, 4])
    c = e.infer(rgb[perm].cuda(), out_channels=1).cpu()
    # not bitwise: the GroupNorm partial sums are added in a different (still fixed) order when the images move to
    # other CTAs, and 16-bit activations turn that 1e-6 perturbation into the network's fp16 noise floor — the same
    # magnitude as the engine-vs-oracle error, with the maximum taken over 4.7 M pixels here
    dl = (c - a[perm]).abs()
    print(f"768x768 batch-8 permutation: max|delta| = {dl.max().item():.3e} mean = {dl.mean().item():.3e}")
    assert dl.mean().item() < 1.5e-3 and dl.max().item() < 4e-2
    n3 = e.infer(rgb[:2].cuda(), out_channels=3).cpu()
    assert n3.shape == (2, 3, 768, 768) and n3.min() >= 0 and n3.max() <= 1
    dd = engines["dpt"].infer(rgb[:2].cuda()).cpu()
    for i in range(2):
        assert dd[i].min().item() == 0.0 and dd[i].max().item() == 1.0
