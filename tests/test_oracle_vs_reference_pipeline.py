"""Pins the oracle's orchestration (oracle/pipeline.py) against the REFERENCE'S OWN ``GenPerceptPipeline.single_infer`` /
``encode_rgb`` / ``decode_pred`` (genpercept/genpercept_pipeline.py:375-526 of the reference), its UNet forward, its
scheduler constants, its host image helpers and its first release's pipeline.

tests/golden/make_golden_reference.py executes the reference's code around the oracle's own VAE / UNet modules and
one-step scheduler (behind thin adapters, plus the reference's DPT head class) on seeded inputs and stores the outputs
in tests/golden/reference_pipeline.npz.  Everything between those modules — latent scaling, the mean half of the
moments, the scheduler call and ``pred_original_sample``, ``/ scale`` + post_quant_conv + decoder, the channel mean,
clip and shift, the DPT feature order and min-max — is therefore the reference's code, not a restatement; here the
oracle recomputes the same inputs and must match it.  (What stays unpinned is the inside of the diffusers blocks; see
oracle/__init__.py.)"""
import os

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
UNET_SIZES = ((8, 8), (9, 11), (12, 10))        # as in make_golden_reference.py
FEAT_STRIDE = 8
RESIZE_EDGES = (64, 128, 200)


@pytest.fixture(scope="module")
def ref():
    z = np.load(os.path.join(GOLDEN, "reference_pipeline.npz"))
    return {k: z[k] for k in z.files}


def _t(a):
    return torch.from_numpy(np.asarray(a))


def test_single_infer_glue_matches_the_reference(ref, synth_state, text_embed):
    from oracle.pipeline import OraclePipeline
    g = torch.Generator().manual_seed(21)
    rgb = torch.rand((1, 3, 64, 64), generator=g) * 2 - 1
    # VAE readout, 1- and 3-channel modes
    op = OraclePipeline(synth_state, text_embed)
    for mode in ("depth", "normal"):
        r = _t(ref[f"glue_{mode}"])
        mine = op.single_infer(rgb, mode=mode)
        assert r.shape == mine.shape and torch.allclose(r, mine, atol=1e-6, rtol=0), float((r - mine).abs().max())
    with torch.no_grad():
        assert torch.allclose(_t(ref["glue_latent"]), op.encode_rgb(rgb), atol=1e-7)
    # --fix_timesteps: the reference feeds that timestep to the UNet instead of the scheduler's
    assert torch.allclose(_t(ref["glue_fix7"]), op.single_infer(rgb, mode="normal", fix_timesteps=7), atol=1e-6, rtol=0)
    # DPT readout (the reference's own head class)
    od = OraclePipeline(synth_state, text_embed, use_dpt=True)
    r = _t(ref["glue_dpt"])
    mine = od.single_infer(rgb, mode="depth")
    assert r.shape == mine.shape and torch.allclose(r, mine, atol=2e-6, rtol=0), float((r - mine).abs().max())


def test_unet_dataflow_matches_the_reference_forward(ref, synth_state, text_embed):
    """genpercept/models/custom_unet.py:34-427 of the reference (its own UNet forward: skip stack, the `upsample_size`
    forwarding for odd extents, the DPT feature taps, conv_norm_out / conv_out) executed around the ORACLE's blocks,
    against oracle.unet's forward (feature taps: every FEAT_STRIDE-th channel is stored)."""
    from oracle.pipeline import OraclePipeline
    ou = OraclePipeline(synth_state, text_embed).unet
    g = torch.Generator().manual_seed(4)
    ctx = text_embed.float().reshape(1, -1, 1024)
    for i, (h, w) in enumerate(UNET_SIZES):                    # multiples of 8, odd extents, 8 does not divide
        x = torch.randn((1, 4, h, w), generator=g)
        with torch.no_grad():
            r = _t(ref[f"unet{i}_sample"])
            mine = ou(x, torch.tensor([1]), ctx)
            assert torch.allclose(r, mine, atol=1e-6, rtol=0), (h, w, float((r - mine).abs().max()))
            mf = ou(x, torch.tensor([1]), ctx, return_feature=True)
            rf = [_t(ref[f"unet{i}_feat{k}"]) for k in range(4) if f"unet{i}_feat{k}" in ref]
            assert len(rf) == len(mf) == 4
            for a, b in zip(rf, mf):
                b = b[:, ::FEAT_STRIDE]
                assert a.shape == b.shape and torch.allclose(a, b, atol=1e-5, rtol=0)


def test_scheduler_constants_match_the_reference_class(ref):
    """src/customized_modules/ddim.py:144-217 of the reference (DDIMSchedulerCustomized.__init__ — the part of the
    scheduler that IS in the reference tree; set_timesteps / step are diffusers') instantiated from the reference's own
    hf_configs/scheduler_beta_1.0_1.0/scheduler_config.json, against oracle.scheduler.DDIMOneStep."""
    from oracle.scheduler import DDIMOneStep
    mine = DDIMOneStep()
    assert torch.equal(_t(ref["sched_betas"]), mine.betas) and torch.equal(_t(ref["sched_alphas_cumprod"]), mine.alphas_cumprod)
    assert torch.equal(_t(ref["sched_final_alpha_cumprod"]), torch.as_tensor(mine.final_alpha_cumprod))
    assert float(ref["sched_alphas_cumprod"][1]) == 0.0 and float(ref["sched_init_noise_sigma"]) == 1.0   # beta = 1: x_t carries no signal
    # one DDIM step at the single timestep the pipeline uses (t = 1, leading spacing + offset 1): x0 = -v
    ts = mine.set_timesteps(1)
    assert ts.tolist() == [1]
    g = torch.Generator().manual_seed(0)
    v, x = torch.randn((1, 4, 8, 8), generator=g), torch.randn((1, 4, 8, 8), generator=g)
    prev, x0 = mine.step(v, 1, x)
    assert torch.equal(x0, -v)


def test_host_image_helpers_match_the_reference_functions(ref):
    """genpercept_b200.image_util (host mirror) and oracle.imgproc against the reference's own
    genpercept/util/image_util.py: resize_max_res (:75-105), get_tv_resample_method (:108-119), chw2hwc (:66-72)."""
    from genpercept_b200 import image_util as mine
    from oracle import imgproc as IP
    g = torch.Generator().manual_seed(8)
    x = torch.randint(0, 256, (1, 3, 90, 160), generator=g, dtype=torch.uint8)
    for edge in RESIZE_EDGES:
        r = _t(ref[f"resize{edge}"])
        assert torch.equal(mine.resize_max_res(x, edge), r)
        assert tuple(r.shape[-2:]) == IP.resize_max_res_shape(90, 160, edge)
        d = np.abs(IP.resize_aa(x.numpy(), *r.shape[-2:]).astype(np.int32) - r.numpy().astype(np.int32))
        assert d.max() <= 1 and (d > 0).mean() <= 1e-3
    for m in ("bilinear", "bicubic", "nearest"):
        assert str(mine.get_tv_resample_method(m)) == str(ref[f"tv_{m}"])
    with pytest.raises(ValueError):
        mine.get_tv_resample_method("lanczos")
    assert bool(ref["tv_lanczos_raises"])
    c = torch.rand((3, 4, 5), generator=g)
    assert torch.equal(mine.chw2hwc(c), _t(ref["chw2hwc"])) and np.array_equal(mine.chw2hwc(c.numpy()), ref["chw2hwc"])


def test_legacy_v1_pipeline_closed_form_matches(ref, synth_state):
    """GenPercept_v1/genpercept/pipeline_genpercept.py:263-354 of the reference — the first release hard-codes what the
    v2 scheduler collapses to (t = 1, pred_latent = -unet_pred, no scheduler object) and feeds the full 77-token padded
    empty-prompt embedding (GenPercept_v1/empty_text_embed.npy).  Its single_infer around the oracle's modules must equal
    the oracle run with that 77-token context (range [-1,1] there, [0,1] in v2); the embedding is stored as
    tests/golden/empty_text_embed_77x1024.npy."""
    from oracle.pipeline import OraclePipeline
    te = torch.from_numpy(np.load(os.path.join(GOLDEN, "empty_text_embed_77x1024.npy")).astype(np.float32))[None]
    op = OraclePipeline(synth_state, te)
    g = torch.Generator().manual_seed(31)
    rgb = torch.rand((1, 3, 64, 64), generator=g) * 2 - 1
    r = _t(ref["v1_depth"])
    mine = op.single_infer(rgb, mode="depth") * 2.0 - 1.0
    # (x + 1) / 2 * 2 - 1 and the different place of the channel mean cost a few fp32 ulps of values up to 1
    assert r.shape == mine.shape and torch.allclose(r, mine, atol=2e-5, rtol=0), float((r - mine).abs().max())
