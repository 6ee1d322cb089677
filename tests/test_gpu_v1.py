"""GenPercept v1 on the GPU: Pillow-exact resizing (gp_resize_pil), v1's post-processing (gp_v1_postprocess) against
v1's torch expressions, the v1 pipeline against the reference's own v1 ``__call__`` (tests/golden/v1_call.npz, made by
tests/golden/make_golden_v1.py), the 77-token context in the high-precision mode, and the torch.hub entry points."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = {"depth": 8e-3, "normal": 1.3e-2}          # the fp16 engine against the fp32 reference (tests/test_gpu_e2e.py)


def _embed77(golden_dir):
    return torch.from_numpy(np.load(os.path.join(golden_dir, "empty_text_embed_77x1024.npy")).astype(np.float32))[None]


def _photo(W, H, seed):
    g = torch.Generator().manual_seed(seed)
    base = torch.rand((1, 3, 12, 16), generator=g)
    img = F.interpolate(base, size=(H, W), mode="bicubic", align_corners=False)[0]
    img = (img + 0.1 * torch.rand((3, H, W), generator=g)).clamp(0, 1)
    return (img.permute(1, 2, 0).numpy() * 255).astype(np.uint8)


# (W, H) -> (OW, OH), as PIL's size tuples
RESIZE_CASES = [((4032, 3024), (768, 576)), ((1920, 1080), (768, 432)), ((100, 75), (768, 576)), ((97, 131), (64, 86)),
                ((200, 120), (77, 120)), ((200, 120), (200, 51)), ((150, 90), (150, 90)), ((300, 1), (97, 1))]


@pytest.mark.parametrize("src,dst", RESIZE_CASES)
def test_resize_pil_is_byte_exact(src, dst):
    from genpercept_b200 import engine as E
    a = _photo(src[0], src[1], seed=src[0] + 7 * src[1])
    ref = np.asarray(Image.fromarray(a).resize(dst))                         # BICUBIC, Pillow's default
    got = E.resize_pil(a, dst[1], dst[0])
    assert got.is_cuda and got.shape == (3, dst[1], dst[0])
    assert np.array_equal(got.cpu().numpy().transpose(1, 2, 0), ref)
    host = E.resize_pil(torch.from_numpy(a), dst[1], dst[0], device="cpu")    # host buffers in and out
    assert torch.equal(host, got.cpu())
    dev_in = E.resize_pil(torch.from_numpy(a).cuda(), dst[1], dst[0])          # a device image
    assert torch.equal(dev_in, got)


def _v1_torch(y, task, size):
    """v1's expressions (pipeline_genpercept.py __call__ / image_util.norm_to_rgb) on p = 2 y - 1, on the device."""
    p = y * 2 - 1
    if size is not None:
        p = F.interpolate(p, size, mode="nearest" if task in ("seg", "sr") else "bilinear")
    if task == "depth":
        p = p[:, 0]
        B = p.shape[0]
        mn = p.view(B, -1).min(dim=1)[0]
        mx = p.view(B, -1).max(dim=1)[0]
        return (p - mn[:, None, None]) / (mx[:, None, None] - mn[:, None, None]), None
    if task == "normal":
        n = p.clip(-1, 1)
        rgb = np.clip(((n.cpu().numpy() + 1) * 0.5) * 255, 0, 255).astype(np.uint8)
        return n, np.moveaxis(rgb, 1, -1)
    return None, ((p + 1.0) / 2.0 * 255).clip(0, 255).cpu().numpy().astype(np.uint8)


@pytest.mark.parametrize("task", ["depth", "normal", "seg", "sr"])
@pytest.mark.parametrize("shapes", [((2, 96, 64), (150, 97)), ((1, 48, 64), (77, 101)), ((3, 64, 64), (64, 64)),
                                    ((1, 72, 96), None), ((1, 40, 56), (23, 300))])
def test_v1_postprocess_matches_torch(task, shapes):
    from genpercept_b200 import engine as E
    (B, h, w), size = shapes
    C = 1 if task == "depth" else 3
    g = torch.Generator().manual_seed(B * 1000 + h + w)
    y = torch.rand((B, C, h, w), generator=g).cuda()
    f32, u8 = E.v1_postprocess(y, task, size)
    rf, ru = _v1_torch(y, task, size)
    if rf is not None:
        err = (f32 - rf).abs().max().item()
        print(f"{task} {shapes}: max|err| = {err:.3e}")
        assert f32.shape == rf.shape and err <= 2e-6
    if task == "normal":
        d = np.abs(u8.cpu().numpy().astype(int) - ru.astype(int))
        assert d.max() <= 1 and (d > 0).mean() <= 1e-4
    elif ru is not None:
        assert np.array_equal(u8.cpu().numpy(), ru)


def test_v1_postprocess_constant_depth_is_nan_like_torch():
    from genpercept_b200 import engine as E
    y = torch.full((2, 1, 40, 48), 0.25, device="cuda")
    y[1] = torch.rand((1, 40, 48), generator=torch.Generator().manual_seed(3)).cuda()
    f32, _ = E.v1_postprocess(y, "depth", (61, 33))
    rf, _ = _v1_torch(y, "depth", (61, 33))
    assert torch.equal(torch.isnan(f32), torch.isnan(rf)) and torch.isnan(f32[0]).all()
    assert (f32[1] - rf[1]).abs().max().item() <= 2e-6


def _cases(z):
    return [k[3:] for k in z.files if k.startswith("in_")]


def _call(pipe, z, name):
    kw = json.loads(str(z[f"kw_{name}"]))
    x = z[f"in_{name}"]
    x = torch.from_numpy(x) if x.dtype == np.float32 else Image.fromarray(x)
    return pipe(x, show_progress_bar=False, **kw), kw


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "v1_call.npz"))


@pytest.fixture(scope="module", params=["high", "fp16"])
def v1_pipe(request, synth_state, golden_dir):
    from genpercept_b200.v1 import GenPerceptPipeline
    cast = (lambda sd: sd) if request.param == "high" else (lambda sd: {k: v.half() for k, v in sd.items()})
    p = GenPerceptPipeline(cast(synth_state["unet"]), cast(synth_state["vae"]), None, _embed77(golden_dir))
    assert p.precision == ("high" if request.param == "high" else "default")
    yield request.param, p
    p._engine.close()


def test_v1_call_matches_the_reference(v1_pipe, golden):
    from genpercept_b200 import engine as E
    mode_name, pipe = v1_pipe
    for name in _cases(golden):
        out, kw = _call(pipe, golden, name)
        ref, ref_col = golden[f"pred_{name}"], golden[f"colored_{name}"]
        assert out.pred_np.shape == ref.shape and out.pred_np.dtype == ref.dtype, name
        col = out.pred_colored if isinstance(out.pred_colored, list) else [out.pred_colored]
        col = np.squeeze(np.stack([np.asarray(c) for c in col]))
        assert col.shape == ref_col.shape and col.dtype == ref_col.dtype, name
        err = np.abs(out.pred_np.astype(np.float64) - ref.astype(np.float64))
        task = kw["mode"]
        if task == "depth":
            # the min-max divides the error of p = 2 y - 1 by the stored range; TOL["depth"] bounds the [0, 1] map y,
            # so in p it is twice that.  The high-precision bound is stated for p directly.
            rng = golden[f"range_{name}"]
            bound = (1e-3 if mode_name == "high" else 2 * TOL["depth"]) / float(rng.min())
        elif task == "normal":
            bound = 1e-3 if mode_name == "high" else TOL["normal"]
        else:
            bound = 1 if mode_name == "high" else 4
        print(f"{mode_name} {name}: max|err| = {err.max():.3e} (bound {bound:.3e})")
        assert err.max() <= bound, name
        if f"resized_{name}" in golden.files:        # the engine saw Pillow's bytes
            small = golden[f"resized_{name}"]
            hw = small.shape[:2]
            a = golden[f"in_{name}"]
            assert np.array_equal(E.resize_pil(a, hw[0], hw[1]).cpu().numpy().transpose(1, 2, 0), small)
        if task == "seg":                             # the image is the map, channel-last
            assert np.array_equal(col, np.moveaxis(out.pred_np, 0, -1))
        if task == "normal":
            assert np.abs(col.astype(int) - np.moveaxis(
                np.clip(((out.pred_np + 1) * 0.5) * 255, 0, 255).astype(np.uint8), 0, -1).astype(int)).max() <= 1


def test_v1_batching_and_tensor_input(v1_pipe, golden):
    """batch_size=1 chunks a batch; batch_size=0 runs it in one call: equal up to the GroupNorm summation order."""
    mode_name, pipe = v1_pipe
    x = torch.from_numpy(golden["in_depth_tensor"])
    one = pipe(x, mode="normal", batch_size=1, show_progress_bar=False)
    all_ = pipe(x, mode="normal", batch_size=0, show_progress_bar=False)
    assert one.pred_np.shape == (2, 3, 64, 64) and isinstance(one.pred_colored, list) and len(one.pred_colored) == 2
    assert np.abs(one.pred_np - all_.pred_np).max() < (1e-4 if mode_name == "high" else 1.2e-2)


def test_v1_77_token_context_in_high_precision(synth_state, golden_dir):
    from genpercept_b200.v1 import GenPerceptPipeline
    from oracle.pipeline import OraclePipeline
    te = _embed77(golden_dir)
    p = GenPerceptPipeline(synth_state["unet"], synth_state["vae"], None, te)
    try:
        g = torch.Generator().manual_seed(77)
        rgb = torch.randint(0, 256, (2, 3, 64, 96), generator=g, dtype=torch.uint8)
        for mode in ("depth", "normal"):
            got = p.single_infer(rgb.cuda(), mode=mode)
            assert got.dtype == torch.float32 and got.shape[1] == (1 if mode == "depth" else 3)
            ref = OraclePipeline(synth_state, te).single_infer(rgb.float() / 255.0 * 2.0 - 1.0, mode=mode).numpy()
            err = np.abs((got.cpu().numpy() + 1) / 2 - ref).max()
            print(f"high, 77 tokens, {mode}: max|err| = {err:.3e}")
            assert err < 1e-3
    finally:
        p._engine.close()


def _write_local_dir(tmp_path, synth_state, golden_dir):
    from safetensors.torch import save_file
    for sub in ("unet_depth_v1", "unet_normal_v1", "unet_dis_v1"):
        (tmp_path / sub).mkdir()
    (tmp_path / "vae").mkdir()
    save_file({k: v.contiguous() for k, v in synth_state["unet"].items()},
              str(tmp_path / "unet_depth_v1" / "diffusion_pytorch_model.safetensors"))
    for sub in ("unet_normal_v1", "unet_dis_v1"):
        os.link(tmp_path / "unet_depth_v1" / "diffusion_pytorch_model.safetensors",
                tmp_path / sub / "diffusion_pytorch_model.safetensors")
    save_file({k: v.contiguous() for k, v in synth_state["vae"].items()}, str(tmp_path / "vae" / "diffusion_pytorch_model.safetensors"))
    np.save(tmp_path / "empty_text_embed.npy", _embed77(golden_dir)[0].numpy())


def test_hub_entry_points(tmp_path, synth_state, golden_dir):
    import cv2
    from genpercept_b200 import hub
    _write_local_dir(tmp_path, synth_state, golden_dir)
    g = np.random.default_rng(5)
    bgr = cv2.resize(g.integers(0, 256, (9, 12, 3), dtype=np.uint8), (150, 110), interpolation=cv2.INTER_CUBIC)
    for entry, mode in (("GenPercept_Depth", "depth"), ("GenPercept_Normal", "normal"), ("GenPercept_Segmentation", "seg")):
        pred = torch.hub.load(ROOT, entry, source="local", local_dir=str(tmp_path), device="cuda")
        try:
            assert pred.model.precision == "high"
            got = pred.infer_cv2(bgr)
            img = cv2.cvtColor(hub.resize_image(hub.HWC3(bgr), 768), cv2.COLOR_BGR2RGB)
            out = pred.model(Image.fromarray(img), processing_res=768, match_input_res=True, batch_size=1,
                             color_map="Spectral", show_progress_bar=False, mode=mode)
            assert np.array_equal(got, cv2.cvtColor(np.asarray(out.pred_colored), cv2.COLOR_RGB2BGR)), entry
            assert got.shape == img.shape and got.dtype == np.uint8
        finally:
            pred.model._engine.close()
    os.remove(tmp_path / "vae" / "diffusion_pytorch_model.safetensors")
    with pytest.raises(FileNotFoundError, match="vae"):
        torch.hub.load(ROOT, "GenPercept_Depth", source="local", local_dir=str(tmp_path))
