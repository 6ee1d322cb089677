"""CPU tests of genpercept_b200.multitask: the construction checks of MultiTaskPipeline and the post-processing it shares
with GenPerceptPipeline.__call__ (host tensors; the GPU kernels it calls are replaced by their host definitions)."""
import numpy as np
import pytest
import torch
from PIL import Image

from genpercept_b200 import engine as E
from genpercept_b200 import weights as W
from genpercept_b200.image_util import _lut
from genpercept_b200.multitask import MultiTaskPipeline
from genpercept_b200.pipeline import GenPerceptOutput, GenPerceptPipeline, postprocess


def _vae(seed=0):
    g = torch.Generator().manual_seed(seed)
    return {"encoder.conv_in.weight": torch.randn((8, 3, 3, 3), generator=g),
            "encoder.mid_block.attentions.0.to_q.weight": torch.randn((8, 8), generator=g),
            "quant_conv.weight": torch.randn((8, 8, 1, 1), generator=g),
            "decoder.conv_in.weight": torch.randn((8, 4, 3, 3), generator=g),
            "post_quant_conv.weight": torch.randn((4, 4, 1, 1), generator=g)}


def _pipe(vae=None, dtype=torch.float16, precision="default", device=torch.device("cuda", 0), one_step=True):
    """A GenPerceptPipeline as the checks see it, without an engine (construction needs a GPU)."""
    p = object.__new__(GenPerceptPipeline)
    p.genpercept_pipeline = one_step
    p.dtype, p.precision, p.device = dtype, precision, device
    p._encoder_state = W.encoder_state(vae if vae is not None else _vae())
    return p


def _modes(pipes):
    return {k: "depth" for k in pipes}


def test_accepts_equal_encoders_with_different_decoders_and_storage():
    base = {k: v.half().float() for k, v in _vae().items()}                            # values exact in fp16
    new_decoder = {**base, "decoder.conv_in.weight": base["decoder.conv_in.weight"] + 1.0}   # a vae_decoder/ override
    as_fp16 = {k: v.half() for k, v in base.items()}                                   # the same values, stored as fp16
    pipes = {"depth": _pipe(base), "normal": _pipe(new_decoder), "seg": _pipe(as_fp16)}
    m = MultiTaskPipeline(pipes, _modes(pipes))
    assert list(m.pipelines) == ["depth", "normal", "seg"]


@pytest.mark.parametrize("key", ["encoder.conv_in.weight", "encoder.mid_block.attentions.0.to_q.weight", "quant_conv.weight"])
def test_mismatched_encoder_tensor_names_task_and_key(key):
    bad = _vae()
    bad[key] = bad[key].clone()
    bad[key].view(-1)[3] += 1e-3
    pipes = {"depth": _pipe(), "normal": _pipe(bad)}
    with pytest.raises(ValueError, match=rf"'normal'.*vae\.{key}"):
        MultiTaskPipeline(pipes, _modes(pipes))


def test_missing_encoder_tensor_names_task_and_key():
    bad = _vae()
    del bad["quant_conv.weight"]
    pipes = {"depth": _pipe(), "seg": _pipe(bad)}
    with pytest.raises(ValueError, match=r"'seg'.*vae\.quant_conv\.weight"):
        MultiTaskPipeline(pipes, _modes(pipes))


def test_mismatched_dtype_names_task():
    pipes = {"depth": _pipe(), "normal": _pipe(dtype=torch.bfloat16)}
    with pytest.raises(ValueError, match=r"'normal'.*dtype"):
        MultiTaskPipeline(pipes, _modes(pipes))


def test_mismatched_precision_names_task():
    pipes = {"depth": _pipe(dtype=torch.float32, precision="high"), "normal": _pipe(dtype=torch.float32, precision="default")}
    with pytest.raises(ValueError, match=r"'normal'.*precision"):
        MultiTaskPipeline(pipes, _modes(pipes))


def test_multi_step_pipeline_names_task():
    pipes = {"depth": _pipe(), "marigold": _pipe(one_step=False)}
    with pytest.raises(ValueError, match=r"'marigold'.*multi-step"):
        MultiTaskPipeline(pipes, _modes(pipes))


def test_mismatched_device_names_task():
    pipes = {"depth": _pipe(), "disparity": _pipe(device=torch.device("cuda", 1))}
    with pytest.raises(ValueError, match=r"'disparity'.*device"):
        MultiTaskPipeline(pipes, _modes(pipes))


def test_modes_must_name_the_tasks():
    pipes = {"depth": _pipe(), "normal": _pipe()}
    with pytest.raises(ValueError, match="modes"):
        MultiTaskPipeline(pipes, {"depth": "depth"})
    with pytest.raises(ValueError):
        MultiTaskPipeline({}, {})


# ---------------------------------------------------------------- post-processing shared with __call__
def _host_colorize(pred, lut_u8, vmin=0.0, vmax=1.0, to_host=True):       # gp_colorize's definition (the header)
    idx = np.clip(np.floor((pred.numpy() - vmin) / (vmax - vmin) * 256), 0, 255).astype(np.int64)
    return torch.from_numpy(np.ascontiguousarray(lut_u8[idx]))


def _host_quantize(pred, bits=16, to_host=True):                           # (pred * 255).astype(uint8)
    return (pred.numpy() * (255 if bits == 8 else 65535)).astype(np.uint8 if bits == 8 else np.uint16)


@pytest.fixture
def host_kernels(monkeypatch):
    monkeypatch.setattr(E, "colorize", _host_colorize)
    monkeypatch.setattr(E, "quantize", _host_quantize)


def _maps(B, C, H, W, seed=3):
    g = torch.Generator().manual_seed(seed)
    return torch.rand((B, C, H, W), generator=g) * 1.2 - 0.1       # beyond [0, 1]: the clip matters


def _expected(pred, color_map):
    """__call__'s tail as the reference writes it (genpercept_pipeline.py:301-323), for maps already at the input size."""
    p = pred.clamp(0, 1).numpy()
    if color_map is not None:
        lut = (_lut(color_map) * 255).astype(np.uint8)
        col = lut[np.clip(np.floor(p[:, 0] * 256), 0, 255).astype(np.int64)]
    else:
        col = (p * 255).astype(np.uint8)
        col = col[:, 0] if p.shape[1] == 1 else np.transpose(col, (0, 2, 3, 1))
    if p.shape[0] > 1:
        arr = p[:, 0] if p.shape[1] == 1 else np.transpose(p, (0, 2, 3, 1))
        return arr, [np.asarray(Image.fromarray(c)) for c in col]
    arr = p[0, 0] if p.shape[1] == 1 else np.transpose(p[0], (1, 2, 0))
    return arr, np.asarray(Image.fromarray(col[0]))


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("C,mode,color_map", [(1, "depth", "Spectral"), (1, "depth", None), (3, "normal", None)])
def test_postprocess_matches_call_tail(host_kernels, B, C, mode, color_map):
    pred = _maps(B, C, 24, 40)
    out = postprocess(pred, (B, 3, 24, 40), True, "bilinear", color_map, mode)
    assert isinstance(out, GenPerceptOutput)
    arr, img = _expected(pred, color_map)
    assert np.array_equal(out.pred_np, arr)
    if B == 1:
        assert isinstance(out.pred_colored, Image.Image)
        assert np.array_equal(np.asarray(out.pred_colored), img)
    else:
        assert len(out.pred_colored) == B
        for got, want in zip(out.pred_colored, img):
            assert np.array_equal(np.asarray(got), want)


@pytest.mark.parametrize("C", [1, 3])
def test_postprocess_resizes_back_on_the_host_path(host_kernels, C):
    """nearest resampling keeps torchvision's host resize back to the input size (genpercept_pipeline.py:301-307;
    "nearest" is NEAREST_EXACT, image_util.get_tv_resample_method)."""
    from torchvision.transforms import InterpolationMode
    from torchvision.transforms.functional import resize
    pred = _maps(1, C, 16, 24)
    out = postprocess(pred, (1, 3, 33, 47), True, "nearest", None, "normal" if C == 3 else "depth")
    arr, img = _expected(resize(pred, [33, 47], interpolation=InterpolationMode.NEAREST_EXACT, antialias=True), None)
    assert np.array_equal(out.pred_np, arr) and np.array_equal(np.asarray(out.pred_colored), img)
    kept = postprocess(pred, (1, 3, 33, 47), False, "nearest", None, "depth" if C == 1 else "normal")
    assert kept.pred_np.shape[:2] == (16, 24)


def test_postprocess_colorizes_only_depth_and_disparity(host_kernels):
    with pytest.raises(AssertionError):
        postprocess(_maps(1, 3, 8, 8), (1, 3, 8, 8), True, "bilinear", "Spectral", "normal")
