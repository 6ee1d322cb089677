"""GenPercept v1's torch.hub predictors (GenPercept_v1/hubconf.py) on the native engine.

    predictor = torch.hub.load("/path/to/this/checkout", "GenPercept_Depth", source="local", local_dir="/path/to/weights")
    bgr_depth = predictor.infer_cv2(cv2.imread("photo.jpg"))

``local_dir`` holds the released v1 layout: ``unet_{depth,normal,dis}_v1/diffusion_pytorch_model.safetensors`` and
``vae/diffusion_pytorch_model.safetensors``, plus ``empty_text_embed.npy`` (GenPercept_v1/empty_text_embed.npy) unless
the embedding is passed as ``empty_text_embed=``.  Files are read locally only: this module never downloads, and a
missing file raises FileNotFoundError naming it.  As in v1, the weights are taken as fp32 (the modules v1 builds are
fp32), which selects the engine's high-precision mode.

``infer_cv2``'s host steps stay as v1 has them: HWC3, OpenCV's Lanczos-4 / area resize to multiples of 64 and the
colour conversions (cv2, imported when used).
"""
import os
from typing import Optional

import numpy as np
import torch
from PIL import Image

from .v1 import GenPerceptPipeline

_VAE = os.path.join("vae", "diffusion_pytorch_model.safetensors")


def HWC3(x):
    assert x.dtype == np.uint8
    if x.ndim == 2:
        x = x[:, :, None]
    assert x.ndim == 3
    H, W, C = x.shape
    assert C == 1 or C == 3 or C == 4
    if C == 3:
        return x
    if C == 1:
        return np.concatenate([x, x, x], axis=2)
    color = x[:, :, 0:3].astype(np.float32)
    alpha = x[:, :, 3:4].astype(np.float32) / 255.0
    y = color * alpha + 255.0 * (1.0 - alpha)
    return y.clip(0, 255).astype(np.uint8)


def resize_image(input_image, resolution):
    """The short side to `resolution`, both sides rounded to multiples of 64 (Lanczos-4 up, area down)."""
    import cv2
    H, W, C = input_image.shape
    H = float(H)
    W = float(W)
    k = float(resolution) / min(H, W)
    H *= k
    W *= k
    H = int(np.round(H / 64.0)) * 64
    W = int(np.round(W / 64.0)) * 64
    return cv2.resize(input_image, (W, H), interpolation=cv2.INTER_LANCZOS4 if k > 1 else cv2.INTER_AREA)


class BasePredictor:
    mode = None

    def __init__(self, model, device="cuda"):
        self.model = model
        self.device = device

    def infer_cv2(self, image, image_resolution=768):
        """BGR uint8 image -> BGR uint8 prediction.  As in v1, `image_resolution` sets only the OpenCV resize: the
        pipeline call inside infer_pil keeps its processing resolution of 768."""
        import cv2
        raw_image = HWC3(image)
        img = resize_image(raw_image, image_resolution)
        img = cv2.cvtColor(img, cv2.COLOR_BGR2RGB)
        return self.infer_pil(Image.fromarray(img))

    def infer_pil(self, image, image_resolution=768):
        import cv2
        with torch.no_grad():
            pipe_out = self.model(image, processing_res=image_resolution, match_input_res=True, batch_size=1,
                                  color_map="Spectral", show_progress_bar=True, mode=self.mode)
            pred = np.asarray(pipe_out.pred_colored)
            return cv2.cvtColor(pred, cv2.COLOR_RGB2BGR)


class NormalPredictor(BasePredictor):
    mode = "normal"


class DepthPredictor(BasePredictor):
    mode = "depth"


class SegmentationPredictor(BasePredictor):
    mode = "seg"


def _device_index(device):
    d = torch.device(device)
    if d.type != "cuda":
        raise ValueError(f"the engine runs on a CUDA device, not {device!r}")
    return d.index if d.index is not None else torch.cuda.current_device()


def load_model(unet_subfolder, device="cuda", local_dir=None, empty_text_embed=None):
    """The v1 pipeline from `local_dir`'s files (see the module docstring)."""
    if local_dir is None:
        raise FileNotFoundError("local_dir= is required: the weights are read from local files, never downloaded")
    unet_path = os.path.join(local_dir, unet_subfolder, "diffusion_pytorch_model.safetensors")
    vae_path = os.path.join(local_dir, _VAE)
    for p in (unet_path, vae_path):
        if not os.path.isfile(p):
            raise FileNotFoundError(p)
    if empty_text_embed is None:
        p = os.path.join(local_dir, "empty_text_embed.npy")
        if not os.path.isfile(p):
            raise FileNotFoundError(p)
        empty_text_embed = torch.from_numpy(np.load(p)).float()[None]
    from safetensors.torch import load_file
    fp32 = lambda sd: {k: v.float() for k, v in sd.items()}     # v1 loads them into fp32 modules
    return GenPerceptPipeline(fp32(load_file(unet_path)), fp32(load_file(vae_path)), None, empty_text_embed,
                              device=_device_index(device))


def GenPercept_Normal(local_dir: Optional[str] = None, device="cuda", repo_id="guangkaixu/GenPercept", empty_text_embed=None):
    return NormalPredictor(load_model("unet_normal_v1", device, local_dir, empty_text_embed), device)


def GenPercept_Depth(local_dir: Optional[str] = None, device="cuda", repo_id="guangkaixu/GenPercept", empty_text_embed=None):
    return DepthPredictor(load_model("unet_depth_v1", device, local_dir, empty_text_embed), device)


def GenPercept_Segmentation(local_dir: Optional[str] = None, device="cuda", repo_id="guangkaixu/GenPercept",
                            empty_text_embed=None):
    return SegmentationPredictor(load_model("unet_dis_v1", device, local_dir, empty_text_embed), device)
