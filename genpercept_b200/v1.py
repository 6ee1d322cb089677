"""GenPercept's first release on the native engine: the ``GenPerceptPipeline`` of
GenPercept_v1/genpercept/pipeline_genpercept.py, with v1's constructor, ``__call__`` signature, defaults, asserts,
``task_infos`` and result shapes.

What differs from the v2 pipeline (genpercept_b200/pipeline.py), as v1 does:
  * the context is the 77-token padded empty prompt (``empty_text_embed`` [1,77,1024], required: v1 never encodes
    text); it runs through the engine's general cross-attention path;
  * a PIL image reaches the processing size through Pillow's ``Image.resize`` (BICUBIC), reproduced byte for byte on
    the GPU (gp_resize_pil); a [B,3,H,W] tensor in [-1,1] is not resized;
  * the map goes back to the input size through plain ``F.interpolate`` (bilinear for depth / normal, nearest for
    seg / sr), then depth is min-max normalised per image without a clamp, normals are clipped and coloured by
    ``norm_to_rgb``, and seg / sr become uint8 — all on the GPU (gp_v1_postprocess);
  * ``pred_np`` is channel-first for the 3-channel modes.

The precision follows the modules, as v1 has no ``torch_dtype``: fp32 parameters (what v1's tool and torch.hub
entry points build) select the engine's high-precision mode, fp16 16-bit storage, bf16 bf16 storage.

Not offered: v1's ELU-terminated DPT head (``customized_head``, dpt_head_elu.py), for which no weights are released.
"""
from typing import Union

import numpy as np
import torch
from PIL import Image

from . import engine as E
from . import weights as W
from .engine import Engine
from .image_util import _lut
from .pipeline import GenPerceptOutput, _as_state_dict

__all__ = ["GenPerceptPipeline", "GenPerceptOutput"]


def _weights_dtype(sd):
    """The dtype of the first floating-point tensor of a state dict (v1's modules carry one dtype throughout)."""
    for v in sd.values():
        if torch.is_tensor(v) and v.is_floating_point():
            return v.dtype
    return torch.float32


class GenPerceptPipeline:
    vae_scale_factor = 0.18215
    task_infos = {
        "depth": dict(task_channel_num=1, interpolate="bilinear"),
        "seg": dict(task_channel_num=3, interpolate="nearest"),
        "sr": dict(task_channel_num=3, interpolate="nearest"),
        "normal": dict(task_channel_num=3, interpolate="bilinear"),
    }

    def __init__(self, unet, vae, customized_head=None, empty_text_embed=None, *, device=0, cuda_graph="auto"):
        """unet / vae: modules, state dicts or checkpoint paths (as the v2 pipeline takes them).  empty_text_embed:
        [1,77,1024] (any dtype or device).  The weights are folded and uploaded here, with the embedding."""
        if customized_head is not None:
            raise NotImplementedError(
                "GenPercept v1's customized_head (DPTNeckHeadForUnetAfterUpsample, genpercept/models/dpt_head_elu.py) is "
                "not offered by this engine: no v1 DPT weights are released; use the VAE decoder readout")
        if empty_text_embed is None:
            raise ValueError("empty_text_embed ([1,77,1024], GenPercept_v1/empty_text_embed.npy) is required: "
                             "v1 never encodes text")
        unet_sd = dict(_as_state_dict(unet))
        vae_sd = W.remap_legacy_vae_keys(_as_state_dict(vae))
        if not any(k.startswith("conv_out.") for k in unet_sd):
            raise NotImplementedError("a UNet without conv_out feeds a customized head, which this engine does not offer")
        if not any(k.startswith("decoder.") for k in vae_sd):
            raise NotImplementedError("a VAE without a decoder feeds a customized head, which this engine does not offer")
        self.dtype = _weights_dtype(unet_sd)
        self.precision = "high" if self.dtype == torch.float32 else "default"
        storage = torch.bfloat16 if self.dtype == torch.bfloat16 else torch.float16
        self._engine = Engine(dtype=storage, readout="vae", timestep=1, device=device, cuda_graph=cuda_graph,
                              precision=self.precision)
        self._engine.load_state("unet", unet_sd)
        self._engine.load_state("vae", vae_sd)
        e = torch.as_tensor(empty_text_embed).detach().float().cpu().reshape(1, -1, 1024)
        self._engine.set_text_embed(e)
        self._engine.finalize()
        self.empty_text_embed = e.to(self.dtype)
        self.customized_head = None

    # ------------------------------------------------------------------ diffusers-pipeline surface
    @property
    def device(self):
        return self._engine.device

    def to(self, *a, **k):
        return self

    def set_progress_bar_config(self, **k):
        return None

    def enable_xformers_memory_efficient_attention(self, *a, **k):
        """In the high-precision mode every attention runs fused and stores no T x T score matrix (the 16-bit modes
        already bound it).  Valid before or after the first inference."""
        self._engine.set_memory_efficient_attention(True)

    def disable_xformers_memory_efficient_attention(self):
        self._engine.set_memory_efficient_attention(False)

    # ------------------------------------------------------------------ v1 helpers
    @torch.no_grad()
    def single_infer(self, rgb_in: torch.Tensor, mode: str = "depth") -> torch.Tensor:
        """rgb_in: [B,3,H,W] uint8 (0..255) or float in [-1,1].  Returns v1's clip(pred, -1, 1), [B,1|3,H,W] on the GPU
        in ``self.dtype`` (the channel mean for depth)."""
        ch = self.task_infos[mode]["task_channel_num"]
        return (self._engine.infer(rgb_in, out_channels=ch) * 2.0 - 1.0).to(self.dtype)

    @torch.no_grad()
    def encode_rgb(self, rgb_in: torch.Tensor) -> torch.Tensor:
        """mean(quant_conv(encoder(rgb_in))) * 0.18215 on the GPU in ``self.dtype``."""
        return self._engine.encode(rgb_in).to(self.dtype)

    @torch.no_grad()
    def decode_pred(self, pred_latent: torch.Tensor) -> torch.Tensor:
        """decoder(post_quant_conv(pred_latent / 0.18215)), [B,3,8h,8w] on the GPU.  The engine's last kernel fuses the
        clip to [-1, 1] that single_infer applies next, so values beyond it are not recoverable."""
        return (self._engine.decode(pred_latent.float(), out_channels=3) * 2.0 - 1.0).to(self.dtype)

    def _pil_input(self, img: Image.Image, processing_res: int, resize_hard: bool) -> torch.Tensor:
        """v1's resize_max_res / resize_res + convert("RGB") -> uint8 [1,3,h,w] on the GPU.  An RGB image is resized on
        the GPU (gp_resize_pil, Pillow's bytes); other modes take Pillow's own resize in their mode first, as v1 does
        (Pillow resizes RGBA premultiplied and P / 1 with NEAREST), then only the upload and layout change."""
        w, h = img.size
        if processing_res > 0:
            if resize_hard:
                size = (processing_res, processing_res)
            else:
                f = min(processing_res / w, processing_res / h)
                size = (int(w * f), int(h * f))
        else:
            size = (w, h)
        if img.mode != "RGB":
            if size != (w, h):
                img = img.resize(size)
            img = img.convert("RGB")
        return E.resize_pil(np.asarray(img), size[1], size[0], device=self.device)[None]

    # ------------------------------------------------------------------ the v1 call
    @torch.no_grad()
    def __call__(self, input_image: Union[Image.Image, torch.Tensor], mode: str = "depth", resize_hard=False,
                 processing_res: int = 768, match_input_res: bool = True, batch_size: int = 0,
                 color_map: str = "Spectral", show_progress_bar: bool = True) -> GenPerceptOutput:
        """GenPercept v1's ``__call__``.  ``batch_size > 0`` runs the batch in chunks of that size; ``batch_size=0`` runs
        it in one engine call (v1 asks ``find_batch_size(ensemble_size=1, ...)``, which always answers 1).  A batch's
        maps differ from one-image maps only by the GroupNorm summation order.  ``show_progress_bar`` is accepted and
        ignored.  Returns ``GenPerceptOutput(pred_np, pred_colored)`` with v1's shapes: ``np.squeeze`` of depth [B,H,W]
        (fp32 in [0,1]), normal [B,3,H,W] (fp32 in [-1,1]) or seg / sr [B,3,H,W] (uint8); ``pred_colored`` one PIL image,
        or a list of them when B > 1."""
        task_channel_num = self.task_infos[mode]["task_channel_num"]
        if not match_input_res:
            assert processing_res is not None, "Value error: `resize_output_back` is only valid with "
        assert processing_res >= 0

        if type(input_image) == torch.Tensor:                     # [B, 3, H, W] in [-1, 1], not resized
            rgb = input_image.to(self.device)
            input_size = tuple(input_image.shape[2:])
            bs_imgs = rgb.shape[0]
            assert rgb.min() >= -1.0 and rgb.max() <= 1.0
            rgb = rgb.to(self.dtype)
        else:
            input_size = (input_image.size[1], input_image.size[0])
            rgb = self._pil_input(input_image, processing_res, resize_hard)
            bs_imgs = 1

        bs = batch_size if batch_size > 0 else bs_imgs
        preds = [self._engine.infer(rgb[lo:lo + bs], out_channels=task_channel_num) for lo in range(0, bs_imgs, bs)]
        pred = preds[0] if len(preds) == 1 else torch.cat(preds, dim=0)
        return self._postprocess(pred, mode, input_size if match_input_res else None, color_map)

    def _postprocess(self, pred, mode, size, color_map) -> GenPerceptOutput:
        f32, u8 = E.v1_postprocess(pred, mode, size)
        if mode == "depth":
            lut = (_lut(color_map) * 255).astype(np.uint8)          # (colorize_depth_maps(...) * 255).astype(uint8)
            colored = [Image.fromarray(c) for c in E.colorize(f32, lut, 0.0, 1.0).numpy()]
            preds = f32.cpu().numpy()
        elif mode == "normal":
            colored = [Image.fromarray(c) for c in u8.cpu().numpy()]
            preds = f32.cpu().numpy()
        else:                                                        # seg / sr: uint8 CHW, chw2hwc for the image
            preds = u8.cpu().numpy()
            colored = [Image.fromarray(np.ascontiguousarray(np.moveaxis(p, 0, -1))) for p in preds]
        return GenPerceptOutput(pred_np=np.squeeze(preds), pred_colored=colored[0] if len(colored) == 1 else colored)
