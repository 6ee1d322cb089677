"""Drop-in for ``genpercept.GenPerceptPipeline`` / ``GenPerceptOutput``
(/root/reference/genpercept/genpercept_pipeline.py:50-62, :64-526) on top of the native engine.

Same constructor kwargs, ``__call__`` kwargs/defaults (:146-162), helper methods
(``single_infer`` :375, ``encode_rgb`` :488, ``decode_pred`` :507, ``encode_text`` :360) and error
behaviour (asserts / TypeError / ValueError at the same points).  Below this file nothing is
PyTorch: ``single_infer`` is one ``gp_infer`` call into libgenpercept_b200.so.

Extensions (SURVEY.md F10): ``input_image`` may be a uint8 tensor [B,3,H,W] with B > 1 (the
reference's ``expand(ensemble_size)`` admits only B == 1); outputs then carry a leading batch dim.
Multi-GPU: ``genpercept_b200.parallel.sharded_infer`` shards the batch over ranks.
"""
import logging
import os
from dataclasses import dataclass
from typing import Dict, Optional, Union

import numpy as np
import torch
from PIL import Image
from torchvision.transforms.functional import pil_to_tensor, resize

from . import engine as E
from . import weights as W
from .engine import Engine
from .image_util import _lut, decode_unloaded_jpeg, get_tv_resample_method, resize_max_res

ONE_CHANNEL_MODES = ("depth", "matting", "dis", "disparity")     # genpercept_pipeline.py:523
_NO_SCHEDULER = "the multi-step archs need a scheduler (hf_configs/scheduler_beta_*/scheduler_config.json)"


def _checkpoint_scheduler(root, kw):
    """diffusers' from_pretrained loads ``<root>/scheduler/`` when no scheduler is passed: the multi-step archs
    (genpercept_pipeline=False) take the folder's scheduler_config.json, as run.py's default invocation expects
    (run.py:361-368).  A missing file raises the ValueError of a missing scheduler, naming the path."""
    if kw.get("genpercept_pipeline", True) or kw.get("scheduler") is not None:
        return
    path = os.path.join(str(root), "scheduler", "scheduler_config.json")
    if not os.path.isfile(path):
        raise ValueError(f"{_NO_SCHEDULER}: {path} does not exist")
    kw["scheduler"] = path


def _checkpoint_text_tower(root, kw):
    """The SD-2.1 folder's text tower when no text_embed / text_encoder is passed: ``<root>/text_encoder/`` as a path,
    which the pipeline reads as a state dict (model.safetensors or .bin, honouring `variant`) for the engine's own tower,
    and transformers' CLIPTokenizer from ``<root>/tokenizer`` unless a tokenizer is passed.  No CLIPTextModel is built."""
    if kw.get("text_embed") is not None or kw.get("text_encoder") is not None:
        return
    folder = os.path.join(root, "text_encoder")
    if not os.path.isdir(folder):
        return
    kw["text_encoder"] = folder
    if kw.get("tokenizer") is None:
        from transformers import CLIPTokenizer
        kw["tokenizer"] = CLIPTokenizer.from_pretrained(os.path.join(root, "tokenizer"))


@dataclass
class GenPerceptOutput:
    """pred_np: result in [0,1]; pred_colored: PIL image or None (genpercept_pipeline.py:50-62)."""
    pred_np: np.ndarray
    pred_colored: Union[None, Image.Image, list]

    def __getitem__(self, k):
        return (self.pred_np, self.pred_colored)[k] if isinstance(k, int) else getattr(self, k)


def _as_state_dict(m, variant=None):
    """Accept a module (anything with .state_dict()), a dict, or a path to a checkpoint file/dir."""
    if m is None:
        return None
    if isinstance(m, dict):
        return m
    if isinstance(m, (str, os.PathLike)):
        return load_checkpoint(m, variant)
    if hasattr(m, "state_dict"):
        return m.state_dict()
    raise TypeError(f"cannot take weights from {type(m)}")


def load_checkpoint(path, variant=None):
    """diffusers folder layouts the reference reads (run.py:283-343): a dir holding
    diffusion_pytorch_model.{safetensors,bin} / model.safetensors, or such a file directly.  `variant` ("fp16")
    prefers ``diffusion_pytorch_model.<variant>.safetensors`` like ``from_pretrained(variant=...)`` (run.py:374)."""
    path = str(path)
    if os.path.isdir(path):
        names = []
        for stem in ("diffusion_pytorch_model", "model"):
            for ext in ("safetensors", "bin"):
                if variant:
                    names.append(f"{stem}.{variant}.{ext}")
                names.append(f"{stem}.{ext}")
        names.sort(key=lambda n: (n.endswith(".bin"), variant is None or f".{variant}." not in n))
        for n in names:
            if os.path.exists(os.path.join(path, n)):
                path = os.path.join(path, n)
                break
        else:
            raise FileNotFoundError(f"no checkpoint file under {path}")
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        return load_file(path)
    return torch.load(path, map_location="cpu", weights_only=True)      # tensors only: no pickled code


class GenPerceptPipeline:
    latent_scale_factor = 0.18215                                 # genpercept_pipeline.py:96

    def __init__(self, unet, vae, scheduler=None, text_encoder=None, tokenizer=None,
                 default_denoising_steps: Optional[int] = 10, default_processing_resolution: Optional[int] = 768,
                 rgb_blending=False, customized_head=None, genpercept_pipeline=True, *, text_embed=None,
                 torch_dtype=torch.float16, device=0, cuda_graph="auto", fix_timesteps=None, precision=None,
                 variant=None):
        self.genpercept_pipeline = genpercept_pipeline
        if genpercept_pipeline:                       # genpercept_pipeline.py:122-125
            default_denoising_steps = 1
            rgb_blending = True
            cfg = getattr(scheduler, "config", scheduler)
            bs = cfg.get("beta_start") if isinstance(cfg, dict) else getattr(cfg, "beta_start", None)
            be = cfg.get("beta_end") if isinstance(cfg, dict) else getattr(cfg, "beta_end", None)
            if bs is not None:
                assert bs == 1 and be == 1, \
                    "the one-step collapse x0 = -v needs the beta=1 scheduler (hf_configs/scheduler_beta_1.0_1.0)"
        else:
            # multi-step archs (run.py --archs marigold / rgb_blending, SURVEY.md §8 f4): real DDIM steps around the UNet.
            # `scheduler`: a scheduler_config.json path / folder / dict, a DDIMSchedule, or any object whose .config
            # carries the reference's scheduler fields (the reference passes its DDIMSchedulerCustomized).
            # The scheduler must be a DDIM one (scheduler.check_scheduler_class): the config's _class_name, else the
            # object's class name.
            from .scheduler import DDIMSchedule, check_scheduler_class
            if customized_head is not None:
                raise ValueError("the DPT readout is one-step (genpercept_pipeline.py:474-483)")
            if scheduler is None:
                raise ValueError(_NO_SCHEDULER)
            if not isinstance(scheduler, DDIMSchedule):
                cfg = getattr(scheduler, "config", scheduler)
                if not isinstance(cfg, (str, os.PathLike)):
                    cfg = dict(cfg)
                    if not isinstance(scheduler, dict) and cfg.get("_class_name") is None:
                        check_scheduler_class(type(scheduler).__name__)
                scheduler = DDIMSchedule.from_config(cfg)
        self.scheduler = scheduler
        self.text_encoder = text_encoder
        self.tokenizer = tokenizer
        self.default_denoising_steps = default_denoising_steps
        self.default_processing_resolution = default_processing_resolution
        self.rgb_blending = rgb_blending
        self.customized_head = customized_head
        self.text_embed = None
        # run.py:273-281: fp32 unless --half_precision.  torch_dtype=float32 (the reference default) selects the
        # engine's high-precision mode — every operand an fp16 (hi, lo) pair, three tensor-core passes, fp32
        # accumulate: fp32-class results at ~3x the tensor work; float16 / bfloat16 select 16-bit storage.
        self.dtype = torch.float32 if torch_dtype is None else torch_dtype
        if precision is None:
            precision = "high" if self.dtype == torch.float32 else "default"
        self.precision = precision
        storage = torch.bfloat16 if self.dtype == torch.bfloat16 else torch.float16
        self._timestep = int(fix_timesteps) if fix_timesteps else 1
        self._engine = Engine(dtype=storage, readout="dpt" if customized_head is not None else "vae",
                              timestep=self._timestep, device=device, cuda_graph=cuda_graph, precision=precision,
                              arch="genpercept" if genpercept_pipeline else "multistep")
        self.device = self._engine.device
        unet_sd = dict(_as_state_dict(unet, variant))
        vae_sd = W.remap_legacy_vae_keys(_as_state_dict(vae, variant))
        self._encoder_state = W.encoder_state(vae_sd)      # references, compared by multitask.MultiTaskPipeline
        if customized_head is not None:          # run.py:322-331 drops these for the DPT readout
            unet_sd = {k: v for k, v in unet_sd.items() if not k.startswith(("conv_out", "conv_norm_out"))}
            self._engine.load_state("dpt", _as_state_dict(customized_head))
        self._engine.load_state("unet", unet_sd)
        self._engine.load_state("vae", vae_sd)
        # the text tower's weights only (a module's forward never runs): encode_text runs SD-2.1's CLIP tower on the
        # engine, in its mode
        if text_encoder is not None and text_embed is None:
            self._engine.load_state("text", _as_state_dict(text_encoder, variant))
        self._finalized = False
        if text_embed is not None:
            self._set_text_embed(text_embed)

    # ------------------------------------------------------------------ diffusers-pipeline surface
    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, variant=None, torch_dtype=None, **kw):
        """Mirrors ``GenPerceptPipeline.from_pretrained(sd21_dir, variant=…, torch_dtype=…,
        genpercept_pipeline=True, unet=…, scheduler=…, [customized_head|vae]=…)`` (run.py:374-376):
        vae / text_encoder / tokenizer come from the SD-2.1 folder unless passed, and so does the scheduler
        (``scheduler/scheduler_config.json``) of the multi-step archs (genpercept_pipeline=False)."""
        root = str(pretrained_model_name_or_path)
        _checkpoint_scheduler(root, kw)
        if kw.get("vae") is None:
            kw["vae"] = os.path.join(root, "vae")
        if kw.get("unet") is None:
            kw["unet"] = os.path.join(root, "unet")
        _checkpoint_text_tower(root, kw)
        return cls(torch_dtype=torch_dtype, variant=variant, **kw)

    @classmethod
    def from_run_args(cls, checkpoint, unet=None, lora_rank=0, **kw):
        """The model section of the reference CLI (run.py:273-376, infer.py:299-405) in one call:
        ``--checkpoint`` (SD-2.1 folder), ``--unet`` (fine-tuned UNet folder in either layout, with an optional
        ``dpt_head_identity/`` or ``vae_decoder/`` + ``vae_post_quant_conv/`` next to it) and ``--lora_rank``.
        See genpercept_b200/loader.py for the layouts."""
        from . import loader
        _checkpoint_scheduler(checkpoint, kw)
        parts = loader.assemble(checkpoint, unet=unet, lora_rank=lora_rank, variant=kw.get("variant"))
        _checkpoint_text_tower(str(checkpoint), kw)
        return cls(unet=parts["unet"], vae=parts["vae"], customized_head=parts["customized_head"], **kw)

    def to(self, *a, **k):
        return self

    def enable_xformers_memory_efficient_attention(self, *a, **k):   # run.py:382-385, infer.py:400-403
        """Memory-efficient attention: in the high-precision mode (torch_dtype=float32) every attention runs fused and
        stores no T x T score matrix, so native-resolution photos fit.  The 16-bit modes already bound it.  Valid before
        or after the first inference."""
        self._engine.set_memory_efficient_attention(True)

    def disable_xformers_memory_efficient_attention(self):
        """Back to the default: the high-precision mode stores the score matrices (the plans ``bench.py`` measures)."""
        self._engine.set_memory_efficient_attention(False)

    def enable_shared_arena(self):
        """Take this pipeline's activation memory from the device's one shared pool, so several pipelines (or several
        native-resolution shapes) in one process need the largest arena among them, not the sum, as the reference's
        pipelines share PyTorch's caching allocator.  Outputs are unchanged.  Valid before or after the first inference."""
        self._engine.set_shared_arena(True)

    def disable_shared_arena(self):
        """Back to the default: every plan owns its activation arena."""
        self._engine.set_shared_arena(False)

    def set_progress_bar_config(self, **k):
        return None

    # ------------------------------------------------------------------ text embedding
    def _set_text_embed(self, e):
        e = torch.as_tensor(e).detach().float().cpu().reshape(1, -1, 1024)
        if self._finalized:
            raise RuntimeError("the text embedding is folded into the weights at first use; build a new pipeline")
        self.text_embed = e.to(self.dtype)
        self._engine.set_text_embed(e)

    def encode_text(self, prompt):
        """genpercept_pipeline.py:360-372: tokenizer(prompt, padding='do_not_pad') on the host, then SD-2.1's CLIP text
        tower on the engine (gp_encode_text, in the engine's mode) -> [1, n, 1024]; the empty prompt gives n = 2."""
        if self.text_encoder is None or self.tokenizer is None:
            raise RuntimeError("no text_encoder/tokenizer given: pass text_embed= (e.g. the fixture "
                               "tests/golden/empty_text_embed_2x1024.npy)")
        ti = self.tokenizer(prompt, padding="do_not_pad", max_length=self.tokenizer.model_max_length,
                            truncation=True, return_tensors="pt")
        self._set_text_embed(self._engine.encode_text(ti.input_ids))

    def _ensure_ready(self, prompt=""):
        if self.text_embed is None:
            self.encode_text(prompt)
        if not self._finalized:
            self._engine.finalize()
            self._finalized = True

    # ------------------------------------------------------------------ the hot path
    @torch.no_grad()
    def single_infer(self, rgb_in, num_inference_steps=1, generator=None, show_pbar=False, fix_timesteps=None,
                     prompt="", mode=None):
        """rgb_in: [B,3,H,W] uint8 (0..255) or float in [-1,1].  Returns fp32 [B,1|3,H,W] in [0,1] (cuda)."""
        if not self.genpercept_pipeline:
            return self._single_infer_steps(rgb_in, num_inference_steps, generator, fix_timesteps, prompt, mode)
        assert num_inference_steps == 1, "GenPercept only forward once."
        return self._engine.infer(rgb_in, out_channels=self._one_step_setup(fix_timesteps, prompt, mode))

    def _one_step_setup(self, fix_timesteps, prompt, mode):
        """Readies the one-step engine for a call (text embedding, timestep); returns the map's channel count."""
        self._ensure_ready(prompt)
        # :405-408: a per-call fix_timesteps replaces the scheduler's [1] for THIS call only
        self._engine.set_timestep(int(fix_timesteps) if fix_timesteps else self._timestep)
        return 1 if (self.customized_head is not None or self._mode(mode) in ONE_CHANNEL_MODES) else 3

    def _single_infer_steps(self, rgb_in, num_inference_steps, generator, fix_timesteps, prompt, mode):
        """genpercept_pipeline.py:399-472 with genpercept_pipeline=False: set_timesteps, pred_latent = randn (marigold) or
        rgb_latent (rgb_blending), the denoising loop with the scheduler's DDIM step, decode(pred_original_sample)."""
        self._ensure_ready(prompt)
        ts = self.scheduler.set_timesteps(int(num_inference_steps))
        # :405-408: fix_timesteps replaces EVERY timestep of the loop — the UNet's and the scheduler step's (:453-460)
        t_unet = [int(fix_timesteps)] * len(ts) if fix_timesteps else [int(t) for t in ts]
        coeffs = [self.scheduler.step_coefficients(t) for t in t_unet]
        B, _, H, W = rgb_in.shape
        noise = None
        if not self.rgb_blending:                                            # :418-425
            gdev = generator.device if generator is not None else self.device
            noise = torch.randn((B, 4, H // 8, W // 8), device=gdev, dtype=torch.float32, generator=generator)
        ch = 1 if self._mode(mode) in ONE_CHANNEL_MODES else 3
        return self._engine.infer_steps(rgb_in, t_unet, coeffs, noise=noise, out_channels=ch)

    def _mode(self, mode=None):
        """``self.mode`` is set by __call__ (:199-200); the helpers read it like the reference does (AttributeError if unset)."""
        return mode if mode is not None else self.mode

    @torch.no_grad()
    def encode_rgb(self, rgb_in):
        """:488-505, device-resident (gp_encode): rgb_in [B,3,H,W] uint8 (0..255) or float in [-1,1], cuda or cpu
        -> latent [B,4,H/8,W/8] on the GPU in ``self.dtype``."""
        self._ensure_ready()
        return self._engine.encode(rgb_in).to(self.dtype)

    @torch.no_grad()
    def decode_pred(self, pred_latent, post_quant=True):
        """:507-526, device-resident (gp_decode): ``vae.post_quant_conv(pred_latent / 0.18215)`` -> decoder -> channel
        mean for the one-channel modes, as the reference.  ``post_quant=False`` is for a latent that already went
        through post_quant_conv (the engine's own "z").  The result is clipped to [-1, 1]: the engine's last kernel
        fuses the clip the reference applies on the very next line (:470), so values beyond it are not recoverable."""
        if self.customized_head is not None:
            raise ValueError("decode_pred is undefined for the DPT readout")
        self._ensure_ready()
        ch = 1 if self._mode() in ONE_CHANNEL_MODES else 3
        out = self._engine.decode(pred_latent.float(), out_channels=ch, post_quant=bool(post_quant))
        return out * 2.0 - 1.0

    @torch.no_grad()
    def __call__(self, input_image, denoising_steps: Optional[int] = None, ensemble_size: int = 1,
                 processing_res: Optional[int] = None, match_input_res: bool = True, resample_method: str = "bilinear",
                 batch_size: int = 0, generator=None, color_map: str = "Spectral", show_progress_bar: bool = True,
                 ensemble_kwargs: Dict = None, mode=None, fix_timesteps=None, prompt="") -> GenPerceptOutput:
        assert mode is not None, "mode of GenPerceptPipeline can be chosen from ['depth', 'normal', 'seg', 'matting', 'dis']."
        self.mode = mode
        if denoising_steps is None:
            denoising_steps = self.default_denoising_steps
        if processing_res is None:
            processing_res = self.default_processing_resolution
        assert processing_res >= 0
        assert ensemble_size >= 1
        if self.genpercept_pipeline:                  # :211-213
            assert ensemble_size == 1
            assert denoising_steps == 1
        else:
            assert denoising_steps >= 1
        rgb, input_size = preprocess(input_image, processing_res, resample_method, self.device)
        if self.genpercept_pipeline or ensemble_size == 1:
            pred = self.single_infer(rgb, num_inference_steps=denoising_steps, generator=generator,
                                     show_pbar=show_progress_bar, fix_timesteps=fix_timesteps, prompt=prompt, mode=mode)
        else:
            # :250-296: the image repeated ensemble_size times, inferred in batches, then ensemble_depth
            assert rgb.shape[0] == 1, "ensembling takes one image (the reference expands it ensemble_size times)"
            from .ensemble import ensemble_depth
            bs = batch_size if batch_size > 0 else min(ensemble_size, 8)
            members = []
            for lo in range(0, ensemble_size, bs):
                n = min(bs, ensemble_size - lo)
                members.append(self.single_infer(rgb.expand(n, -1, -1, -1), num_inference_steps=denoising_steps,
                                                 generator=generator, show_pbar=show_progress_bar, fix_timesteps=fix_timesteps,
                                                 prompt=prompt, mode=mode))
            pred, _ = ensemble_depth(torch.cat(members, dim=0), scale_invariant=True, shift_invariant=True, max_res=50,
                                     **(ensemble_kwargs or {}))
        return postprocess(pred, input_size, match_input_res, resample_method, color_map, self.mode)


# Pre/post-processing of ``__call__`` (shared with multitask.MultiTaskPipeline).  It runs on the GPU (gp_resize_aa /
# gp_colorize / gp_quantize, SURVEY.md §8 f1) for the anti-aliased bilinear / bicubic filters; the nearest modes keep
# torchvision's host path.
def preprocess(input_image, processing_res, resample_method, device):
    """The image intake of ``__call__``: a PIL image or a [B,3,H,W] tensor -> (the engine's rgb input, the input's
    shape).  uint8 stays uint8 (the engine maps x/255*2-1 and casts, :245-246); a float image in [0,255] comes back
    on `device` in [-1,1]."""
    resample = get_tv_resample_method(resample_method)
    if isinstance(input_image, Image.Image):
        rgb = None
        if processing_res <= 0 or resample_method in E.RESIZE_MODES:   # the nearest modes resize on the host
            rgb = decode_unloaded_jpeg(input_image, device, "chw")      # None: Pillow decodes, as the reference does
        rgb = (pil_to_tensor(input_image.convert("RGB")) if rgb is None else rgb).unsqueeze(0)
    elif isinstance(input_image, torch.Tensor):
        rgb = input_image
    else:
        raise TypeError(f"Unknown input type: {type(input_image) = }")
    input_size = rgb.shape
    assert 4 == rgb.dim() and 3 == input_size[-3], f"Wrong input shape {input_size}, expected [1, rgb, H, W]"
    if rgb.dtype != torch.uint8:
        assert rgb.min() >= 0 and rgb.max() <= 255
        rgb = rgb.float() if rgb.is_floating_point() else rgb.to(torch.uint8)
    if processing_res > 0:
        if resample_method in E.RESIZE_MODES:
            h0, w0 = rgb.shape[-2:]
            f = min(processing_res / w0, processing_res / h0)                    # image_util.py:98-102
            rgb = E.resize_aa(rgb, int(h0 * f), int(w0 * f), resample_method, device=device)
        else:
            rgb = resize_max_res(rgb, max_edge_resolution=processing_res, resample_method=resample)
    if rgb.dtype != torch.uint8:                       # float image in [0,255]: the reference keeps it float (:245)
        rgb = rgb.to(device) / 255.0 * 2.0 - 1.0
    return rgb, input_size


def postprocess(pred, input_size, match_input_res, resample_method, color_map, mode) -> GenPerceptOutput:
    """The tail of ``__call__`` (:301-323): pred [B,C,h,w] in [0,1] -> resized back to `input_size`, clipped, and
    colorized (`color_map`, depth / disparity) or quantized to uint8."""
    if match_input_res and tuple(pred.shape[-2:]) != tuple(input_size[-2:]):
        if resample_method in E.RESIZE_MODES:
            pred = E.resize_aa(pred, int(input_size[-2]), int(input_size[-1]), resample_method)
        else:
            pred = resize(pred, list(input_size[-2:]), interpolation=get_tv_resample_method(resample_method), antialias=True)
    pred = pred.clamp(0, 1)                            # :310 (a bicubic resize can overshoot)
    batched = pred.shape[0] > 1
    one_ch = pred.shape[1] == 1
    if color_map is not None:
        assert mode in ["depth", "disparity"]
        lut = (_lut(color_map) * 255).astype(np.uint8)                          # (c * 255).astype(uint8), :318-321
        col = E.colorize(pred[:, 0].contiguous(), lut, 0.0, 1.0).numpy()      # [B,H,W,3] uint8 on the host
    else:
        col = E.quantize(pred, 8)                                               # (p * 255).astype(uint8)
        col = col[:, 0] if one_ch else np.transpose(col, (0, 2, 3, 1))
    colored = [Image.fromarray(c) for c in col]
    pred_np = pred.cpu().numpy()
    pred_np = pred_np.squeeze() if not batched else (pred_np[:, 0] if one_ch else pred_np)
    if batched:
        if pred_np.ndim == 4 and pred_np.shape[1] == 3:
            pred_np = np.transpose(pred_np, (0, 2, 3, 1))
        return GenPerceptOutput(pred_np=pred_np, pred_colored=colored)
    if pred_np.ndim == 3 and pred_np.shape[0] == 3:
        pred_np = np.transpose(pred_np, (1, 2, 0))
    return GenPerceptOutput(pred_np=pred_np, pred_colored=colored[0])
