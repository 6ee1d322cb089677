"""Several GenPercept tasks on one image with one VAE encode.

Every released GenPercept checkpoint (depth, normal, segmentation, matting, dichotomous segmentation, disparity, with
the VAE or the DPT readout) runs on the same frozen SD-2.1 VAE encoder: the reference takes ``vae/`` from the SD-2.1
folder and overrides at most the decoder (run.py:283-376).  ``MultiTaskPipeline`` pre-processes an image once, encodes
it once on the first task's engine (``Engine.encode_exact``) and runs every task's UNet and readout from that latent
(``Engine.infer_latent``).  Each task's maps are bit for bit those of its own ``GenPerceptPipeline.__call__``.
"""
from typing import Dict, Optional

import torch

from .pipeline import GenPerceptOutput, GenPerceptPipeline, postprocess, preprocess

COLORIZED_MODES = ("depth", "disparity")       # the modes __call__ colorizes (genpercept_pipeline.py:316-321)


def _equal(x, y):
    """Equal weights as an engine holds them (fp32), whatever dtype or device they came in."""
    if x is y:
        return True
    return tuple(x.shape) == tuple(y.shape) and torch.equal(x.detach().to("cpu", torch.float32), y.detach().to("cpu", torch.float32))


class MultiTaskPipeline:
    """``pipelines``: {task name: one-step GenPerceptPipeline}; ``modes``: {task name: mode} (the ``mode`` each task's
    ``__call__`` would get: depth, normal, seg, matting, dis, disparity).

    The pipelines must run the one-step arch on one device with one dtype and precision mode, and hold equal VAE encoder
    weights (vae.encoder.*, vae.quant_conv.*, compared by value); their decoders, DPT heads, UNets, timesteps and text
    embeddings are their own.  Otherwise construction raises ValueError naming the task and what differs.

    ``share_arena=True`` turns on the shared activation arena (``GenPerceptPipeline.enable_shared_arena``) of every task's
    engine, so the tasks need one inference's worth of activation memory instead of one per task; the maps are unchanged.
    """

    def __init__(self, pipelines: Dict[str, GenPerceptPipeline], modes: Dict[str, str], share_arena: bool = False):
        if not pipelines:
            raise ValueError("MultiTaskPipeline needs at least one task")
        if set(modes) != set(pipelines):
            raise ValueError(f"modes must name exactly the tasks {sorted(pipelines)}; got {sorted(modes)}")
        names = list(pipelines)
        first = pipelines[names[0]]
        for name in names:
            p = pipelines[name]
            if not p.genpercept_pipeline:
                raise ValueError(f"task {name!r}: a multi-step pipeline (genpercept_pipeline=False); only one-step "
                                 "pipelines run from a shared latent")
            for attr in ("device", "dtype", "precision"):
                if getattr(p, attr) != getattr(first, attr):
                    raise ValueError(f"task {name!r}: {attr} {getattr(p, attr)} differs from task {names[0]!r}'s "
                                     f"{getattr(first, attr)}")
            a, b = first._encoder_state, p._encoder_state
            for k in sorted(set(a) | set(b)):
                if k not in a or k not in b or not _equal(a[k], b[k]):
                    raise ValueError(f"task {name!r}: vae.{k} differs from task {names[0]!r}'s; one encode serves only "
                                     "tasks that share the VAE encoder")
        self.pipelines = dict(pipelines)
        self.modes = dict(modes)
        if share_arena:
            for p in self.pipelines.values():
                p.enable_shared_arena()

    @torch.no_grad()
    def __call__(self, input_image, processing_res: Optional[int] = None, match_input_res: bool = True,
                 resample_method: str = "bilinear", color_map: Optional[str] = "Spectral",
                 fix_timesteps=None) -> Dict[str, GenPerceptOutput]:
        """``GenPerceptPipeline.__call__`` for every task at once -> {task name: GenPerceptOutput}.  `input_image`: a
        PIL image or a uint8 / float [B,3,H,W] tensor, as ``__call__`` takes it.  `processing_res` defaults to the first
        task's ``default_processing_resolution``.  `color_map` colorizes the depth and disparity tasks (None: quantize
        them too); the other modes are always quantized.  `fix_timesteps` (None: each task's own) applies to every task."""
        names = list(self.pipelines)
        enc = self.pipelines[names[0]]
        if enc.precision == "high":
            # the encoder's VAE mid-block attention follows the switch: a latent made with the other setting differs
            for name in names:
                if self.pipelines[name]._engine.memory_efficient_attention != enc._engine.memory_efficient_attention:
                    raise ValueError(f"task {name!r}: memory-efficient attention differs from task {names[0]!r}'s")
        if processing_res is None:
            processing_res = enc.default_processing_resolution
        assert processing_res >= 0
        rgb, input_size = preprocess(input_image, processing_res, resample_method, enc.device)
        B, _, H, W = rgb.shape
        enc._ensure_ready()
        latent = enc._engine.encode_exact(rgb)
        out = {}
        for name in names:
            p, mode = self.pipelines[name], self.modes[name]
            p.mode = mode                                    # as __call__ leaves it (genpercept_pipeline.py:199-200)
            ch = p._one_step_setup(fix_timesteps, "", mode)
            eng = p._engine
            if eng.plan_shape != (B, H, W):
                eng.plan(B, H, W)
            pred = eng.infer_latent(latent, out_channels=ch)
            out[name] = postprocess(pred, input_size, match_input_res, resample_method,
                                    color_map if mode in COLORIZED_MODES else None, mode)
        return out
