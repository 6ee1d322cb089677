"""Regenerates tests/golden/reference_pipeline.npz: outputs of the REFERENCE'S OWN code (a GenPercept checkout, whose
path is the first argument) around the oracle's modules, on the seeded inputs that tests/test_oracle_vs_reference_pipeline.py
and tests/test_oracle.py recreate.  Those tests compare the oracle with these arrays, so they need no reference tree.

  python tests/golden/make_golden_reference.py /path/to/GenPercept

The reference modules are imported through a minimal ``diffusers`` / ``matplotlib`` shim (base classes and type names
only: diffusers is not a dependency of this project) and instantiated with the oracle's VAE / UNet modules and one-step
scheduler behind thin adapters, plus the reference's own DPT head class.  Everything between those modules — latent
scaling, the mean half of the moments, the scheduler call and ``pred_original_sample``, ``/ scale`` + post_quant_conv +
decoder, the channel mean, clip and shift, the DPT feature order and min-max — is then the reference's code.

Entries (float32 unless noted):
  glue_depth, glue_normal, glue_latent, glue_fix7, glue_dpt   genpercept/genpercept_pipeline.py:375-526 single_infer /
                                                              encode_rgb on a seeded 64x64 batch (seed 21)
  unet{i}_sample, unet{i}_feat{k}                             genpercept/models/custom_unet.py:34-427 forward around the
                                                              oracle's blocks, sizes 8x8, 9x11, 12x10 (seed 4); of the
                                                              DPT feature taps every FEAT_STRIDE-th channel (file size)
  sched_betas, sched_alphas_cumprod, sched_final_alpha_cumprod, sched_init_noise_sigma
                                                              src/customized_modules/ddim.py:144-217 from
                                                              hf_configs/scheduler_beta_1.0_1.0/scheduler_config.json
  resize{edge} (uint8), tv_{mode} (str), tv_lanczos_raises, chw2hwc
                                                              genpercept/util/image_util.py:66-119 (seed 8)
  v1_depth                                                    GenPercept_v1/genpercept/pipeline_genpercept.py:263-354 with
                                                              GenPercept_v1/empty_text_embed.npy (seed 31), which is
                                                              copied to tests/golden/empty_text_embed_77x1024.npy
  up_weight, up_bias, up_x, up_out, up_out_{h}x{w}            the Upsample2D vendored in genpercept/models/dpt_head.py:92-210
"""
import importlib
import importlib.util
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
UNET_SIZES = ((8, 8), (9, 11), (12, 10))
FEAT_STRIDE = 8
RESIZE_EDGES = (64, 128, 200)
UPSAMPLE_SIZES = ((13, 17), (14, 18), (13, 18))


def install_shims(ref):
    import torch.nn as nn
    if "diffusers" not in sys.modules or not hasattr(sys.modules["diffusers"], "DiffusionPipeline"):
        d = sys.modules.get("diffusers") or types.ModuleType("diffusers")

        class DiffusionPipeline:
            def __init__(self):
                self._cfg = {}

            def register_modules(self, **kw):
                for k, v in kw.items():
                    setattr(self, k, v)

            def register_to_config(self, **kw):
                self._cfg.update(kw)

            @property
            def device(self):
                return torch.device("cpu")

            @property
            def dtype(self):
                return torch.float32

        for name in ("AutoencoderKL", "DDIMScheduler", "LCMScheduler", "UNet2DConditionModel"):
            setattr(d, name, type(name, (), {}))
        d.DiffusionPipeline = DiffusionPipeline
        du = sys.modules.get("diffusers.utils") or types.ModuleType("diffusers.utils")
        du.BaseOutput = type("BaseOutput", (), {})
        du.USE_PEFT_BACKEND = True
        dm = sys.modules.get("diffusers.models") or types.ModuleType("diffusers.models")
        dl = sys.modules.get("diffusers.models.lora") or types.ModuleType("diffusers.models.lora")
        dl.LoRACompatibleConv = nn.Conv2d
        d.utils, d.models, dm.lora = du, dm, dl
        sys.modules.update({"diffusers": d, "diffusers.utils": du, "diffusers.models": dm, "diffusers.models.lora": dl})
    if "matplotlib" not in sys.modules:
        m = types.ModuleType("matplotlib")
        mp = types.ModuleType("matplotlib.pyplot")
        m.pyplot = mp
        sys.modules.update({"matplotlib": m, "matplotlib.pyplot": mp})
    if ref not in sys.path:
        sys.path.insert(0, ref)


class UNetAdapter:
    def __init__(self, unet):
        self.unet = unet

    def __call__(self, x, t, encoder_hidden_states=None, return_feature=False):
        t = torch.as_tensor(t).reshape(-1)[:1]
        out = self.unet(x, t, encoder_hidden_states, return_feature=return_feature)
        return types.SimpleNamespace(multi_level_feats=out) if return_feature else types.SimpleNamespace(sample=out)


class SchedulerAdapter:
    beta_start = 1
    beta_end = 1

    def __init__(self, s):
        self.s = s

    def set_timesteps(self, n, device=None):
        self.timesteps = self.s.set_timesteps(n)

    def step(self, model_output, t, sample, generator=None):
        prev, x0 = self.s.step(model_output, int(t), sample)
        return types.SimpleNamespace(prev_sample=prev, pred_original_sample=x0)


def glue(ref, state, te, out):
    from oracle.pipeline import OraclePipeline
    install_shims(ref)
    mod = importlib.import_module("genpercept.genpercept_pipeline")
    g = torch.Generator().manual_seed(21)
    rgb = torch.rand((1, 3, 64, 64), generator=g) * 2 - 1
    op = OraclePipeline(state, te)
    rp = mod.GenPerceptPipeline(unet=UNetAdapter(op.unet), vae=op.vae, scheduler=SchedulerAdapter(op.scheduler),
                                text_encoder=None, tokenizer=None, genpercept_pipeline=True)
    rp.text_embed = op.text_embed
    with torch.no_grad():
        for mode in ("depth", "normal"):
            rp.mode = mode
            out[f"glue_{mode}"] = rp.single_infer(rgb, 1, None, False)
        out["glue_latent"] = rp.encode_rgb(rgb)
        out["glue_fix7"] = rp.single_infer(rgb, 1, None, False, fix_timesteps=7)     # rp.mode is "normal" here
    # DPT readout with the reference's own head class (isinstance check at genpercept_pipeline.py:475)
    od = OraclePipeline(state, te, use_dpt=True)
    head_mod = sys.modules["genpercept.models.dpt_head"]
    # transformers >= 4.4x refuses ModelOutput subclasses that are not dataclasses; the reference's output container
    # (dpt_head.py:24-49, written for an older transformers) is replaced by a plain attribute bag — no arithmetic involved
    head_mod.DepthEstimatorOutput = lambda **kw: types.SimpleNamespace(**kw)
    from transformers import DPTConfig
    head = head_mod.DPTNeckHeadForUnetAfterUpsampleIdentity(
        DPTConfig.from_pretrained(f"{ref}/hf_configs/dpt-sd2.1-unet-after-upsample-general")).eval()
    head.load_state_dict(state["dpt"], strict=True)
    rd = mod.GenPerceptPipeline(unet=UNetAdapter(od.unet), vae=od.vae, scheduler=SchedulerAdapter(od.scheduler),
                                text_encoder=None, tokenizer=None, customized_head=head, genpercept_pipeline=True)
    rd.text_embed = od.text_embed
    rd.mode = "depth"
    with torch.no_grad():
        out["glue_dpt"] = rd.single_infer(rgb, 1, None, False)


def unet(ref, state, te, out):
    import torch.nn as nn
    install_shims(ref)
    d = sys.modules["diffusers"]
    d.UNet2DConditionModel = type("UNet2DConditionModel", (nn.Module,), {})
    du = sys.modules["diffusers.utils"]
    du.deprecate = lambda *a, **k: None
    du.logging = types.SimpleNamespace(get_logger=lambda *a, **k: None)
    du.scale_lora_layers = lambda *a, **k: None
    du.unscale_lora_layers = lambda *a, **k: None
    unets = types.ModuleType("diffusers.models.unets")
    u2d = types.ModuleType("diffusers.models.unets.unet_2d_condition")
    u2d.UNet2DConditionOutput = type("UNet2DConditionOutput", (), {})
    sys.modules.update({"diffusers.models.unets": unets, "diffusers.models.unets.unet_2d_condition": u2d})
    spec = importlib.util.spec_from_file_location("ref_custom_unet", f"{ref}/genpercept/models/custom_unet.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    from oracle.pipeline import OraclePipeline
    ou = OraclePipeline(state, te).unet

    class Down(nn.Module):
        def __init__(self, blk, cross):
            super().__init__()
            self.blk, self.has_cross_attention = blk, cross

        def forward(self, hidden_states, temb, encoder_hidden_states=None, **kw):
            return self.blk(hidden_states, temb, encoder_hidden_states)

    class Mid(nn.Module):
        has_cross_attention = True

        def __init__(self, blk):
            super().__init__()
            self.blk = blk

        def forward(self, sample, emb, encoder_hidden_states=None, **kw):
            return self.blk(sample, emb, encoder_hidden_states)

    class Up(nn.Module):
        def __init__(self, blk):
            super().__init__()
            self.blk, self.has_cross_attention, self.resnets = blk, blk.attentions is not None, blk.resnets

        def forward(self, hidden_states, temb, res_hidden_states_tuple, encoder_hidden_states=None, upsample_size=None, **kw):
            return self.blk(hidden_states, res_hidden_states_tuple, temb, encoder_hidden_states, upsample_size)

    class TimeEmb(nn.Module):
        def __init__(self, m):
            super().__init__()
            self.m = m

        def forward(self, t_emb, cond=None):
            return self.m(t_emb)

    ru = mod.CustomUNet2DConditionModel()
    ru.num_upsamplers = 3
    ru.config = types.SimpleNamespace(center_input_sample=False, class_embed_type=None, addition_embed_type=None,
                                      class_embeddings_concat=False, encoder_hid_dim_type=None)
    ru.class_embedding = ru.time_embed_act = ru.encoder_hid_proj = None
    ru.time_proj, ru.time_embedding = ou.time_proj, TimeEmb(ou.time_embedding)
    ru.conv_in, ru.conv_norm_out, ru.conv_act, ru.conv_out = ou.conv_in, ou.conv_norm_out, nn.SiLU(), ou.conv_out
    ru.down_blocks = nn.ModuleList([Down(b, i < 3) for i, b in enumerate(ou.down_blocks)])
    ru.mid_block = Mid(ou.mid_block)
    ru.up_blocks = nn.ModuleList([Up(b) for b in ou.up_blocks])
    ru.eval()
    g = torch.Generator().manual_seed(4)
    ctx = te.float().reshape(1, -1, 1024)
    for i, (h, w) in enumerate(UNET_SIZES):
        x = torch.randn((1, 4, h, w), generator=g)
        with torch.no_grad():
            out[f"unet{i}_sample"] = ru(x, 1, ctx).sample
            for k, f in enumerate(ru(x, torch.tensor([1]), ctx, return_feature=True).multi_level_feats):
                out[f"unet{i}_feat{k}"] = f[:, ::FEAT_STRIDE].contiguous()


def scheduler(ref, out):
    install_shims(ref)
    d = sys.modules["diffusers"]
    d.DDIMScheduler = getattr(d, "DDIMScheduler", type("DDIMScheduler", (), {}))
    d.DDPMScheduler = type("DDPMScheduler", (), {})
    cu = types.ModuleType("diffusers.configuration_utils")
    cu.ConfigMixin = type("ConfigMixin", (), {})
    cu.register_to_config = lambda f: f
    sys.modules["diffusers.configuration_utils"] = cu
    spec = importlib.util.spec_from_file_location("ref_ddim", f"{ref}/src/customized_modules/ddim.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    cfg = json.load(open(f"{ref}/hf_configs/scheduler_beta_1.0_1.0/scheduler_config.json"))
    kw = {k: v for k, v in cfg.items() if not k.startswith("_") and k != "skip_prk_steps"}
    s = mod.DDIMSchedulerCustomized(**kw)
    out["sched_betas"] = s.betas
    out["sched_alphas_cumprod"] = s.alphas_cumprod
    out["sched_final_alpha_cumprod"] = torch.as_tensor(s.final_alpha_cumprod)
    out["sched_init_noise_sigma"] = torch.as_tensor(float(s.init_noise_sigma))


def image_helpers(ref, out):
    install_shims(ref)
    mod = importlib.import_module("genpercept.util.image_util")
    g = torch.Generator().manual_seed(8)
    x = torch.randint(0, 256, (1, 3, 90, 160), generator=g, dtype=torch.uint8)
    for edge in RESIZE_EDGES:
        out[f"resize{edge}"] = mod.resize_max_res(x, edge)
    for m in ("bilinear", "bicubic", "nearest"):
        out[f"tv_{m}"] = np.array(str(mod.get_tv_resample_method(m)))
    try:
        mod.get_tv_resample_method("lanczos")
        out["tv_lanczos_raises"] = np.array(False)
    except ValueError:
        out["tv_lanczos_raises"] = np.array(True)
    c = torch.rand((3, 4, 5), generator=g)
    out["chw2hwc"] = mod.chw2hwc(c)


def legacy_v1(ref, state, out):
    from oracle.pipeline import OraclePipeline
    install_shims(ref)
    v1_root = f"{ref}/GenPercept_v1"
    spec = importlib.util.spec_from_file_location("genpercept_v1", f"{v1_root}/genpercept/__init__.py",
                                                  submodule_search_locations=[f"{v1_root}/genpercept"])
    pkg = importlib.util.module_from_spec(spec)
    sys.modules["genpercept_v1"] = pkg
    spec.loader.exec_module(pkg)
    mod = importlib.import_module("genpercept_v1.pipeline_genpercept")
    e = np.load(f"{v1_root}/empty_text_embed.npy")
    np.save(os.path.join(HERE, "empty_text_embed_77x1024.npy"), e)
    te = torch.from_numpy(e.astype(np.float32))[None]     # [1, 77, 1024]
    op = OraclePipeline(state, te)
    p1 = mod.GenPerceptPipeline(unet=UNetAdapter(op.unet), vae=op.vae, empty_text_embed=te)
    g = torch.Generator().manual_seed(31)
    rgb = torch.rand((1, 3, 64, 64), generator=g) * 2 - 1
    with torch.no_grad():
        out["v1_depth"] = p1.single_infer(rgb, mode="depth")


def upsample(out):
    import make_golden
    make_golden.load_reference_dpt()
    ref_mod = sys.modules["ref_dpt_head"]
    torch.manual_seed(3)
    up = ref_mod.Upsample2D(24, use_conv=True).eval()
    x = torch.randn(2, 24, 7, 9)
    out["up_weight"], out["up_bias"], out["up_x"] = up.conv.weight, up.conv.bias, x
    with torch.no_grad():
        out["up_out"] = up(x)
        for h, w in UPSAMPLE_SIZES:
            out[f"up_out_{h}x{w}"] = up(x, output_size=(h, w))


def main(ref):
    import make_golden
    from genpercept_b200 import weights as W
    make_golden.REF = ref
    state = W.synth_state(1234)
    te = torch.from_numpy(np.load(os.path.join(HERE, "empty_text_embed_2x1024.npy")).astype(np.float32))[None]
    out = {}
    glue(ref, state, te, out)
    unet(ref, state, te, out)
    scheduler(ref, out)
    image_helpers(ref, out)
    legacy_v1(ref, state, out)
    upsample(out)
    arrays = {k: (v.detach().numpy() if torch.is_tensor(v) else v) for k, v in out.items()}
    path = os.path.join(HERE, "reference_pipeline.npz")
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path), "bytes,", len(arrays), "arrays")


if __name__ == "__main__":
    main(sys.argv[1])
