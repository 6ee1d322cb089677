"""Checkpoint key/shape specification of the SD-2.1 GenPercept models and a seeded synthetic
weight generator.

The key names are the diffusers on-disk names that the reference loads
(/root/reference/run.py:314-343 UNet, :296-301 DPT head, :308-312 VAE decoder override), so a real
``diffusion_pytorch_model.safetensors`` drops in through the same ``load_state`` path.  No
weights ship with the reference (SURVEY.md F4); tests and bench use ``synth_state``.
"""
from collections import OrderedDict

import numpy as np
import torch

UNET_BLOCK_OUT = (320, 640, 1280, 1280)
UNET_HEADS = (5, 10, 20, 20)
CROSS_DIM = 1024
TEMB = 1280


def _conv(spec, name, cin, cout, k, bias=True):
    spec[name + ".weight"] = ((cout, cin, k, k), "conv")
    if bias:
        spec[name + ".bias"] = ((cout,), "bias")


def _lin(spec, name, cin, cout, bias=True):
    spec[name + ".weight"] = ((cout, cin), "linear")
    if bias:
        spec[name + ".bias"] = ((cout,), "bias")


def _norm(spec, name, c):
    spec[name + ".weight"] = ((c,), "gamma")
    spec[name + ".bias"] = ((c,), "beta")


def _resnet(spec, p, cin, cout, temb=True):
    _norm(spec, p + ".norm1", cin)
    _conv(spec, p + ".conv1", cin, cout, 3)
    if temb:
        _lin(spec, p + ".time_emb_proj", TEMB, cout)
    _norm(spec, p + ".norm2", cout)
    _conv(spec, p + ".conv2", cout, cout, 3)
    if cin != cout:
        _conv(spec, p + ".conv_shortcut", cin, cout, 1)


def _transformer(spec, p, c):
    _norm(spec, p + ".norm", c)
    _lin(spec, p + ".proj_in", c, c)
    b = p + ".transformer_blocks.0"
    _norm(spec, b + ".norm1", c)
    for n in ("to_q", "to_k", "to_v"):
        _lin(spec, b + ".attn1." + n, c, c, bias=False)
    _lin(spec, b + ".attn1.to_out.0", c, c)
    _norm(spec, b + ".norm2", c)
    _lin(spec, b + ".attn2.to_q", c, c, bias=False)
    _lin(spec, b + ".attn2.to_k", CROSS_DIM, c, bias=False)
    _lin(spec, b + ".attn2.to_v", CROSS_DIM, c, bias=False)
    _lin(spec, b + ".attn2.to_out.0", c, c)
    _norm(spec, b + ".norm3", c)
    _lin(spec, b + ".ff.net.0.proj", c, 8 * c)
    _lin(spec, b + ".ff.net.2", 4 * c, c)
    _lin(spec, p + ".proj_out", c, c)


def unet_spec(in_channels=4, out_channels=4):
    """SURVEY.md App. A.2."""
    s = OrderedDict()
    _conv(s, "conv_in", in_channels, 320, 3)
    _lin(s, "time_embedding.linear_1", 320, TEMB)
    _lin(s, "time_embedding.linear_2", TEMB, TEMB)
    cin = 320
    for i, cout in enumerate(UNET_BLOCK_OUT):
        for j in range(2):
            _resnet(s, f"down_blocks.{i}.resnets.{j}", cin if j == 0 else cout, cout)
            if i < 3:
                _transformer(s, f"down_blocks.{i}.attentions.{j}", cout)
        if i < 3:
            _conv(s, f"down_blocks.{i}.downsamplers.0.conv", cout, cout, 3)
        cin = cout
    _resnet(s, "mid_block.resnets.0", 1280, 1280)
    _transformer(s, "mid_block.attentions.0", 1280)
    _resnet(s, "mid_block.resnets.1", 1280, 1280)
    up = [(1280, 1280, (1280, 1280, 1280), False), (1280, 1280, (1280, 1280, 640), True),
          (1280, 640, (640, 640, 320), True), (640, 320, (320, 320, 320), True)]
    for i, (cprev, cout, skips, attn) in enumerate(up):
        for j in range(3):
            _resnet(s, f"up_blocks.{i}.resnets.{j}", (cprev if j == 0 else cout) + skips[j], cout)
            if attn:
                _transformer(s, f"up_blocks.{i}.attentions.{j}", cout)
        if i < 3:
            _conv(s, f"up_blocks.{i}.upsamplers.0.conv", cout, cout, 3)
    _norm(s, "conv_norm_out", 320)
    _conv(s, "conv_out", 320, out_channels, 3)
    return s


def _vae_mid(s, p):
    _resnet(s, p + ".resnets.0", 512, 512, temb=False)
    a = p + ".attentions.0"
    _norm(s, a + ".group_norm", 512)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        _lin(s, a + "." + n, 512, 512)
    _resnet(s, p + ".resnets.1", 512, 512, temb=False)


def vae_spec():
    """SURVEY.md App. A.3."""
    s = OrderedDict()
    _conv(s, "encoder.conv_in", 3, 128, 3)
    chans = (128, 128, 256, 512, 512)
    for i in range(4):
        for j in range(2):
            _resnet(s, f"encoder.down_blocks.{i}.resnets.{j}", chans[i] if j == 0 else chans[i + 1],
                    chans[i + 1], temb=False)
        if i < 3:
            _conv(s, f"encoder.down_blocks.{i}.downsamplers.0.conv", chans[i + 1], chans[i + 1], 3)
    _vae_mid(s, "encoder.mid_block")
    _norm(s, "encoder.conv_norm_out", 512)
    _conv(s, "encoder.conv_out", 512, 8, 3)
    _conv(s, "decoder.conv_in", 4, 512, 3)
    _vae_mid(s, "decoder.mid_block")
    prev = (512, 512, 512, 256)
    outc = (512, 512, 256, 128)
    for i in range(4):
        for j in range(3):
            _resnet(s, f"decoder.up_blocks.{i}.resnets.{j}", prev[i] if j == 0 else outc[i], outc[i],
                    temb=False)
        if i < 3:
            _conv(s, f"decoder.up_blocks.{i}.upsamplers.0.conv", outc[i], outc[i], 3)
    _norm(s, "decoder.conv_norm_out", 128)
    _conv(s, "decoder.conv_out", 128, 3, 3)
    _conv(s, "quant_conv", 8, 8, 1)
    _conv(s, "post_quant_conv", 4, 4, 1)
    return s


def dpt_spec():
    """SURVEY.md App. A.4 (dpt_head.py + hf_configs/dpt-sd2.1-unet-after-upsample-general)."""
    s = OrderedDict()
    _conv(s, "feature_upsample_0.conv", 320, 320, 3)
    for i, c in enumerate((320, 640, 1280, 1280)):
        _conv(s, f"neck.convs.{i}", c, 256, 3, bias=False)
    for i in range(4):
        p = f"neck.fusion_stage.layers.{i}"
        _conv(s, p + ".projection", 256, 256, 1)
        for r in (("residual_layer1",) if i > 0 else ()) + ("residual_layer2",):
            _conv(s, f"{p}.{r}.convolution1", 256, 256, 3, bias=False)
            _conv(s, f"{p}.{r}.convolution2", 256, 256, 3, bias=False)
    _conv(s, "head.projection", 256, 256, 3)
    _conv(s, "head.head.0", 256, 128, 3)
    _conv(s, "head.head.2", 128, 32, 3)
    _conv(s, "head.head.4", 32, 1, 1)
    return s


# legacy SD checkpoints name the VAE attention params differently (diffusers remaps on load)
_LEGACY_VAE_ATTN = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}


def remap_legacy_vae_keys(sd):
    out = {}
    for k, v in sd.items():
        parts = k.split(".")
        if "attentions" in parts:
            for old, new in _LEGACY_VAE_ATTN.items():
                if parts[-2] == old:
                    k = ".".join(parts[:-2] + [new, parts[-1]])
                    if v.dim() == 4:            # 1x1 conv form -> linear
                        v = v[:, :, 0, 0]
        out[k] = v
    return out


def encoder_state(vae_sd):
    """The VAE's encode side (encoder.*, quant_conv.*: everything encode_rgb reads) of a diffusers-layout state dict:
    the same tensors, not copies."""
    return {k: v for k, v in vae_sd.items() if k.startswith(("encoder.", "quant_conv."))}


def synth_unet(seed, in_channels=4):
    """A seeded synthetic UNet alone (the gains of ``synth_state``): task engines that share one VAE."""
    return _synth(unet_spec(in_channels=in_channels), torch.Generator().manual_seed(seed), gain=1.0, out_gain={"conv_out": 2.0})


def _synth(spec, gen, gain=1.0, out_gain=None):
    sd = OrderedDict()
    for k, (shape, kind) in spec.items():
        if kind in ("conv", "linear"):
            fan_in = int(np.prod(shape[1:]))
            g = gain
            if out_gain is not None and any(k.startswith(p) for p in out_gain):
                g = [v for p, v in out_gain.items() if k.startswith(p)][0]
            w = torch.randn(shape, generator=gen, dtype=torch.float32) * (g / fan_in ** 0.5)
        elif kind == "bias":
            w = torch.randn(shape, generator=gen, dtype=torch.float32) * 0.05
        elif kind == "gamma":
            w = 1.0 + 0.1 * (2 * torch.rand(shape, generator=gen, dtype=torch.float32) - 1)
        elif kind == "beta":
            w = 0.1 * (2 * torch.rand(shape, generator=gen, dtype=torch.float32) - 1)
        else:
            raise ValueError(kind)
        sd[k] = w
    return sd


def synth_state(seed=1234, with_dpt=True, unet_in_channels=4):
    """Seeded synthetic fp32 weights with the exact SD-2.1 topology (SURVEY.md 8d).

    Gains are chosen so activations stay O(1) through the depth of the graph and the final maps
    spread over [0,1] instead of collapsing to a constant (checked in tests/test_oracle.py)."""
    gen = torch.Generator().manual_seed(seed)
    state = {
        "vae": _synth(vae_spec(), gen, gain=1.0,
                      out_gain={"decoder.conv_out": 1.5, "encoder.conv_out": 2.0, "quant_conv": 1.5}),
        "unet": _synth(unet_spec(in_channels=unet_in_channels), gen, gain=1.0, out_gain={"conv_out": 2.0}),
    }
    if with_dpt:
        state["dpt"] = _synth(dpt_spec(), gen, gain=1.0)
    return state


def synth_text_embed(seed=1234, n_tokens=2):
    """Stand-in for the cached empty-prompt embedding ([1, 2, 1024], genpercept_pipeline.py:427-429)
    when the fixture tests/golden/empty_text_embed_2x1024.npy is not used."""
    gen = torch.Generator().manual_seed(seed + 77)
    return torch.randn((1, n_tokens, 1024), generator=gen, dtype=torch.float32)


TEXT_VOCAB, TEXT_POSITIONS, TEXT_DIM, TEXT_LAYERS, TEXT_MLP = 49408, 77, 1024, 23, 4096


def text_spec():
    """SD-2.1's CLIP text tower (transformers' CLIPTextModel, SURVEY.md App. A) under its own state-dict keys."""
    s = OrderedDict()
    m = "text_model."
    s[m + "embeddings.token_embedding.weight"] = ((TEXT_VOCAB, TEXT_DIM), "embedding")
    s[m + "embeddings.position_embedding.weight"] = ((TEXT_POSITIONS, TEXT_DIM), "embedding")
    for i in range(TEXT_LAYERS):
        p = f"{m}encoder.layers.{i}."
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            _lin(s, p + "self_attn." + n, TEXT_DIM, TEXT_DIM)
        _norm(s, p + "layer_norm1", TEXT_DIM)
        _lin(s, p + "mlp.fc1", TEXT_DIM, TEXT_MLP)
        _lin(s, p + "mlp.fc2", TEXT_MLP, TEXT_DIM)
        _norm(s, p + "layer_norm2", TEXT_DIM)
    _norm(s, m + "final_layer_norm", TEXT_DIM)
    return s


def synth_text_state(seed=1234):
    """Seeded synthetic fp32 weights of SD-2.1's CLIP text tower (``text_spec``), from a generator of their own, so no
    other fixture's stream moves.  Embedding rows have std 0.5, so token and position both matter after the first
    LayerNorm; the linear layers keep O(1) activations as in ``synth_state``."""
    sd = OrderedDict()
    gen = torch.Generator().manual_seed(seed + 4242)
    for k, (shape, kind) in text_spec().items():
        if kind == "embedding":
            sd[k] = torch.randn(shape, generator=gen, dtype=torch.float32) * 0.5
        else:
            sd.update(_synth(OrderedDict([(k, (shape, kind))]), gen))
    return sd


def param_count(spec):
    return sum(int(np.prod(s)) for s, _ in spec.values())
