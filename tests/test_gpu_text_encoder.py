"""SD-2.1's CLIP text tower on the engine (gp_encode_text) and its kernels (gp_causal_attention, gp_gelu).

Per kernel: each entry point against fp64 on exactly the operands it sees (16-bit-rounded, or hi + lo of the pair).  The
whole tower: Engine.encode_text against oracle/clip.py in fp64 on synth_text_state weights.  Bounds, with u_s the storage
unit (2^-11 fp16, 2^-8 bf16, 2^-22 for an fp16 (hi, lo) pair) and u = 2^-24:
  attention 16-bit  C16 u_s max|ref|: one output ulp of the magnitude (scores, softmax and P V are fp32)
            pair    C_ATTN u (|ref| + (1 + max_j |s_ij|) max|v|): the fp32 scores' error moves P by u |s| relative
  GELU      16-bit  C16 u_s |ref| + 2^-24 (fp16's subnormal spacing)
            pair    C_GELU u |ref| (1 + x^2) + 2^-24: erfc's relative error grows with its argument; the lo plane's fp16
                    subnormal spacing bounds the pair's absolute precision
  tower     16-bit  C_TOWER16 u_s max|ref|: 23 layers of 16-bit activations and weights
            pair    C_TOWER_PAIR u max|ref|; the observed max|err| / (u max|ref|) is printed.  It is the high-precision
                    mode's level (the three-pass products and the tensor cores' fp32 accumulation over K = 4096, as in
                    the UNet), about 30 times transformers' fp32 tower against fp64 (9 u) and 1/100 of the fp16 mode's.

Calibrated on an NVIDIA H100 80GB HBM3 (700 W power limit).  Worst |err| / bound at the constants below (fp16 / bf16 /
pair): causal attention 0.30 / 0.30 / 0.033 (n = 2); GELU 0.50 / 0.49 / 0.50; tower 0.61 / 0.52 / 0.28
(max|err| = 264 - 291 u max|ref| over n = 2, 7, 77).

Discrimination (CPU, test_bounds_discriminate_*): fp64 outputs of plausible wrong kernels break each bound at least
DISCRIMINATION times: for the attention bound no causal mask, the mask off by one and the softmax scale not folded; for
the GELU bound the tanh form; for the tower bound positions offset by one, the final LayerNorm skipped and the tanh GELU.
Not asserted (the ratios are printed), because a precision cannot separate it:
  - the tanh GELU in the whole tower, in every mode: it moves the output by about 2e-4 of its largest value, under the
    16-bit bounds (0.03x) and 3.6x the pair layout's.  Per kernel the GELU bound separates it in every mode (61x and
    more), since there it is elementwise.
"""
import functools
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import clip

U = 2.0 ** -24
C16 = 2.0
C_ATTN = 64.0
C_GELU = 16.0
C_TOWER16 = {"f16": 8.0, "bf16": 8.0}
C_TOWER_PAIR = 1024.0
DISCRIMINATION = 10.0

DTYPES = {"f16": torch.float16, "bf16": torch.bfloat16, "pair": torch.float32}
US = {"f16": 2.0 ** -11, "bf16": 2.0 ** -8, "pair": 2.0 ** -22}
PROMPT_IDS = [49406, 320, 1205, 3027, 12875, 2867, 49407]       # "a high quality rgb image" as CLIPTokenizer gives it
TOWER_CASES = {2: [49406, 49407], 7: PROMPT_IDS, 77: [49406] + [(1000 + 613 * i) % 49408 for i in range(75)] + [49407]}
ATTN_N = (1, 2, 3, 16, 77)


@functools.lru_cache(maxsize=1)
def _text_sd():
    from genpercept_b200 import weights as W
    return W.synth_text_state(1234)


def _split(t):
    from genpercept_b200.engine import split_hi_lo
    hi, lo = split_hi_lo(t)
    return hi.double(), lo.double()


def _seen(t, dt):
    """fp32 t as the kernel sees it in layout dt: the 16-bit value, or hi + lo of the pair (fp64)."""
    if dt == "pair":
        hi, lo = _split(t)
        return hi + lo
    return t.to(DTYPES[dt]).double()


def _arg(t, dt):
    return t if dt == "pair" else t.to(DTYPES[dt])


def _report(name, err, bound):
    ratio = (err / bound).max().item()
    print(f"{name}: max|err|/bound = {ratio:.3f}")
    assert torch.isfinite(err).all(), name + ": non-finite output"
    assert ratio <= 1.0, f"{name}: |err| exceeds the bound {ratio:.3f}x"


def _discriminates(name, bound, wrong, exempt=()):
    for v, d in wrong:
        r = (d / bound).max().item()
        print(f"{name}: {v} breaks the bound {r:.1f}x" + (" (not asserted)" if v in exempt else ""))
        assert v in exempt or r >= DISCRIMINATION, f"{name}: {v} stays within {DISCRIMINATION}x of the bound ({r:.2f})"


# ------------------------------------------------------------------------------------------------ causal attention
def _attn_operands(n, gen, heads=16, d=64):
    C = heads * d
    q = torch.randn((n, C), generator=gen) * 0.25       # the scale already folded: scores of a few units
    k = torch.randn((n, C), generator=gen)
    v = torch.randn((n, C), generator=gen)
    return torch.cat([q, k, v], dim=-1), heads


def _attn_bound(qkv_seen, ref, heads, dt):
    n, c3 = qkv_seen.shape
    C = c3 // 3
    if dt != "pair":
        return torch.full_like(ref, C16 * US[dt] * ref.abs().max().item())
    d = C // heads
    q, k, v = (t.reshape(n, heads, d).transpose(0, 1) for t in qkv_seen.split(C, dim=-1))
    smax = (q @ k.transpose(1, 2)).abs().tril().amax(dim=-1)                 # [heads, n]
    vmax = v.abs().amax(dim=(1, 2))[:, None]                                # [heads, 1]
    extra = ((1.0 + smax) * vmax).transpose(0, 1).repeat_interleave(d, dim=1)  # [n, C]
    return C_ATTN * U * (ref.abs() + extra)


def _attn_case(n, dt, gen):
    qkv, heads = _attn_operands(n, gen)
    qs = _seen(qkv, dt)
    ref = clip.causal_attention(qs, heads)
    return qkv, qs, ref, heads, _attn_bound(qs, ref, heads, dt)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("n", ATTN_N)
def test_causal_attention(n, dt):
    from genpercept_b200 import engine as E
    qkv, qs, ref, heads, bound = _attn_case(n, dt, torch.Generator().manual_seed(n))
    y = E.causal_attention(_arg(qkv, dt).cuda(), heads).double().cpu()
    _report(f"causal_attention {dt} n{n}", (y - ref).abs(), bound)


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("n", [n for n in ATTN_N if n > 1])
def test_bounds_discriminate_causal_attention(n, dt):
    _, qs, ref, heads, bound = _attn_case(n, dt, torch.Generator().manual_seed(n))
    wrong = [(v, (clip.causal_attention(qs, heads, v) - ref).abs()) for v in ("no_mask", "mask_off_by_one", "unscaled")]
    _discriminates(f"causal_attention {dt} n{n}", bound, wrong)


# ------------------------------------------------------------------------------------------------ GELU
def _gelu_case(dt, gen):
    x = torch.cat([torch.randn((77 * 4096 - 16,), generator=gen) * 3.0,
                   torch.tensor([0.0, -0.0, 1e-3, -1e-3, 8.0, -8.0, 12.0, -12.0, 0.5, -0.5, 3.0, -3.0, 5.5, -5.5, 1.0, -1.0])])
    xs = _seen(x, dt)
    ref = F.gelu(xs)
    if dt == "pair":
        bound = C_GELU * U * ref.abs() * (1.0 + xs * xs) + 2.0 ** -24
    else:
        bound = C16 * US[dt] * ref.abs() + 2.0 ** -24
    return x, xs, ref, bound


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DTYPES))
def test_gelu(dt):
    from genpercept_b200 import engine as E
    x, _, ref, bound = _gelu_case(dt, torch.Generator().manual_seed(7))
    y = E.gelu(_arg(x, dt).cuda()).double().cpu()
    _report(f"gelu {dt}", (y - ref).abs(), bound)


@pytest.mark.parametrize("dt", list(DTYPES))
def test_bounds_discriminate_gelu(dt):
    _, xs, ref, bound = _gelu_case(dt, torch.Generator().manual_seed(7))
    wrong = [("tanh_gelu", (F.gelu(xs, approximate="tanh") - ref).abs())]
    _discriminates(f"gelu {dt}", bound, wrong)


# ------------------------------------------------------------------------------------------------ the whole tower
@functools.lru_cache(maxsize=None)
def _tower_ref(n, variant=None):
    return clip.text_tower(_text_sd(), TOWER_CASES[n], variant=variant)[0]


def _tower_bound(ref, dt):
    c = C_TOWER_PAIR * U if dt == "pair" else C_TOWER16[dt] * US[dt]
    return torch.full_like(ref, c * ref.abs().max().item())


def _engine(dt, **kw):
    from genpercept_b200.engine import Engine
    return Engine(dtype=torch.bfloat16 if dt == "bf16" else torch.float16, precision="high" if dt == "pair" else "default", **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", list(DTYPES))
def test_tower(dt):
    e = _engine(dt)
    e.load_state("text", _text_sd())
    for n in TOWER_CASES:
        out = e.encode_text(TOWER_CASES[n])
        assert out.dtype == torch.float32 and tuple(out.shape) == (1, n, 1024)
        ref = _tower_ref(n)
        err = (out[0].double() - ref).abs()
        if dt == "pair":
            print(f"tower pair n{n}: max|err| / (u max|ref|) = {err.max().item() / (U * ref.abs().max().item()):.1f}")
        _report(f"tower {dt} n{n}", err, _tower_bound(ref, dt))
    e.close()


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("n", list(TOWER_CASES))
def test_bounds_discriminate_tower(n, dt):
    ref = _tower_ref(n)
    bound = _tower_bound(ref, dt)
    variants = ("positions_offset", "no_final_ln", "tanh_gelu")
    wrong = [(v, (_tower_ref(n, v) - ref).abs()) for v in variants]
    _discriminates(f"tower {dt} n{n}", bound, wrong, ("tanh_gelu",))


# ------------------------------------------------------------------------------------------------ pipeline
class _StubTokenizer:
    """CLIPTokenizer's call surface with fixed ids."""
    model_max_length = 77

    def __init__(self, ids):
        self.ids = ids

    def __call__(self, prompt, padding=None, max_length=None, truncation=None, return_tensors=None):
        assert padding == "do_not_pad" and return_tensors == "pt"
        return types.SimpleNamespace(input_ids=torch.tensor([self.ids]))


@pytest.mark.gpu
def test_pipeline_prompt_on_the_engine(synth_state):
    from genpercept_b200.pipeline import GenPerceptPipeline
    g = torch.Generator().manual_seed(3)
    img = torch.randint(0, 256, (1, 3, 64, 96), generator=g, dtype=torch.uint8)
    kw = dict(unet=synth_state["unet"], vae=synth_state["vae"], torch_dtype=torch.float16)
    call = dict(mode="depth", prompt="a high quality rgb image", processing_res=0)
    pipe = GenPerceptPipeline(text_encoder=_text_sd(), tokenizer=_StubTokenizer(PROMPT_IDS), **kw)
    got = pipe(img, **call)
    e = _engine("f16")
    e.load_state("text", _text_sd())
    embed = e.encode_text(PROMPT_IDS)
    e.close()
    want = GenPerceptPipeline(text_embed=embed, **kw)(img, **call)
    assert np.array_equal(got.pred_np, want.pred_np), "the prompt path differs from the same embedding passed in"
    ref = _tower_ref(7)
    _report("pipeline embedding f16", (pipe.text_embed[0].double() - ref).abs(), _tower_bound(ref, "f16"))
    with pytest.raises(RuntimeError):
        pipe.encode_text("another prompt")          # the context is folded in at the first call


# ------------------------------------------------------------------------------------------------ errors and lifetime
@pytest.mark.gpu
def test_errors_leave_the_engine_usable():
    import ctypes
    e = _engine("f16")
    st = lambda ids, n: e.L.gp_encode_text(e.h, (ctypes.c_int32 * max(len(ids), 1))(*ids), n,
                                           np.empty((max(n, 1), 1024), np.float32).ctypes.data_as(ctypes.c_void_p), None)
    assert st([49406, 49407], 2) == 2                                # GP_ERR_MISSING: no text weights
    sd = _text_sd()
    e.load_state("text", {k: v for k, v in sd.items() if "layers.22.mlp.fc2.bias" not in k})
    assert st([49406, 49407], 2) == 2                                # GP_ERR_MISSING: one tensor short
    e.load_state("text", {"text_model.encoder.layers.22.mlp.fc2.bias": sd["text_model.encoder.layers.22.mlp.fc2.bias"],
                          "text_model.embeddings.position_ids": torch.arange(77)[None]})
    good = e.encode_text([49406, 49407])
    assert st([49406, 49408], 2) == 1 and st([-1, 49407], 2) == 1     # GP_ERR_INVALID: ids outside the vocabulary
    assert st([], 0) == 1 and st([49406] * 78, 78) == 1                # GP_ERR_INVALID: n outside [1, 77]
    with pytest.raises(RuntimeError, match="GP_ERR_INVALID"):
        e.load_state("text", {"text_model.final_layer_norm.weight": torch.ones(768)})   # SD-1.x's width
    assert torch.equal(e.encode_text([49406, 49407]), good)
    e.close()


@pytest.mark.gpu
def test_finalize_returns_the_tower_memory(synth_state, text_embed):
    def engine():
        e = _engine("f16")
        e.load_state("unet", synth_state["unet"])
        e.load_state("vae", synth_state["vae"])
        e.set_text_embed(text_embed)
        return e

    free = lambda: (torch.cuda.synchronize(), torch.cuda.mem_get_info()[0])[1]
    plain = engine()
    f0 = free()
    plain.finalize()
    weights = f0 - free()
    plain.plan(1, 64, 64)
    info_plain = plain.plan_info()
    plain.close()

    e = engine()
    e.load_state("text", _text_sd())
    f0 = free()
    e.encode_text(PROMPT_IDS)
    tower = f0 - free()
    assert tower > 600 << 20, tower                     # 340M weights in fp16 plus the fp32 embedding tables
    e.finalize()
    returned = f0 - weights - free()
    print(f"tower {tower / 2**20:.0f} MiB, image weights {weights / 2**20:.0f} MiB, still held {returned / 2**20:.1f} MiB")
    assert returned < 64 << 20, returned
    with pytest.raises(RuntimeError, match="GP_ERR_STATE"):
        e.encode_text(PROMPT_IDS)
    e.plan(1, 64, 64)
    assert e.plan_info()["weight_bytes"] == info_plain["weight_bytes"]
    e.close()
