"""SD-2.1's CLIP text tower (transformers' CLIPTextModel with SD-2.1's text_encoder config, SURVEY.md App. A) restated in
plain PyTorch on the CPU, for the tests only: token + position embedding, 23 pre-LN layers of causal self-attention (16
heads of 64) and an exact-erf GELU MLP (4096), final LayerNorm; LN eps 1e-5.  The input is a token id sequence without
padding (the reference tokenizes with padding='do_not_pad'), so the causal mask is the only mask.

`variant` builds the plausible wrong towers the discrimination tests measure the bounds against:
  "no_mask"           every key visible
  "mask_off_by_one"   key j visible for j <= i + 1
  "unscaled"          the softmax scale 1/8 never applied to the scores
  "positions_offset"  position row t + 1 (mod 77) added to token t
  "no_final_ln"       last_hidden_state before final_layer_norm
  "tanh_gelu"         the tanh approximation of GELU
"""
import torch
import torch.nn.functional as F

LAYERS, HEADS, DIM = 23, 16, 1024
EPS = 1e-5
PREFIX = "text_model."


def causal_attention(qkv, heads, variant=None):
    """qkv [n, 3C] = per token [q | k | v], the softmax scale already in q -> [n, C]: softmax(q k^T) v per head over keys
    j <= i, in qkv's dtype."""
    n, c3 = qkv.shape
    C = c3 // 3
    d = C // heads
    q, k, v = (t.reshape(n, heads, d).transpose(0, 1) for t in qkv.split(C, dim=-1))
    if variant == "unscaled":
        q = q * d ** 0.5
    s = q @ k.transpose(1, 2)
    i = torch.arange(n)[:, None]
    j = torch.arange(n)[None, :]
    keep = {"no_mask": torch.ones(n, n, dtype=torch.bool), "mask_off_by_one": j <= i + 1}.get(variant, j <= i)
    p = torch.softmax(s.masked_fill(~keep, float("-inf")), dim=-1)
    return (p @ v).transpose(0, 1).reshape(n, C)


def gelu(x, variant=None):
    return F.gelu(x, approximate="tanh" if variant == "tanh_gelu" else "none")


def text_tower(sd, ids, dtype=torch.float64, variant=None):
    """last_hidden_state [1, n, 1024] of CLIPTextModel with state dict `sd` (its own keys, "text_model. ...") for the token
    ids `ids` (n <= 77), computed in `dtype`."""
    ids = torch.as_tensor(ids).reshape(-1).long()
    n = ids.numel()
    w = lambda k: sd[PREFIX + k].to(dtype)
    pos_rows = torch.arange(n)
    if variant == "positions_offset":
        pos_rows = (pos_rows + 1) % sd[PREFIX + "embeddings.position_embedding.weight"].shape[0]
    x = sd[PREFIX + "embeddings.token_embedding.weight"][ids].to(dtype) + w("embeddings.position_embedding.weight")[pos_rows]
    scale = (DIM // HEADS) ** -0.5
    for li in range(LAYERS):
        p = f"encoder.layers.{li}."
        h = F.layer_norm(x, (DIM,), w(p + "layer_norm1.weight"), w(p + "layer_norm1.bias"), EPS)
        q, k, v = (F.linear(h, w(f"{p}self_attn.{m}.weight"), w(f"{p}self_attn.{m}.bias")) for m in ("q_proj", "k_proj", "v_proj"))
        a = causal_attention(torch.cat([q * scale, k, v], dim=-1), HEADS, variant)
        x = x + F.linear(a, w(p + "self_attn.out_proj.weight"), w(p + "self_attn.out_proj.bias"))
        h = F.layer_norm(x, (DIM,), w(p + "layer_norm2.weight"), w(p + "layer_norm2.bias"), EPS)
        h = gelu(F.linear(h, w(p + "mlp.fc1.weight"), w(p + "mlp.fc1.bias")), variant)
        x = x + F.linear(h, w(p + "mlp.fc2.weight"), w(p + "mlp.fc2.bias"))
    if variant != "no_final_ln":
        x = F.layer_norm(x, (DIM,), w("final_layer_norm.weight"), w("final_layer_norm.bias"), EPS)
    return x[None]
