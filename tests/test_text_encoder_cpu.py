"""CPU tests of the text tower's host side: oracle/clip.py against transformers' CLIPTextModel, and from_pretrained
reading an SD-2.1 folder's text_encoder/ as weights for the engine without building a CLIPTextModel."""
import functools
import os
import types

import pytest
import torch

from oracle import clip

IDS = {2: [49406, 49407], 7: [49406, 320, 1205, 3027, 12875, 2867, 49407],
       77: [49406] + [(1000 + 613 * i) % 49408 for i in range(75)] + [49407]}


@functools.lru_cache(maxsize=1)
def _text_sd():
    from genpercept_b200 import weights as W
    return W.synth_text_state(1234)


def test_synth_text_state_has_sd21_shapes():
    from genpercept_b200 import weights as W
    sd = _text_sd()
    assert list(sd) == list(W.text_spec())
    assert tuple(sd["text_model.embeddings.token_embedding.weight"].shape) == (49408, 1024)
    assert tuple(sd["text_model.encoder.layers.22.mlp.fc1.weight"].shape) == (4096, 1024)
    assert not any(".layers.23." in k for k in sd)
    assert W.param_count(W.text_spec()) == sum(v.numel() for v in sd.values())


@pytest.mark.parametrize("n", list(IDS))
def test_oracle_matches_transformers_clip_text_model(n):
    transformers = pytest.importorskip("transformers")
    cfg = transformers.CLIPTextConfig(vocab_size=49408, hidden_size=1024, intermediate_size=4096, num_hidden_layers=23,
                                      num_attention_heads=16, max_position_embeddings=77, hidden_act="gelu",
                                      layer_norm_eps=1e-5, projection_dim=512)
    model = transformers.CLIPTextModel(cfg).eval()
    missing, unexpected = model.load_state_dict(_text_sd(), strict=False)
    assert not unexpected and all(k.endswith("position_ids") for k in missing)
    with torch.no_grad():
        hf = model(torch.tensor([IDS[n]])).last_hidden_state.double()
    ref = clip.text_tower(_text_sd(), IDS[n])
    rel = (hf - ref).abs().max().item() / ref.abs().max().item()
    print(f"n = {n}: max|transformers - oracle| / max|oracle| = {rel:.2e}")
    assert rel < 2e-6, rel          # fp32 against fp64 over 23 layers: 5.6e-7 measured


class _RecordingEngine:
    """Stands in for the native engine: records what the pipeline loads."""
    loaded = {}

    def __init__(self, *a, **k):
        self.device = torch.device("cpu")

    def load_state(self, component, sd):
        _RecordingEngine.loaded[component] = dict(sd)

    def set_text_embed(self, e):
        pass


def test_from_pretrained_reads_the_text_encoder_folder(tmp_path, monkeypatch):
    from safetensors.torch import save_file
    from genpercept_b200 import pipeline as P
    transformers = pytest.importorskip("transformers")

    def no_model(*a, **k):
        raise AssertionError("CLIPTextModel must not be constructed")

    monkeypatch.setattr(transformers, "CLIPTextModel", types.SimpleNamespace(from_pretrained=no_model, __call__=no_model))
    monkeypatch.setattr(P, "Engine", _RecordingEngine)
    _RecordingEngine.loaded = {}
    sd = {k: v.half() for k, v in list(_text_sd().items())[:6]}       # any text_model.* tensors: the file is read as is
    os.makedirs(tmp_path / "text_encoder")
    save_file({k: v.contiguous() for k, v in sd.items()}, str(tmp_path / "text_encoder" / "model.fp16.safetensors"))
    save_file({"text_model.final_layer_norm.weight": torch.ones(1024)}, str(tmp_path / "text_encoder" / "model.safetensors"))
    tok = types.SimpleNamespace(model_max_length=77)
    pipe = P.GenPerceptPipeline.from_pretrained(str(tmp_path), variant="fp16", unet={}, vae={}, tokenizer=tok)
    assert set(_RecordingEngine.loaded["text"]) == set(sd)
    assert all(torch.equal(_RecordingEngine.loaded["text"][k], v) for k, v in sd.items())
    assert pipe.tokenizer is tok and pipe.text_embed is None

    _RecordingEngine.loaded = {}
    P.GenPerceptPipeline.from_pretrained(str(tmp_path), unet={}, vae={}, tokenizer=tok)
    assert list(_RecordingEngine.loaded["text"]) == ["text_model.final_layer_norm.weight"]

    _RecordingEngine.loaded = {}
    P.GenPerceptPipeline.from_pretrained(str(tmp_path), unet={}, vae={}, text_embed=torch.zeros(1, 2, 1024))
    assert "text" not in _RecordingEngine.loaded                     # text_embed= takes precedence


def test_encode_text_without_weights_keeps_its_error(monkeypatch):
    from genpercept_b200 import pipeline as P
    monkeypatch.setattr(P, "Engine", _RecordingEngine)
    pipe = P.GenPerceptPipeline(unet={}, vae={})
    with pytest.raises(RuntimeError, match="no text_encoder/tokenizer given"):
        pipe.encode_text("")
