"""One VAE encode for several tasks (seeded synthetic weights): Engine.encode_exact -> Engine.infer_latent gives
gp_infer's maps bit for bit in every storage mode and readout, eagerly and through CUDA graphs, and MultiTaskPipeline
gives each task's own GenPerceptPipeline.__call__ output from one encode."""
import numpy as np
import pytest
import torch
from PIL import Image

from genpercept_b200 import weights as W
from genpercept_b200.engine import Engine
from genpercept_b200.multitask import MultiTaskPipeline
from genpercept_b200.pipeline import GenPerceptPipeline

pytestmark = pytest.mark.gpu

SHAPES = [(1, 64, 64), (1, 200, 328), (3, 64, 64)]
# fp16 runs before bf16 in one process: the large-shared-memory kernels' attributes must hold for both storage types
MODES = {"fp16": (torch.float16, "default"), "bf16": (torch.bfloat16, "default"), "high": (torch.float16, "high")}


def _engine(state, te, dtype=torch.float16, precision="default", readout="vae", cuda_graph=False, arch="genpercept",
            unet=None):
    e = Engine(dtype=dtype, readout=readout, precision=precision, cuda_graph=cuda_graph, arch=arch)
    e.load_state("unet", unet if unet is not None else state["unet"])
    e.load_state("vae", state["vae"])
    if readout == "dpt":
        e.load_state("dpt", state["dpt"])
    e.set_text_embed(te)
    e.finalize()
    return e


def _rgb(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (B, 3, H, W), generator=g, dtype=torch.uint8).cuda()


@pytest.mark.parametrize("cuda_graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("readout", ["vae", "dpt"])
@pytest.mark.parametrize("mode", list(MODES))
def test_infer_latent_equals_infer(synth_state, text_embed, mode, readout, cuda_graph):
    dtype, precision = MODES[mode]
    e = _engine(synth_state, text_embed, dtype, precision, readout, cuda_graph)
    try:
        for i, (B, H, W) in enumerate(SHAPES):
            x = _rgb(B, H, W, 100 + i)
            for C in ((1,) if readout == "dpt" else (1, 3)):
                # twice each: the first pass runs eagerly, the second replays the graphs when they are on
                ref = [e.infer(x, out_channels=C).cpu().numpy() for _ in range(2)]
                lat = e.encode_exact(x)
                assert tuple(lat.shape) == (B, 8 if precision == "high" else 4, H // 8, W // 8)
                got = [e.infer_latent(lat, out_channels=C).cpu().numpy() for _ in range(2)]
                again = e.infer(x, out_channels=C).cpu().numpy()     # the full graph is left as it was
                for r in ref[1:] + got + [again]:
                    assert np.array_equal(r, ref[0]), (mode, readout, cuda_graph, (B, H, W), C)
                assert 0.0 <= ref[0].min() and ref[0].max() <= 1.0 and ref[0].std() > 1e-3
    finally:
        e.close()


def test_infer_latent_from_another_engine(synth_state, text_embed):
    """The hand-off between engines: a latent encoded by a DPT engine drives a VAE-readout engine's UNet."""
    a = _engine(synth_state, text_embed, readout="dpt")
    b = _engine(synth_state, text_embed, readout="vae")
    try:
        x = _rgb(2, 96, 160, 7)
        lat = a.encode_exact(x)
        b.plan(2, 96, 160)
        assert np.array_equal(b.infer_latent(lat, out_channels=3).cpu().numpy(), b.infer(x, out_channels=3).cpu().numpy())
        host = torch.empty((2, 3, 96, 160), dtype=torch.float32)
        b.infer_latent(lat, out_channels=3, out=host)
        assert np.array_equal(host.numpy(), b.infer(x, out_channels=3).cpu().numpy())
    finally:
        a.close()
        b.close()


@pytest.fixture(scope="module")
def task_unets():
    return {"depth": W.synth_unet(11), "normal": W.synth_unet(12), "disparity": W.synth_unet(13)}


@pytest.mark.parametrize("mode", ["fp16", "high"])
def test_multitask_pipeline_equals_each_task(synth_state, text_embed, task_unets, mode, monkeypatch):
    dtype = torch.float32 if mode == "high" else torch.float16
    vae = synth_state["vae"]
    pipes = {
        "depth": GenPerceptPipeline(unet=task_unets["depth"], vae=vae, text_embed=text_embed, torch_dtype=dtype),
        "normal": GenPerceptPipeline(unet=task_unets["normal"], vae=vae, text_embed=text_embed, torch_dtype=dtype),
        "disparity": GenPerceptPipeline(unet=task_unets["disparity"], vae=vae, customized_head=synth_state["dpt"],
                                        text_embed=text_embed, torch_dtype=dtype),
    }
    modes = {"depth": "depth", "normal": "normal", "disparity": "disparity"}
    mt = MultiTaskPipeline(pipes, modes)
    g = np.random.default_rng(5)
    inputs = [
        (Image.fromarray(g.integers(0, 256, (77, 101, 3), dtype=np.uint8)), dict(processing_res=96)),   # odd-sized PIL
        (torch.from_numpy(g.integers(0, 256, (2, 3, 64, 96), dtype=np.uint8)), dict(processing_res=0)),  # batched uint8
        (torch.from_numpy(g.integers(0, 256, (1, 3, 80, 120), dtype=np.uint8)).cuda(),
         dict(processing_res=64, resample_method="bicubic")),
    ]
    calls = []
    for meth in ("encode", "encode_exact", "infer", "infer_latent"):
        def counted(self, *a, _f=getattr(Engine, meth), _m=meth, **k):
            calls.append((_m, self))
            return _f(self, *a, **k)
        monkeypatch.setattr(Engine, meth, counted)
    try:
        for img, kw in inputs:
            calls.clear()
            res = mt(img, **kw)
            # one encode on the first task's engine, then each engine from the UNet on: no full pass
            assert calls == [("encode_exact", pipes["depth"]._engine)] + [("infer_latent", p._engine) for p in pipes.values()]
            assert set(res) == set(pipes)
            maps = {}
            for name, p in pipes.items():
                cm = "Spectral" if modes[name] != "normal" else None
                own = p(img, mode=modes[name], color_map=cm, **kw)
                got = res[name]
                assert np.array_equal(got.pred_np, own.pred_np), (name, kw)
                gc = got.pred_colored if isinstance(got.pred_colored, list) else [got.pred_colored]
                oc = own.pred_colored if isinstance(own.pred_colored, list) else [own.pred_colored]
                assert len(gc) == len(oc)
                for a, b in zip(gc, oc):
                    assert np.array_equal(np.asarray(a), np.asarray(b)), (name, kw)
                maps[name] = got.pred_np
            if isinstance(img, Image.Image):
                assert maps["depth"].shape == (77, 101) and maps["normal"].shape == (77, 101, 3)
            assert not np.array_equal(maps["depth"], maps["disparity"])      # the tasks' own UNets ran
    finally:
        for p in pipes.values():
            p._engine.close()


def test_multitask_pipeline_rejects_different_encoders(synth_state, text_embed, task_unets):
    vae2 = dict(synth_state["vae"])
    vae2["encoder.conv_in.bias"] = vae2["encoder.conv_in.bias"] + 0.5
    a = GenPerceptPipeline(unet=task_unets["depth"], vae=synth_state["vae"], text_embed=text_embed)
    b = GenPerceptPipeline(unet=task_unets["normal"], vae=vae2, text_embed=text_embed)
    try:
        with pytest.raises(ValueError, match=r"'normal'.*vae\.encoder\.conv_in\.bias"):
            MultiTaskPipeline({"depth": a, "normal": b}, {"depth": "depth", "normal": "normal"})
    finally:
        a._engine.close()
        b._engine.close()


def test_infer_latent_errors_leave_the_engine_usable(synth_state, text_embed):
    x = _rgb(1, 64, 96, 3)
    e = _engine(synth_state, text_embed)
    try:
        with pytest.raises(RuntimeError, match="GP_ERR_NO_PLAN"):
            e.infer_latent(torch.zeros((1, 4, 8, 12), device="cuda"))
        lat = e.encode_exact(x)
        ref = e.infer(x).cpu().numpy()
        for bad in (lat[:, :, :7], lat[:, :, :, :11].contiguous(), torch.cat([lat, lat]), lat.repeat(1, 2, 1, 1)):
            with pytest.raises(RuntimeError, match="GP_ERR_INVALID"):
                e.infer_latent(bad)
        assert np.array_equal(e.infer(x).cpu().numpy(), ref)
        assert np.array_equal(e.infer_latent(lat).cpu().numpy(), ref)
    finally:
        e.close()
    h = _engine(synth_state, text_embed, precision="high")
    try:
        ref = h.infer(x).cpu().numpy()
        with pytest.raises(RuntimeError, match="GP_ERR_INVALID"):      # gp_encode's fp32 sum is not the (hi, lo) pair
            h.infer_latent(h.encode(x))
        assert np.array_equal(h.infer(x).cpu().numpy(), ref)
    finally:
        h.close()
    m = _engine(synth_state, text_embed, arch="multistep")
    try:
        m.plan(1, 64, 96)
        with pytest.raises(RuntimeError, match="GP_ERR_INVALID"):
            m.infer_latent(torch.zeros((1, 4, 8, 12), device="cuda"))
        out = m.infer_steps(x, [999], [[1.0, 0.0, 1.0, 0.0]])
        assert out.shape == (1, 1, 64, 96) and torch.isfinite(out).all()
    finally:
        m.close()
