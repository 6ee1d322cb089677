"""The shared activation arena (seeded synthetic weights): engines that take their plans' arenas from the device's one
pool give the bits of engines with arenas of their own, through every run entry point, whatever another engine did to
the pool in between (a larger plan that grows it, a byte pattern written over it, work on another stream), and the pool
maps the largest arena among its plans, not the sum."""
import numpy as np
import pytest
import torch
from PIL import Image

from genpercept_b200 import engine as E
from genpercept_b200 import weights as W
from genpercept_b200.multitask import MultiTaskPipeline
from genpercept_b200.pipeline import GenPerceptPipeline
from genpercept_b200.scheduler import DDIMSchedule
from test_gpu_multitask import _engine, _rgb

pytestmark = pytest.mark.gpu

GRAN = 2 << 20          # the H100's minimum allocation granularity for device memory
FILLS = (None, 0xFF, 0x00)   # 0xFF is a NaN in fp16 and bf16: any op that reads a byte it did not write shows it


def _shared(state, te, **kw):
    e = _engine(state, te, **kw)
    e.set_shared_arena(True)
    return e


def _fill(byte):
    if byte is not None:
        E.shared_arena_fill(byte)


def _one_step_calls(e, x, readout, fill):
    """Every one-step entry point twice (eager, then a graph replay where graphs are on), into device and host buffers,
    with `fill` written over the pool before each call.  -> list of numpy results."""
    B, _, H, W_ = x.shape
    res = []
    for C in ((1,) if readout == "dpt" else (1, 3)):
        for _ in range(2):
            _fill(fill)
            res.append(e.infer(x, out_channels=C).cpu().numpy())
            _fill(fill)
            host = torch.empty((B, C, H, W_), dtype=torch.float32)
            res.append(e.infer(x, out_channels=C, out=host).numpy())
        for _ in range(2):
            _fill(fill)
            lat = e.encode_exact(x)
            res.append(lat.cpu().numpy())
            _fill(fill)
            res.append(e.infer_latent(lat, out_channels=C).cpu().numpy())
            _fill(fill)
            host = torch.empty((B, C, H, W_), dtype=torch.float32)
            res.append(e.infer_latent(lat, out_channels=C, out=host).numpy())
        if readout == "vae":
            _fill(fill)
            z = e.encode(x)
            res.append(z.cpu().numpy())
            _fill(fill)
            res.append(e.decode(z, out_channels=C).cpu().numpy())
            e.plan(B, H, W_)
    return res


@pytest.mark.parametrize("cuda_graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("readout", ["vae", "dpt"])
@pytest.mark.parametrize("mode", ["fp16", "high"])
def test_one_step_entry_points_equal_private_arena(synth_state, text_embed, mode, readout, cuda_graph):
    kw = dict(readout=readout, cuda_graph=cuda_graph, precision="high" if mode == "high" else "default")
    ref_e = _engine(synth_state, text_embed, **kw)
    e = _shared(synth_state, text_embed, **kw)
    try:
        if mode == "high":
            ref_e.set_memory_efficient_attention(True)
            e.set_memory_efficient_attention(True)
        x = _rgb(2, 64, 96, 11)
        ref = _one_step_calls(ref_e, x, readout, None)
        assert all(np.isfinite(r).all() for r in ref) and ref[0].std() > 1e-3
        for fill in FILLS:
            got = _one_step_calls(e, x, readout, fill)
            for i, (a, b) in enumerate(zip(ref, got)):
                assert np.array_equal(a, b), (mode, readout, cuda_graph, fill, i)
        assert E.shared_arena_info()["live_plans"] == e.plan_count()
    finally:
        ref_e.close()
        e.close()
    assert E.shared_arena_info()["mapped_bytes"] == 0


@pytest.mark.parametrize("mode", ["fp16", "high"])
@pytest.mark.parametrize("arch", ["marigold", "rgb_blending"])
def test_infer_steps_equals_private_arena(text_embed, arch, mode):
    blending = arch == "rgb_blending"
    state = W.synth_state(4321, with_dpt=False, unet_in_channels=4 if blending else 8)
    kw = dict(arch="multistep", precision="high" if mode == "high" else "default")
    ref_e = _engine(state, text_embed, **kw)
    e = _shared(state, text_embed, **kw)
    try:
        B, H, W_, C = 2, 64, 96, 3
        sched = DDIMSchedule(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                             set_alpha_to_one=False, steps_offset=1, prediction_type="v_prediction", timestep_spacing="leading")
        ts = [int(t) for t in sched.set_timesteps(2)]
        coeffs = [sched.step_coefficients(t) for t in ts]
        x = _rgb(B, H, W_, 41)
        noise = None if blending else torch.randn((B, 4, H // 8, W_ // 8), generator=torch.Generator().manual_seed(42))
        ref = ref_e.infer_steps(x, ts, coeffs, noise=noise, out_channels=C).cpu().numpy()
        assert np.isfinite(ref).all() and ref.std() > 1e-3
        for fill in FILLS:
            _fill(fill)
            assert np.array_equal(e.infer_steps(x, ts, coeffs, noise=noise, out_channels=C).cpu().numpy(), ref), fill
            _fill(fill)
            host = torch.empty((B, C, H, W_), dtype=torch.float32)
            assert np.array_equal(e.infer_steps(x, ts, coeffs, noise=noise, out_channels=C, out=host).numpy(), ref), fill
    finally:
        ref_e.close()
        e.close()


def test_growth_keeps_graphs_captured_before_it(synth_state, text_embed):
    pa = _engine(synth_state, text_embed, cuda_graph=True)
    pb = _engine(synth_state, text_embed, readout="dpt", cuda_graph=True)
    a = _shared(synth_state, text_embed, cuda_graph=True)
    b = _shared(synth_state, text_embed, readout="dpt", cuda_graph=True)
    try:
        xa, xb = _rgb(1, 64, 96, 21), _rgb(1, 256, 256, 22)
        ref_a, ref_b = pa.infer(xa, out_channels=3).cpu().numpy(), pb.infer(xb).cpu().numpy()
        got = [a.infer(xa, out_channels=3).cpu().numpy() for _ in range(2)]      # eager, then the captured graph
        small = E.shared_arena_info()["mapped_bytes"]
        got_b = [b.infer(xb).cpu().numpy() for _ in range(2)]
        assert E.shared_arena_info()["mapped_bytes"] > small                     # B's plan grew the pool
        got += [a.infer(xa, out_channels=3).cpu().numpy() for _ in range(2)]     # A's graph from before the growth
        for r in got:
            assert np.array_equal(r, ref_a)
        for r in got_b:
            assert np.array_equal(r, ref_b)
    finally:
        for e in (pa, pb, a, b):
            e.close()


def test_engines_on_two_streams_without_host_sync(synth_state, text_embed):
    a = _shared(synth_state, text_embed)
    b = _shared(synth_state, text_embed, readout="dpt")
    try:
        xa, xb = _rgb(2, 128, 192, 31), _rgb(2, 192, 128, 32)
        ref_a, ref_b = a.infer(xa, out_channels=3).clone(), b.infer(xb).clone()
        outs_a = [torch.empty_like(ref_a) for _ in range(3)]
        outs_b = [torch.empty_like(ref_b) for _ in range(3)]
        sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
        torch.cuda.synchronize()
        for oa, ob in zip(outs_a, outs_b):
            with torch.cuda.stream(sa):
                a.infer(xa, out_channels=3, out=oa)
            with torch.cuda.stream(sb):
                b.infer(xb, out=ob)
        torch.cuda.synchronize()
        for oa, ob in zip(outs_a, outs_b):
            assert torch.equal(oa, ref_a) and torch.equal(ob, ref_b)
    finally:
        a.close()
        b.close()


def _round(n):
    return (n + GRAN - 1) // GRAN * GRAN


def test_pool_maps_the_largest_arena_and_gives_everything_back(synth_state, text_embed):
    warm = _engine(synth_state, text_embed)      # loads the library's kernels before the baseline is taken
    warm.infer(_rgb(1, 64, 64, 1))
    warm.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    shapes = [(1, 128, 128), (4, 512, 512), (2, 256, 256)]
    engines = [_shared(synth_state, text_embed) for _ in shapes]
    try:
        sizes = []
        for e, (B, H, W_) in zip(engines, shapes):
            e.infer(_rgb(B, H, W_, 41))
            sizes.append(e.plan_info()["arena_bytes"])
        info = E.shared_arena_info()
        assert info["mapped_bytes"] == _round(max(sizes)) < sum(sizes)
        assert info["live_plans"] == 3 and info["reserved_bytes"] >= torch.cuda.mem_get_info()[1]
        engines[1].set_shared_arena(False)                     # the largest plan leaves: the pool shrinks
        assert engines[1].plan_count() == 0
        assert E.shared_arena_info()["mapped_bytes"] == _round(max(sizes[0], sizes[2]))
        engines[1].set_shared_arena(True)
        one = engines[0]
        sizes = []
        for B, H, W_ in [(1, 64, 64), (2, 256, 256), (1, 128, 192), (4, 512, 512)]:    # four cached plans in one engine
            one.infer(_rgb(B, H, W_, 42))
            sizes.append(one.plan_info()["arena_bytes"])
        assert one.plan_count() == 4
        assert E.shared_arena_info()["mapped_bytes"] == _round(max(sizes + [engines[2].plan_info()["arena_bytes"]]))
    finally:
        for e in engines:
            e.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    assert E.shared_arena_info() == {"mapped_bytes": 0, "reserved_bytes": 0, "live_plans": 0}
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 64 << 20


def test_toggle_drops_plans_and_keeps_bits(synth_state, text_embed):
    e = _engine(synth_state, text_embed, cuda_graph=True)
    try:
        x = _rgb(1, 64, 96, 51)
        ref = e.infer(x).cpu().numpy()
        for flag in (True, False, True):
            e.set_shared_arena(flag)
            assert e.plan_count() == 0
            assert E.shared_arena_info()["live_plans"] == 0
            for _ in range(2):
                assert np.array_equal(e.infer(x).cpu().numpy(), ref), flag
            assert E.shared_arena_info()["live_plans"] == (1 if flag else 0)
    finally:
        e.close()


def test_multitask_native_resolution_high_precision(synth_state, text_embed):
    """Three tasks on a 4032 x 3024 photo in the high-precision mode with memory-efficient attention: 33.7 GiB of arena
    each, so only a shared arena holds all three plans on an 80 GB card."""
    vae = synth_state["vae"]
    pipes = {
        "depth": GenPerceptPipeline(unet=W.synth_unet(11), vae=vae, text_embed=text_embed, torch_dtype=torch.float32),
        "normal": GenPerceptPipeline(unet=W.synth_unet(12), vae=vae, text_embed=text_embed, torch_dtype=torch.float32),
        "disparity": GenPerceptPipeline(unet=W.synth_unet(13), vae=vae, customized_head=synth_state["dpt"],
                                        text_embed=text_embed, torch_dtype=torch.float32),
    }
    for p in pipes.values():
        p.enable_xformers_memory_efficient_attention()
    modes = {"depth": "depth", "normal": "normal", "disparity": "disparity"}
    try:
        mt = MultiTaskPipeline(pipes, modes, share_arena=True)
        img = Image.fromarray(np.random.default_rng(9).integers(0, 256, (3024, 4032, 3), dtype=np.uint8))
        res = mt(img, processing_res=0, color_map=None)
        assert E.shared_arena_info()["live_plans"] == 3
        for name, p in pipes.items():
            own = p(img, mode=modes[name], processing_res=0, color_map=None)
            assert res[name].pred_np.shape[:2] == (3024, 4032)
            assert np.array_equal(res[name].pred_np, own.pred_np), name
    finally:
        for p in pipes.values():
            p._engine.close()
