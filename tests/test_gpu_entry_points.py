"""The engine's run entry points (seeded synthetic weights, small shapes): every route to a result gives the same bits,
whether the result goes to a device or a host buffer, runs eagerly or replays a CUDA graph, starts from the image or from
its latent, or follows another plan or entry point; and each entry point reports a missing plan or the wrong arch with
its status code, leaving the engine usable."""
from ctypes import c_void_p

import numpy as np
import pytest
import torch

from genpercept_b200 import engine as E
from genpercept_b200 import weights as W
from genpercept_b200.scheduler import DDIMSchedule
from test_gpu_multitask import _engine, _rgb

pytestmark = pytest.mark.gpu

GP_ERR_INVALID, GP_ERR_NO_PLAN, GP_ERR_STATE = 1, 3, 5


def _host(shape):
    return torch.full(shape, float("nan"), dtype=torch.float32)


@pytest.mark.parametrize("cuda_graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("readout", ["vae", "dpt"])
def test_infer_and_infer_latent_into_device_and_host_out(synth_state, text_embed, readout, cuda_graph):
    e = _engine(synth_state, text_embed, readout=readout, cuda_graph=cuda_graph)
    try:
        B, H, W_ = 2, 64, 96
        x = _rgb(B, H, W_, 21)
        for C in ((1,) if readout == "dpt" else (1, 3)):
            def both(f, arg):
                # three passes each (the first eager, then graph replays when they are on), into device and host buffers
                res = [f(arg, out_channels=C).cpu().numpy() for _ in range(3)]
                for _ in range(3):
                    host = _host((B, C, H, W_))
                    assert f(arg, out_channels=C, out=host) is host
                    res.append(host.numpy())
                return res
            ref = e.infer(x, out_channels=C).cpu().numpy()
            assert 0.0 <= ref.min() and ref.max() <= 1.0 and ref.std() > 1e-3
            lat = e.encode_exact(x)
            got = both(e.infer, x) + both(e.infer_latent, lat)
            # interleaved in either order, neither route disturbs the other's buffers or graphs
            got += [e.infer_latent(lat, out_channels=C).cpu().numpy(), e.infer(x, out_channels=C).cpu().numpy(),
                    e.infer(x, out_channels=C).cpu().numpy(), e.infer_latent(lat, out_channels=C).cpu().numpy()]
            for i, r in enumerate(got):
                assert np.array_equal(r, ref), (readout, cuda_graph, C, i)
    finally:
        e.close()


def test_plan_switch_keeps_results_and_plan(synth_state, text_embed):
    e = _engine(synth_state, text_embed, cuda_graph=True)
    try:
        a, b = _rgb(1, 64, 96, 31), _rgb(1, 64, 128, 32)
        first = [e.infer(a).cpu().numpy() for _ in range(2)]
        info = e.plan_info()
        other = e.infer(b).cpu().numpy()
        assert other.shape == (1, 1, 64, 128)
        again = e.infer(a).cpu().numpy()
        assert np.array_equal(first[1], first[0]) and np.array_equal(again, first[0])
        after = e.plan_info()
        assert {k: after[k] for k in ("ops", "launches", "arena_bytes")} == \
            {k: info[k] for k in ("ops", "launches", "arena_bytes")}
        assert e.plan_count() == 2
    finally:
        e.close()


@pytest.mark.parametrize("arch", ["marigold", "rgb_blending"])
def test_infer_steps_device_and_host_buffers(text_embed, arch):
    blending = arch == "rgb_blending"
    state = W.synth_state(4321, with_dpt=False, unet_in_channels=4 if blending else 8)
    e = _engine(state, text_embed, arch="multistep")
    try:
        B, H, W_, C = 2, 64, 96, 3
        sched = DDIMSchedule(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                             set_alpha_to_one=False, steps_offset=1, prediction_type="v_prediction", timestep_spacing="leading")
        ts = [int(t) for t in sched.set_timesteps(2)]
        coeffs = [sched.step_coefficients(t) for t in ts]
        x = _rgb(B, H, W_, 41)
        noise = None if blending else torch.randn((B, 4, H // 8, W_ // 8), generator=torch.Generator().manual_seed(42))
        noises = [None] if blending else [noise, noise.cuda()]       # on the host, then on the device
        ref = None
        for nz in noises:
            dev = e.infer_steps(x, ts, coeffs, noise=nz, out_channels=C)
            host = _host((B, C, H, W_))
            assert e.infer_steps(x, ts, coeffs, noise=nz, out_channels=C, out=host) is host
            for r in (dev.cpu().numpy(), host.numpy()):
                if ref is None:
                    ref = r
                    assert tuple(ref.shape) == (B, C, H, W_) and np.isfinite(ref).all() and ref.std() > 1e-3
                assert np.array_equal(r, ref), (arch, nz is not None and nz.is_cuda)
    finally:
        e.close()


@pytest.mark.parametrize("mode", ["fp16", "high"])
def test_encode_and_encode_exact(synth_state, text_embed, mode):
    e = _engine(synth_state, text_embed, precision="high" if mode == "high" else "default")
    try:
        x = _rgb(2, 64, 96, 51)
        lat = e.encode(x).cpu()
        exact = e.encode_exact(x).cpu()
        assert tuple(lat.shape) == (2, 4, 8, 12)
        if mode == "high":      # the fp32 sum of each (hi, lo) pair
            assert tuple(exact.shape) == (2, 8, 8, 12)
            exact = exact[:, :4] + exact[:, 4:]
        assert np.array_equal(lat.numpy(), exact.numpy())
        assert lat.std() > 1e-3
    finally:
        e.close()


def test_infer_steps_rejects_a_wrong_out(text_embed):
    state = W.synth_state(4321, with_dpt=False, unet_in_channels=4)
    e = _engine(state, text_embed, arch="multistep")
    try:
        B, H, W_, C = 1, 64, 96, 1
        x = _rgb(B, H, W_, 61)
        e.plan(B, H, W_)
        for out in (torch.full((B, C, H + 8, W_), 7.0, device="cuda"), _host((B, C, H + 8, W_)).fill_(7.0)):
            with pytest.raises(AssertionError, match="out must be"):
                e.infer_steps(x, [999], [[1.0, 0.0, 1.0, 0.0]], out_channels=C, out=out)
            assert bool((out == 7.0).all())      # the library never saw the buffer
    finally:
        e.close()


def test_status_codes(synth_state, text_embed):
    L = E.lib()
    s = c_void_p(torch.cuda.current_stream().cuda_stream)
    rgb = torch.zeros((1, 3, 64, 96), dtype=torch.uint8, device="cuda")
    lat = torch.zeros((1, 4, 8, 12), device="cuda")
    out = torch.zeros((1, 1, 64, 96), device="cuda")
    p = lambda t: c_void_p(t.data_ptr())
    infer = lambda e: L.gp_infer(e.h, p(rgb), E.GP_U8, 0, p(out), 0, 1, s)
    infer_latent = lambda e: L.gp_infer_latent(e.h, p(lat), 1, 4, 8, 12, p(out), 0, 1, s)

    e = _engine(synth_state, text_embed)
    try:
        assert infer(e) == GP_ERR_NO_PLAN
        assert infer_latent(e) == GP_ERR_NO_PLAN
        assert L.gp_encode(e.h, p(rgb), E.GP_U8, 0, p(lat), s) == GP_ERR_NO_PLAN
        assert L.gp_encode_exact(e.h, p(rgb), E.GP_U8, 0, p(lat), s) == GP_ERR_NO_PLAN
        assert L.gp_decode(e.h, p(lat), 1, p(out), 1, s) == GP_ERR_NO_PLAN
        assert L.gp_run_stage(e.h, E.STAGE_READOUT, 1, s) == GP_ERR_NO_PLAN
        x = _rgb(1, 64, 96, 71)
        got = e.infer(x).cpu().numpy()
        assert got.shape == (1, 1, 64, 96) and np.isfinite(got).all() and got.std() > 1e-3
        assert np.array_equal(e.infer(x).cpu().numpy(), got)
    finally:
        e.close()

    m = _engine(W.synth_state(4321, with_dpt=False, unet_in_channels=8), text_embed, arch="multistep")
    try:
        assert infer_latent(m) == GP_ERR_INVALID
        m.plan(1, 64, 96)
        assert infer(m) == GP_ERR_STATE
        assert infer_latent(m) == GP_ERR_INVALID
    finally:
        m.close()
