"""gp_infer_steps on the caller's stream: per-step biases and DDIM coefficients travel to the device with the call, and with
CUDA graphs on, every call after the first of its (n_steps, noise, out_channels) replays one graph of the whole loop.

The maps of a replayed loop must equal those of a cuda_graph=False engine bit for bit, whatever the steps' timesteps
(nothing of a call may be baked into a graph), and a call must return without waiting for the device."""
import numpy as np
import pytest
import torch

from genpercept_b200 import weights as W
from genpercept_b200.engine import STAGE_UNET, Engine
from genpercept_b200.scheduler import DDIMSchedule

pytestmark = pytest.mark.gpu
SCHED = {"num_train_timesteps": 1000, "beta_start": 0.00085, "beta_end": 0.012, "beta_schedule": "scaled_linear",
         "clip_sample": False, "set_alpha_to_one": False, "steps_offset": 1, "prediction_type": "v_prediction",
         "timestep_spacing": "leading"}
ARCHS = ("marigold", "rgb_blending")
PRECISIONS = ("default", "high")
SHAPES = ((2, 64, 64), (1, 96, 128))
SLEEP_CYCLES = 100_000_000          # about 50-60 ms at the H100's 1.6-2.0 GHz SM clock


@pytest.fixture(scope="module")
def states():
    return {a: W.synth_state(4321, with_dpt=False, unet_in_channels=8 if a == "marigold" else 4) for a in ARCHS}


@pytest.fixture(scope="module")
def engines(states, text_embed):
    """make(arch, precision, graph, shared=False) -> a finalized multi-step engine, cached for the module."""
    made = {}

    def make(arch, precision, graph, shared=False):
        key = (arch, precision, graph, shared)
        if key not in made:
            e = Engine(dtype=torch.float16, precision=precision, arch="multistep", cuda_graph="auto" if graph else False,
                       shared_arena=shared)
            e.load_state("unet", states[arch]["unet"])
            e.load_state("vae", states[arch]["vae"])
            e.set_text_embed(text_embed)
            e.finalize()
            made[key] = e
        return made[key]

    yield make
    for e in made.values():
        e.close()


def _schedule(n, fix=None):
    s = DDIMSchedule(**SCHED)
    ts = [int(fix)] * n if fix else [int(t) for t in s.set_timesteps(n)]
    s.set_timesteps(n)
    return ts, [s.step_coefficients(t) for t in ts]


def _inputs(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    rgb = torch.randint(0, 256, (B, 3, H, W), generator=g, dtype=torch.uint8)
    noise = torch.randn((B, 4, H // 8, W // 8), generator=g)
    return rgb, noise


def _run(e, arch, rgb, noise, n, fix=None, noise_dev=True, out_dev=True, ch=1):
    ts, cf = _schedule(n, fix)
    nz = None
    if arch == "marigold":
        nz = noise.cuda() if noise_dev else noise
    out = None if out_dev else torch.empty((rgb.shape[0], ch) + tuple(rgb.shape[2:]), dtype=torch.float32)
    r = e.infer_steps(rgb.cuda(), ts, cf, noise=nz, out_channels=ch, out=out)
    if out_dev:
        torch.cuda.synchronize()
    return r.cpu().numpy()


# (n_steps, fix_timesteps, noise on the device, out on the device, out_channels)
CASES = ((1, None, False, True, 1), (3, None, True, False, 1), (10, None, True, True, 1), (3, 400, False, False, 3),
         (10, 250, True, True, 3))


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("arch", ARCHS)
def test_replayed_loop_matches_eager(arch, precision, shape, engines):
    eager, graph = engines(arch, precision, False), engines(arch, precision, True)
    rgb, noise = _inputs(*shape, seed=11)
    for n, fix, nd, od, ch in CASES:
        ref = _run(eager, arch, rgb, noise, n, fix, nd, od, ch)
        assert np.isfinite(ref).all() and ref.std() > 1e-4
        for call in range(3):       # eager, then captured and replayed, then replayed
            got = _run(graph, arch, rgb, noise, n, fix, nd, od, ch)
            assert np.array_equal(got, ref), f"n={n} fix={fix} call {call + 1}: max|diff| = {np.abs(got - ref).max():.3e}"


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("arch", ARCHS)
def test_interleaved_keys_keep_their_own_results(arch, precision, engines):
    """One graph per (n_steps, noise, out_channels), replayed with other timesteps and coefficients than its capture's."""
    eager, graph = engines(arch, precision, False), engines(arch, precision, True)
    rgb, noise = _inputs(2, 64, 64, seed=23)
    calls = [(3, None, 1), (10, None, 1), (3, 400, 1), (1, 700, 3), (3, 900, 3), (10, 100, 1), (3, None, 1), (1, None, 3),
             (3, 400, 1), (10, None, 1)]
    refs = {c: _run(eager, arch, rgb, noise, c[0], c[1], ch=c[2]) for c in set(calls)}
    for c in calls + calls:
        got = _run(graph, arch, rgb, noise, c[0], c[1], ch=c[2])
        assert np.array_equal(got, refs[c]), f"{c}: max|diff| = {np.abs(got - refs[c]).max():.3e}"
    assert not np.array_equal(refs[(3, None, 1)], refs[(3, 400, 1)])      # the timesteps do reach the maps


@pytest.mark.parametrize("arch", ARCHS)
def test_set_timestep_after_a_multistep_call(arch, engines):
    """After a call, the UNet holds the last step's timestep, and gp_set_timestep knows it."""
    eager, graph = engines(arch, "default", False), engines(arch, "default", True)
    rgb, noise = _inputs(2, 64, 64, seed=31)
    ref = _run(eager, arch, rgb, noise, 3)
    for _ in range(2):
        assert np.array_equal(_run(graph, arch, rgb, noise, 3), ref)      # last step at t = 1 (leading spacing, offset 1)
        _run(graph, arch, rgb, noise, 2, fix=600)                          # the bias buffers now hold t = 600
        graph.set_timestep(1)                                              # must re-upload: 600 is live, not 1
        graph.run_stage(STAGE_UNET)
        a = graph.read_tensor("noise_pred")
        graph.set_timestep(600)
        graph.set_timestep(1)
        graph.run_stage(STAGE_UNET)
        b = graph.read_tensor("noise_pred")
        assert np.array_equal(a, b)
        assert np.array_equal(_run(graph, arch, rgb, noise, 3), ref)


def _device_call(e, rgb, noise, ts, cf, out):
    e.infer_steps(rgb, ts, cf, noise=noise, out_channels=1, out=out)


def test_call_returns_while_another_stream_sleeps(engines):
    """No device-wide synchronisation: a call on stream A does not wait for stream B's queued work."""
    e, eager = engines("marigold", "default", True), engines("marigold", "default", False)
    rgb, noise = _inputs(2, 64, 64, seed=41)
    ref = _run(eager, "marigold", rgb, noise, 3)
    ts, cf = _schedule(3)
    rgb_d, noise_d = rgb.cuda(), noise.cuda()
    out = torch.empty((2, 1, 64, 64), dtype=torch.float32, device="cuda")
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(a):
        for _ in range(2):                       # the first pass of the key runs eagerly, the second captures
            _device_call(e, rgb_d, noise_d, ts, cf, out)
    torch.cuda.synchronize()
    with torch.cuda.stream(b):
        torch.cuda._sleep(SLEEP_CYCLES)
    with torch.cuda.stream(a):
        _device_call(e, rgb_d, noise_d, ts, cf, out)
    busy = not b.query()
    torch.cuda.synchronize()
    assert busy, "the call waited for another stream's work"
    assert np.array_equal(out.cpu().numpy(), ref)


def test_call_returns_before_its_own_stream_completes(engines):
    """Asynchronous on its stream: with a sleep queued ahead of it, the call returns before the stream drains."""
    e, eager = engines("rgb_blending", "default", True), engines("rgb_blending", "default", False)
    rgb, noise = _inputs(2, 64, 64, seed=43)
    ref = _run(eager, "rgb_blending", rgb, noise, 3)
    ts, cf = _schedule(3)
    rgb_d = rgb.cuda()
    out = torch.empty((2, 1, 64, 64), dtype=torch.float32, device="cuda")
    a = torch.cuda.Stream()
    with torch.cuda.stream(a):
        for _ in range(2):
            _device_call(e, rgb_d, None, ts, cf, out)
    torch.cuda.synchronize()
    with torch.cuda.stream(a):
        torch.cuda._sleep(SLEEP_CYCLES)
        _device_call(e, rgb_d, None, ts, cf, out)
    busy = not a.query()
    torch.cuda.synchronize()
    assert busy, "the call waited for its stream"
    assert np.array_equal(out.cpu().numpy(), ref)


def test_shared_arena_engines_on_two_streams(engines):
    """A multi-step engine and a second shared-arena engine on another stream take turns in the pool: the maps equal
    those of engines with private arenas."""
    m_priv, r_priv = engines("marigold", "default", True), engines("rgb_blending", "default", True)
    m, r = engines("marigold", "default", True, shared=True), engines("rgb_blending", "default", True, shared=True)
    rgb, noise = _inputs(2, 64, 64, seed=53)
    rgb2, _ = _inputs(1, 96, 128, seed=59)
    ts3, cf3 = _schedule(3)
    ts2, cf2 = _schedule(2, fix=500)
    ref_m = _run(m_priv, "marigold", rgb, noise, 3)
    ref_r = _run(r_priv, "rgb_blending", rgb2, None, 2, fix=500)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    rgb_d, noise_d, rgb2_d = rgb.cuda(), noise.cuda(), rgb2.cuda()
    outs = []
    for _ in range(4):
        om = torch.empty((2, 1, 64, 64), dtype=torch.float32, device="cuda")
        orr = torch.empty((1, 1, 96, 128), dtype=torch.float32, device="cuda")
        with torch.cuda.stream(sa):
            m.infer_steps(rgb_d, ts3, cf3, noise=noise_d, out_channels=1, out=om)
        with torch.cuda.stream(sb):
            r.infer_steps(rgb2_d, ts2, cf2, noise=None, out_channels=1, out=orr)
        outs.append((om, orr))
    torch.cuda.synchronize()
    for om, orr in outs:
        assert np.array_equal(om.cpu().numpy(), ref_m)
        assert np.array_equal(orr.cpu().numpy(), ref_r)
