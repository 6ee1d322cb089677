"""The GPU baseline-JPEG decoder (engine.decode_jpeg) against Pillow's own bytes, its rejection of corrupt streams,
and the pipelines' use of it for unloaded JPEGs."""
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image, ImageFile

from genpercept_b200 import engine as E

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURES = ["jpeg_dis_bag.jpg", "jpeg_depth_4.jpg"]


def encode(h, w, q, subsampling, seed, kind="photo", **kw):
    g = np.random.default_rng(seed)
    if kind == "noise":                                   # long codes, many 0xFF bytes, clamped pixels
        a = g.integers(0, 256, (h, w, 3)).astype(np.float64)
    else:
        yy, xx = np.mgrid[0:h, 0:w]
        a = np.stack([np.sin(xx / 37.0 + c) * np.cos(yy / 53.0 - c) for c in range(3)], -1) * 100 + 128
        if kind == "photo":
            a = a + g.normal(0, 12, a.shape)
    buf = io.BytesIO()
    Image.fromarray(np.clip(a, 0, 255).astype(np.uint8)).save(buf, "JPEG", quality=q, subsampling=subsampling, **kw)
    return buf.getvalue()


def pillow(data):
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def check(data, layout="hwc"):
    got = E.decode_jpeg(data, layout=layout).cpu().numpy()
    ref = pillow(data)
    if layout == "chw":
        ref = ref.transpose(2, 0, 1)
    assert got.shape == ref.shape
    if not np.array_equal(got, ref):
        d = got.astype(int) - ref
        raise AssertionError(f"{(d != 0).sum()} bytes differ, max |d| = {np.abs(d).max()}")


@pytest.mark.parametrize("subsampling", [0, 1, 2])
@pytest.mark.parametrize("q", [50, 75, 90, 95, 100])
def test_samplings_and_qualities(subsampling, q):
    for kind in ("photo", "noise", "gradient"):
        check(encode(131, 197, q, subsampling, seed=q + subsampling, kind=kind))


@pytest.mark.parametrize("size", [(1, 1), (7, 9), (17, 33), (2, 3), (1200, 686)])
@pytest.mark.parametrize("subsampling", [0, 1, 2])
def test_odd_sizes(size, subsampling):
    for kind in ("photo", "noise"):
        check(encode(*size, 90, subsampling, seed=size[0] + size[1], kind=kind))


@pytest.mark.parametrize("restart", [{"restart_marker_blocks": 1}, {"restart_marker_blocks": 7},
                                     {"restart_marker_rows": 1}])
@pytest.mark.parametrize("subsampling", [0, 1, 2])
def test_restart_intervals(restart, subsampling):
    for kind in ("photo", "noise", "gradient"):
        check(encode(97, 161, 90, subsampling, seed=3, kind=kind, **restart))


def test_4032x3024():
    check(encode(3024, 4032, 90, 2, seed=1))
    check(encode(3024, 4032, 95, 0, seed=2, restart_marker_rows=1), layout="chw")


@pytest.mark.parametrize("name", FIXTURES)
@pytest.mark.parametrize("layout", ["hwc", "chw"])
def test_fixtures(name, layout):
    check(open(os.path.join(GOLDEN, name), "rb").read(), layout)


def _pillow_outcome(data):
    try:
        return "ok", pillow(data)
    except Exception as ex:                               # noqa: BLE001 - whatever Pillow raises is the outcome
        return "error", type(ex)


def _pipeline_outcome(data, tmp_path):
    from genpercept_b200.pipeline import preprocess
    p = tmp_path / "x.jpg"
    p.write_bytes(data)
    try:
        rgb, _ = preprocess(Image.open(p), 0, "bilinear", "cuda")
        return "ok", rgb[0].cpu().numpy().transpose(1, 2, 0)
    except Exception as ex:                               # noqa: BLE001
        return "error", type(ex)


def _same(a, b):
    return a[0] == b[0] and (np.array_equal(a[1], b[1]) if a[0] == "ok" else a[1] is b[1])


def test_truncated_entropy_segment(tmp_path, monkeypatch):
    d = encode(400, 480, 90, 2, seed=4)                   # above JPEG_GPU_MIN_PIXELS: the pipeline tries the GPU
    for cut in (d[:len(d) * 2 // 3], d[:len(d) * 2 // 3] + b"\xff\xd9"):
        with pytest.raises(ValueError):
            E.decode_jpeg(cut)
        assert _same(_pipeline_outcome(cut, tmp_path), _pillow_outcome(cut))
        monkeypatch.setattr(ImageFile, "LOAD_TRUNCATED_IMAGES", True)
        assert _same(_pipeline_outcome(cut, tmp_path), _pillow_outcome(cut))
        monkeypatch.setattr(ImageFile, "LOAD_TRUNCATED_IMAGES", False)


def test_garbage_entropy_segment(tmp_path):
    base = encode(400, 480, 90, 2, seed=5)
    sos = base.index(b"\xff\xda")
    start = sos + 2 + (base[sos + 2] << 8 | base[sos + 3])
    g = np.random.default_rng(6)
    for trial in range(6):
        n = len(base) - 2 - start
        junk = g.integers(0, 256, n, dtype=np.uint8)
        if trial % 2:                                     # without markers: stuffed 0xFF only
            junk[junk == 0xFF] = 0x7F
        d = base[:start] + junk.tobytes() + b"\xff\xd9"
        try:
            got = E.decode_jpeg(d, layout="hwc").cpu().numpy()
            assert np.array_equal(got, pillow(d))
        except ValueError:
            pass
        assert _same(_pipeline_outcome(d, tmp_path), _pillow_outcome(d))


def test_out_of_window_idct_takes_pillows_path(tmp_path):
    """Well-formed streams whose IDCT values leave the window where libjpeg-turbo's C and SIMD IDCTs agree (every
    quantisation entry rewritten to 8 on a q100 noise image; single-bit flips that shift the DC of every later block):
    the device decode raises ValueError, and the pipeline gives Pillow's own bytes."""
    from test_oracle_jpeg import FLIP_PHOTO, OUT_OF_WINDOW_FLIPS, flipped, with_dqt
    from test_oracle_jpeg import encode as oracle_encode
    cases = [with_dqt(oracle_encode(h, w, 100, 0, seed=1, kind="noise"), 8) for h, w in ((64, 64), (400, 480))]
    base = oracle_encode(**FLIP_PHOTO)
    cases += [flipped(base, off, bit) for off, bit in OUT_OF_WINDOW_FLIPS]
    for d in cases:
        pillow(d)                                         # Pillow decodes each of them
        with pytest.raises(ValueError, match="IDCT"):
            E.decode_jpeg(d)
        assert _same(_pipeline_outcome(d, tmp_path), _pillow_outcome(d))


def test_bit_flips_match_pillow_or_are_rejected(tmp_path):
    from test_oracle_jpeg import FLIP_PHOTO, flipped
    from test_oracle_jpeg import encode as oracle_encode
    base = oracle_encode(**FLIP_PHOTO)
    sos = base.index(b"\xff\xda")
    n = len(base) - (sos + 2 + (base[sos + 2] << 8 | base[sos + 3])) - 2
    g = np.random.default_rng(1)
    accepted = 0
    for _ in range(200):
        d = flipped(base, int(g.integers(0, n)), int(g.integers(0, 8)))
        try:
            got = E.decode_jpeg(d, layout="hwc").cpu().numpy()
        except ValueError:
            continue
        accepted += 1
        assert _same(("ok", got), _pillow_outcome(d))
    assert accepted > 20


# ------------------------------------------------------------------------------------------------ the pipelines
def _files(tmp_path):
    paths = []
    for i, (h, w, ss) in enumerate([(481, 601, 2), (384, 512, 0), (420, 480, 1)]):   # above JPEG_GPU_MIN_PIXELS
        p = tmp_path / f"in{i}.jpg"
        p.write_bytes(encode(h, w, 90, ss, seed=i))
        paths.append(str(p))
    return paths


def _no_load(monkeypatch):
    def fail(self, *a, **k):
        raise AssertionError("Pillow decoded an image the GPU decoder should have taken")
    monkeypatch.setattr(ImageFile.ImageFile, "load", fail)


def _eq(a, b):
    assert np.array_equal(a.pred_np, b.pred_np)
    ac = a.pred_colored if isinstance(a.pred_colored, list) else [a.pred_colored]
    bc = b.pred_colored if isinstance(b.pred_colored, list) else [b.pred_colored]
    for x, y in zip(ac, bc):
        assert np.array_equal(np.asarray(x), np.asarray(y))


def test_pipelines_take_unloaded_jpegs(synth_state, text_embed, golden_dir, tmp_path, monkeypatch):
    from genpercept_b200 import v1
    from genpercept_b200.multitask import MultiTaskPipeline
    from genpercept_b200.pipeline import GenPerceptPipeline
    pipe = GenPerceptPipeline(unet=synth_state["unet"], vae=synth_state["vae"], text_embed=text_embed,
                              torch_dtype=torch.float16)
    mt = MultiTaskPipeline({"depth": pipe}, {"depth": "depth"})
    te77 = torch.from_numpy(np.load(os.path.join(golden_dir, "empty_text_embed_77x1024.npy")).astype(np.float32))[None]
    half = lambda sd: {k: v.half() for k, v in sd.items()}          # noqa: E731
    vp = v1.GenPerceptPipeline(half(synth_state["unet"]), half(synth_state["vae"]), None, te77)
    runs = [
        lambda im: pipe(im, mode="depth", processing_res=64, show_progress_bar=False),
        lambda im: pipe(im, mode="depth", processing_res=0, show_progress_bar=False),
        lambda im: mt(im, processing_res=64)["depth"],
        lambda im: vp(im, processing_res=64, show_progress_bar=False),
        lambda im: vp(im, mode="normal", processing_res=0, show_progress_bar=False),
    ]
    try:
        paths = _files(tmp_path)
        refs = [[run(Image.open(p).convert("RGB")) for run in runs] for p in paths]
        with monkeypatch.context() as m:
            _no_load(m)
            for p, ref in zip(paths, refs):
                for run, r in zip(runs, ref):
                    im = Image.open(p)
                    _eq(run(im), r)
                    assert im.tile                                    # still unloaded
        # below JPEG_GPU_MIN_PIXELS Pillow's host decode is the faster one, and the pipelines take it
        from genpercept_b200.image_util import JPEG_GPU_MIN_PIXELS
        small = tmp_path / "small.jpg"
        small.write_bytes(encode(240, 320, 90, 2, seed=8))
        assert 240 * 320 < JPEG_GPU_MIN_PIXELS
        for run in runs:
            im = Image.open(small)
            _eq(run(im), run(Image.open(small).convert("RGB")))
            assert not im.tile                                        # Pillow loaded it
        # the nearest modes resize with torchvision on the host, so Pillow decodes for them as before
        nearest = lambda im: pipe(im, mode="depth", processing_res=64, resample_method="nearest",  # noqa: E731
                                  show_progress_bar=False)
        _eq(nearest(Image.open(paths[0])), nearest(Image.open(paths[0]).convert("RGB")))
        # streams the GPU decoder leaves to Pillow still run, through Pillow
        for kw in ({"progressive": True}, {}):
            p = tmp_path / "other.jpg"
            img = Image.fromarray(np.random.default_rng(9).integers(0, 256, (400, 480, 3), dtype=np.uint8))
            (img if kw else img.convert("L")).save(p, "JPEG", **kw)
            for run in runs:
                _eq(run(Image.open(p)), run(Image.open(p).convert("RGB")))
    finally:
        pipe._engine.close()
        vp._engine.close()
