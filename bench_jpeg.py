"""Times JPEG decoding for the pipelines' input: Pillow's host decode against the GPU decoder, and the whole
``pipe(Image.open(path))`` call with each.

Per photo:
  pillow       Image.open(path).convert("RGB") on the host (median of --host-iters)
  gpu          engine.decode_jpeg(bytes): the upload of the file bytes, the decode and the status read (median of
               --iters after --warmup)
  call pillow  pipe(im) at processing_res=768 in fp16 with im = Image.open(path).convert("RGB") done inside the timed
               region (the path before the GPU decoder)
  call gpu     pipe(Image.open(path)): the pipeline decodes on the GPU from image_util.JPEG_GPU_MIN_PIXELS pixels on,
               and through Pillow below that
The two call arms alternate, and their maps are asserted equal.  The weights are seeded (weights.synth_state): the
engine's time does not depend on their values.

Photos: the two fixtures under tests/golden (a 2592 x 3872 photo and a 686 x 1200 one whose width is not a multiple of
16), seeded photo-like 4032 x 3024 images at q90 4:2:0 and q95 4:4:4 with and without restart markers, and 1920 x 1080
down to 160 x 120, on both sides of JPEG_GPU_MIN_PIXELS.  Prints the card and its power limit, the host CPU and its core
count, one JSON line per photo and a table.
Everything it writes goes to a temporary directory.
"""
import argparse
import io
import json
import os
import platform
import statistics
import subprocess
import tempfile
import time

import numpy as np
import torch
from PIL import Image

from genpercept_b200 import engine as E
from genpercept_b200 import weights as W
from genpercept_b200.pipeline import GenPerceptPipeline

ROOT = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _photo(h, w, seed):
    """Smooth shapes with texture and noise: JPEG statistics close to a camera photo's."""
    g = np.random.default_rng(seed)
    base = torch.from_numpy(g.random((1, 3, 24, 32)).astype(np.float32))
    img = torch.nn.functional.interpolate(base, size=(h, w), mode="bicubic", align_corners=False)[0].numpy()
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    img = img + 0.08 * np.sin(xx / 3.1)[None] * np.cos(yy / 4.7)[None] + g.normal(0, 0.03, img.shape)
    return (np.clip(img.transpose(1, 2, 0), 0, 1) * 255).astype(np.uint8)


def _cpu():
    name = None
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name"):
                name = line.split(":", 1)[1].strip()
                break
    except OSError:
        pass
    if not name:
        try:
            out = subprocess.run(["lscpu"], capture_output=True, text=True).stdout
            name = next((ln.split(":", 1)[1].strip() for ln in out.splitlines() if ln.startswith("Model name")), None)
        except OSError:
            pass
    return name or platform.machine(), len(os.sched_getaffinity(0))


def _median_ms(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        t = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t) * 1e3)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-iters", type=int, default=5)
    ap.add_argument("--call-iters", type=int, default=5)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    cpu, cores = _cpu()
    print(f"card: {card}")
    print(f"host: {cpu}, {cores} cores")
    tmp = tempfile.mkdtemp(prefix="bench_jpeg_")
    photos = [("fixture 2592x3872 (DIS bag)", os.path.join(GOLDEN, "jpeg_dis_bag.jpg")),
              ("fixture 686x1200 (depth/4)", os.path.join(GOLDEN, "jpeg_depth_4.jpg"))]
    for name, h, w, q, ss, kw in [("4032x3024 q90 4:2:0", 3024, 4032, 90, 2, {}),
                                  ("4032x3024 q90 4:2:0 RST", 3024, 4032, 90, 2, {"restart_marker_rows": 1}),
                                  ("4032x3024 q95 4:4:4", 3024, 4032, 95, 0, {}),
                                  ("4032x3024 q95 4:4:4 RST", 3024, 4032, 95, 0, {"restart_marker_rows": 1}),
                                  ("1920x1080 q90 4:2:0", 1080, 1920, 90, 2, {}),
                                  ("640x480 q90 4:2:0", 480, 640, 90, 2, {}),
                                  ("480x360 q90 4:2:0", 360, 480, 90, 2, {}),
                                  ("320x240 q90 4:2:0", 240, 320, 90, 2, {}),
                                  ("160x120 q90 4:2:0", 120, 160, 90, 2, {})]:
        p = os.path.join(tmp, name.replace(" ", "_").replace(":", "") + ".jpg")
        Image.fromarray(_photo(h, w, h + w + q)).save(p, "JPEG", quality=q, subsampling=ss, **kw)
        photos.append((name, p))

    state = W.synth_state(1234, with_dpt=False)
    te = torch.from_numpy(np.load(os.path.join(GOLDEN, "empty_text_embed_2x1024.npy")).astype(np.float32))[None]
    pipe = GenPerceptPipeline(unet=state["unet"], vae=state["vae"], text_embed=te, torch_dtype=torch.float16)
    rows = []
    for name, p in photos:
        data = open(p, "rb").read()
        ref = np.asarray(Image.open(p).convert("RGB"))
        got = E.decode_jpeg(data, layout="hwc").cpu().numpy()
        assert np.array_equal(got, ref), name
        t_pil = _median_ms(lambda: Image.open(p).convert("RGB"), 1, a.host_iters)
        t_gpu = _median_ms(lambda: E.decode_jpeg(data), a.warmup, a.iters)

        def call_pillow():
            out = pipe(Image.open(p).convert("RGB"), mode="depth", processing_res=768, show_progress_bar=False)
            torch.cuda.synchronize()
            return out

        def call_gpu():
            out = pipe(Image.open(p), mode="depth", processing_res=768, show_progress_bar=False)
            torch.cuda.synchronize()
            return out
        a_out, b_out = call_pillow(), call_gpu()
        assert np.array_equal(a_out.pred_np, b_out.pred_np), name
        ta, tb = [], []
        for _ in range(a.call_iters):
            for fn, ts in ((call_pillow, ta), (call_gpu, tb)):
                t = time.perf_counter()
                fn()
                ts.append((time.perf_counter() - t) * 1e3)
        row = dict(photo=name, bytes=len(data), H=int(ref.shape[0]), W=int(ref.shape[1]), pillow_ms=round(t_pil, 2),
                   gpu_ms=round(t_gpu, 2), call_pillow_ms=round(statistics.median(ta), 2),
                   call_gpu_ms=round(statistics.median(tb), 2), card=card, host=f"{cpu} ({cores} cores)")
        print(json.dumps(row), flush=True)
        rows.append(row)
    pipe._engine.close()
    print("\n| photo | size | Pillow decode (ms) | GPU decode (ms) | call, Pillow decode (ms) | "
          "call, GPU decode (ms) |")
    print("|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['photo']} | {r['bytes'] / 1e6:.2f} MB | {r['pillow_ms']} | {r['gpu_ms']} | "
              f"{r['call_pillow_ms']} | {r['call_gpu_ms']} |")


if __name__ == "__main__":
    main()
