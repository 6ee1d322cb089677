#!/usr/bin/env python
"""Measurement behind GenPercept v1 on the engine (genpercept_b200/v1.py): where the time of a v1 ``__call__`` goes, and
what the 77-token context costs.

  python bench_v1.py [--reps N] [--warmup W] [--precisions fp16,high]

Prints ONE JSON line:

  call       v1 __call__ on a seeded synthetic PIL photo of 4032x3024, 1920x1080 and 640x480 at processing_res=768, in
             depth and normal, per precision (fp16 storage / the high-precision mode v1's fp32 modules select).  Two arms
             alternate in one process on the same engine:
               host    the reference's steps: Pillow's Image.resize on the CPU, the numpy normalisation and upload, then
                       torch's F.interpolate and min-max (depth) or clip on the device as v1 runs them, .cpu(), and the
                       colour step on the CPU (a 256-entry Spectral table indexed as matplotlib's colormap indexes, which
                       stands in for matplotlib; norm_to_rgb for normals)
               device  the pipeline's path: gp_resize_pil, gp_v1_postprocess, gp_colorize, one copy to the host
             Milliseconds per image, median over --reps calls after --warmup, host clock around work that ends in a
             device synchronisation, split into pre (image -> engine input on the device), engine (Engine.infer) and
             post (engine map -> pred_np and the colour image on the host).
  context    Engine.infer at 768x768, batch 8, with the 77-token context (the general cross-attention path) and with the
             2-token empty prompt (the closed form), per precision: ms per call, median.
  device     the card's name and power limit, read in the same run.

Weights and inputs are seeded synthetic data; nothing is written to the tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from PIL import Image  # noqa: E402

SIZES = ((4032, 3024), (1920, 1080), (640, 480))      # (W, H), PIL order
MODES = ("depth", "normal")


def device_info():
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"] = float(out[1])
        info["sm_max_mhz"] = float(out[2])
    except Exception as ex:                       # the number is then missing, not guessed
        info["power_limit_error"] = str(ex)
    return info


def photo(W, H, seed):
    g = torch.Generator().manual_seed(seed)
    base = torch.rand((1, 3, 24, 32), generator=g)
    img = F.interpolate(base, size=(H, W), mode="bilinear", align_corners=False)[0]
    img = (img + 0.05 * torch.rand((3, H, W), generator=g)).clamp(0, 1)
    return Image.fromarray((img.permute(1, 2, 0).numpy() * 255).astype(np.uint8))


def _sync():
    torch.cuda.synchronize()
    return time.perf_counter()


def host_arm(pipe, img, mode, lut_f):
    """The reference's own steps around the engine (GenPercept_v1 pipeline_genpercept.py __call__)."""
    ch = pipe.task_infos[mode]["task_channel_num"]
    t0 = _sync()
    w, h = img.size
    f = min(768 / w, 768 / h)
    small = img.resize((int(w * f), int(h * f)))
    rgb = np.transpose(np.asarray(small.convert("RGB")), (2, 0, 1)) / 255.0 * 2.0 - 1.0
    rgb = torch.from_numpy(rgb).to(pipe.dtype)[None].to(pipe.device)
    t1 = _sync()
    y = pipe._engine.infer(rgb, out_channels=ch)
    t2 = _sync()
    preds = F.interpolate(y * 2 - 1, (h, w), mode="bilinear")
    if mode == "depth":
        preds = preds[:, 0]
        mn = preds.view(1, -1).min(dim=1)[0]
        mx = preds.view(1, -1).max(dim=1)[0]
        preds = ((preds - mn[:, None, None]) / (mx[:, None, None] - mn[:, None, None])).cpu().numpy().astype(np.float32)
        idx = (np.clip(preds[0], 0, 1) * 256).astype(np.int64).clip(0, 255)
        colored = (lut_f[idx] * 255).astype(np.uint8)
    else:
        preds = preds.clip(-1, 1).cpu().numpy()
        colored = np.moveaxis(np.clip(((preds[0] + 1) * 0.5) * 255, 0, 255).astype(np.uint8), 0, -1)
    Image.fromarray(colored)
    t3 = _sync()
    return t1 - t0, t2 - t1, t3 - t2


def device_arm(pipe, img, mode):
    """The pipeline's path (the same steps as GenPerceptPipeline.__call__, split for timing)."""
    ch = pipe.task_infos[mode]["task_channel_num"]
    t0 = _sync()
    rgb = pipe._pil_input(img, 768, False)
    t1 = _sync()
    y = pipe._engine.infer(rgb, out_channels=ch)
    t2 = _sync()
    pipe._postprocess(y, mode, (img.size[1], img.size[0]), "Spectral")
    t3 = _sync()
    return t1 - t0, t2 - t1, t3 - t2


def _ms(samples):
    return round(1e3 * statistics.median(samples), 3)


def bench_calls(pipe, reps, warmup, lut_f):
    res = []
    for (W, H) in SIZES:
        img = photo(W, H, seed=W + H)
        for mode in MODES:
            arms = {"host": [], "device": []}
            for i in range(warmup + reps):
                for name, fn in (("host", lambda: host_arm(pipe, img, mode, lut_f)), ("device", lambda: device_arm(pipe, img, mode))):
                    t = fn()
                    if i >= warmup:
                        arms[name].append(t)
            row = {"size": [W, H], "mode": mode}
            for name, ts in arms.items():
                pre, eng, post = (_ms([t[k] for t in ts]) for k in range(3))
                row[name] = {"pre_ms": pre, "engine_ms": eng, "post_ms": post, "total_ms": _ms([sum(t) for t in ts])}
            res.append(row)
            print(json.dumps(row), file=sys.stderr)
    return res


def bench_context(pipe, state, te2, precision, reps, warmup):
    from genpercept_b200.engine import Engine
    storage = torch.float16
    e2 = Engine(dtype=storage, readout="vae", precision="high" if precision == "high" else "default")
    try:
        sd = (lambda d: d) if precision == "high" else (lambda d: {k: v.half() for k, v in d.items()})
        e2.load_state("unet", sd(state["unet"]))
        e2.load_state("vae", sd(state["vae"]))
        e2.set_text_embed(te2)
        e2.finalize()
        g = torch.Generator().manual_seed(768)
        rgb = torch.randint(0, 256, (8, 3, 768, 768), generator=g, dtype=torch.uint8).cuda()
        out = {}
        times = {"77": [], "2": []}
        for i in range(warmup + reps):
            for name, e in (("77", pipe._engine), ("2", e2)):
                t0 = _sync()
                e.infer(rgb, out_channels=1)
                t1 = _sync()
                if i >= warmup:
                    times[name].append(t1 - t0)
        out["tokens77_ms"] = _ms(times["77"])
        out["tokens2_ms"] = _ms(times["2"])
        out["extra_pct"] = round(100.0 * (out["tokens77_ms"] / out["tokens2_ms"] - 1.0), 2)
        return out
    finally:
        e2.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precisions", default="fp16,high")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_v1.py measures on a CUDA device; there is none")
    from genpercept_b200 import weights as W
    from genpercept_b200.image_util import _lut
    from genpercept_b200.v1 import GenPerceptPipeline
    state = W.synth_state(1234, with_dpt=False)
    golden = os.path.join(ROOT, "tests", "golden")
    te77 = torch.from_numpy(np.load(os.path.join(golden, "empty_text_embed_77x1024.npy")).astype(np.float32))[None]
    te2 = torch.from_numpy(np.load(os.path.join(golden, "empty_text_embed_2x1024.npy")).astype(np.float32))[None]
    lut_f = _lut("Spectral")
    result = {"bench": "v1", "reps": args.reps, "warmup": args.warmup, "device": device_info(), "call": {}, "context": {}}
    for prec in args.precisions.split(","):
        sd = (lambda d: d) if prec == "high" else (lambda d: {k: v.half() for k, v in d.items()})
        pipe = GenPerceptPipeline(sd(state["unet"]), sd(state["vae"]), None, te77)
        try:
            result["call"][prec] = bench_calls(pipe, args.reps, args.warmup, lut_f)
            result["context"][prec] = bench_context(pipe, state, te2, prec, args.reps, args.warmup)
            print(json.dumps({prec: result["context"][prec]}), file=sys.stderr)
        finally:
            pipe._engine.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
