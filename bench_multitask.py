#!/usr/bin/env python
"""Several GenPercept tasks on one image: one VAE encode shared by N task engines against N full passes.

  python bench_multitask.py [--precision default|high] [--dtype f16|bf16] [--res 768] [--batch 8] [--tasks 2,5]
                            [--steps 5] [--warmup 2]

Task engine i has its own seeded synthetic UNet (weights.synth_unet(100 + i)); odd-numbered tasks read out through the
DPT head, the others through the VAE decoder, and all of them share the VAE of weights.synth_state(1234).  For each N,
one step over a batch of uint8 images resident in HBM is timed with CUDA events in two ways, alternated round by
round (the median of the rounds is reported):

  full    each of the N engines runs Engine.infer (encode, UNet, readout);
  shared  the first engine runs Engine.encode_exact once, then each engine runs Engine.infer_latent on that latent.

Both arms give bit-identical maps; the script checks that.  The saving expected from the FLOP table
(genpercept_b200/flops.py) is (N - 1) encodes per image over N full passes.  The high-precision mode runs with
memory-efficient attention, so that five engines fit on one 80 GB card; an N that does not fit is reported as not
measured.  Prints one JSON line with the card's name and power limit, read in the same run.  Nothing is written.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from genpercept_b200 import flops as FL  # noqa: E402
from genpercept_b200 import weights as W  # noqa: E402
from genpercept_b200.engine import Engine  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
    except Exception as ex:
        name, power, clock = torch.cuda.get_device_name(0), f"unknown ({ex})", "unknown"
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def text_embed():
    e = np.load(os.path.join(ROOT, "tests", "golden", "empty_text_embed_2x1024.npy")).astype(np.float32)
    return torch.from_numpy(e)[None]


def make_engine(i, state, args):
    readout = "dpt" if i % 2 else "vae"
    e = Engine(dtype=torch.bfloat16 if args.dtype == "bf16" else torch.float16, readout=readout, precision=args.precision,
               cuda_graph=False, memory_efficient_attention=args.precision == "high")
    e.load_state("unet", W.synth_unet(100 + i))
    e.load_state("vae", state["vae"])
    if readout == "dpt":
        e.load_state("dpt", state["dpt"])
    e.set_text_embed(text_embed())
    e.finalize()
    e.plan(args.batch, args.res, args.res)
    return e


def measure(engines, x, outs, args):
    """-> (ms per step full, ms per step shared, bit-identical) for the given engines."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def full():
        for e, o in zip(engines, outs[0]):
            e.infer(x, out=o)

    def shared():
        lat = engines[0].encode_exact(x)
        for e, o in zip(engines, outs[1]):
            e.infer_latent(lat, out=o)          # each engine's one plan, made in make_engine

    def timed(fn):
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(args.steps):
            fn()
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / args.steps

    for _ in range(args.warmup):
        full()
        shared()
    same = all(torch.equal(a, b) for a, b in zip(outs[0], outs[1]))
    t_full, t_shared = [], []
    for _ in range(args.rounds):
        t_full.append(timed(full))
        t_shared.append(timed(shared))
    return statistics.median(t_full), statistics.median(t_shared), same, (min(t_full), max(t_full)), (min(t_shared), max(t_shared))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="default", choices=["default", "high"])
    ap.add_argument("--dtype", default="f16", choices=["f16", "bf16"])
    ap.add_argument("--res", type=int, default=768)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--tasks", default="2,5")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multitask.py needs a CUDA (sm_90a) device")
    ns = sorted(int(n) for n in args.tasks.split(","))
    B, R = args.batch, args.res
    state = W.synth_state(1234)
    g = torch.Generator().manual_seed(1002)
    x = torch.randint(0, 256, (B, 3, R, R), generator=g, dtype=torch.uint8).cuda()
    engines, outs, results = [], [[], []], []
    enc = FL.vae_encoder_flops(R, R)
    for n in ns:
        try:
            while len(engines) < n:
                e = make_engine(len(engines), state, args)
                engines.append(e)
                for k in range(2):
                    outs[k].append(torch.empty((B, 1) + tuple(e.out_hw), dtype=torch.float32, device="cuda"))
            ms_full, ms_shared, same, rf, rs = measure(engines[:n], x, [o[:n] for o in outs], args)
        except RuntimeError as ex:
            results.append({"tasks": n, "measured": False, "reason": f"not measured: {str(ex).splitlines()[0][:200]}"})
            break
        readouts = ["dpt" if i % 2 else "vae" for i in range(n)]
        total = sum(FL.single_infer_flops(R, R, r) for r in readouts)
        results.append({
            "tasks": n, "measured": True, "readouts": readouts,
            "ms_per_image_full": ms_full / B, "ms_per_image_shared": ms_shared / B,
            "ms_per_step_full_range": list(rf), "ms_per_step_shared_range": list(rs),
            "saving_measured": 1.0 - ms_shared / ms_full,
            "saving_flop_table": (n - 1) * enc / total,
            "bit_identical": bool(same),
            "arena_bytes": [e.plan_info()["arena_bytes"] for e in engines[:n]],
            "weight_bytes": [e.plan_info()["weight_bytes"] for e in engines[:n]],
        })
    print(json.dumps({
        "bench": "multitask: one encode + N infer_latent vs N infer", "res": R, "batch": B, "dtype": args.dtype,
        "precision": args.precision, "memory_efficient_attention": args.precision == "high", "steps": args.steps,
        "rounds": args.rounds, "encode_tflop_per_image": enc / 1e12, "card": card(), "results": results,
    }))
    for e in engines:
        e.close()


if __name__ == "__main__":
    main()
