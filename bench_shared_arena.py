#!/usr/bin/env python
"""Device memory and speed of N task engines with and without the shared activation arena.

  python bench_shared_arena.py [--precision default|high] [--dtype f16|bf16] [--size 768x768] [--batch 8]
                               [--tasks 2,5] [--steps 3] [--warmup 1] [--rounds 3]
  python bench_shared_arena.py --three-shapes [--precision default|high]

Task engine i has its own seeded synthetic UNet (weights.synth_unet(100 + i)); odd-numbered tasks read out through the
DPT head, the others through the VAE decoder, and all share the VAE of weights.synth_state(1234), as in
bench_multitask.py.  The high-precision mode runs with memory-efficient attention, as run.py and infer.py turn it on.
One step is what MultiTaskPipeline runs: one encode_exact, then infer_latent on every engine.  The same engines run
both arms, alternated round by round (the arena setting is switched between rounds, which re-plans outside the timed
window):

  private  every plan owns its arena (the default);
  shared   every engine takes its plans' arenas from the device's one pool (Engine.set_shared_arena).

For each arm it reports the activation bytes (the sum of the plans' arenas, or the pool's mapped bytes), the peak of
device memory in use (torch.cuda.mem_get_info, over the whole device, after planning and after each step), the median
ms per image, and whether the arms' maps are np.array_equal.  An arm that does not fit is reported as not measured,
with the error.  --three-shapes instead runs one VAE-readout engine over three native-resolution photo shapes in turn
(4032 x 3024, 3024 x 4032, 3872 x 2592; batch 1), once per arm.  Prints one JSON line with the card's name and power
limit, read in the same run.  Nothing is written.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_multitask import card, text_embed  # noqa: E402
from genpercept_b200 import engine as E  # noqa: E402
from genpercept_b200 import weights as W  # noqa: E402
from genpercept_b200.engine import Engine  # noqa: E402

GIB = 1 << 30
THREE_SHAPES = [(3024, 4032), (4032, 3024), (2592, 3872)]


def make_engine(i, state, args, readout=None):
    readout = readout or ("dpt" if i % 2 else "vae")
    e = Engine(dtype=torch.bfloat16 if args.dtype == "bf16" else torch.float16, readout=readout, precision=args.precision,
               cuda_graph=False, memory_efficient_attention=args.precision == "high")
    e.load_state("unet", W.synth_unet(100 + i))
    e.load_state("vae", state["vae"])
    if readout == "dpt":
        e.load_state("dpt", state["dpt"])
    e.set_text_embed(text_embed())
    e.finalize()
    return e


def used_bytes():
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info()
    return total - free


class Arm:
    """Peak device memory and activation bytes of one arm."""

    def __init__(self, name):
        self.name, self.peak, self.ms, self.error, self.maps = name, 0, [], None, None

    def note(self):
        self.peak = max(self.peak, used_bytes())


def set_arm(engines, shared):
    for e in engines:
        e.set_shared_arena(shared)
    torch.cuda.empty_cache()


def activation_bytes(engines, shared, plans):
    return E.shared_arena_info()["mapped_bytes"] if shared else sum(plans)


def run_tasks(engines, x, outs, args, arms):
    """Alternates the arms round by round over the N engines; -> the per-arm result dicts."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    B = x.shape[0]

    def step():
        lat = engines[0].encode_exact(x)
        for e, o in zip(engines, outs):
            e.infer_latent(lat, out=o)

    res = {}
    for rnd in range(args.rounds):
        for arm in arms:
            if arm.error:
                continue
            shared = arm.name == "shared"
            set_arm(engines, shared)
            try:
                plans = []
                for e in engines:
                    e.plan(*x.shape[:1], *x.shape[2:])
                    plans.append(e.plan_info()["arena_bytes"])
                arm.note()
                for _ in range(args.warmup):
                    step()
                torch.cuda.synchronize()
                ev[0].record()
                for _ in range(args.steps):
                    step()
                ev[1].record()
                torch.cuda.synchronize()
                arm.note()
            except RuntimeError as ex:
                arm.error = f"not measured: {str(ex).splitlines()[0][:240]}"
                continue
            arm.ms.append(ev[0].elapsed_time(ev[1]) / args.steps / B)
            arm.act = activation_bytes(engines, shared, plans)
            arm.maps = [o.cpu().numpy() for o in outs]
    set_arm(engines, False)
    for arm in arms:
        if arm.error:
            res[arm.name] = {"measured": False, "reason": arm.error}
        else:
            res[arm.name] = {"measured": True, "ms_per_image": statistics.median(arm.ms),
                             "ms_per_image_range": [min(arm.ms), max(arm.ms)], "activation_gib": arm.act / GIB,
                             "peak_device_used_gib": arm.peak / GIB}
    a, b = arms
    res["bit_identical"] = None if a.maps is None or b.maps is None else \
        all(np.array_equal(p, q) for p, q in zip(a.maps, b.maps))
    return res


def bench_tasks(args, state):
    H, W_ = (int(v) for v in args.size.split("x"))
    B = args.batch
    g = torch.Generator().manual_seed(1002)
    x = torch.randint(0, 256, (B, 3, H, W_), generator=g, dtype=torch.uint8).cuda()
    results = []
    for n in sorted(int(v) for v in args.tasks.split(",")):
        engines = [make_engine(i, state, args) for i in range(n)]
        set_arm(engines, True)        # the result extents, from plans that fit whichever arm does not
        outs = []
        for e in engines:
            e.plan(B, H, W_)
            outs.append(torch.empty((B, 1) + tuple(e.out_hw), dtype=torch.float32, device="cuda"))
        r = run_tasks(engines, x, outs, args, [Arm("private"), Arm("shared")])
        r.update({"tasks": n, "readouts": [e.readout for e in engines]})
        results.append(r)
        for e in engines:
            e.close()
        del outs
        torch.cuda.empty_cache()
    return {"bench": "shared arena: N task engines, one encode + N infer_latent per step", "size": args.size, "batch": B,
            "results": results}


def bench_three_shapes(args, state):
    e = make_engine(0, state, args, readout="vae")
    g = torch.Generator().manual_seed(1003)
    xs = [torch.randint(0, 256, (1, 3, h, w), generator=g, dtype=torch.uint8).cuda() for h, w in THREE_SHAPES]
    arms = {}
    for shared in (False, True):
        set_arm([e], shared)
        peak, steps, maps = 0, [], []
        for x in xs:
            h, w = x.shape[2:]
            try:
                torch.cuda.synchronize()
                t0 = torch.cuda.Event(enable_timing=True)
                t1 = torch.cuda.Event(enable_timing=True)
                e.plan(1, h, w)
                t0.record()
                out = e.infer(x)
                t1.record()
                peak = max(peak, used_bytes())
                maps.append(out.cpu().numpy())
                steps.append({"shape": f"{h}x{w}", "ok": True, "arena_gib": e.plan_info()["arena_bytes"] / GIB,
                              "s_first_call": t0.elapsed_time(t1) / 1e3, "plans_cached": e.plan_count(),
                              "pool_mapped_gib": E.shared_arena_info()["mapped_bytes"] / GIB})
                del out
            except RuntimeError as ex:
                maps.append(None)
                steps.append({"shape": f"{h}x{w}", "ok": False, "error": str(ex).splitlines()[0][:240]})
        arms["shared" if shared else "private"] = {"steps": steps, "peak_device_used_gib": peak / GIB, "maps": maps}
    set_arm([e], False)
    e.close()
    same = [None if p is None or q is None else bool(np.array_equal(p, q))
            for p, q in zip(arms["private"].pop("maps"), arms["shared"].pop("maps"))]
    return {"bench": "shared arena: one engine, three native-resolution shapes in turn", "arms": arms,
            "bit_identical_per_shape": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="default", choices=["default", "high"])
    ap.add_argument("--dtype", default="f16", choices=["f16", "bf16"])
    ap.add_argument("--size", default="768x768", help="H x W")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--tasks", default="2,5")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--three-shapes", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_shared_arena.py needs a CUDA (sm_90a) device")
    state = W.synth_state(1234)
    base = used_bytes()
    res = bench_three_shapes(args, state) if args.three_shapes else bench_tasks(args, state)
    res.update({"dtype": args.dtype, "precision": args.precision,
                "memory_efficient_attention": args.precision == "high", "steps": args.steps, "rounds": args.rounds,
                "device_used_before_gib": base / GIB, "device_total_gib": torch.cuda.mem_get_info()[1] / GIB,
                "card": card()})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
