#!/usr/bin/env python
"""Speed of the multi-step arch's denoising loop with and without CUDA graphs.

  python bench_multistep.py [--steps 10] [--precision default,high] [--shapes 1x384x384,1x512x512,1x768x768,5x768x768]
                            [--warmup 2] [--calls 3] [--rounds 3]

Times GenPerceptPipeline.single_infer of the marigold arch (8-channel conv_in, noise drawn from a CPU generator, as
run.py's default --archs marigold does) with `--steps` DDIM steps, on seeded synthetic weights (weights.synth_state).
Batch 5 at 768 x 768 is the size of run.py's ensemble (--ensemble_size 5).  Two arms, one engine each:

  eager  cuda_graph=False: every kernel launched from the host, step by step;
  graph  the default engine (cuda_graph="auto"): after the first call, each call replays one graph of the whole loop
         where the plan is small enough (batch x height x width <= 2 x 768 x 768); larger plans run eagerly.

The arms alternate round by round; each round times `--calls` calls between two device synchronisations, after
`--warmup` untimed calls per arm and shape.  It reports the median ms per call of each arm, and checks that both arms'
maps are np.array_equal.  The high-precision mode (torch_dtype=float32) runs with memory-efficient attention, as run.py
turns it on.  The card's name and power limit are read in the same run.  Prints one JSON line at the end; nothing is
written.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
os.environ.setdefault("GP_MAX_PLANS", "1")     # one plan per engine at a time: the largest shapes fit both arms

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_multitask import card, text_embed  # noqa: E402
from genpercept_b200 import weights as W  # noqa: E402
from genpercept_b200.pipeline import GenPerceptPipeline  # noqa: E402

# the reference's hf_configs/scheduler_beta_0.00085_0.012/scheduler_config.json
SCHED = {"_class_name": "DDIMScheduler", "num_train_timesteps": 1000, "beta_start": 0.00085, "beta_end": 0.012,
         "beta_schedule": "scaled_linear", "clip_sample": False, "set_alpha_to_one": False, "steps_offset": 1,
         "prediction_type": "v_prediction", "timestep_spacing": "leading"}
ARMS = ("eager", "graph")


def make_pipeline(state, precision, arm):
    pipe = GenPerceptPipeline(unet=state["unet"], vae=state["vae"], scheduler=dict(SCHED), text_embed=text_embed(),
                              genpercept_pipeline=False, rgb_blending=False,
                              torch_dtype=torch.float32 if precision == "high" else torch.float16,
                              cuda_graph="auto" if arm == "graph" else False)
    if precision == "high":
        pipe.enable_xformers_memory_efficient_attention()
    return pipe


def call(pipe, rgb, steps, seed):
    return pipe.single_infer(rgb, num_inference_steps=steps, generator=torch.Generator().manual_seed(seed), mode="depth")


def time_calls(pipe, rgb, steps, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        call(pipe, rgb, steps, 100 + i)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--precision", default="default,high")
    ap.add_argument("--shapes", default="1x384x384,1x512x512,1x768x768,5x768x768")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multistep.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}, max SM clock {info['max_sm_clock']}", flush=True)
    state = W.synth_state(1234, with_dpt=False, unet_in_channels=8)
    shapes = [tuple(int(v) for v in s.split("x")) for s in args.shapes.split(",")]
    results = []
    for precision in args.precision.split(","):
        pipes = {arm: make_pipeline(state, precision, arm) for arm in ARMS}
        for B, H, W_ in shapes:
            row = {"precision": precision, "batch": B, "height": H, "width": W_, "steps": args.steps}
            try:
                rgb = torch.randint(0, 256, (B, 3, H, W_), generator=torch.Generator().manual_seed(7),
                                    dtype=torch.uint8).cuda()
                maps = {}
                for arm in ARMS:
                    for _ in range(args.warmup):
                        maps[arm] = call(pipes[arm], rgb, args.steps, 1).cpu().numpy()
                ms = {arm: [] for arm in ARMS}
                for _ in range(args.rounds):
                    for arm in ARMS:
                        ms[arm].append(time_calls(pipes[arm], rgb, args.steps, args.calls))
                for arm in ARMS:
                    row[f"{arm}_ms"] = round(statistics.median(ms[arm]), 2)
                    row[f"{arm}_ms_all"] = [round(v, 2) for v in ms[arm]]
                row["speedup"] = round(row["eager_ms"] / row["graph_ms"], 3)
                row["maps_equal"] = bool(np.array_equal(maps["eager"], maps["graph"]))
            except RuntimeError as ex:
                row["error"] = str(ex)
            print(json.dumps(row), flush=True)
            results.append(row)
        for p in pipes.values():
            p._engine.close()
        del pipes
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "multistep", "card": info, "results": results}))
    if any(not r.get("maps_equal", False) for r in results):
        raise SystemExit("the arms' maps differ (or a shape failed)")


if __name__ == "__main__":
    main()
