#!/usr/bin/env python
"""Measurement behind the fused head-dim-512 attention of the VAE mid-block (csrc/fattn512.cu), and with
--precision high behind the high-precision mode's memory-efficient attention (the split-precision instances of
csrc/fattn.cu and csrc/fattn512.cu).

  python bench_native.py [--iters N] [--skip-e2e] [--precision default|high]

Prints ONE JSON line:

  attention    both d = 512 paths (fused kernel, unfused QK^T -> softmax -> P V) at B in {1, 8} and
               T in {9216, 16384, 25600, 36864} tokens, fp16: microseconds per call (CUDA events, after a warm-up call)
               and achieved TFLOP/s of the algorithmic 4 B T^2 512 FLOPs, next to the H100 SXM data-sheet dense fp16
               peak (989 TFLOP/s, not a measured figure).  `s_bytes` is the score matrix the unfused path stores;
               `planner` names the path the planner takes at that size (fused above kFusedAttnMinBytes = 2 GiB, or
               where the unfused path cannot run: rows past 16384 keys with T a multiple of 8, recorded as null).
  native       whole-engine inference (Engine.infer, the single_infer hot path) of one fp16 image at native photo
               sizes: ms per image (median of the timed calls, device-synchronised) and the plan's arena bytes.
  device       the card's name and power limit, read in the same run.

With --precision high the line instead holds
  attention    both high-precision paths (fused split-precision kernel; unfused QK^T -> softmax -> P V over (hi, lo)
               planes) for d = 64 with 5 heads (the UNet's first level) and for d = 512 with one head, at the same B and
               T: microseconds per call and TFLOP/s of the algorithmic 4 B heads T^2 d FLOPs (each takes three
               tensor-core passes per product); null where the unfused path cannot run.
  native       the same native sizes through the high-precision engine with memory-efficient attention on.

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

PEAK_FP16_DENSE_TFLOPS = 989.0        # NVIDIA H100 SXM data sheet, dense fp16 / bf16, 700 W card
FUSED_MIN_BYTES = 2 << 30             # kFusedAttnMinBytes in csrc/builder.cu
SOFTMAX_ROWS_MAX_T = 16384            # kSoftmaxRowsMaxT in csrc/kernels.h: the unfused path's longest row (T % 8 == 0)
TOKENS = (9216, 16384, 25600, 36864)  # 768^2, 1024^2, 1280^2, 1536^2 images
BATCHES = (1, 8)
NATIVE = ((3872, 2592), (2592, 3872), (3024, 4032))   # (H, W)


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


def attention_sweep_high(iters):
    from genpercept_b200 import engine as E
    rows = []
    for heads, d in ((5, 64), (1, 512)):
        for B in BATCHES:
            for T in TOKENS:
                tp = (T + 7) // 8 * 8
                unfused_runs = T % 8 != 0 or T <= SOFTMAX_ROWS_MAX_T
                row = {"heads": heads, "d": d, "B": B, "T": T, "s_bytes": B * heads * T * 2 * tp * 2}
                for path, fused in (("fused", True), ("unfused", False)):
                    if not fused and not unfused_runs:
                        row[path] = None
                        continue
                    us, fl = E.bench_attention_high(B, T, heads, d, fused, iters)
                    row[path] = {"usec": round(us, 1), "tflops": round(fl / us * 1e-6, 1)}
                    torch.cuda.empty_cache()
                if row["unfused"]:
                    row["fused_over_unfused"] = round(row["fused"]["usec"] / row["unfused"]["usec"], 3)
                rows.append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
    return rows


def attention_sweep(iters):
    from genpercept_b200 import engine as E
    rows = []
    for B in BATCHES:
        for T in TOKENS:
            tp = (T + 7) // 8 * 8
            s_bytes = B * T * tp * 2
            unfused_runs = T % 8 != 0 or T <= SOFTMAX_ROWS_MAX_T
            row = {"B": B, "T": T, "s_bytes": s_bytes,
                   "planner": "fused" if s_bytes > FUSED_MIN_BYTES or not unfused_runs else "unfused"}
            for path, fused in (("fused", True), ("unfused", False)):
                if not fused and not unfused_runs:
                    row[path] = None                  # softmax_rows takes rows of at most 16384 keys (T % 8 == 0)
                    continue
                us, fl = E.bench_attention(torch.float16, B, T, fused, iters)
                row[path] = {"usec": round(us, 1), "tflops": round(fl / us * 1e-6, 1)}
                torch.cuda.empty_cache()
            if row["unfused"]:
                row["fused_over_unfused"] = round(row["fused"]["usec"] / row["unfused"]["usec"], 3)
            rows.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
    return rows


def native_sweep(reps, precision="default"):
    from genpercept_b200 import weights as W
    from genpercept_b200.engine import Engine
    state = W.synth_state(1234, with_dpt=False)
    te = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", "empty_text_embed_2x1024.npy")).astype(np.float32))[None]
    high = precision == "high"
    if high:   # the high-precision arenas (~30 GB at these sizes) do not fit the default four cached plans
        os.environ["GP_MAX_PLANS"] = "1"
    e = Engine(dtype=torch.float16, readout="vae", precision=precision, memory_efficient_attention=high)
    e.load_state("unet", state["unet"])
    e.load_state("vae", state["vae"])
    e.set_text_embed(te)
    e.finalize()
    res = []
    try:
        for H, W_ in NATIVE:
            g = torch.Generator().manual_seed(H * W_)
            rgb = torch.randint(0, 256, (1, 3, H, W_), generator=g, dtype=torch.uint8).cuda()
            out = e.infer(rgb)                      # plan + warm-up
            torch.cuda.synchronize()
            ts = []
            for _ in range(reps):
                t0 = time.perf_counter()
                out = e.infer(rgb, out=out)
                torch.cuda.synchronize()
                ts.append((time.perf_counter() - t0) * 1e3)
            info = e.plan_info()
            names = [op["name"] for op in e.profile_ops()]
            r = {"H": H, "W": W_, "T_mid": (H // 8) * (W_ // 8), "ms_per_image": round(statistics.median(ts), 1),
                 "ms_all": [round(t, 1) for t in ts], "arena_bytes": info["arena_bytes"],
                 "fused_attention_ops": sum(n.endswith((".fattn512", ".fattn") if high else ".fattn512") for n in names),
                 "finite": bool(torch.isfinite(out).all().item())}
            res.append(r)
            print(json.dumps(r), file=sys.stderr, flush=True)
    finally:
        e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5, help="timed calls per attention configuration")
    ap.add_argument("--reps", type=int, default=3, help="timed images per native size")
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--precision", choices=("default", "high"), default="default")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_native.py needs a CUDA device (H100)")
    dev = device_info()
    if a.precision == "high":
        line = {"device": dev, "precision": "high", "peak_fp16_dense_tflops_datasheet": PEAK_FP16_DENSE_TFLOPS,
                "attention": attention_sweep_high(a.iters)}
    else:
        line = {"device": dev, "peak_fp16_dense_tflops_datasheet": PEAK_FP16_DENSE_TFLOPS,
                "attention": attention_sweep(a.iters)}
    if not a.skip_e2e:
        line["native"] = native_sweep(a.reps, a.precision)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
