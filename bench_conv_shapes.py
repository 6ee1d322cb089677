#!/usr/bin/env python
"""Per-shape timing of the 3x3 stride-1 convolutions of the default bench.py step (batch 8, 768x768 depth).

  python bench_conv_shapes.py [--iters N] [--dtype f16|bf16] [--json FILE]

Each shape is planned and timed alone through gp_bench_conv (CUDA events over `iters` launches, after warm-up): the VAE
levels at 768^2, 384^2, 192^2 and 96^2 and the UNet levels at 96^2 and 48^2, with the step's channel counts.  For each
shape it prints microseconds per launch, the algorithmic rate (2 * MACs / time) and the kernel and tile the planner
picked.  The 1x1-shortcut ResNet convolutions are not covered: gp_bench_conv takes no shortcut (bench.py --ops-json
times them op by op).  The card name, power limit and SM clocks are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from genpercept_b200 import engine as E  # noqa: E402

# (output side, Cin, Cout, where in the step)
SHAPES = [
    (768, 128, 128, "VAE 768^2: enc/dec ResNets"),
    (768, 256, 128, "VAE dec up3 res0 conv1"),
    (384, 128, 256, "VAE enc down1 res0 conv1"),
    (384, 256, 256, "VAE 384^2 ResNets"),
    (384, 512, 256, "VAE dec up2 res0 conv1"),
    (192, 256, 512, "VAE enc down2 res0 conv1"),
    (192, 512, 512, "VAE 192^2 ResNets"),
    (96, 512, 512, "VAE 96^2: down3, mid, up0"),
    (96, 320, 320, "UNet 96^2 ResNets"),
    (96, 640, 320, "UNet up3 conv1 (skip concat)"),
    (96, 960, 320, "UNet up3 conv1 (skip concat)"),
    (48, 320, 640, "UNet down1 res0 conv1"),
    (48, 640, 640, "UNet 48^2 ResNets"),
    (48, 960, 640, "UNet up2 conv1 (skip concat)"),
    (48, 1280, 640, "UNet up2 conv1 (skip concat)"),
]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as ex:  # noqa: BLE001
        return {"error": str(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--dtype", default="f16", choices=["f16", "bf16"])
    ap.add_argument("--json", default=None, help="also write the table here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_conv_shapes.py needs a CUDA device")
    dt = torch.float16 if args.dtype == "f16" else torch.bfloat16
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    info = card()
    print(json.dumps({"card": info, "sms": sms}))
    rows = []
    print(f"{'HxW':>7} {'Cin':>5} {'Cout':>5} {'us':>9} {'TFLOP/s':>8}  plan")
    for side, cin, cout, where in SHAPES:
        us, fl = E.bench_conv(dt, args.batch, side, side, cin, cout, 3, 0, args.iters)
        plan = E.conv_tile(args.batch, side, side, cin, cout, num_sms=sms) if hasattr(E, "conv_tile") else None
        tag = "n/a"
        if plan is not None:
            tag = (f"patch {plan['tw']}x{plan['th']}" if plan["patch"] else "tap") + f" BN{plan['bn']} MT{plan['mt']}"
        rate = fl / us * 1e-6
        print(f"{side:>3}^2   {cin:>5} {cout:>5} {us:>9.1f} {rate:>8.1f}  {tag:<28} {where}")
        rows.append({"side": side, "cin": cin, "cout": cout, "us": us, "tflops": rate, "plan": plan, "where": where})
    info_after = card()
    print(json.dumps({"card_after": info_after}))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "card_after": info_after, "batch": args.batch, "dtype": args.dtype, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
