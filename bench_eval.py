#!/usr/bin/env python
"""Depth evaluation speed: the fused GPU evaluation (genpercept_b200.evaluation.evaluate -> csrc/evaluate.cu) against
the reference's per-sample path as eval.py runs it (eval.py:168-215): boolean indexing + np.linalg.lstsq on the host,
the host clips, an upload of the aligned map, then one torch call per metric on the GPU, with the host copies
threshold_percentage makes (metric.py:101-115).  The reference path is restated here; the reference is not imported.

  python bench_eval.py [--iters N] [--alignment least_square|least_square_disparity] [--max-res R]

Prints ONE JSON line with, per size (NYUv2 480 x 640, KITTI 352 x 1216, ETH3D 4032 x 6048; batch 1 as eval.py):
  fused_us / reference_us   microseconds per image (host clock around device-synchronised calls; the maps are on
                            the device for the fused path and on the host for the reference path, as each receives them)
  metrics_pass_us           the metrics kernel alone (gp_depth_metrics, CUDA events), its bytes (pred + gt + mask read
                            once) and achieved GB/s next to the H100 SXM data-sheet 3.35 TB/s (not a measured figure)
and the card's name and power limit, read in the same run.  Inputs are seeded synthetic maps; nothing is written.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

SIZES = {"nyuv2": (480, 640), "kitti": (352, 1216), "eth3d": (4032, 6048)}
HBM_DATASHEET_GBS = 3350.0


def reference_path(pred, gt, valid, alignment, max_res, lo, hi, dev):
    """eval.py's per-sample body with the reference's operations (numpy alignment, torch metrics on `dev`)."""
    if alignment == "least_square_disparity":
        pos = gt > 0
        target = np.zeros_like(gt)
        target[pos] = 1.0 / gt[pos]
        mask = valid & pos & (pred > 0)
    else:
        target, mask = gt, valid
    p_fit, g_fit, m_fit = pred, target, mask
    if max_res is not None:
        s = np.min(max_res / np.array(pred.shape[-2:]))
        if s < 1:
            up = torch.nn.Upsample(scale_factor=s, mode="nearest")
            p_fit = up(torch.as_tensor(pred).unsqueeze(0)).numpy()[0]
            g_fit = up(torch.as_tensor(target).unsqueeze(0)).numpy()[0]
            m_fit = up(torch.as_tensor(mask).unsqueeze(0).float()).bool().numpy()[0]
    pm = p_fit[m_fit].reshape(-1, 1)
    A = np.concatenate([pm, np.ones_like(pm)], axis=-1)
    scale, shift = np.linalg.lstsq(A, g_fit[m_fit].reshape(-1, 1), rcond=None)[0]
    d = pred * scale + shift
    if alignment == "least_square_disparity":
        d = np.clip(d, 1e-3, None)
        inv = np.zeros_like(d)
        inv[d > 0] = 1.0 / d[d > 0]
        d = inv
    d = np.clip(np.clip(d, lo, hi), 1e-6, None)
    p, g, m = torch.from_numpy(d).to(dev), torch.from_numpy(gt).to(dev), torch.from_numpy(valid).to(dev)
    n = m.sum((-1, -2))
    out = []

    def masked_mean(x):
        x[~m] = 0
        return torch.sum(x, (-1, -2)) / n
    out.append(masked_mean(torch.abs(p - g) / g).mean().item())
    out.append(masked_mean(torch.pow(torch.abs(p - g), 2) / g).mean().item())
    out.append(torch.sqrt(masked_mean(torch.pow(p - g, 2))).mean().item())
    out.append(torch.sqrt(masked_mean(torch.pow(torch.log(p) - torch.log(g), 2))).mean().item())
    out.append(torch.abs(torch.log10(p[m]) - torch.log10(g[m])).mean().item())
    for k in (1, 2, 3):
        r = torch.max(p / g, g / p)
        bit = torch.where(r.cpu() < 1.25 ** k, torch.ones(*p.shape), torch.zeros(*p.shape))
        bit[~m.cpu()] = 0
        out.append((torch.sum(bit, (-1, -2)) / n.cpu()).mean().item())
    out.append(torch.sqrt(masked_mean(torch.pow(1.0 / p - 1.0 / g, 2))).mean().item())
    ld = torch.log(p) - torch.log(g)
    ld[~m] = 0
    out.append((torch.sqrt(torch.mean(torch.sum(ld ** 2, (-1, -2)) / n - torch.sum(ld, (-1, -2)) ** 2 / n ** 2)) * 100).item())
    return out


def inputs(H, W, seed):
    rng = np.random.default_rng(seed)
    gt = (rng.random((H, W), dtype=np.float32) * 9 + 0.5).astype(np.float32)
    valid = rng.random((H, W)) > 0.2
    pred = ((gt - 0.5) / 9 + rng.normal(0, 0.03, (H, W))).astype(np.float32)
    return pred, gt, valid


def device_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
    except Exception as ex:  # noqa: BLE001
        name, power, clock = torch.cuda.get_device_name(0), f"unknown ({ex})", "unknown"
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--alignment", default="least_square", choices=["least_square", "least_square_disparity"])
    ap.add_argument("--max-res", type=int, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_eval.py measures the GPU evaluation and needs a CUDA device")
    from genpercept_b200 import engine as E
    from genpercept_b200.evaluation import METRICS, evaluate
    dev = torch.device("cuda", 0)
    lo, hi = 1e-5, 80.0
    res = {"alignment": args.alignment, "max_res": args.max_res, "sizes": {}}
    for name, (H, W) in SIZES.items():
        pred, gt, valid = inputs(H, W, 1)
        if args.alignment == "least_square_disparity":
            pred = np.where(gt > 0, 1.0 / gt, 0).astype(np.float32) * 0.8 + 0.01
        p, g, v = (torch.from_numpy(x).to(dev) for x in (pred, gt, valid))
        for _ in range(10):                                                          # warm-up (module load, clocks)
            m, _, _ = evaluate(p, g, v, args.alignment, args.max_res, lo, hi)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.iters):
            m, _, _ = evaluate(p, g, v, args.alignment, args.max_res, lo, hi)
            vals = torch.cat([m[k] for k in METRICS]).cpu()                      # the 10 numbers reach the host
        fused_us = (time.perf_counter() - t0) / args.iters * 1e6
        # the metrics pass alone
        p3, g3, v3 = p[None], g[None], v[None].to(torch.uint8)
        ss, _ = E.depth_align(p3, g3, v3, mode=1 if args.alignment == "least_square_disparity" else 0,
                              max_res=args.max_res or 0)
        mode = 2 if args.alignment == "least_square_disparity" else 1
        E.depth_metrics(p3, g3, v3, mode, ss, lo, hi)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = max(args.iters, 50)
        e0.record()
        for _ in range(reps):
            E.depth_metrics(p3, g3, v3, mode, ss, lo, hi)
        e1.record()
        torch.cuda.synchronize()
        pass_us = e0.elapsed_time(e1) / reps * 1e3
        nbytes = H * W * (4 + 4 + 1)
        ref_iters = 2 if H * W > 4e6 else max(3, args.iters // 4)
        reference_path(pred, gt, valid, args.alignment, args.max_res, lo, hi, dev)      # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(ref_iters):
            ref = reference_path(pred, gt, valid, args.alignment, args.max_res, lo, hi, dev)
        torch.cuda.synchronize()
        ref_us = (time.perf_counter() - t0) / ref_iters * 1e6
        rel = float(np.nanmax(np.abs(vals.numpy() - np.array(ref)) / np.maximum(np.abs(np.array(ref)), 1e-30)))
        res["sizes"][name] = {"H": H, "W": W, "fused_us": round(fused_us, 1), "reference_us": round(ref_us, 1),
                              "speedup": round(ref_us / fused_us, 1), "metrics_pass_us": round(pass_us, 2),
                              "metrics_pass_bytes": nbytes, "metrics_pass_GBs": round(nbytes / pass_us / 1e3, 1),
                              "datasheet_GBs": HBM_DATASHEET_GBS,
                              "metrics_pass_of_datasheet": round(nbytes / pass_us / 1e3 / HBM_DATASHEET_GBS, 3),
                              "max_rel_diff_vs_reference_path": rel}
    res["device"] = device_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
