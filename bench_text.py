"""Times SD-2.1's CLIP text tower (encode_text) at n = 2, 8 and 77 tokens in each engine mode, on synth_text_state weights:

  engine       Engine.encode_text (gp_encode_text): ids in, fp32 [1, n, 1024] out on the host
  host fp32    transformers.CLIPTextModel on the CPU in fp32, the pipeline's path before the tower moved to the engine
  gpu <dtype>  transformers.CLIPTextModel on the GPU in the pipeline's dtype (fp16 / bf16 / fp32), the reference's path
               (run.py's pipe.to(dtype)); skipped without transformers

Each number is the mean of --iters calls after --warmup calls (host clock; every call ends in a device synchronisation).
It also reports the device memory the tower holds before gp_finalize and what the engine holds after it.  Prints the card
and its power limit, one JSON line per measurement and a table.
"""
import argparse
import json
import subprocess
import time

import torch

from genpercept_b200 import weights as W
from genpercept_b200.engine import Engine

MODES = {"fp16": (torch.float16, "default", torch.float16), "bf16": (torch.bfloat16, "default", torch.bfloat16),
         "high": (torch.float16, "high", torch.float32)}
NS = (2, 8, 77)


def _ids(n):
    return [49406] + [(1000 + 613 * i) % 49408 for i in range(n - 2)] + [49407]


def _time(fn, warmup, iters, sync=False):
    for _ in range(warmup):
        fn()
    if sync:
        torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    if sync:
        torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3 / iters


def _free():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-iters", type=int, default=3)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(f"card: {card}")
    sd = W.synth_text_state(1234)
    img = W.synth_state(1234, with_dpt=False)
    rows = []
    for mode, (storage, precision, _) in MODES.items():
        e = Engine(dtype=storage, precision=precision)
        e.load_state("unet", img["unet"])
        e.load_state("vae", img["vae"])
        e.load_state("text", sd)
        f0 = _free()
        for n in NS:
            ms = _time(lambda: e.encode_text(_ids(n)), a.warmup, a.iters)
            rows.append({"path": "engine", "mode": mode, "n": n, "ms": round(ms, 3)})
            print(json.dumps(rows[-1]))
        tower = f0 - _free()
        e.set_text_embed(e.encode_text(_ids(2)))
        e.finalize()
        held = f0 - _free()
        rows.append({"path": "memory", "mode": mode, "tower_mib_before_finalize": round(tower / 2 ** 20, 1),
                     "engine_mib_after_finalize": round(held / 2 ** 20, 1)})
        print(json.dumps(rows[-1]))
        e.close()
    try:
        import transformers
    except ImportError:
        transformers = None
    if transformers is not None:
        cfg = transformers.CLIPTextConfig(vocab_size=49408, hidden_size=1024, intermediate_size=4096, num_hidden_layers=23,
                                          num_attention_heads=16, max_position_embeddings=77, hidden_act="gelu",
                                          layer_norm_eps=1e-5, projection_dim=512)
        model = transformers.CLIPTextModel(cfg).eval()
        model.load_state_dict(sd, strict=False)
        with torch.no_grad():
            for n in NS:
                ids = torch.tensor([_ids(n)])
                ms = _time(lambda: model(ids), 1, a.host_iters)
                rows.append({"path": "host fp32", "mode": "any", "n": n, "ms": round(ms, 3)})
                print(json.dumps(rows[-1]))
            for mode, (_, _, dt) in MODES.items():
                m = model.to("cuda", dt)
                for n in NS:
                    ids = torch.tensor([_ids(n)], device="cuda")
                    ms = _time(lambda: m(ids), a.warmup, a.iters, sync=True)
                    rows.append({"path": f"gpu {str(dt).split('.')[-1]}", "mode": mode, "n": n, "ms": round(ms, 3)})
                    print(json.dumps(rows[-1]))
    print(f"\nencode_text, ms per call ({card}):")
    print("| path | mode | " + " | ".join(f"n = {n}" for n in NS) + " |")
    print("|---|---|" + "---|" * len(NS))
    keys = []
    for r in rows:
        if "ms" in r and (r["path"], r["mode"]) not in keys:
            keys.append((r["path"], r["mode"]))
    for k in keys:
        vals = {r["n"]: r["ms"] for r in rows if "ms" in r and (r["path"], r["mode"]) == k}
        print(f"| {k[0]} | {k[1]} | " + " | ".join(f"{vals[n]:.2f}" for n in NS) + " |")


if __name__ == "__main__":
    main()
