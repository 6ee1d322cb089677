"""Regenerates tests/golden/v1_call.npz: the REFERENCE'S OWN GenPercept v1 ``__call__``
(GenPercept_v1/genpercept/pipeline_genpercept.py, in a GenPercept checkout whose path is the first argument) around the
oracle's modules on ``synth_state(1234)`` with the 77-token ``empty_text_embed_77x1024.npy``.  tests/test_gpu_v1.py and
tests/test_v1_cpu.py compare the v1 pipeline with these arrays, so they need no reference tree.

  python tests/golden/make_golden_v1.py /path/to/GenPercept

The reference is imported through make_golden_reference.py's ``diffusers`` shim and ``UNetAdapter``; two more stand-ins
carry no arithmetic of the pipeline: ``BaseOutput`` takes keyword fields, and ``matplotlib.colormaps["Spectral"]``
(matplotlib is not a dependency here) is the 256-entry Spectral table genpercept_b200.image_util builds, indexed as
matplotlib's ``Colormap.__call__`` indexes a float array.  Everything from the PIL image on — Pillow's resize, the
normalisation, batching, single_infer, F.interpolate, min-max, colorize, norm_to_rgb, the uint8 casts — is the
reference's code on the CPU in float32.

Entries per case c:
  in_{c}        the input: uint8 HWC (a PIL RGB image) or float32 [B,3,H,W] in [-1,1]
  kw_{c}        the keyword arguments of the call (a JSON string)
  resized_{c}   uint8 HWC: the Pillow-resized image the engine sees (PIL inputs)
  pred_{c}      pred_np;  colored_{c}: np.asarray(pred_colored), stacked over a list
  range_{c}     depth: per image max - min of the map before the min-max normalisation
  signature     JSON list of (name, default) of __call__
"""
import importlib
import importlib.util
import inspect
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

# (name, input, kwargs); PIL inputs are (W, H, seed)
CASES = [
    ("depth_pil", (101, 77, 1), dict(mode="depth", processing_res=64)),
    ("normal_pil", (97, 150, 2), dict(mode="normal", processing_res=96)),
    ("seg_pil", (101, 77, 3), dict(mode="seg", processing_res=96)),
    ("depth_hard", (97, 150, 4), dict(mode="depth", processing_res=64, resize_hard=True)),
    ("normal_nomatch", (101, 77, 5), dict(mode="normal", processing_res=96, match_input_res=False)),
    ("depth_tensor", (2, 64, 64, 6), dict(mode="depth")),
]


def pil_image(W, H, seed):
    """A smooth seeded photo-like RGB image with some texture."""
    from PIL import Image
    g = torch.Generator().manual_seed(seed)
    base = torch.rand((1, 3, 9, 11), generator=g)
    img = torch.nn.functional.interpolate(base, size=(H, W), mode="bicubic", align_corners=False)[0]
    img = (img + 0.08 * torch.rand((3, H, W), generator=g)).clamp(0, 1)
    return Image.fromarray((img.permute(1, 2, 0).numpy() * 255).astype(np.uint8))


def tensor_image(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    base = torch.rand((B, 3, 8, 8), generator=g)
    return (torch.nn.functional.interpolate(base, size=(H, W), mode="bilinear", align_corners=False) * 2 - 1).clamp(-1, 1)


class _Spectral:
    def __init__(self):
        from genpercept_b200.image_util import _lut
        self.lut = np.concatenate([_lut("Spectral"), np.ones((256, 1))], axis=1)

    def __call__(self, x, bytes=False):
        xa = np.array(x, dtype=np.float64) * 256
        xa[xa == 256] = 255
        idx = np.clip(xa, -1, 256).astype(int).clip(0, 255)
        return self.lut[idx]


def load_v1(ref):
    import make_golden_reference as R
    R.install_shims(ref)

    class BaseOutput:
        def __init__(self, **kw):
            self.__dict__.update(kw)

    sys.modules["diffusers.utils"].BaseOutput = BaseOutput
    sys.modules["matplotlib"].colormaps = {"Spectral": _Spectral()}
    v1_root = f"{ref}/GenPercept_v1"
    spec = importlib.util.spec_from_file_location("genpercept_v1", f"{v1_root}/genpercept/__init__.py",
                                                  submodule_search_locations=[f"{v1_root}/genpercept"])
    pkg = importlib.util.module_from_spec(spec)
    sys.modules["genpercept_v1"] = pkg
    spec.loader.exec_module(pkg)
    return importlib.import_module("genpercept_v1.pipeline_genpercept"), importlib.import_module("genpercept_v1.util.image_util")


def main(ref):
    import make_golden_reference as R
    from genpercept_b200 import weights as W
    from oracle.pipeline import OraclePipeline
    mod, iu = load_v1(ref)
    state = W.synth_state(1234)
    te = torch.from_numpy(np.load(os.path.join(HERE, "empty_text_embed_77x1024.npy")).astype(np.float32))[None]
    op = OraclePipeline(state, te)
    pipe = mod.GenPerceptPipeline(unet=R.UNetAdapter(op.unet), vae=op.vae, empty_text_embed=te)
    out = {}
    sig = inspect.signature(mod.GenPerceptPipeline.__call__)
    out["signature"] = np.array(json.dumps([(n, None if p.default is inspect.Parameter.empty else p.default)
                                            for n, p in sig.parameters.items() if n != "self"]))
    for name, spec, kw in CASES:
        if name.endswith("tensor"):
            x = tensor_image(*spec)
            out[f"in_{name}"] = x.numpy()
            rgb = x
        else:
            img = pil_image(*spec)
            out[f"in_{name}"] = np.asarray(img)
            x = img
            res = kw["processing_res"]
            small = iu.resize_res(img, res) if kw.get("resize_hard") else iu.resize_max_res(img, res)
            out[f"resized_{name}"] = np.asarray(small)
            rgb = torch.from_numpy(np.transpose(np.asarray(small), (2, 0, 1)) / 255.0 * 2.0 - 1.0).float()[None]
        out[f"kw_{name}"] = np.array(json.dumps(kw))
        with torch.no_grad():
            r = pipe(x, show_progress_bar=False, **kw)
            if kw["mode"] == "depth":
                p = pipe.single_infer(rgb, mode="depth")
                size = x.shape[2:] if torch.is_tensor(x) else (x.size[1], x.size[0])
                if kw.get("match_input_res", True):
                    p = torch.nn.functional.interpolate(p, size, mode="bilinear")
                p = p.reshape(p.shape[0], -1)
                out[f"range_{name}"] = (p.max(1)[0] - p.min(1)[0]).numpy()
        out[f"pred_{name}"] = r.pred_np
        col = r.pred_colored if isinstance(r.pred_colored, list) else [r.pred_colored]
        out[f"colored_{name}"] = np.squeeze(np.stack([np.asarray(c) for c in col]))
        print(name, r.pred_np.shape, r.pred_np.dtype, out[f"colored_{name}"].shape)
    path = os.path.join(HERE, "v1_call.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main(sys.argv[1])
