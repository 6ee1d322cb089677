"""Golden vectors for the depth evaluation (genpercept_b200/evaluation.py, oracle/evaluation.py) from the REFERENCE's own
src/util/alignment.py and src/util/metric.py, run on the CPU in the order eval.py uses them (align, disparity -> depth,
dataset clip, clip at 1e-6, the ten metric functions on torch tensors).  Run where the reference checkout exists (it
does not on the GPU box):   python tests/golden/make_golden_eval.py
Writes tests/golden/depth_eval_ref.npz: per case the reference's (scale, shift), its ten metrics and a checksum of the
inputs.  The inputs themselves are regenerated from seeds by cases() below, which the tests import."""
import importlib.util
import os
import sys

import numpy as np

REF = "/root/reference/src/util"
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "depth_eval_ref.npz")

METRICS = ("abs_relative_difference", "squared_relative_difference", "rmse_linear", "rmse_log", "log10",
           "delta1_acc", "delta2_acc", "delta3_acc", "i_rmse", "silog_rmse")

# name, H, W, seed, alignment, max_res, (min_depth, max_depth), kind
CASES = [
    ("nyu_ls", 480, 640, 1, "least_square", None, (1e-3, 10.0), "relative"),
    ("nyu_ls_max1024", 480, 640, 2, "least_square", 1024, (1e-3, 10.0), "relative"),        # factor 1.6: no downscale
    ("nyu_lsd", 480, 640, 3, "least_square_disparity", None, (1e-3, 10.0), "disparity"),
    ("kitti_ls_max1024", 352, 1216, 4, "least_square", 1024, (1e-5, 80.0), "relative"),
    ("kitti_lsd_max1024", 352, 1216, 5, "least_square_disparity", 1024, (1e-5, 80.0), "disparity"),
    ("kitti_none", 352, 1216, 6, None, None, (1e-5, 80.0), "metric"),
    ("odd_ls_max200", 333, 517, 7, "least_square", 200, (1e-3, 10.0), "relative"),
    ("ragged_lsd_max20", 37, 53, 8, "least_square_disparity", 20, (1e-3, 10.0), "disparity"),
    ("tiny_ls", 3, 5, 9, "least_square", None, (1e-3, 10.0), "relative"),
    ("constant_ls", 64, 96, 10, "least_square", None, (1e-3, 10.0), "constant"),
    ("constant_lsd_max50", 64, 96, 11, "least_square_disparity", 50, (1e-3, 10.0), "constant"),
    ("empty_ls", 48, 64, 12, "least_square", None, (1e-3, 10.0), "empty"),
]


def make_inputs(H, W, seed, kind, scale_m):
    """Seeded (pred fp32, gt fp32, valid bool) of one case: a smooth positive depth field with zeros where the ground
    truth is missing, and a prediction that is an affine map of depth (relative), of inverse depth with some negative
    values (disparity), the depth itself plus noise (metric), or one value (constant); no valid pixel (empty)."""
    rng = np.random.default_rng(seed)
    y = np.linspace(0.0, 1.0, H, dtype=np.float64)[:, None]
    x = np.linspace(0.0, 1.0, W, dtype=np.float64)[None, :]
    f = rng.uniform(1.0, 3.0, 4)
    gt = 1.0 + 0.45 * (np.sin(2 * np.pi * (f[0] * x + f[1] * y)) + 1.0) + 0.3 * np.cos(2 * np.pi * f[2] * x * y)
    gt = gt * scale_m * rng.uniform(0.8, 1.2, (H, W))
    valid = rng.random((H, W)) > 0.2
    gt = np.where(valid | (rng.random((H, W)) < 0.5), gt, 0.0)        # missing ground truth: some zeros, some not
    noise = rng.normal(0.0, 0.05, (H, W))
    if kind in ("relative", "empty"):
        pred = (gt - gt.min()) / (gt.max() - gt.min()) * 0.9 + 0.05 + noise
    elif kind == "disparity":
        pred = np.where(gt > 0, 1.0 / np.maximum(gt, 1e-6), 0.0) * 0.7 + 0.02 + noise * 0.3
        pred = np.where(rng.random((H, W)) < 0.03, -pred, pred)
    elif kind == "metric":
        pred = gt * 1.05 + noise * scale_m
    else:
        pred = np.full((H, W), 0.37)
    if kind == "empty":
        valid = np.zeros((H, W), dtype=bool)
    return pred.astype(np.float32), gt.astype(np.float32), valid


def cases():
    """[(name, pred, gt, valid, alignment, max_res, min_depth, max_depth)] of the golden, regenerated from the seeds."""
    out = []
    for name, H, W, seed, alignment, max_res, (lo, hi), kind in CASES:
        scale_m = 10.0 if name.startswith("kitti") else 2.0
        pred, gt, valid = make_inputs(H, W, seed, kind, scale_m)
        out.append((name, pred, gt, valid, alignment, max_res, lo, hi))
    return out


def checksum(pred, gt, valid):
    return np.array([pred.astype(np.float64).sum(), gt.astype(np.float64).sum(), valid.sum()], dtype=np.float64)


def _load(name):
    spec = importlib.util.spec_from_file_location(f"ref_{name}", os.path.join(REF, f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    import torch
    A, M = _load("alignment"), _load("metric")
    out = {"names": np.array([c[0] for c in CASES])}
    for name, pred, gt, valid, alignment, max_res, lo, hi in cases():
        scale = shift = np.full((1,), np.nan, dtype=np.float32)
        depth = pred
        if alignment == "least_square":
            depth, scale, shift = A.align_depth_least_square(gt_arr=gt, pred_arr=pred, valid_mask_arr=valid,
                                                             return_scale_shift=True, max_resolution=max_res)
        elif alignment == "least_square_disparity":
            gt_disp, gt_pos = A.depth2disparity(depth=gt, return_mask=True)
            disp, scale, shift = A.align_depth_least_square(gt_arr=gt_disp, pred_arr=pred,
                                                            valid_mask_arr=valid & gt_pos & (pred > 0),
                                                            return_scale_shift=True, max_resolution=max_res)
            depth = A.disparity2depth(np.clip(disp, a_min=1e-3, a_max=None))
        depth = np.clip(np.clip(depth, a_min=lo, a_max=hi), a_min=1e-6, a_max=None)
        assert depth.dtype == np.float32 and np.asarray(scale).dtype == np.float32
        p_t, g_t, v_t = torch.from_numpy(depth), torch.from_numpy(gt), torch.from_numpy(valid)
        vals = np.array([getattr(M, m)(p_t, g_t, v_t).item() for m in METRICS], dtype=np.float64)
        out[f"{name}.scale_shift"] = np.array([np.asarray(scale).item(), np.asarray(shift).item()], dtype=np.float32)
        out[f"{name}.metrics"] = vals
        out[f"{name}.checksum"] = checksum(pred, gt, valid)
        print(name, pred.shape, alignment, max_res, out[f"{name}.scale_shift"], vals[[0, 2, 5]])
    np.savez_compressed(GOLDEN, **out)


if __name__ == "__main__":
    sys.exit(main())
