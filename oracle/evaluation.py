"""CPU oracle of the depth evaluation (eval.py's alignment and ten metrics), restated from their definitions.

The aligned map is computed with the reference's float32 rounding (numpy float32: pred * scale, then + shift, then
the clips); the least-squares fit and every metric sum are fp64.  Single images [H, W], numpy or torch inputs."""
import math

import numpy as np
import torch

METRICS = ("abs_relative_difference", "squared_relative_difference", "rmse_linear", "rmse_log", "log10",
           "delta1_acc", "delta2_acc", "delta3_acc", "i_rmse", "silog_rmse")


def fit_grid(H, W, max_res):
    """(fit width, float32 1/s or None) of align_depth_least_square's optional downscale.  s = min(max_res / (H, W)) in
    fp64; below 1 the reference resamples the [1, H, W] map with torch.nn.Upsample(scale_factor=s, mode="nearest"),
    which treats it as one 1-D signal of W samples per row: the rows stay, the width becomes floor(W * s)."""
    if max_res is None:
        return W, None
    s = min(max_res / H, max_res / W)
    if s >= 1:
        return W, None
    return int(math.floor(W * s)), np.float32(1.0 / s)


def nearest_index(in_size, out_size, inv_scale):
    """Source index of each of `out_size` nearest-resampled samples: min(floor(float32(dst) * float32(1/s)), in - 1)."""
    dst = np.arange(out_size, dtype=np.float32)
    return np.minimum(np.floor(dst * np.float32(inv_scale)).astype(np.int64), in_size - 1)


def _np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def least_squares(pred, gt, valid, disparity=False, max_res=None):
    """(scale, shift) as float32: the least-squares fit of gt ~ scale * pred + shift over the valid pixels of the fit
    grid, fp64 (LAPACK gelsd: the minimum-norm solution when the system is rank deficient; (0, 0) when it is empty).
    disparity: the target is 1/gt (float32) where gt > 0, and the mask also needs gt > 0 and pred > 0."""
    p = _np(pred).astype(np.float32)
    g = _np(gt).astype(np.float32)
    m = _np(valid).astype(bool)
    if disparity:
        pos = g > 0
        m = m & pos & (p > 0)
        g = np.where(pos, np.float32(1.0) / np.where(pos, g, np.float32(1.0)), np.float32(0.0)).astype(np.float32)
    fit_w, inv = fit_grid(p.shape[-2], p.shape[-1], max_res)
    if inv is not None:
        idx = nearest_index(p.shape[-1], fit_w, inv)
        p, g, m = p[:, idx], g[:, idx], m[:, idx]
    pv = torch.from_numpy(p[m].astype(np.float64))
    gv = torch.from_numpy(g[m].astype(np.float64))
    if pv.numel() == 0:
        return np.float32(0.0), np.float32(0.0)
    A = torch.stack([pv, torch.ones_like(pv)], dim=1)
    x = torch.linalg.lstsq(A, gv[:, None], driver="gelsd").solution[:, 0]
    return np.float32(x[0].item()), np.float32(x[1].item())


def aligned_depth(pred, scale, shift, alignment, min_depth, max_depth):
    """The map eval.py scores (float32): pred * scale + shift (in disparity: clipped at 1e-3 and inverted), then the
    dataset clip [min_depth, max_depth] and the clip at 1e-6."""
    p = _np(pred).astype(np.float32)
    if alignment is not None:
        p = (p * np.float32(scale)).astype(np.float32) + np.float32(shift)
        if alignment == "least_square_disparity":
            p = np.maximum(p, np.float32(1e-3))
            p = np.float32(1.0) / p
    p = np.minimum(np.maximum(p, np.float32(min_depth)), np.float32(max_depth))
    return np.maximum(p, np.float32(1e-6)).astype(np.float32)


def metrics(pred, gt, valid):
    """The ten metrics of one image from their definitions, fp64 over the valid pixels (n of them):
    mean |p-g|/g, mean (p-g)^2/g, sqrt mean (p-g)^2, sqrt mean (ln p - ln g)^2, mean |log10 p - log10 g|,
    fraction with max(p/g, g/p) < 1.25^k (the ratio in float32, k = 1..3), sqrt mean (1/p - 1/g)^2,
    100 sqrt(mean l^2 - (mean l)^2) with l = ln p - ln g.  No valid pixel: NaN."""
    m = torch.from_numpy(_np(valid).astype(bool))
    p32 = torch.from_numpy(_np(pred).astype(np.float32))[m]
    g32 = torch.from_numpy(_np(gt).astype(np.float32))[m]
    p, g = p32.double(), g32.double()
    n = float(m.sum())
    if n == 0:
        return {k: float("nan") for k in METRICS}
    d = p - g
    lg = torch.log(p) - torch.log(g)
    ratio = torch.maximum(p32 / g32, g32 / p32)
    out = {
        "abs_relative_difference": (d.abs() / g).sum() / n,
        "squared_relative_difference": (d * d / g).sum() / n,
        "rmse_linear": torch.sqrt((d * d).sum() / n),
        "rmse_log": torch.sqrt((lg * lg).sum() / n),
        "log10": (torch.log10(p) - torch.log10(g)).abs().sum() / n,
        "delta1_acc": (ratio < 1.25).sum() / n,
        "delta2_acc": (ratio < 1.25 ** 2).sum() / n,
        "delta3_acc": (ratio < 1.25 ** 3).sum() / n,
        "i_rmse": torch.sqrt(((1.0 / p - 1.0 / g) ** 2).sum() / n),
        "silog_rmse": torch.sqrt((lg * lg).sum() / n - (lg.sum() / n) ** 2) * 100,
    }
    return {k: float(v) for k, v in out.items()}


def evaluate(pred, gt, valid, alignment=None, max_res=None, min_depth=0.0, max_depth=1e8):
    """One image [H, W] through eval.py's steps.  Returns (metrics dict, scale, shift); (1, 0) without alignment."""
    scale, shift = np.float32(1.0), np.float32(0.0)
    if alignment is not None:
        scale, shift = least_squares(pred, gt, valid, alignment == "least_square_disparity", max_res)
    p = aligned_depth(pred, scale, shift, alignment, min_depth, max_depth)
    return metrics(p, gt, valid), scale, shift
