"""Host-side image helpers mirroring /root/reference/genpercept/util/image_util.py
(resize_max_res :75, get_tv_resample_method :108, colorize_depth_maps :25, chw2hwc :66)."""
import numpy as np
import torch
from torchvision.transforms import InterpolationMode
from torchvision.transforms.functional import resize

# ColorBrewer "Spectral" (11 classes) — the anchors of matplotlib's 'Spectral' colormap; the
# reference calls matplotlib.colormaps['Spectral'] (image_util.py:44) which interpolates them
# linearly into a 256-entry LUT.  matplotlib is not a dependency here.
_SPECTRAL = np.array([(158, 1, 66), (213, 62, 79), (244, 109, 67), (253, 174, 97), (254, 224, 139),
                      (255, 255, 191), (230, 245, 152), (171, 221, 164), (102, 194, 165), (50, 136, 189),
                      (94, 79, 162)], dtype=np.float64) / 255.0


def _lut(cmap):
    try:
        import matplotlib
        cm = matplotlib.colormaps[cmap]
        return cm(np.linspace(0, 1, 256))[:, :3]
    except Exception:
        if cmap != "Spectral":
            raise ValueError(f"colormap {cmap!r} needs matplotlib; only 'Spectral' is built in")
        x = np.linspace(0, 1, 256)
        xp = np.linspace(0, 1, len(_SPECTRAL))
        return np.stack([np.interp(x, xp, _SPECTRAL[:, c]) for c in range(3)], axis=1)


def colorize_depth_maps(depth_map, min_depth, max_depth, cmap="Spectral", valid_mask=None):
    assert len(depth_map.shape) >= 2, "Invalid dimension"
    if isinstance(depth_map, torch.Tensor):
        depth = depth_map.detach().squeeze().cpu().numpy()
    else:
        depth = np.asarray(depth_map).copy().squeeze()
    if depth.ndim < 3:
        depth = depth[np.newaxis, :, :]
    depth = ((depth - min_depth) / (max_depth - min_depth)).clip(0, 1)
    lut = _lut(cmap)
    idx = (depth * 256).astype(np.int64).clip(0, 255)       # matplotlib: floor(x*N), x==1 -> N-1
    img = np.rollaxis(lut[idx], 3, 1)                        # [B,3,H,W], values 0..1
    if valid_mask is not None:
        vm = np.asarray(valid_mask).squeeze()
        vm = vm[np.newaxis, np.newaxis] if vm.ndim < 3 else vm[:, np.newaxis]
        img[~np.repeat(vm, 3, axis=1)] = 0
    return torch.from_numpy(img).float() if isinstance(depth_map, torch.Tensor) else img


def chw2hwc(chw):
    assert 3 == len(chw.shape)
    if isinstance(chw, torch.Tensor):
        return torch.permute(chw, (1, 2, 0))
    return np.moveaxis(chw, 0, -1)


def resize_max_res(img, max_edge_resolution, resample_method=InterpolationMode.BILINEAR):
    assert 4 == img.dim(), f"Invalid input shape {img.shape}"
    h, w = img.shape[-2:]
    f = min(max_edge_resolution / w, max_edge_resolution / h)
    return resize(img, (int(h * f), int(w * f)), resample_method, antialias=True)


def get_tv_resample_method(method_str):
    d = {"bilinear": InterpolationMode.BILINEAR, "bicubic": InterpolationMode.BICUBIC,
         "nearest": InterpolationMode.NEAREST_EXACT, "nearest-exact": InterpolationMode.NEAREST_EXACT}
    m = d.get(method_str, None)
    if m is None:
        raise ValueError(f"Unknown resampling method: {m}")
    return m


# Below this many pixels Pillow's host decode is the faster one: the GPU decode (upload, about 20 launches, two status
# reads) has a floor of about 1.5 ms.  bench_jpeg.py, two runs on an NVIDIA H100 80GB HBM3 at 700 W with an 8-core host,
# q90 4:2:0, GPU / Pillow: 640 x 480 2.01-2.02 / 3.90-5.02 ms, 480 x 360 2.08-2.11 / 2.17-3.82 ms, 320 x 240
# 1.71-1.78 / 1.26-1.30 ms, 160 x 120 1.40-1.51 / 0.80-1.34 ms.
JPEG_GPU_MIN_PIXELS = 480 * 360


def decode_unloaded_jpeg(img, device, layout):
    """The RGB bytes of ``img.convert("RGB")`` decoded on the GPU (engine.decode_jpeg) when `img` is a JPEG that PIL
    opened but has not loaded (format JPEG, mode RGB, one pending tile, no ``draft()``), has at least
    JPEG_GPU_MIN_PIXELS pixels, and whose stream the GPU decoder takes; None otherwise, and when the device decode rejects the stream (corrupt, or not converged), so the caller
    runs Pillow's own decode and the user sees Pillow's result or error.  The file's bytes are read without loading
    the image, and its position is restored.  Returns uint8 [3,H,W] ("chw") or [H,W,3] ("hwc") on `device`."""
    from PIL import JpegImagePlugin
    from . import engine as E
    if not (isinstance(img, JpegImagePlugin.JpegImageFile) and img.format == "JPEG" and img.mode == "RGB"
            and len(img.tile) == 1 and img.tile[0][0] == "jpeg" and not img.decoderconfig
            and getattr(img, "fp", None) is not None and img.size[0] * img.size[1] >= JPEG_GPU_MIN_PIXELS):
        return None
    fp = img.fp
    pos = fp.tell()
    try:
        fp.seek(img.tile[0][2])
        data = fp.read()
    finally:
        fp.seek(pos)
    try:
        E.jpeg_probe(data)
    except ValueError:
        return None
    try:
        return E.decode_jpeg(data, device=device, layout=layout)
    except ValueError:
        return None
