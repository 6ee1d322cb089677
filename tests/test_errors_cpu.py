"""The error path of the C-ABI calls that take no engine: calls that fail before any device call return their status,
leave a reason in gp_last_call_error(), and the Python wrappers raise with both the status name and that reason.  A
successful call clears the reason.  No device is needed."""
from ctypes import byref, c_int, c_void_p

import numpy as np
import pytest
import torch

from genpercept_b200 import build
from genpercept_b200 import engine as E

P = c_void_p(16)   # a non-null pointer the calls below reject before they read it
F32 = torch.float32


def _zeros(*shape, dtype=F32):
    return torch.zeros(shape, dtype=dtype)


# (status, a fragment of the reason, the raw call, the Python wrapper's call or None).  A wrapper that checks the
# argument of the raw call on the host first is driven with another argument the library rejects with the same reason.
CASES = {
    "resize_aa_mode": (1, "gp_resize_aa",
                       lambda L: L.gp_resize_aa(P, E.GP_U8, 1, 1, 4, 4, P, E.GP_U8, 1, 2, 2, 2, None),
                       lambda: E.resize_aa(_zeros(4, 4, dtype=torch.uint8), 0, 2)),
    "colorize_range": (1, "gp_colorize",
                       lambda L: L.gp_colorize(P, 1, 1, 4, 4, 1.0, 0.0, P, P, 1, None),
                       lambda: E.colorize(_zeros(1, 4, 4), np.zeros((256, 3), np.uint8), vmin=1.0, vmax=0.0)),
    "quantize_bits": (1, "gp_quantize", lambda L: L.gp_quantize(P, 1, 16, 7, P, 1, None), None),
    "resize_pil_null": (1, "gp_resize_pil",
                        lambda L: L.gp_resize_pil(None, 1, 4, 4, P, 1, 2, 2, None),
                        lambda: E.resize_pil(np.zeros((4, 4, 3), np.uint8), 0, 2, device="cpu")),
    "v1_postprocess_task": (1, "gp_v1_postprocess",
                            lambda L: L.gp_v1_postprocess(P, 1, 1, 4, 4, 3, 8, 8, P, P, None), None),
    "depth_align_mode": (1, "gp_depth_align",
                         lambda L: L.gp_depth_align(P, P, None, 1, 4, 4, 2, 0, P, None, None),
                         lambda: E.depth_align(_zeros(1, 4, 4), _zeros(1, 4, 4), None, mode=2)),
    "depth_metrics_mode": (1, "gp_depth_metrics",
                           lambda L: L.gp_depth_metrics(P, P, None, 1, 4, 4, 3, P, 0.0, 1.0, P, None),
                           lambda: E.depth_metrics(_zeros(1, 4, 4), _zeros(1, 4, 4), None, mode=3)),
    "jpeg_probe_short": (1, "no SOI",
                         lambda L: L.gp_jpeg_probe(b"xx", 2, None, None, None),
                         lambda: E.jpeg_probe(b"xx")),
    "conv2d_ks": (1, "gp_conv2d",
                  lambda L: L.gp_conv2d(E.GP_F16, P, 1, 4, 4, 8, P, None, 8, 2, 0, None, 0, P, 0, None),
                  lambda: E.conv2d(_zeros(1, 4, 4, 8, dtype=torch.float16), _zeros(8, 8, 2, 2))),
    "groupnorm_groups": (1, "gp_groupnorm",
                         lambda L: L.gp_groupnorm(E.GP_F16, P, 1, 4, 4, 8, 0, P, P, 1e-5, 0, P, None),
                         lambda: E.groupnorm(_zeros(1, 4, 4, 8, dtype=torch.float16), 0, _zeros(8), _zeros(8), 1e-5,
                                             False)),
    "tile_shape_cout": (1, "gp_tile_shape",
                        lambda L: L.gp_tile_shape(0, 128, 3, 8, 768, 768, 0, 132, byref(c_int()), byref(c_int())),
                        lambda: E.tile_shape(0, 128, 3, 8, 768, 768)),
    "conv_tile_cout": (1, "gp_conv_tile",
                       lambda L: L.gp_conv_tile(128, 0, 0, 8, 96, 96, 132, byref(c_int()), byref(c_int()),
                                                byref(c_int())),
                       lambda: E.conv_tile(8, 96, 96, 128, 0)),
    "step_bias_layout_null": (1, "gp_step_bias_layout", lambda L: L.gp_step_bias_layout(0, None, None, None), None),
    "shared_arena_fill_no_pool": (5, "no engine on device 999",
                                  lambda L: L.gp_shared_arena_fill(999, 0, None),
                                  lambda: E.shared_arena_fill(0, device=999)),
    "create_f32": (1, "gp_create",
                   lambda L: L.gp_create(byref(E._Config(0, E.GP_F32, 0, 1, 0)), byref(c_void_p())),
                   lambda: E.Engine(dtype=F32)),
}


@pytest.fixture(scope="module")
def L():
    build.build()
    return E.lib()


@pytest.fixture
def no_device_needed(monkeypatch):
    """Lets the wrappers reach the library without a device: the failing calls never use the stream."""
    monkeypatch.setattr(E, "_stream_ptr", lambda device=None: None)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)


@pytest.mark.parametrize("case", list(CASES))
def test_failure_status_and_reason(L, no_device_needed, case):
    status, fragment, raw, wrapper = CASES[case]
    assert raw(L) == status
    reason = L.gp_last_call_error().decode()
    assert fragment in reason, reason
    if wrapper is None:
        return
    with pytest.raises((RuntimeError, ValueError)) as ex:
        wrapper()
    assert E._STATUS[status] in str(ex.value) and reason in str(ex.value), str(ex.value)


def test_success_clears_the_reason(L):
    assert L.gp_tile_shape(0, 128, 3, 8, 768, 768, 0, 132, byref(c_int()), byref(c_int())) == 1
    assert L.gp_last_call_error().decode() != ""
    bn, mt = c_int(), c_int()
    assert L.gp_tile_shape(128, 128, 3, 8, 768, 768, 0, 132, byref(bn), byref(mt)) == 0
    assert L.gp_last_call_error().decode() == ""
    assert (bn.value, mt.value) == (128, 1)

