"""ctypes binding of libgenpercept_b200.so (include/genpercept_b200.h).

PyTorch is used only for device memory, streams and dtype bookkeeping; every numerical op of the
hot path runs inside the native library.  There is no CPU fallback: if the library or a CUDA device
is missing, construction raises.
"""
import ctypes
import os
import warnings
from ctypes import POINTER, byref, c_char_p, c_double, c_float, c_int, c_int64, c_size_t, c_void_p

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgenpercept_b200.so")

GP_F32, GP_F16, GP_BF16, GP_U8, GP_F16_PAIR = 0, 1, 2, 3, 4
GP_READOUT_VAE, GP_READOUT_DPT = 0, 1
STAGE_PRE, STAGE_VAE_ENCODE, STAGE_UNET, STAGE_READOUT = 0, 1, 2, 3
_STATUS = {0: "GP_OK", 1: "GP_ERR_INVALID", 2: "GP_ERR_MISSING", 3: "GP_ERR_NO_PLAN", 4: "GP_ERR_CUDA",
           5: "GP_ERR_STATE"}


class _Config(ctypes.Structure):
    _fields_ = [("device", c_int), ("dtype", c_int), ("readout", c_int), ("timestep", c_int),
                ("use_cuda_graph", c_int), ("precision", c_int), ("arch", c_int)]


_lib = None


def lib():
    """Loads the native library (fails loudly when it has not been built)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} not built: run `python -m genpercept_b200.build` "
                           "(or __graft_entry__.build()); there is no fallback path")
    L = ctypes.CDLL(LIB_PATH)
    L.gp_create.argtypes = [POINTER(_Config), POINTER(c_void_p)]
    L.gp_destroy.argtypes = [c_void_p]
    L.gp_destroy.restype = None
    L.gp_last_error.argtypes = [c_void_p]
    L.gp_last_error.restype = c_char_p
    L.gp_load_tensor.argtypes = [c_void_p, c_char_p, c_void_p, c_int, POINTER(c_int64), c_int]
    L.gp_set_text_embed.argtypes = [c_void_p, c_void_p, c_int, c_int]
    L.gp_finalize.argtypes = [c_void_p]
    L.gp_plan.argtypes = [c_void_p, c_int, c_int, c_int]
    L.gp_infer.argtypes = [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p]
    L.gp_run_stage.argtypes = [c_void_p, c_int, c_int, c_void_p]
    L.gp_encode.argtypes = [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]
    L.gp_decode.argtypes = [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p]
    L.gp_encode_exact.argtypes = [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]
    L.gp_infer_latent.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p]
    L.gp_set_timestep.argtypes = [c_void_p, c_int]
    L.gp_infer_steps.argtypes = [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, POINTER(c_int), POINTER(c_float), c_int, c_void_p,
                                 c_int, c_int, c_void_p]
    L.gp_ensemble_reduce.argtypes = [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]
    L.gp_plan_count.argtypes = [c_void_p]
    L.gp_set_memory_efficient_attention.argtypes = [c_void_p, c_int]
    L.gp_set_shared_arena.argtypes = [c_void_p, c_int]
    L.gp_shared_arena_info.argtypes = [c_int, POINTER(c_int64), POINTER(c_int64), POINTER(c_int64)]
    L.gp_shared_arena_fill.argtypes = [c_int, c_int, c_void_p]
    L.gp_tile_shape.argtypes = [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_int), POINTER(c_int)]
    L.gp_tensor_shape.argtypes = [c_void_p, c_char_p, POINTER(c_int64)]
    L.gp_read_tensor.argtypes = [c_void_p, c_char_p, c_void_p, c_size_t]
    L.gp_write_tensor.argtypes = [c_void_p, c_char_p, c_void_p, c_size_t]
    L.gp_plan_info.argtypes = [c_void_p, POINTER(c_int64), POINTER(c_int64), POINTER(c_int64), POINTER(c_int64),
                               POINTER(c_double)]
    L.gp_profile_ops.argtypes = [c_void_p, c_int, c_void_p]
    L.gp_op_info.argtypes = [c_void_p, c_int64, c_char_p, c_size_t, POINTER(c_double), POINTER(c_double),
                             POINTER(c_double), POINTER(c_int), POINTER(c_double)]
    L.gp_conv2d.argtypes = [c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                            c_void_p, c_int, c_void_p, c_int, c_void_p]
    L.gp_groupnorm.argtypes = [c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float,
                               c_int, c_void_p, c_void_p]
    L.gp_gn_conv3x3.argtypes = [c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_int,
                                c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                c_void_p]
    L.gp_conv_groupnorm.argtypes = [c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int,
                                    c_int, c_void_p, c_void_p, c_float, c_int, c_void_p, c_void_p, c_void_p]
    L.gp_layernorm.argtypes = [c_int, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_float, c_void_p, c_void_p]
    L.gp_attention.argtypes = [c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p,
                               c_void_p]
    L.gp_bilinear_up2x.argtypes = [c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]
    L.gp_bench_conv.argtypes = [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_double),
                                POINTER(c_double)]
    L.gp_bench_attention.argtypes = [c_int, c_int, c_int, c_int, c_int, POINTER(c_double), POINTER(c_double)]
    L.gp_attention_high.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]
    L.gp_bench_attention_high.argtypes = [c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_double), POINTER(c_double)]
    L.gp_resize_aa.argtypes = [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int,
                               c_int, c_void_p]
    L.gp_colorize.argtypes = [c_void_p, c_int, c_int, c_int, c_int, c_float, c_float, c_void_p, c_void_p, c_int,
                              c_void_p]
    L.gp_quantize.argtypes = [c_void_p, c_int, c_size_t, c_int, c_void_p, c_int, c_void_p]
    L.gp_resize_pil.argtypes = [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_int, c_void_p]
    L.gp_v1_postprocess.argtypes = [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                    c_void_p]
    L.gp_depth_align.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                 c_void_p]
    L.gp_depth_metrics.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_float, c_float,
                                   c_void_p, c_void_p]
    _lib = L
    return L


def _gp_dtype(t):
    return {torch.float32: GP_F32, torch.float16: GP_F16, torch.bfloat16: GP_BF16, torch.uint8: GP_U8}[t]


def _stream_ptr(device=None):
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _on_host(t):
    """The C-ABI's on-host flag of a buffer."""
    return 0 if t.is_cuda else 1


def _rgb_arg(rgb):
    """An rgb batch as the C-ABI takes it: contiguous, with bf16 (which it does not take) as fp32."""
    return (rgb.float() if rgb.dtype == torch.bfloat16 else rgb).contiguous()


def _check_free(st, what):
    if st != 0:
        raise RuntimeError(f"{what} failed: {_STATUS.get(st, st)} (see stderr)")


class Engine:
    """One engine per (process, GPU).  Mirrors the C-ABI one to one."""

    def __init__(self, dtype=torch.float16, readout="vae", timestep=1, device=0, cuda_graph="auto",
                 precision="default", arch="genpercept", memory_efficient_attention=False, shared_arena=False):
        if not torch.cuda.is_available():
            raise RuntimeError("genpercept_b200 needs a CUDA (sm_90a) device; there is no CPU fallback")
        self.L = lib()
        self.torch_dtype = dtype
        self.readout = readout
        self.device = torch.device("cuda", device)
        cfg = _Config(device, _gp_dtype(dtype), GP_READOUT_DPT if readout == "dpt" else GP_READOUT_VAE, timestep,
                      2 if cuda_graph == "auto" else (1 if cuda_graph else 0),   # auto: graphs for small plans
                      {"default": 0, "high": 1}[precision], {"genpercept": 0, "multistep": 1}[arch])
        self.precision = precision
        self.arch = arch
        self.h = c_void_p()
        st = self.L.gp_create(byref(cfg), byref(self.h))
        if st != 0:
            raise RuntimeError(f"gp_create failed: {_STATUS.get(st, st)} (no sm_90a device?)")
        self.plan_shape = None
        self.out_hw = None
        self.memory_efficient_attention = False
        if memory_efficient_attention:
            self.set_memory_efficient_attention(True)
        self.shared_arena = False
        if shared_arena:
            self.set_shared_arena(True)

    def set_memory_efficient_attention(self, flag):
        """High-precision mode: run every attention fused, storing no T x T score matrix (gp_set_memory_efficient_attention).
        The 16-bit modes ignore it.  A change drops the cached plans; the next call plans again."""
        self._ck(self.L.gp_set_memory_efficient_attention(self.h, 1 if flag else 0), "gp_set_memory_efficient_attention")
        if bool(flag) != self.memory_efficient_attention:
            self.plan_shape = None
            self.out_hw = None
        self.memory_efficient_attention = bool(flag)

    def set_shared_arena(self, flag):
        """Take the activation arena of every plan from the device's one shared pool (gp_set_shared_arena), so engines
        and cached plans that opt in need the largest arena among them, not the sum.  A shared plan's kept tensors
        (``read_tensor``) are meaningful only straight after its own call.  A change drops the cached plans."""
        self._ck(self.L.gp_set_shared_arena(self.h, 1 if flag else 0), "gp_set_shared_arena")
        if bool(flag) != self.shared_arena:
            self.plan_shape = None
            self.out_hw = None
        self.shared_arena = bool(flag)

    def close(self):
        if getattr(self, "h", None):
            self.L.gp_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, st, what):
        if st != 0:
            msg = self.L.gp_last_error(self.h).decode()
            raise RuntimeError(f"{what}: {_STATUS.get(st, st)}: {msg}")

    def load_state(self, component, sd):
        """component in {unet, vae, dpt}; sd: {diffusers key: tensor}."""
        for k, v in sd.items():
            t = v.detach().to("cpu")
            if t.dtype not in (torch.float32, torch.float16, torch.bfloat16):
                t = t.float()
            t = t.contiguous()
            shape = (c_int64 * t.dim())(*t.shape)
            self._ck(self.L.gp_load_tensor(self.h, f"{component}.{k}".encode(), c_void_p(t.data_ptr()),
                                           _gp_dtype(t.dtype), shape, t.dim()), f"gp_load_tensor({k})")

    def set_text_embed(self, embed):
        e = torch.as_tensor(embed).detach().float().cpu().reshape(-1, 1024).contiguous()
        self._ck(self.L.gp_set_text_embed(self.h, c_void_p(e.data_ptr()), e.shape[0], 1024), "gp_set_text_embed")

    def finalize(self):
        self._ck(self.L.gp_finalize(self.h), "gp_finalize")

    def plan(self, batch, height, width):
        self._ck(self.L.gp_plan(self.h, batch, height, width), "gp_plan")
        self.plan_shape = (batch, height, width)
        self.out_hw = self.tensor_shape("out")[2:]      # == (height, width) for multiples of 8 (VAE) / 64 (DPT)

    def plan_count(self):
        return int(self.L.gp_plan_count(self.h))

    def set_timestep(self, t):
        """Per-call ``fix_timesteps`` (genpercept_pipeline.py:405-408): re-folds the ResNet biases (cached per t)."""
        self._ck(self.L.gp_set_timestep(self.h, int(t)), "gp_set_timestep")

    def _sp(self):
        return _stream_ptr(self.device)

    def _plan_for(self, B, H, W):
        if self.plan_shape != (B, H, W):
            self.plan(B, H, W)

    def _out(self, out, B, C):
        """The caller's `out`, checked, or a new device buffer: contiguous fp32 [B, C, *out_hw]."""
        shape = (B, C) + tuple(self.out_hw or (0, 0))      # no plan (infer_latent): the library reports GP_ERR_NO_PLAN
        if out is None:
            out = torch.empty(shape, dtype=torch.float32, device=self.device)
        assert out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == shape, \
            f"out must be contiguous fp32 {shape}"
        return out

    def encode(self, rgb):
        """encode_rgb on the device: [B,3,H,W] uint8 / float -> fp32 latent [B,4,H/8,W/8] (cuda)."""
        B, _, H, W = rgb.shape
        self._plan_for(B, H, W)
        rgb = _rgb_arg(rgb)
        lat = torch.empty((B, 4) + self.tensor_shape("rgb_latent")[2:], dtype=torch.float32, device=self.device)
        self._ck(self.L.gp_encode(self.h, c_void_p(rgb.data_ptr()), _gp_dtype(rgb.dtype), _on_host(rgb),
                                  c_void_p(lat.data_ptr()), self._sp()), "gp_encode")
        return lat

    def decode(self, latent, out_channels=1, post_quant=True):
        """decode_pred + clip + shift on the device: fp32 latent [B,4,h,w] -> fp32 [B,C,8h,8w] in [0,1] (cuda)."""
        B, _, h, w = latent.shape
        if self.plan_shape is None or self.plan_shape[0] != B or tuple(self.tensor_shape("z")[2:]) != (h, w):
            self.plan(B, 8 * h, 8 * w)
        latent = latent.to(self.device, torch.float32).contiguous()
        out = torch.empty((B, out_channels, 8 * h, 8 * w), dtype=torch.float32, device=self.device)
        self._ck(self.L.gp_decode(self.h, c_void_p(latent.data_ptr()), 1 if post_quant else 0, c_void_p(out.data_ptr()),
                                  out_channels, self._sp()), "gp_decode")
        return out

    def infer(self, rgb, out_channels=1, out=None):
        """rgb: [B,3,H,W] uint8 (0..255) or float16/float32 in [-1,1]; cuda or cpu tensor.
        Returns fp32 [B,C,H,W] in [0,1] on the device of `out` (default: cuda)."""
        assert rgb.dim() == 4 and rgb.shape[1] == 3
        B, _, H, W = rgb.shape
        self._plan_for(B, H, W)
        rgb = _rgb_arg(rgb)
        C = 1 if self.readout == "dpt" else out_channels
        out = self._out(out, B, C)
        self._ck(self.L.gp_infer(self.h, c_void_p(rgb.data_ptr()), _gp_dtype(rgb.dtype), _on_host(rgb),
                                 c_void_p(out.data_ptr()), _on_host(out), C, self._sp()), "gp_infer")
        return out

    def encode_exact(self, rgb):
        """The latent ``infer_latent`` takes, without loss (gp_encode_exact): [B,3,H,W] uint8 / float -> fp32
        [B,4,H/8,W/8] (cuda) in the 16-bit modes, the same as ``encode``; in the high-precision mode fp32 [B,8,H/8,W/8] =
        [hi | lo], the (hi, lo) pair of every value.  Plans (B, H, W) like ``infer``."""
        B, _, H, W = rgb.shape
        self._plan_for(B, H, W)
        rgb = _rgb_arg(rgb)
        c = 8 if self.precision == "high" else 4
        lat = torch.empty((B, c) + self.tensor_shape("rgb_latent")[2:], dtype=torch.float32, device=self.device)
        self._ck(self.L.gp_encode_exact(self.h, c_void_p(rgb.data_ptr()), _gp_dtype(rgb.dtype), _on_host(rgb),
                                        c_void_p(lat.data_ptr()), self._sp()), "gp_encode_exact")
        return lat

    def infer_latent(self, latent, out_channels=1, out=None):
        """``infer`` from the UNet on (gp_infer_latent): `latent` as ``encode_exact`` returns it, from this engine or another
        with the same dtype, precision and VAE encoder.  It runs on the CURRENT plan, the one ``plan(B, H, W)`` (or
        ``encode_exact`` / ``infer``) made for the image the latent came from: a latent's extent does not fix the image's,
        and the image's sets the result's.  Returns fp32 [B,C,H,W] in [0,1] on the device of `out`, equal to ``infer``'s."""
        assert latent.dim() == 4, "latent must be [B,C,h,w]"
        B, c, h, w = latent.shape
        latent = latent.to(self.device, torch.float32).contiguous()
        C = 1 if self.readout == "dpt" else out_channels
        out = self._out(out, B, C)
        self._ck(self.L.gp_infer_latent(self.h, c_void_p(latent.data_ptr()), B, c, h, w, c_void_p(out.data_ptr()),
                                        _on_host(out), C, self._sp()), "gp_infer_latent")
        return out

    def infer_steps(self, rgb, timesteps, coeffs, noise=None, out_channels=1, out=None):
        """Multi-step archs (gp_infer_steps): `timesteps` [n] ints, `coeffs` [n,4] DDIM coefficients
        (scheduler.DDIMSchedule.step_coefficients), `noise` fp32 [B,4,h,w] (marigold) or None (rgb_blending)."""
        assert rgb.dim() == 4 and rgb.shape[1] == 3
        B, _, H, W = rgb.shape
        self._plan_for(B, H, W)
        rgb = _rgb_arg(rgb)
        out = self._out(out, B, out_channels)
        n = len(timesteps)
        ts = (c_int * n)(*[int(t) for t in timesteps])
        cf = (c_float * (4 * n))(*[float(v) for row in coeffs for v in row])
        nz = None
        if noise is not None:
            nz = noise.detach().to(torch.float32).contiguous()
            assert tuple(nz.shape) == (B, 4) + tuple(self.tensor_shape("rgb_latent")[2:]), "noise must be [B,4,H/8,W/8]"
        self._ck(self.L.gp_infer_steps(self.h, c_void_p(rgb.data_ptr()), _gp_dtype(rgb.dtype), _on_host(rgb),
                                       c_void_p(nz.data_ptr()) if nz is not None else None, _on_host(nz) if nz is not None else 0,
                                       ts, cf, n, c_void_p(out.data_ptr()), _on_host(out), out_channels, self._sp()),
                 "gp_infer_steps")
        return out

    def run_stage(self, stage, out_channels=1):
        self._ck(self.L.gp_run_stage(self.h, stage, out_channels, self._sp()), "gp_run_stage")

    def tensor_shape(self, name):
        s = (c_int64 * 4)()
        self._ck(self.L.gp_tensor_shape(self.h, name.encode(), s), f"gp_tensor_shape({name})")
        return tuple(int(x) for x in s)

    def read_tensor(self, name):
        shape = self.tensor_shape(name)
        a = np.empty(shape, dtype=np.float32)
        self._ck(self.L.gp_read_tensor(self.h, name.encode(), a.ctypes.data_as(c_void_p), a.size), "gp_read_tensor")
        return a

    def write_tensor(self, name, arr):
        a = np.ascontiguousarray(arr, dtype=np.float32)
        self._ck(self.L.gp_write_tensor(self.h, name.encode(), a.ctypes.data_as(c_void_p), a.size), "gp_write_tensor")

    def plan_info(self):
        n_ops, n_l, ab, wb, fl = c_int64(), c_int64(), c_int64(), c_int64(), c_double()
        self._ck(self.L.gp_plan_info(self.h, byref(n_ops), byref(n_l), byref(ab), byref(wb), byref(fl)), "gp_plan_info")
        return {"ops": n_ops.value, "launches": n_l.value, "arena_bytes": ab.value, "weight_bytes": wb.value,
                "flops": fl.value}

    def profile_ops(self, out_channels=1):
        self._ck(self.L.gp_profile_ops(self.h, out_channels, self._sp()), "gp_profile_ops")
        res = []
        buf = ctypes.create_string_buffer(256)
        us, fl, by, kd, fx = c_double(), c_double(), c_double(), c_int(), c_double()
        for i in range(self.plan_info()["ops"]):
            self._ck(self.L.gp_op_info(self.h, i, buf, 256, byref(us), byref(fl), byref(by), byref(kd), byref(fx)), "gp_op_info")
            res.append({"name": buf.value.decode(), "usec": us.value, "flops": fl.value, "bytes": by.value,
                        "kind": kd.value, "flops_exec": fx.value})
        return res


def shared_arena_info(device=0):
    """The device's shared activation pool: {"mapped_bytes", "reserved_bytes", "live_plans"} (all 0 when no engine on
    `device` shares it)."""
    m, r, n = c_int64(), c_int64(), c_int64()
    _check_free(lib().gp_shared_arena_info(int(device), byref(m), byref(r), byref(n)), "gp_shared_arena_info")
    return {"mapped_bytes": m.value, "reserved_bytes": r.value, "live_plans": n.value}


def shared_arena_fill(byte, device=0):
    """Tests: write `byte` over the shared pool's mapped range, on the current stream and ordered after every earlier
    user of the pool (gp_shared_arena_fill)."""
    _check_free(lib().gp_shared_arena_fill(int(device), int(byte), _stream_ptr(device)), "gp_shared_arena_fill")


# ---------------------------------------------------------------- per-kernel entry points (tests)
# An fp32 activation selects the high-precision mode's layout (GP_F16_PAIR): it is split into its (hi, lo) fp16 pair,
# stored [hi C | lo C] per pixel, and the result comes back as float64 hi + lo, the exact stored value (an fp32 sum is not
# exact where lo is far below hi's last bit).  f16 / bf16 activations run the 16-bit modes and come back as they are.
def _nhwc(x):
    """NCHW torch tensor -> contiguous NHWC (same dtype)."""
    return x.permute(0, 2, 3, 1).contiguous()


def _layout(x):
    """The C-ABI dtype of a per-kernel call on activation `x`."""
    return GP_F16_PAIR if x.dtype == torch.float32 else _gp_dtype(x.dtype)


def _arg(t, dt):
    """Activation `t` (or None) as the kernels take it in layout `dt`: contiguous, fp32 split into [hi | lo] channels."""
    if t is None:
        return None
    if dt == GP_F16_PAIR:
        assert t.dtype == torch.float32, "every activation of a high-precision call is fp32"
        return torch.cat(split_hi_lo(t), dim=-1).contiguous()
    assert t.dtype != torch.float32, "fp32 activations select the high-precision layout for every operand"
    return t.contiguous()


def _out(shape, dt, device):
    """An output buffer of logical `shape` (channels last) in layout `dt`."""
    if dt == GP_F16_PAIR:
        return torch.zeros(tuple(shape[:-1]) + (2 * shape[-1],), dtype=torch.float16, device=device)
    return torch.zeros(tuple(shape), dtype=torch.bfloat16 if dt == GP_BF16 else torch.float16, device=device)


def _result(y, dt):
    """An output buffer as the caller sees it: float64 hi + lo in the pair layout."""
    if dt == GP_F16_PAIR:
        c = y.shape[-1] // 2
        return y[..., :c].double() + y[..., c:].double()
    return y


def conv2d(x_nhwc, w, bias=None, mode=0, residual=None, relu=False, direct=False):
    """x_nhwc: cuda [N,H,W,Cin] f16/bf16, or fp32 (the (hi, lo) pair layout); w: cpu fp32 [Cout,Cin,ks,ks]. Returns NHWC
    (float64 for an fp32 input)."""
    dt = _layout(x_nhwc)
    N, H, W, Cin = x_nhwc.shape
    Cout, _, ks, _ = w.shape
    Ho, Wo = H, W
    if mode == 1:
        Ho, Wo = (H + 2 - 3) // 2 + 1, (W + 2 - 3) // 2 + 1
    elif mode == 2:
        Ho, Wo = (H + 1 - 3) // 2 + 1, (W + 1 - 3) // 2 + 1
    elif mode == 3:
        Ho, Wo = 2 * H, 2 * W
    y = _out((N, Ho, Wo, Cout), dt, x_nhwc.device)
    x, res = _arg(x_nhwc, dt), _arg(residual, dt)
    w = w.detach().float().cpu().contiguous()
    b = bias.detach().float().cpu().contiguous() if bias is not None else None
    st = lib().gp_conv2d(dt, c_void_p(x.data_ptr()), N, H, W, Cin, c_void_p(w.data_ptr()),
                         c_void_p(b.data_ptr()) if b is not None else None, Cout, ks, mode, _ptr(res), 1 if relu else 0,
                         c_void_p(y.data_ptr()), 1 if direct else 0, _stream_ptr())
    _check_free(st, "gp_conv2d")
    return _result(y, dt)


def groupnorm(x_nhwc, groups, gamma, beta, eps, silu):
    """GroupNorm(+SiLU) on NHWC x (f16/bf16, or fp32: the pair layout, float64 result)."""
    dt = _layout(x_nhwc)
    N, H, W, C = x_nhwc.shape
    x = _arg(x_nhwc, dt)
    y = _out((N, H, W, C), dt, x_nhwc.device)
    g = gamma.detach().float().cpu().contiguous()
    b = beta.detach().float().cpu().contiguous()
    st = lib().gp_groupnorm(dt, c_void_p(x.data_ptr()), N, H, W, C, groups, c_void_p(g.data_ptr()), c_void_p(b.data_ptr()),
                            eps, 1 if silu else 0, c_void_p(y.data_ptr()), _stream_ptr())
    _check_free(st, "gp_groupnorm")
    return _result(y, dt)


def gn_conv3x3(x_nhwc, groups, gamma, beta, eps, silu, w, bias=None, sc_x=None, sc_w=None, sc_b=None, residual=None,
               out_f32=False):
    """GroupNorm(+SiLU) -> 3x3 conv (+ 1x1 shortcut over raw sc_x, + residual) through gp_gn_conv3x3.  An fp32 x selects
    the pair layout (sc_x and residual fp32 too) and a float64 NHWC result; out_f32: an fp32 NCHW map either way."""
    dt = _layout(x_nhwc)
    N, H, W, Cin = x_nhwc.shape
    Cout = w.shape[0]
    f = lambda t: None if t is None else t.detach().float().cpu().contiguous()
    g, b_, w_, bias_, scw, scb = f(gamma), f(beta), f(w), f(bias), f(sc_w), f(sc_b)
    x, scx, res = _arg(x_nhwc, dt), _arg(sc_x, dt), _arg(residual, dt)
    if out_f32:
        y = torch.zeros((N, Cout, H, W), dtype=torch.float32, device=x_nhwc.device)
    else:
        y = _out((N, H, W, Cout), dt, x_nhwc.device)
    st = lib().gp_gn_conv3x3(dt, _ptr(x), N, H, W, Cin, groups, _ptr(g), _ptr(b_), eps, 1 if silu else 0,
                             _ptr(w_), _ptr(bias_), Cout, _ptr(scx), 0 if sc_x is None else sc_x.shape[-1], _ptr(scw), _ptr(scb),
                             _ptr(res), _ptr(y), 1 if out_f32 else 0, _stream_ptr())
    _check_free(st, "gp_gn_conv3x3")
    return y if out_f32 else _result(y, dt)


def conv_groupnorm(x_nhwc, w, bias, groups, gamma, beta, eps, silu, skip=None):
    """3x3 stride-1 conv x -> y_conv, then GroupNorm(+SiLU) over concat(y_conv, skip) -> y (gp_conv_groupnorm).  Returns
    (y_conv, y) NHWC; an fp32 x (and skip) selects the pair layout and float64 results."""
    dt = _layout(x_nhwc)
    N, H, W, Cin = x_nhwc.shape
    Cout = w.shape[0]
    Cskip = 0 if skip is None else skip.shape[-1]
    f = lambda t: None if t is None else t.detach().float().cpu().contiguous()
    w_, b_, g, bt = f(w), f(bias), f(gamma), f(beta)
    x, sk = _arg(x_nhwc, dt), _arg(skip, dt)
    yc = _out((N, H, W, Cout), dt, x_nhwc.device)
    y = _out((N, H, W, Cout + Cskip), dt, x_nhwc.device)
    st = lib().gp_conv_groupnorm(dt, _ptr(x), N, H, W, Cin, _ptr(w_), _ptr(b_), Cout, _ptr(sk), Cskip, groups, _ptr(g), _ptr(bt),
                                 eps, 1 if silu else 0, _ptr(yc), _ptr(y), _stream_ptr())
    _check_free(st, "gp_conv_groupnorm")
    return _result(yc, dt), _result(y, dt)


def ensemble_reduce(pred, scale, shift, median=True, normalise=1):
    """gp_ensemble_reduce: pred fp32 [B,1,H,W] (cuda) -> [1,1,H,W] (cuda); scale / shift: numpy [B]."""
    assert pred.is_cuda and pred.dtype == torch.float32 and pred.dim() == 4 and pred.shape[1] == 1
    pred = pred.contiguous()
    B, _, H, W = pred.shape
    sc = np.ascontiguousarray(scale, dtype=np.float32)
    sh = np.ascontiguousarray(shift, dtype=np.float32)
    out = torch.empty((1, 1, H, W), dtype=torch.float32, device=pred.device)
    st = lib().gp_ensemble_reduce(c_void_p(pred.data_ptr()), B, H, W, sc.ctypes.data_as(c_void_p), sh.ctypes.data_as(c_void_p),
                                  1 if median else 0, int(normalise), c_void_p(out.data_ptr()), _stream_ptr(pred.device))
    _check_free(st, "gp_ensemble_reduce")
    return out


def layernorm(x, gamma, beta, eps=1e-5):
    """LayerNorm over the last axis of cuda x (f16/bf16, or fp32: the pair layout, float64 result)."""
    dt = _layout(x)
    C = x.shape[-1]
    xa = _arg(x, dt)
    y = _out(tuple(x.shape), dt, x.device)
    g = gamma.detach().float().cpu().contiguous()
    b = beta.detach().float().cpu().contiguous()
    st = lib().gp_layernorm(dt, c_void_p(xa.data_ptr()), x.numel() // C, C, c_void_p(g.data_ptr()),
                            c_void_p(b.data_ptr()), eps, c_void_p(y.data_ptr()), _stream_ptr())
    _check_free(st, "gp_layernorm")
    return _result(y, dt)


def attention(q, k, v, heads, scale):
    """q,k,v: cuda [B,T,heads*d]."""
    B, T, C = q.shape
    o = torch.zeros_like(q)
    st = lib().gp_attention(_gp_dtype(q.dtype), c_void_p(q.data_ptr()), c_void_p(k.data_ptr()), c_void_p(v.data_ptr()),
                            B, T, heads, C // heads, scale, c_void_p(o.data_ptr()), _stream_ptr())
    _check_free(st, "gp_attention")
    return o


def split_hi_lo(x):
    """fp32 -> its fp16 (hi, lo) pair, value = hi + lo: the high-precision mode's operand format."""
    x = x.float()
    hi = x.half()
    return hi, (x - hi.float()).half()


def attention_high(q, k, v, heads, scale, fused):
    """High-precision attention (gp_attention_high): q, k, v cuda fp32 [B,T,heads*d] -> fp32 o = hi + lo.  scale * q
    is split into its (hi, lo) pair, as are k and v; `fused` picks the fused split-precision kernel or the unfused path."""
    B, T, C = q.shape
    qh, ql = split_hi_lo(q * scale)
    kh, kl = split_hi_lo(k)
    vh, vl = split_hi_lo(v)
    qk = torch.cat([qh, kh, ql, kl], dim=-1).contiguous()
    vv = torch.cat([vh, vl], dim=-1).contiguous()
    o = torch.zeros((B, T, 2 * C), dtype=torch.float16, device=q.device)
    st = lib().gp_attention_high(c_void_p(qk.data_ptr()), c_void_p(vv.data_ptr()), B, T, heads, C // heads, 1 if fused else 0,
                                 c_void_p(o.data_ptr()), _stream_ptr(q.device))
    _check_free(st, "gp_attention_high")
    return o[..., :C].float() + o[..., C:].float()


def bilinear_up2x(x_nhwc):
    """Bilinear 2x (align_corners=True) on NHWC x (f16/bf16, or fp32: the pair layout, float64 result)."""
    dt = _layout(x_nhwc)
    N, H, W, C = x_nhwc.shape
    x = _arg(x_nhwc, dt)
    y = _out((N, 2 * H, 2 * W, C), dt, x_nhwc.device)
    st = lib().gp_bilinear_up2x(dt, c_void_p(x.data_ptr()), N, H, W, C, c_void_p(y.data_ptr()), _stream_ptr())
    _check_free(st, "gp_bilinear_up2x")
    return _result(y, dt)


RESIZE_MODES = {"bilinear": 0, "bicubic": 1}


def resize_aa(x, out_h, out_w, mode="bilinear", device=None):
    """torchvision ``resize(tensor, [out_h, out_w], interpolation, antialias=True)`` on the GPU
    (gp_resize_aa).  x: [..., H, W] uint8 or float32, cuda or cpu; the result lives where x lives
    unless `device` says otherwise ("cuda" uploads a host image and keeps the result on the GPU)."""
    assert x.dtype in (torch.uint8, torch.float32) and x.dim() >= 2
    x = x.contiguous()
    H, W = x.shape[-2:]
    N = x.numel() // (H * W)
    out_dev = x.device if device is None else torch.device(device)
    if out_dev.type == "cuda" and out_dev.index is None:
        out_dev = torch.device("cuda", torch.cuda.current_device())
    y = torch.empty(tuple(x.shape[:-2]) + (out_h, out_w), dtype=x.dtype, device=out_dev)
    st = lib().gp_resize_aa(c_void_p(x.data_ptr()), _gp_dtype(x.dtype), 0 if x.is_cuda else 1, N, H, W,
                            c_void_p(y.data_ptr()), _gp_dtype(y.dtype), 0 if y.is_cuda else 1, out_h, out_w,
                            RESIZE_MODES[mode], _stream_ptr())
    _check_free(st, "gp_resize_aa")
    return y


def colorize(pred, lut_u8, vmin=0.0, vmax=1.0, to_host=True):
    """pred: float32 [B,H,W] (cuda or cpu) -> uint8 [B,H,W,3] through a 256x3 uint8 LUT (gp_colorize)."""
    assert pred.dtype == torch.float32 and pred.dim() == 3
    pred = pred.contiguous()
    B, H, W = pred.shape
    lut = np.ascontiguousarray(lut_u8, dtype=np.uint8)
    assert lut.shape == (256, 3)
    out = torch.empty((B, H, W, 3), dtype=torch.uint8, device="cpu" if to_host else pred.device)
    st = lib().gp_colorize(c_void_p(pred.data_ptr()), 0 if pred.is_cuda else 1, B, H, W, vmin, vmax,
                           lut.ctypes.data_as(c_void_p), c_void_p(out.data_ptr()), 0 if out.is_cuda else 1, _stream_ptr())
    _check_free(st, "gp_colorize")
    return out


def quantize(pred, bits=16, to_host=True):
    """(pred * 65535).astype(uint16) / (pred * 255).astype(uint8) (gp_quantize); uint16 comes back as int16 storage
    viewed through numpy on the host."""
    assert pred.dtype == torch.float32 and bits in (8, 16)
    pred = pred.contiguous()
    if to_host:
        out = np.empty(tuple(pred.shape), dtype=np.uint16 if bits == 16 else np.uint8)
        ptr, on_host = out.ctypes.data_as(c_void_p), 1
    else:
        out = torch.empty(tuple(pred.shape), dtype=torch.uint16 if bits == 16 else torch.uint8, device=pred.device)
        ptr, on_host = c_void_p(out.data_ptr()), 0
    st = lib().gp_quantize(c_void_p(pred.data_ptr()), 0 if pred.is_cuda else 1, pred.numel(), bits, ptr, on_host,
                           _stream_ptr())
    _check_free(st, "gp_quantize")
    return out


def resize_pil(img_hwc, out_h, out_w, device=None):
    """``PIL.Image.Image.resize((out_w, out_h))`` (BICUBIC) of an RGB image, byte for byte, on the GPU (gp_resize_pil).
    img_hwc: uint8 [H,W,3] numpy array (``np.asarray(pil_image)``) or tensor, host or cuda.  Returns uint8 [3,out_h,out_w]
    (CHW) on `device` (default: the current cuda device)."""
    if isinstance(img_hwc, np.ndarray):
        with warnings.catch_warnings():          # np.asarray of a PIL image is read-only; it is only read here
            warnings.simplefilter("ignore", UserWarning)
            x = torch.from_numpy(np.ascontiguousarray(img_hwc))
    else:
        x = img_hwc
    assert x.dtype == torch.uint8 and x.dim() == 3 and x.shape[2] == 3, "an RGB image as uint8 [H,W,3]"
    x = x.contiguous()
    H, W = x.shape[:2]
    out_dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if out_dev.type == "cuda" and out_dev.index is None:
        out_dev = torch.device("cuda", torch.cuda.current_device())
    y = torch.empty((3, out_h, out_w), dtype=torch.uint8, device=out_dev)
    st = lib().gp_resize_pil(c_void_p(x.data_ptr()), _on_host(x), H, W, c_void_p(y.data_ptr()), _on_host(y), out_h, out_w,
                             _stream_ptr())
    _check_free(st, "gp_resize_pil")
    return y


V1_TASKS = {"depth": 0, "normal": 1, "seg": 2, "sr": 2}


def v1_postprocess(pred, task, size=None):
    """GenPercept v1's post-processing of the engine's map (gp_v1_postprocess).  pred: cuda fp32 [B,C,h,w] in [0,1];
    `size` (H, W) or None (no interpolation).  Returns, on the device: depth -> (fp32 [B,H,W] min-max normalised, None);
    normal -> (fp32 [B,3,H,W] in [-1,1], uint8 [B,H,W,3] norm_to_rgb); seg / sr -> (None, uint8 [B,3,H,W])."""
    assert pred.is_cuda and pred.dtype == torch.float32 and pred.dim() == 4
    pred = pred.contiguous()
    B, C, h, w = pred.shape
    H, W = (h, w) if size is None else (int(size[0]), int(size[1]))
    t = V1_TASKS[task]
    f32 = u8 = None
    if t == 0:
        f32 = torch.empty((B, H, W), dtype=torch.float32, device=pred.device)
    elif t == 1:
        f32 = torch.empty((B, 3, H, W), dtype=torch.float32, device=pred.device)
        u8 = torch.empty((B, H, W, 3), dtype=torch.uint8, device=pred.device)
    else:
        u8 = torch.empty((B, 3, H, W), dtype=torch.uint8, device=pred.device)
    st = lib().gp_v1_postprocess(c_void_p(pred.data_ptr()), B, C, h, w, t, H, W, _ptr(f32), _ptr(u8),
                                 _stream_ptr(pred.device))
    _check_free(st, "gp_v1_postprocess")
    return f32, u8


def _ptr(t):
    return None if t is None else c_void_p(t.data_ptr())


def depth_align(pred, gt, valid, mode=0, max_res=0, aligned=False):
    """gp_depth_align: pred / gt contiguous cuda fp32 [B,H,W], valid cuda uint8 [B,H,W] or None (all valid); mode 0
    (fit gt) or 1 (disparity of gt).  Returns (scale_shift fp32 [B,2], aligned fp32 [B,H,W] or None), on the device."""
    B, H, W = pred.shape
    ss = torch.empty((B, 2), dtype=torch.float32, device=pred.device)
    out = torch.empty_like(pred) if aligned else None
    st = lib().gp_depth_align(_ptr(pred), _ptr(gt), _ptr(valid), B, H, W, int(mode), int(max_res), _ptr(ss), _ptr(out),
                              _stream_ptr(pred.device))
    _check_free(st, "gp_depth_align")
    return ss, out


def depth_metrics(pred, gt, valid, mode=0, scale_shift=None, min_depth=0.0, max_depth=1e8):
    """gp_depth_metrics: the ten eval.py metrics per image -> fp64 [B,10] on the device.  mode 0 none, 1 least squares,
    2 least squares in disparity (scale_shift fp32 [B,2] on the device)."""
    B, H, W = pred.shape
    out = torch.empty((B, 10), dtype=torch.float64, device=pred.device)
    st = lib().gp_depth_metrics(_ptr(pred), _ptr(gt), _ptr(valid), B, H, W, int(mode), _ptr(scale_shift), float(min_depth),
                                float(max_depth), _ptr(out), _stream_ptr(pred.device))
    _check_free(st, "gp_depth_metrics")
    return out


def tile_shape(cout, cin, ks, images, h, w, tokens_mode=False, num_sms=132):
    """(BN, MT) the planner gives a stride-1 layer (host-only; the rule is tile_shape_for in csrc/builder.cu)."""
    bn, mt = c_int(), c_int()
    st = lib().gp_tile_shape(cout, cin, ks, images, h, w, 1 if tokens_mode else 0, num_sms, byref(bn), byref(mt))
    _check_free(st, "gp_tile_shape")
    return bn.value, mt.value


def bench_conv(dtype, N, H, W, Cin, Cout, ks=3, mode=0, iters=10):
    us, fl = c_double(), c_double()
    st = lib().gp_bench_conv(_gp_dtype(dtype), N, H, W, Cin, Cout, ks, mode, iters, byref(us), byref(fl))
    _check_free(st, "gp_bench_conv")
    return us.value, fl.value


def bench_attention(dtype, B, T, fused, iters=10):
    """Time the fused or the unfused single-head d = 512 attention (VAE mid-block) at B x T tokens, whichever path the
    planner would choose there.  Returns (microseconds per call, FLOPs per call)."""
    us, fl = c_double(), c_double()
    st = lib().gp_bench_attention(_gp_dtype(dtype), B, T, 1 if fused else 0, iters, byref(us), byref(fl))
    _check_free(st, "gp_bench_attention")
    return us.value, fl.value


def bench_attention_high(B, T, heads, d, fused, iters=10):
    """Time the fused or the unfused high-precision attention (d = 64 with `heads` heads, or d = 512 with one) at B x T
    tokens.  Returns (microseconds per call, FLOPs per call)."""
    us, fl = c_double(), c_double()
    st = lib().gp_bench_attention_high(B, T, heads, d, 1 if fused else 0, iters, byref(us), byref(fl))
    _check_free(st, "gp_bench_attention_high")
    return us.value, fl.value
