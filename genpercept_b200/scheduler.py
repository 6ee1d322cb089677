"""Host side of the DDIM schedule for the multi-step archs (SURVEY.md §8 f4: ``--archs marigold`` / ``rgb_blending``).

Mirrors ``DDIMSchedulerCustomized`` (/root/reference/src/customized_modules/ddim.py:144-217: beta schedules
``linear`` / ``scaled_linear`` / ``scaled_linear_power``, ``final_alpha_cumprod``) and the parts of diffusers'
``DDIMScheduler`` it inherits and the pipeline calls (``set_timesteps`` with leading / trailing / linspace spacing and
``steps_offset``; ``step`` with eta = 0 for the ``v_prediction`` / ``epsilon`` / ``sample`` prediction types), driven by the
reference's ``hf_configs/scheduler_beta_*/scheduler_config.json`` files.  Only scalars are computed here: per step the
four coefficients of

    x0   = c_x0_s * sample + c_x0_m * model_output            (pred_original_sample)
    prev = c_pv_s * sample + c_pv_m * model_output            (prev_sample, eta = 0)

which the engine's ``ddim_step`` kernel applies to the latents on the device (gp_infer_steps).
"""
import json
import os

import numpy as np

# The scheduler classes whose step this module restates: diffusers' DDIMScheduler and the reference's subclass of it.
DDIM_CLASSES = ("DDIMScheduler", "DDIMSchedulerCustomized")


def check_scheduler_class(name):
    """Raises NotImplementedError unless `name` (a config's ``_class_name`` or a scheduler object's class name) is one of
    DDIM_CLASSES; None (a config that names no class) passes."""
    if name is not None and name not in DDIM_CLASSES:
        raise NotImplementedError(f"scheduler class {name!r} is not supported: the multi-step archs run DDIM steps "
                                  f"({' or '.join(DDIM_CLASSES)})")


class DDIMSchedule:
    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 trained_betas=None, clip_sample=True, set_alpha_to_one=True, steps_offset=0, prediction_type="epsilon",
                 thresholding=False, timestep_spacing="leading", rescale_betas_zero_snr=False, power_beta_curve=1.0,
                 **_ignored):
        n = int(num_train_timesteps)
        if trained_betas is not None:
            betas = np.asarray(trained_betas, dtype=np.float32)
        elif beta_schedule == "linear":
            betas = np.linspace(beta_start, beta_end, n, dtype=np.float32)
        elif beta_schedule == "scaled_linear":                   # ddim.py:170-172
            betas = np.linspace(np.float32(beta_start) ** 0.5, np.float32(beta_end) ** 0.5, n, dtype=np.float32) ** 2
        elif beta_schedule == "scaled_linear_power":             # ddim.py:173-175
            p = float(power_beta_curve)
            betas = np.linspace(np.float32(beta_start) ** (1 / p), np.float32(beta_end) ** (1 / p), n, dtype=np.float32) ** p
        else:
            raise NotImplementedError(f"{beta_schedule} is not implemented for {type(self).__name__}")
        if rescale_betas_zero_snr or thresholding:
            raise NotImplementedError("rescale_betas_zero_snr / thresholding are not used by the reference's configs")
        if clip_sample:
            raise NotImplementedError("clip_sample=True is not used by the reference's scheduler configs (all set it false)")
        self.num_train_timesteps = n
        self.beta_start, self.beta_end = float(beta_start), float(beta_end)
        self.betas = betas.astype(np.float32)
        self.alphas_cumprod = np.cumprod((1.0 - self.betas).astype(np.float32), dtype=np.float32)
        self.final_alpha_cumprod = np.float32(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.steps_offset = int(steps_offset)
        self.prediction_type = prediction_type
        self.timestep_spacing = timestep_spacing
        self.num_inference_steps = None
        self.timesteps = np.arange(0, n)[::-1].copy().astype(np.int64)

    @classmethod
    def from_config(cls, path_or_dict):
        """A ``scheduler_config.json`` file, the folder holding one, or the parsed dict.  Its ``_class_name``, when
        given, must be a DDIM class (check_scheduler_class)."""
        cfg = path_or_dict
        if not isinstance(cfg, dict):
            p = str(path_or_dict)
            if os.path.isdir(p):
                p = os.path.join(p, "scheduler_config.json")
            with open(p) as f:
                cfg = json.load(f)
        check_scheduler_class(cfg.get("_class_name"))
        return cls(**{k: v for k, v in cfg.items() if not k.startswith("_")})

    def set_timesteps(self, num_inference_steps, device=None):
        n, T = int(num_inference_steps), self.num_train_timesteps
        if n > T:
            raise ValueError(f"num_inference_steps ({n}) cannot exceed num_train_timesteps ({T})")
        self.num_inference_steps = n
        if self.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n).round()[::-1].copy().astype(np.int64)
        elif self.timestep_spacing == "leading":
            ts = (np.arange(0, n) * (T // n)).round()[::-1].copy().astype(np.int64) + self.steps_offset
        elif self.timestep_spacing == "trailing":
            ts = np.round(np.arange(T, 0, -T / n)).astype(np.int64) - 1
        else:
            raise ValueError(f"unsupported timestep_spacing {self.timestep_spacing!r}")
        self.timesteps = ts
        return ts

    def step_coefficients(self, timestep):
        """-> (c_x0_s, c_x0_m, c_pv_s, c_pv_m) for DDIMScheduler.step(model_output, timestep, sample) with eta = 0."""
        t = int(timestep)
        prev_t = t - self.num_train_timesteps // self.num_inference_steps
        a_t = float(self.alphas_cumprod[t])
        a_p = float(self.alphas_cumprod[prev_t]) if prev_t >= 0 else float(self.final_alpha_cumprod)
        b_t = 1.0 - a_t
        if self.prediction_type == "v_prediction":
            x0_s, x0_m = a_t ** 0.5, -(b_t ** 0.5)
            ep_s, ep_m = b_t ** 0.5, a_t ** 0.5
        elif self.prediction_type == "epsilon":
            x0_s, x0_m = 1.0 / a_t ** 0.5, -(b_t ** 0.5) / a_t ** 0.5
            ep_s, ep_m = 0.0, 1.0
        elif self.prediction_type == "sample":
            x0_s, x0_m = 0.0, 1.0
            ep_s, ep_m = 1.0 / b_t ** 0.5, -(a_t ** 0.5) / b_t ** 0.5
        else:
            raise ValueError(f"unsupported prediction_type {self.prediction_type!r}")
        d = (1.0 - a_p) ** 0.5                                   # direction pointing to x_t (std_dev_t = 0)
        return x0_s, x0_m, a_p ** 0.5 * x0_s + d * ep_s, a_p ** 0.5 * x0_m + d * ep_m
