"""CPU tests of the multi-step archs' host side: the checkpoint's own scheduler folder, the scheduler class check, and the
layout of the per-step bias table that gp_infer_steps scatters on the device."""
import json
import os
import re
import types

import pytest
import torch

# the contents of the reference's hf_configs/scheduler_beta_0.00085_0.012/scheduler_config.json
SCHED = {"_class_name": "DDIMScheduler", "_diffusers_version": "0.29.2", "beta_end": 0.012, "beta_schedule": "scaled_linear",
         "beta_start": 0.00085, "clip_sample": False, "clip_sample_range": 1.0, "dynamic_thresholding_ratio": 0.995,
         "num_train_timesteps": 1000, "prediction_type": "v_prediction", "rescale_betas_zero_snr": False,
         "sample_max_value": 1.0, "set_alpha_to_one": False, "skip_prk_steps": True, "steps_offset": 1,
         "thresholding": False, "timestep_spacing": "leading", "trained_betas": None}


class _HostEngine:
    """Stands in for the native engine, so the pipeline's constructor runs without a device."""

    def __init__(self, **kw):
        self.device = torch.device("cpu")

    def load_state(self, component, sd):
        pass


@pytest.fixture
def no_engine(monkeypatch):
    from genpercept_b200 import pipeline
    monkeypatch.setattr(pipeline, "Engine", _HostEngine)
    return pipeline.GenPerceptPipeline


def _checkpoint(tmp_path, cfg):
    d = tmp_path / "scheduler"
    d.mkdir()
    (d / "scheduler_config.json").write_text(json.dumps(cfg))
    return str(tmp_path)


def test_from_pretrained_reads_the_checkpoint_scheduler(tmp_path, no_engine):
    from genpercept_b200.scheduler import DDIMSchedule
    root = _checkpoint(tmp_path, SCHED)
    pipe = no_engine.from_pretrained(root, genpercept_pipeline=False, unet={}, vae={})
    s = pipe.scheduler
    assert isinstance(s, DDIMSchedule)
    assert (s.beta_start, s.beta_end, s.prediction_type, s.steps_offset) == (0.00085, 0.012, "v_prediction", 1)
    assert s.set_timesteps(10).tolist() == [901, 801, 701, 601, 501, 401, 301, 201, 101, 1]
    ref = DDIMSchedule.from_config(dict(SCHED))
    ref.set_timesteps(10)
    assert s.step_coefficients(501) == ref.step_coefficients(501)


def test_from_run_args_reads_the_checkpoint_scheduler(tmp_path, no_engine, monkeypatch):
    from genpercept_b200 import loader
    from genpercept_b200.scheduler import DDIMSchedule
    monkeypatch.setattr(loader, "assemble", lambda *a, **k: {"unet": {}, "vae": {}, "customized_head": None})
    root = _checkpoint(tmp_path, SCHED)
    pipe = no_engine.from_run_args(root, genpercept_pipeline=False)
    assert isinstance(pipe.scheduler, DDIMSchedule) and pipe.scheduler.beta_end == 0.012


def test_a_passed_scheduler_wins_over_the_folder(tmp_path, no_engine):
    root = _checkpoint(tmp_path, dict(SCHED, _class_name="LCMScheduler"))      # never read
    pipe = no_engine.from_pretrained(root, genpercept_pipeline=False, unet={}, vae={}, scheduler=dict(SCHED, beta_end=0.02))
    assert pipe.scheduler.beta_end == 0.02


def test_missing_scheduler_folder_names_the_path(tmp_path, no_engine):
    path = os.path.join(str(tmp_path), "scheduler", "scheduler_config.json")
    with pytest.raises(ValueError, match=re.escape(path)):
        no_engine.from_pretrained(str(tmp_path), genpercept_pipeline=False, unet={}, vae={})
    with pytest.raises(ValueError, match=re.escape(path)):
        no_engine.from_run_args(str(tmp_path), genpercept_pipeline=False)


def test_one_step_pipeline_does_not_read_the_folder(tmp_path, no_engine):
    pipe = no_engine.from_pretrained(str(tmp_path), unet={}, vae={})      # genpercept_pipeline=True: no scheduler/ needed
    assert pipe.scheduler is None


def test_other_scheduler_classes_are_refused(tmp_path, no_engine):
    from genpercept_b200.scheduler import DDIMSchedule
    lcm = dict(SCHED, _class_name="LCMScheduler")
    with pytest.raises(NotImplementedError, match="LCMScheduler"):
        DDIMSchedule.from_config(lcm)
    with pytest.raises(NotImplementedError, match="LCMScheduler"):
        no_engine(unet={}, vae={}, scheduler=lcm, genpercept_pipeline=False)
    with pytest.raises(NotImplementedError, match="LCMScheduler"):
        no_engine.from_pretrained(_checkpoint(tmp_path, lcm), genpercept_pipeline=False, unet={}, vae={})
    cfg = {k: v for k, v in SCHED.items() if not k.startswith("_")}
    LCMScheduler = type("LCMScheduler", (), {})
    obj = LCMScheduler()
    obj.config = cfg                                     # no _class_name in the config: the object's class decides
    with pytest.raises(NotImplementedError, match="LCMScheduler"):
        no_engine(unet={}, vae={}, scheduler=obj, genpercept_pipeline=False)


def test_ddim_scheduler_classes_are_accepted(no_engine):
    from genpercept_b200.scheduler import DDIMSchedule
    cfg = {k: v for k, v in SCHED.items() if not k.startswith("_")}
    for name in ("DDIMScheduler", "DDIMSchedulerCustomized"):
        assert DDIMSchedule.from_config(dict(cfg, _class_name=name)).beta_start == 0.00085
        obj = type(name, (), {})()
        obj.config = cfg
        assert no_engine(unet={}, vae={}, scheduler=obj, genpercept_pipeline=False).scheduler.beta_end == 0.012
    assert DDIMSchedule.from_config(cfg).prediction_type == "v_prediction"          # no _class_name: accepted
    ns = types.SimpleNamespace(config=dict(cfg, _class_name="DDIMSchedulerCustomized"))   # the config's name decides
    assert no_engine(unet={}, vae={}, scheduler=ns, genpercept_pipeline=False).scheduler.steps_offset == 1


def test_step_bias_layout_covers_every_time_embedded_resnet_once():
    """The row of gp_infer_steps' bias table: one segment per time-embedded UNet ResNet, back to back, 20160 floats."""
    from genpercept_b200 import build, engine
    build.build()
    layout = engine.step_bias_layout()
    assert len(layout) == 22
    off = 0
    for o, n in layout:
        assert o == off and n > 0
        off += n
    assert off == 20160
    # down blocks (2 per level), mid block, up blocks (3 per level) in the order unet() emits them
    assert [n for _, n in layout] == [320] * 2 + [640] * 2 + [1280] * 4 + [1280] * 2 + [1280] * 6 + [640] * 3 + [320] * 3
