"""CPU tests of the GenPercept v1 surface: the drop-in for tools/inference_genpercept.py, v1's __call__ signature, the
argument checks of the v1 C-ABI entry points and the hub's local-files-only loading."""
import inspect
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V1_REF = "/root/reference/GenPercept_v1"


def _run(args, cwd):
    p = subprocess.run([sys.executable] + args, cwd=cwd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True,
                       text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    return p.stdout


def _fake_v1_tree(tmp_path):
    pkg = tmp_path / "genpercept"
    (pkg / "util").mkdir(parents=True)
    (pkg / "__init__.py").write_text("")
    (pkg / "pipeline_genpercept.py").write_text("import diffusers_that_is_not_installed\n")
    (pkg / "util" / "__init__.py").write_text("")
    (pkg / "util" / "image_util.py").write_text("MARK = 'reference util'\n")
    (tmp_path / "tools").mkdir()
    (tmp_path / "tools" / "inference_genpercept.py").write_text(
        "import sys\nfrom genpercept.util.image_util import MARK\nfrom genpercept.pipeline_genpercept import GenPerceptPipeline\n"
        "print(GenPerceptPipeline.__module__, MARK, sys.argv[1:])\n")
    (tmp_path / "run.py").write_text("import sys\nprint('v1 seeded:', 'genpercept.pipeline_genpercept' in sys.modules)\n")


def test_install_v1_seeds_and_rebinds(tmp_path):
    _fake_v1_tree(tmp_path)
    code = ("import genpercept, genpercept.util.image_util as u; import genpercept_b200.dropin as d; m = d.install_v1(); "
            "assert d.install_v1() is m; from genpercept.pipeline_genpercept import GenPerceptPipeline as P; "
            "print(P.__module__, genpercept.pipeline_genpercept.GenPerceptPipeline.__module__, u.MARK)")
    out = _run(["-c", code], tmp_path)           # the parent package was imported first
    assert "genpercept_b200.v1 genpercept_b200.v1 reference util" in out
    if os.path.isdir(os.path.join(V1_REF, "genpercept")):       # and the real v1 checkout where it exists
        code = ("import genpercept_b200.dropin as d; d.install_v1(); import genpercept; "
                "from genpercept.pipeline_genpercept import GenPerceptPipeline as P; print(P.__module__, genpercept.__file__)")
        assert f"genpercept_b200.v1 {V1_REF}/genpercept/__init__.py" in _run(["-c", code], V1_REF)


def test_main_seeds_v1_only_for_the_v1_tool(tmp_path):
    _fake_v1_tree(tmp_path)
    out = _run(["-m", "genpercept_b200.dropin", "tools/inference_genpercept.py", "--mode", "depth"], tmp_path)
    assert "genpercept_b200.v1 reference util ['--mode', 'depth']" in out
    assert "v1 seeded: False" in _run(["-m", "genpercept_b200.dropin", "run.py"], tmp_path)


def test_call_signature_matches_v1(golden_dir):
    from genpercept_b200.v1 import GenPerceptPipeline
    ref = json.loads(str(np.load(os.path.join(golden_dir, "v1_call.npz"))["signature"]))
    sig = inspect.signature(GenPerceptPipeline.__call__)
    got = [(n, None if p.default is inspect.Parameter.empty else p.default) for n, p in sig.parameters.items() if n != "self"]
    assert [list(x) for x in got] == ref
    assert set(GenPerceptPipeline.task_infos) == {"depth", "seg", "sr", "normal"}
    init = inspect.signature(GenPerceptPipeline.__init__)
    assert list(init.parameters)[1:5] == ["unet", "vae", "customized_head", "empty_text_embed"]


def test_v1_entry_points_reject_bad_arguments_without_a_device():
    """Shape, mode and pointer checks come before any device call: GP_ERR_INVALID (1)."""
    from ctypes import c_void_p
    from genpercept_b200 import build, engine
    build.build()
    L = engine.lib()
    p = c_void_p(16)
    assert L.gp_resize_pil(None, 1, 4, 4, p, 0, 2, 2, None) == 1
    assert L.gp_resize_pil(p, 1, 4, 4, None, 0, 2, 2, None) == 1
    assert L.gp_resize_pil(p, 1, 0, 4, p, 0, 2, 2, None) == 1
    assert L.gp_resize_pil(p, 1, 4, 4, p, 0, 2, 0, None) == 1
    assert L.gp_v1_postprocess(None, 1, 1, 4, 4, 0, 8, 8, p, None, None) == 1
    assert L.gp_v1_postprocess(p, 1, 1, 4, 4, 3, 8, 8, p, p, None) == 1        # unknown task
    assert L.gp_v1_postprocess(p, 1, 3, 4, 4, 0, 8, 8, p, None, None) == 1     # depth takes one channel
    assert L.gp_v1_postprocess(p, 1, 1, 4, 4, 1, 8, 8, p, p, None) == 1        # normal takes three
    assert L.gp_v1_postprocess(p, 1, 3, 4, 4, 1, 8, 8, p, None, None) == 1     # normal writes both outputs
    assert L.gp_v1_postprocess(p, 1, 3, 4, 4, 2, 8, 8, p, None, None) == 1     # seg writes the uint8 map
    assert L.gp_v1_postprocess(p, 0, 1, 4, 4, 0, 8, 8, p, None, None) == 1
    assert L.gp_v1_postprocess(p, 1, 1, 4, 4, 0, 8, 0, p, None, None) == 1


def test_v1_pipeline_refuses_what_it_does_not_offer():
    from genpercept_b200.v1 import GenPerceptPipeline
    with pytest.raises(NotImplementedError, match="DPTNeckHeadForUnetAfterUpsample"):
        GenPerceptPipeline({}, {}, customized_head=object(), empty_text_embed=np.zeros((1, 77, 1024)))
    with pytest.raises(ValueError, match="empty_text_embed"):
        GenPerceptPipeline({}, {})
    import torch
    with pytest.raises(NotImplementedError, match="conv_out"):
        GenPerceptPipeline({"conv_in.weight": torch.zeros(1)}, {"decoder.conv_in.weight": torch.zeros(1)}, None,
                           np.zeros((1, 77, 1024)))
    with pytest.raises(NotImplementedError, match="decoder"):
        GenPerceptPipeline({"conv_out.weight": torch.zeros(1)}, {"encoder.conv_in.weight": torch.zeros(1)}, None,
                           np.zeros((1, 77, 1024)))


def test_hub_reads_local_files_only(tmp_path):
    from genpercept_b200 import hub
    src = open(os.path.join(ROOT, "genpercept_b200", "hub.py")).read()
    assert "huggingface_hub" not in src
    with pytest.raises(FileNotFoundError, match="unet_depth_v1"):
        hub.GenPercept_Depth(local_dir=str(tmp_path))
    (tmp_path / "unet_normal_v1").mkdir()
    (tmp_path / "unet_normal_v1" / "diffusion_pytorch_model.safetensors").write_bytes(b"")
    with pytest.raises(FileNotFoundError, match="vae"):
        hub.GenPercept_Normal(local_dir=str(tmp_path))
    with pytest.raises(FileNotFoundError):
        hub.GenPercept_Segmentation()
    hubconf = open(os.path.join(ROOT, "hubconf.py")).read()
    for name in ("GenPercept_Depth", "GenPercept_Normal", "GenPercept_Segmentation"):
        assert name in hubconf
