"""CPU tests of the depth evaluation: the oracle (oracle/evaluation.py) against the reference's own alignment and metrics
(tests/golden/depth_eval_ref.npz), the nearest-downscale rule against torch, the pandas-free MetricTracker, argument
checks of the C-ABI, and the eval.py drop-in import route."""
import importlib.util
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("make_golden_eval", os.path.join(ROOT, "tests", "golden", "make_golden_eval.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)
CASES = {c[0]: c for c in G.cases()}
DELTAS = ("delta1_acc", "delta2_acc", "delta3_acc")


@pytest.fixture(scope="module")
def golden():
    return np.load(G.GOLDEN)


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_reproduces_the_reference(name, golden):
    from oracle import evaluation as O
    _, pred, gt, valid, alignment, max_res, lo, hi = CASES[name]
    np.testing.assert_array_equal(G.checksum(pred, gt, valid), golden[f"{name}.checksum"])     # same seeded inputs
    got, scale, shift = O.evaluate(pred, gt, valid, alignment, max_res, lo, hi)
    if alignment is not None:
        ref_s, ref_t = golden[f"{name}.scale_shift"]
        assert scale.dtype == np.float32 and shift.dtype == np.float32
        assert math.isclose(scale, ref_s, rel_tol=1e-6, abs_tol=0) or scale == ref_s == 0
        assert math.isclose(shift, ref_t, rel_tol=1e-6, abs_tol=0) or shift == ref_t == 0
    n = int(valid.sum())
    for k, ref in zip(O.METRICS, golden[f"{name}.metrics"]):
        if n == 0:
            assert math.isnan(got[k]) and math.isnan(ref), k
        elif k in DELTAS:
            assert round(got[k] * n) == round(float(ref) * n), (k, got[k], ref)          # exact counts
        else:
            assert math.isclose(got[k], ref, rel_tol=1e-6), (k, got[k], ref)


def test_golden_covers_the_cases_the_evaluation_meets():
    kinds = {(c[4], c[5]) for c in CASES.values()}
    assert ("least_square", None) in kinds and ("least_square_disparity", None) in kinds and (None, None) in kinds
    from oracle.evaluation import fit_grid
    sized = [(c[1].shape, c[5]) for c in CASES.values() if c[5] is not None]
    assert any(fit_grid(*s, m)[1] is None for s, m in sized)                 # a max_res that does not downscale
    assert any(fit_grid(*s, m)[1] is not None for s, m in sized)
    assert any(c[3].sum() == 0 for c in CASES.values())                        # a mask with no valid pixel
    assert any(np.unique(c[1]).size == 1 for c in CASES.values())              # a constant prediction
    assert any((c[1] < 0).any() and c[4] == "least_square_disparity" for c in CASES.values())


@pytest.mark.parametrize("H,W,max_res", [(480, 640, 1024), (352, 1216, 1024), (333, 517, 200), (37, 53, 20),
                                         (64, 96, 50), (4032, 6048, 1024), (1080, 1920, 700), (5, 100, 20)])
def test_nearest_rule_matches_torch(H, W, max_res):
    """align_depth_least_square resamples the squeezed [H,W] map as `Upsample(...)(map.unsqueeze(0))`: a 3-D input,
    so torch runs a 1-D nearest resample along W with the fp64 factor min(max_res / (H, W))."""
    from oracle.evaluation import fit_grid, nearest_index
    s = float(np.min(max_res / np.array([H, W])))
    fit_w, inv = fit_grid(H, W, max_res)
    if s >= 1:
        assert inv is None and fit_w == W
        return
    src = torch.arange(W, dtype=torch.float32).expand(H, W).contiguous()
    out = torch.nn.Upsample(scale_factor=s, mode="nearest")(src.unsqueeze(0))[0]
    assert tuple(out.shape) == (H, fit_w)
    ref = torch.nn.functional.interpolate(src[:1][None], scale_factor=s, mode="nearest")[0, 0]
    np.testing.assert_array_equal(out[0].numpy().astype(np.int64), nearest_index(W, fit_w, inv))
    np.testing.assert_array_equal(ref.numpy().astype(np.int64), nearest_index(W, fit_w, inv))


def test_metric_tracker_without_pandas():
    from genpercept_b200.evaluation import MetricTracker
    t = MetricTracker("a", "b")
    t.update("a", 1.0)
    t.update("a", 4.0, n=3)
    assert t.avg("a") == pytest.approx(13.0 / 4) and t.avg("b") == 0
    assert t.result() == {"a": pytest.approx(3.25), "b": 0}
    t.reset()
    assert t.result() == {"a": 0, "b": 0}


def test_depth2disparity_keeps_the_kind():
    from genpercept_b200.evaluation import depth2disparity, disparity2depth
    a = np.array([[2.0, 0.0], [-1.0, 0.5]], dtype=np.float32)
    d, m = depth2disparity(a, return_mask=True)
    assert isinstance(d, np.ndarray) and d.dtype == np.float32
    np.testing.assert_array_equal(d, [[0.5, 0.0], [0.0, 2.0]])
    np.testing.assert_array_equal(m, a > 0)
    t = disparity2depth(torch.from_numpy(a))
    assert isinstance(t, torch.Tensor) and torch.equal(t, torch.from_numpy(d))


def test_c_abi_rejects_bad_arguments_without_a_device():
    """Shape and mode checks come before any device call: GP_ERR_INVALID (1) everywhere."""
    from ctypes import c_void_p
    from genpercept_b200 import build, engine
    build.build()
    L = engine.lib()
    p = c_void_p(16)
    assert L.gp_depth_align(None, p, None, 1, 4, 4, 0, 0, p, None, None) == 1
    assert L.gp_depth_align(p, p, None, 1, 4, 4, 2, 0, p, None, None) == 1        # unknown mode
    assert L.gp_depth_align(p, p, None, 0, 4, 4, 0, 0, p, None, None) == 1        # B < 1
    assert L.gp_depth_align(p, p, None, 1, 1000, 2, 0, 10, p, None, None) == 1    # max_res leaves no column
    assert L.gp_depth_metrics(p, p, None, 1, 4, 4, 3, p, 0.0, 1.0, p, None) == 1  # unknown mode
    assert L.gp_depth_metrics(p, p, None, 1, 4, 4, 1, None, 0.0, 1.0, p, None) == 1   # alignment without scale/shift
    assert L.gp_depth_metrics(p, p, None, 1, 0, 4, 0, None, 0.0, 1.0, p, None) == 1


def _make_reference_style_tree(tmp_path):
    (tmp_path / "src" / "util").mkdir(parents=True)
    (tmp_path / "src" / "dataset").mkdir()
    (tmp_path / "src" / "__init__.py").write_text("")
    (tmp_path / "src" / "util" / "metric.py").write_text("import pandas_that_is_not_installed\n")
    (tmp_path / "src" / "util" / "alignment.py").write_text("MARK = 'reference alignment'\n")
    (tmp_path / "src" / "dataset" / "__init__.py").write_text("MARK = 'reference dataset'\n")
    body = ("import sys\nfrom src.dataset import MARK\nfrom src.util import metric\n"
            "from src.util.alignment import align_depth_least_square as A\nfrom src.util.metric import MetricTracker\n"
            "print(metric.__name__, A.__module__, MetricTracker.__module__, getattr(metric, 'delta1_acc').__name__, MARK)\n")
    (tmp_path / "eval.py").write_text(body)
    (tmp_path / "run.py").write_text("import sys\nfrom src.util.alignment import MARK\n"
                                     "print(MARK, 'src.util.metric' in sys.modules)\n")


def test_dropin_seeds_the_eval_import_path(tmp_path):
    """eval.py does `from src.util import metric`, `from src.util.alignment import ...` and `from src.util.metric import
    MetricTracker`; under the drop-in all three resolve to genpercept_b200.evaluation (the reference's metric.py, which
    needs pandas, never runs) while src.dataset comes from the checkout.  run.py seeds nothing new."""
    _make_reference_style_tree(tmp_path)
    env = dict(os.environ, PYTHONPATH=ROOT)
    p = subprocess.run([sys.executable, "-m", "genpercept_b200.dropin", "eval.py", "--alignment", "least_square"],
                       cwd=tmp_path, env=env, capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    mod = "genpercept_b200.evaluation"
    assert f"{mod} {mod} {mod} delta1_acc reference dataset" in p.stdout
    q = subprocess.run([sys.executable, "-m", "genpercept_b200.dropin", "run.py"], cwd=tmp_path, env=env,
                       capture_output=True, text=True, timeout=300)
    assert q.returncode == 0, q.stderr[-2000:]
    assert "reference alignment False" in q.stdout
    ref = "/root/reference"
    if os.path.isfile(os.path.join(ref, "src", "util", "metric.py")):     # and against the real checkout where it exists
        code = ("import genpercept_b200.dropin as d; d.install_evaluation(); import src; from src.util import metric; "
                "from src.util.alignment import align_depth_least_square as A; "
                "print(metric.__name__, A.__module__, src.__file__)")
        r = subprocess.run([sys.executable, "-c", code], cwd=ref, env=env, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr[-2000:]
        assert f"{mod} {mod} {ref}/src/__init__.py" in r.stdout
