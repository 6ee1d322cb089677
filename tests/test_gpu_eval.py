"""GPU depth evaluation (csrc/evaluate.cu through genpercept_b200.evaluation) against the CPU oracle
(oracle/evaluation.py, pinned on the reference in tests/test_eval_cpu.py): every golden case, a batch of four,
determinism, 24 MP maps, the engine's own output, and the alignment.py / metric.py replacements."""
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("make_golden_eval", os.path.join(ROOT, "tests", "golden", "make_golden_eval.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)
CASES = {c[0]: c for c in G.cases()}
DELTAS = ("delta1_acc", "delta2_acc", "delta3_acc")


def _ulps(a, b):
    a, b = np.float32(a), np.float32(b)
    return abs(int(a.view(np.int32)) - int(b.view(np.int32))) if np.sign(a) == np.sign(b) else (0 if a == b else 1 << 30)


def _check(got, scale, shift, ref, ref_scale, ref_shift, n, alignment):
    from oracle.evaluation import METRICS
    if alignment is not None:
        assert _ulps(scale, ref_scale) <= 1, (scale, ref_scale)
        assert _ulps(shift, ref_shift) <= 1, (shift, ref_shift)
    for k in METRICS:
        g, r = float(got[k]), ref[k]
        if n == 0:
            assert math.isnan(g) and math.isnan(r), k
        elif k in DELTAS:
            assert abs(g - r) <= 2.0 / n, (k, g, r)
        else:
            assert math.isclose(g, r, rel_tol=1e-5), (k, g, r)


@pytest.mark.parametrize("name", list(CASES))
def test_kernel_matches_the_oracle(name):
    from genpercept_b200.evaluation import evaluate
    from oracle import evaluation as O
    _, pred, gt, valid, alignment, max_res, lo, hi = CASES[name]
    ref, rs, rt = O.evaluate(pred, gt, valid, alignment, max_res, lo, hi)
    m, s, t = evaluate(torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda(), torch.from_numpy(valid).cuda(),
                       alignment, max_res, lo, hi)
    assert m["rmse_linear"].is_cuda and m["rmse_linear"].dtype == torch.float64 and s.dtype == torch.float32
    _check({k: v[0].item() for k, v in m.items()}, s[0].item(), t[0].item(), ref, rs, rt, int(valid.sum()), alignment)
    if int(valid.sum()) == 0 and alignment is not None:
        assert s[0].item() == 0 and t[0].item() == 0          # np.linalg.lstsq of an empty system


@pytest.mark.parametrize("alignment,max_res", [("least_square", None), ("least_square_disparity", 1024), (None, None)])
def test_batch_of_four(alignment, max_res):
    from genpercept_b200.evaluation import evaluate
    from oracle import evaluation as O
    kind = "disparity" if alignment == "least_square_disparity" else ("metric" if alignment is None else "relative")
    ins = [G.make_inputs(352, 1216, 100 + i, kind, 10.0) for i in range(4)]
    stack = lambda j: torch.from_numpy(np.stack([x[j] for x in ins])).cuda()
    m, s, t = evaluate(stack(0), stack(1), stack(2), alignment, max_res, 1e-5, 80.0)
    for i, (p, g, v) in enumerate(ins):
        ref, rs, rt = O.evaluate(p, g, v, alignment, max_res, 1e-5, 80.0)
        _check({k: x[i].item() for k, x in m.items()}, s[i].item(), t[i].item(), ref, rs, rt, int(v.sum()), alignment)


def test_two_calls_are_bit_identical():
    from genpercept_b200.evaluation import evaluate
    ins = [G.make_inputs(480, 640, 200 + i, "disparity", 2.0) for i in range(4)]
    args = [torch.from_numpy(np.stack([x[j] for x in ins])).cuda() for j in range(3)]
    a = evaluate(*args, "least_square_disparity", 300, 1e-3, 10.0)
    b = evaluate(*args, "least_square_disparity", 300, 1e-3, 10.0)
    for k in a[0]:
        assert torch.equal(a[0][k], b[0][k]), k
    assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


@pytest.mark.parametrize("max_res", [1024, None])
def test_24mp_batch_of_two(max_res):
    """ETH3D-sized ground truth (4032 x 6048), batch 2, made on the device; image 0 against the oracle."""
    from genpercept_b200.evaluation import evaluate
    from oracle import evaluation as O
    g = torch.Generator(device="cuda").manual_seed(7)
    H, W = 4032, 6048
    gt = torch.rand((2, H, W), generator=g, device="cuda") * 20 + 0.5
    valid = torch.rand((2, H, W), generator=g, device="cuda") > 0.3
    pred = (gt - 0.5) / 20 + torch.randn((2, H, W), generator=g, device="cuda") * 0.02
    m, s, t = evaluate(pred, gt, valid, "least_square", max_res, 1e-5, float("inf"))
    torch.cuda.synchronize()
    ref, rs, rt = O.evaluate(pred[0].cpu(), gt[0].cpu(), valid[0].cpu(), "least_square", max_res, 1e-5, float("inf"))
    _check({k: x[0].item() for k, x in m.items()}, s[0].item(), t[0].item(), ref, rs, rt, int(valid[0].sum()),
           "least_square")
    assert abs(s[1].item() - 20) < 0.5 and abs(t[1].item() - 0.5) < 0.5


def test_engine_output_straight_into_evaluate(synth_state, text_embed, golden_dir):
    """The engine's 64² map, resized on the GPU to a 96 x 80 ground truth, evaluated without leaving the device."""
    from genpercept_b200 import engine as E
    from genpercept_b200.evaluation import evaluate
    from oracle import evaluation as O
    gd = np.load(os.path.join(golden_dir, "oracle_e2e_64.npz"))
    e = E.Engine(dtype=torch.float16, readout="vae")
    e.load_state("unet", synth_state["unet"])
    e.load_state("vae", synth_state["vae"])
    e.set_text_embed(text_embed)
    e.finalize()
    depth = E.resize_aa(e.infer(torch.from_numpy(gd["rgb"]).cuda(), out_channels=1)[:, 0], 96, 80)
    e.close()
    g = torch.Generator().manual_seed(3)
    gt = (torch.rand((2, 96, 80), generator=g) * 5 + 0.5).cuda()
    valid = (torch.rand((2, 96, 80), generator=g) > 0.1).cuda()
    for alignment in ("least_square", "least_square_disparity"):
        m, s, t = evaluate(depth, gt, valid, alignment, None, 1e-3, 10.0)
        for i in range(2):
            ref, rs, rt = O.evaluate(depth[i].cpu(), gt[i].cpu(), valid[i].cpu(), alignment, None, 1e-3, 10.0)
            _check({k: x[i].item() for k, x in m.items()}, s[i].item(), t[i].item(), ref, rs, rt,
                   int(valid[i].sum()), alignment)


def test_alignment_and_metric_functions_keep_the_reference_interface(golden_dir):
    """align_depth_least_square / metric functions as eval.py calls them: numpy in, numpy out (aligned map bit-equal to
    pred * scale + shift in numpy float32); CUDA in, CUDA out; metrics as 0-d tensors."""
    from genpercept_b200 import evaluation as EV
    from oracle import evaluation as O
    golden = np.load(G.GOLDEN)
    _, pred, gt, valid, _, max_res, lo, hi = CASES["kitti_ls_max1024"]
    aligned, scale, shift = EV.align_depth_least_square(gt, pred, valid, True, max_res)
    assert isinstance(aligned, np.ndarray) and aligned.dtype == np.float32 and scale.shape == (1,) and shift.shape == (1,)
    rs, rt = golden["kitti_ls_max1024.scale_shift"]
    assert _ulps(scale[0], rs) <= 1 and _ulps(shift[0], rt) <= 1
    assert np.array_equal(aligned, pred * scale + shift)
    a2, s2, t2 = EV.align_depth_least_square(torch.from_numpy(gt).cuda(), torch.from_numpy(pred).cuda()[None],
                                             torch.from_numpy(valid).cuda(), max_resolution=max_res)
    assert a2.is_cuda and tuple(a2.shape) == (1,) + pred.shape and s2.is_cuda
    assert np.array_equal(a2.cpu().numpy()[0], aligned)
    depth = np.clip(np.clip(aligned, lo, hi), 1e-6, None)
    ref = O.metrics(depth, gt, valid)
    p_t, g_t, v_t = (torch.from_numpy(x).cuda() for x in (depth, gt, valid))
    for k in O.METRICS:
        v = getattr(EV, k)(p_t, g_t, v_t)
        assert v.dim() == 0 and v.is_cuda and getattr(EV, k).__name__ == k
        assert math.isclose(v.item(), ref[k], rel_tol=1e-5, abs_tol=2.0 / valid.sum() if k in DELTAS else 0), k
    # a batch: log10 is the mean over all valid pixels of the batch, the others means of per-image values
    p2, g2, v2 = (torch.stack([x, x.flip(-1)]) for x in (p_t, g_t, v_t))
    both = np.concatenate([depth, depth[:, ::-1]], axis=1)
    assert math.isclose(EV.log10(p2, g2, v2).item(), O.metrics(both, np.concatenate([gt, gt[:, ::-1]], 1),
                                                               np.concatenate([valid, valid[:, ::-1]], 1))["log10"],
                        rel_tol=1e-5)
    assert math.isclose(EV.rmse_linear(p2, g2, v2).item(), ref["rmse_linear"], rel_tol=1e-5)
