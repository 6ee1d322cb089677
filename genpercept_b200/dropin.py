"""Zero-edit drop-in for the reference's drivers.

The reference's CLIs import the pipeline as ``from genpercept import GenPerceptPipeline``
(/root/reference/run.py:33, /root/reference/infer.py) and ``genpercept/__init__.py:18`` resolves that through
``from .genpercept_pipeline import GenPerceptPipeline, GenPerceptOutput``.  Python looks a submodule up in
``sys.modules`` before it looks on disk, so seeding ``sys.modules["genpercept.genpercept_pipeline"]`` with a module
that exports this package's classes makes the unmodified ``run.py`` / ``infer.py`` construct the native engine — while
``genpercept.models.*`` / ``genpercept.util.*`` (which run.py also imports) keep coming from the reference checkout.

    cd /path/to/GenPercept
    PYTHONPATH=/path/to/genpercept_b200_repo python -m genpercept_b200.dropin run.py --checkpoint ... --unet ...

or, from Python, ``import genpercept_b200.dropin; genpercept_b200.dropin.install()`` before the first
``import genpercept``.

For ``eval.py`` (and only for it) the drop-in also seeds ``sys.modules["src.util.alignment"]`` and
``sys.modules["src.util.metric"]`` with ``genpercept_b200.evaluation``, so eval.py's ``from src.util import metric``,
``getattr(metric, name)``, ``MetricTracker`` and ``align_depth_least_square`` run on the GPU while ``src.dataset`` keeps
coming from the reference checkout:

    PYTHONPATH=/path/to/genpercept_b200_repo python -m genpercept_b200.dropin eval.py --prediction_dir ... --alignment ...

For GenPercept v1's tool (``tools/inference_genpercept.py``, which imports
``from genpercept.pipeline_genpercept import GenPerceptPipeline``), and only for it, the drop-in also seeds
``sys.modules["genpercept.pipeline_genpercept"]`` with ``genpercept_b200.v1``'s classes.  From ``GenPercept_v1/``:

    PYTHONPATH=/path/to/genpercept_b200_repo python -m genpercept_b200.dropin tools/inference_genpercept.py \
        --input_rgb_dir input/depth --output_dir output/depth --mode depth \
        --checkpoint weights/v1 --unet_ckpt_path weights/v1/unet_depth_v1
"""
import runpy
import sys
import types

_NAME = "genpercept.genpercept_pipeline"
_EVAL_NAMES = ("src.util.alignment", "src.util.metric")
_V1_NAME = "genpercept.pipeline_genpercept"


def install():
    """Idempotent.  Returns the seeded module."""
    mod = sys.modules.get(_NAME)
    if mod is not None and getattr(mod, "__genpercept_b200__", False):
        return mod
    from .pipeline import GenPerceptOutput, GenPerceptPipeline
    mod = types.ModuleType(_NAME, "genpercept_b200 drop-in for genpercept/genpercept_pipeline.py")
    mod.GenPerceptPipeline = GenPerceptPipeline
    mod.GenPerceptOutput = GenPerceptOutput
    mod.__genpercept_b200__ = True
    sys.modules[_NAME] = mod
    parent = sys.modules.get("genpercept")
    if parent is not None:            # the reference package was imported first: rebind what its __init__ re-exported
        parent.genpercept_pipeline = mod
        parent.GenPerceptPipeline = GenPerceptPipeline
        parent.GenPerceptOutput = GenPerceptOutput
    return mod


def install_v1():
    """Idempotent.  Seeds genpercept.pipeline_genpercept (GenPercept v1) with genpercept_b200.v1's classes; returns it."""
    mod = sys.modules.get(_V1_NAME)
    if mod is not None and getattr(mod, "__genpercept_b200__", False):
        return mod
    from .v1 import GenPerceptOutput, GenPerceptPipeline
    mod = types.ModuleType(_V1_NAME, "genpercept_b200 drop-in for GenPercept_v1/genpercept/pipeline_genpercept.py")
    mod.GenPerceptPipeline = GenPerceptPipeline
    mod.GenPerceptOutput = GenPerceptOutput
    mod.__genpercept_b200__ = True
    sys.modules[_V1_NAME] = mod
    parent = sys.modules.get("genpercept")
    if parent is not None:            # the v1 package was imported first: rebind its submodule attribute
        parent.pipeline_genpercept = mod
    return mod


def install_evaluation():
    """Idempotent.  Seeds src.util.alignment / src.util.metric with genpercept_b200.evaluation; returns it."""
    from . import evaluation
    for name in _EVAL_NAMES:
        sys.modules[name] = evaluation
        parent = sys.modules.get("src.util")
        if parent is not None:        # src.util was imported first: rebind its submodule attributes too
            setattr(parent, name.rsplit(".", 1)[1], evaluation)
    return evaluation


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv:
        sys.exit("usage: python -m genpercept_b200.dropin <run.py|infer.py|eval.py|tools/inference_genpercept.py> "
                 "[its arguments ...]")
    install()
    script = argv[0]
    import os
    if os.path.basename(script) == "eval.py":
        install_evaluation()
    if os.path.basename(script) == "inference_genpercept.py":
        install_v1()
    sys.argv = argv
    sys.path.insert(0, os.path.dirname(os.path.abspath(script)))      # what `python script.py` would have done
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main()
