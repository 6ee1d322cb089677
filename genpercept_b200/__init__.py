"""genpercept_b200 — H100-native (sm_90a) engine behind the GenPerceptPipeline API.

``from genpercept_b200 import GenPerceptPipeline, GenPerceptOutput`` mirrors
``from genpercept import GenPerceptPipeline, GenPerceptOutput``
(/root/reference/genpercept/__init__.py:18).  Importing the package does not need a GPU; building
a pipeline does (there is no CPU fallback).
"""
__all__ = ["GenPerceptPipeline", "GenPerceptOutput"]


def __getattr__(name):
    if name in __all__:
        from . import pipeline
        return getattr(pipeline, name)
    raise AttributeError(name)
