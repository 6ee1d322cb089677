"""CPU tests of the shared activation arena's surface: the library exports its entry points, and
MultiTaskPipeline(share_arena=...) turns sharing on for every task's engine (stub engines; no device needed)."""
import ctypes

import pytest

from genpercept_b200 import engine as E
from genpercept_b200.multitask import MultiTaskPipeline
from test_multitask_cpu import _modes, _pipe


def test_library_exports_the_shared_arena_entry_points():
    L = ctypes.CDLL(E.LIB_PATH)
    for name in ("gp_set_shared_arena", "gp_shared_arena_info", "gp_shared_arena_fill"):
        assert hasattr(L, name), name


class _StubEngine:
    def __init__(self):
        self.calls = []

    def set_shared_arena(self, flag):
        self.calls.append(bool(flag))


@pytest.mark.parametrize("share", [False, True])
def test_multitask_share_arena_reaches_every_engine(share):
    pipes = {"depth": _pipe(), "normal": _pipe(), "seg": _pipe()}
    for p in pipes.values():
        p._engine = _StubEngine()
    MultiTaskPipeline(pipes, _modes(pipes), share_arena=share)
    for name, p in pipes.items():
        assert p._engine.calls == ([True] if share else []), name


def test_multitask_checks_run_before_any_engine_changes():
    pipes = {"depth": _pipe(), "normal": _pipe(one_step=False)}
    for p in pipes.values():
        p._engine = _StubEngine()
    with pytest.raises(ValueError, match="'normal'"):
        MultiTaskPipeline(pipes, _modes(pipes), share_arena=True)
    assert all(p._engine.calls == [] for p in pipes.values())
