"""The apply predicate every Python front end shares (no GPU): the pure-Python ``is_apply_step`` agrees with the C
library's ``gaccum_is_apply_step``, and the all-reduce data-parallel driver takes its branch from it."""
import pytest
import torch

import gaccum_b200 as g
from gaccum_b200 import _lib, distributed

SMALL_N = [1, 2, 3, 4, 7, 8]
EDGE_STEPS = [2**31 - 1, 2**31, 2**31 + 1, 2**32, 2**32 + 1, -1, -2**31, 2**40 + 5, 2**63 - 1]


@pytest.mark.parametrize("n", SMALL_N + [2**31 - 1, 0, -1])
def test_python_predicate_matches_the_c_library(n):
    c_pred = _lib._load().gaccum_is_apply_step
    steps = (list(range(3 * n + 1)) if n in SMALL_N else []) + EDGE_STEPS + [2**32 + n]
    for s in steps:
        got = g.is_apply_step(s, n)
        assert isinstance(got, bool) and got == bool(c_pred(s, n)), (s, n)


class FakeEngine:
    """Just the engine interface DataParallelTrainOp may use (what tests/test_dp_gloo.py's OracleEngine has)."""

    def __init__(self, N, global_step, calls):
        self.N, self.global_step, self.calls = N, global_step, calls
        self.accum = torch.zeros(8)
        self.names = ["w"]
        self.hp = type("HP", (), {"variant": 0})()

    def run(self, grads):
        self.calls.append("run")
        applied = _lib.is_apply_step(self.global_step, self.N)
        self.global_step += 1
        return applied

    def accumulate_only(self, grads):
        self.calls.append("accumulate_only")

    def apply_only(self, grads):
        assert grads is None
        self.calls.append("apply_only")


@pytest.mark.parametrize("step,applies", [
    (2**32, True),          # int32(2^32) = 0: the reference applies although 2^32 % 3 == 1
    (2**32 + 1, False),     # both readings accumulate
    (2**32 + 2, False),     # int32 gives 2: the reference accumulates although (2^32 + 2) % 3 == 0
])
def test_allreduce_driver_branches_on_the_int32_step(monkeypatch, step, applies):
    calls = []
    monkeypatch.setattr(distributed.dist, "all_reduce", lambda t, op=None, group=None: calls.append("all_reduce"))
    dp = distributed.DataParallelTrainOp(FakeEngine(3, step, calls), None)
    dp.world = 2
    assert dp.run([torch.zeros(8)]) is applies
    if applies:
        assert calls == ["accumulate_only", "all_reduce", "apply_only"] and dp.allreduces == 1
    else:
        assert calls == ["run"] and dp.allreduces == 0
    assert dp.engine.global_step == step + 1
