"""The keyed `collect` restatement (tests/key_collect_oracle.py) against rows of the reference's own, unmodified
`_CollectLogic` (tests/golden/key_collect_cases.json, made by tools/gen_key_collect_golden.py), which `collect` calls
carry a GPU plan, and the host engine's rows for the reference's own examples."""

import json
import os
from datetime import timedelta

import pytest

from oracle.streams import rows_digest
from tests import key_collect_oracle as ko

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "key_collect_cases.json")

with open(GOLDEN) as _f:
    CASE_NAMES = sorted(json.load(_f)["cases"])


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_case_list(golden):
    want = {"test_collect", "docstring", "max_size_1", "max_size_0", "max_size_negative", "exact_multiples",
            "many_lists_one_batch", "carry_across_activations", "timeout_zero_same_activation",
            "timeout_negative_same_activation", "timeout_at_later_notify", "due_key_epoch_advances", "due_key_same_epoch",
            "reopened_after_timeout", "eof", "numeric_text_order", "interned_keys", "timeout_at_utc_max",
            "timeout_at_past_utc_max", "overflow_first_batch", "max_size_past_u64"}
    assert want <= set(golden["cases"])
    assert set(golden["digests"]) == {str(s) for s in ko.SEEDS}


@pytest.mark.parametrize("name", CASE_NAMES)
def test_hand_built_case(golden, name):
    case = golden["cases"][name]
    assert ko.run_oracle(case) == case["rows"]


@pytest.mark.parametrize("seed", ko.SEEDS)
def test_seeded_digests(golden, seed):
    assert rows_digest(ko.run_oracle(ko.seeded_case(seed))) == golden["digests"][str(seed)]


def test_seeded_streams_cover_every_shape():
    """Across the seeds: every max_size and timeout choice, lists cut by size, by timeout and at EOF, interned keys."""
    cases = [ko.seeded_case(s) for s in ko.SEEDS]
    assert {c["max_size"] for c in cases} == {1, 2, 3, 5, 16, 0, -3, 2**70}
    assert {c["timeout_us"] for c in cases} == {0, -ko.S, ko.S, 3 * ko.S, 10 * ko.S, 10**6 * ko.S}
    tags = {chunk[0] for c in cases for act in ko.run_oracle(c) for chunk in act}
    assert tags == {"B", "N", "E"}


def _flow(max_size, timeout=timedelta(seconds=10)):
    from bytewax_b200.dataflow import Dataflow
    from bytewax_b200.testing import TestingSource
    import bytewax_b200.operators as op

    flow = Dataflow("kc")
    s = op.input("inp", flow, TestingSource(list(range(10))))
    s = op.key_on("key", s, lambda _x: "ALL")
    op.collect("collect", s, timeout, max_size)
    return flow


def _plan(flow):
    from bytewax_b200.engine import _core_steps

    steps = [st for st in _core_steps(flow) if type(st).__name__ == "stateful_batch"]
    assert len(steps) == 1
    return getattr(steps[0].builder, "_gpu_plan", None)


@pytest.mark.parametrize("max_size, stored", [(3, 3), (1, 1), (0, 1), (-5, 1), (2**64 - 1, 2**64 - 1), (2**64, 2**64 - 1),
                                              (2**70, 2**64 - 1), (True, 1)])
def test_plan_for_int_max_size(max_size, stored):
    from bytewax_b200.operators import GpuCollectPlan

    plan = _plan(_flow(max_size, timedelta(seconds=3)))
    assert plan == GpuCollectPlan(timedelta(seconds=3), stored)


@pytest.mark.parametrize("max_size", [3.0, 2.5, None, "3"])
def test_no_plan_for_other_max_size(max_size):
    assert _plan(_flow(max_size)) is None


def test_host_engine_test_collect():
    """pytests/operators/test_collect.py::test_collect on the host engine."""
    from bytewax_b200.dataflow import Dataflow
    from bytewax_b200.testing import TestingSink, TestingSource, run_main
    import bytewax_b200.operators as op

    out = []
    flow = Dataflow("test_df")
    s = op.input("inp", flow, TestingSource(list(range(10))))
    s = op.key_on("key", s, lambda _x: "ALL")
    s = op.collect("collect", s, timedelta(seconds=10), 3)
    op.output("out", s, TestingSink(out))
    run_main(flow)
    assert out == [("ALL", [0, 1, 2]), ("ALL", [3, 4, 5]), ("ALL", [6, 7, 8]), ("ALL", [9])]


def test_host_engine_docstring_example():
    """The docstring example of `collect` (operators/__init__.py:1167-1204) on the host engine."""
    from bytewax_b200.dataflow import Dataflow
    from bytewax_b200.testing import TestingSink, TestingSource, run_main
    import bytewax_b200.operators as op

    source = [{"key": "ab"[i % 2], "val": i + 1} for i in range(8)]
    out = []
    flow = Dataflow("collect_eg")
    nums = op.input("nums", flow, TestingSource(source))
    keyed = op.key_on("key", nums, lambda x: x["key"])
    collected = op.collect("collect", keyed, timedelta(seconds=1), max_size=2)
    op.output("out", collected, TestingSink(out))
    run_main(flow)
    assert out == [("a", [source[0], source[2]]), ("b", [source[1], source[3]]), ("a", [source[4], source[6]]),
                   ("b", [source[5], source[7]])]
