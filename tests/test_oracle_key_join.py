"""The keyed join restatement (tests/key_join_oracle.py) against rows of the reference's own, unmodified `_JoinLogic`
(tests/golden/key_join_cases.json, made by tools/gen_key_join_golden.py), which `join` calls carry which GPU plan, and
the host engine's rows for the reference's own `op.join` examples."""

import json
import os

import pytest

from oracle.streams import rows_digest
from tests import key_join_oracle as ko

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "key_join_cases.json")

with open(GOLDEN) as _f:
    CASE_NAMES = sorted(json.load(_f)["cases"])


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_case_list(golden):
    want = {f"{i}_{e}_{n}" for i in ko.INSERTS for e in ko.EMITS for n in range(1, 5)}
    want |= {"test_join_product_final", "test_join_last_running", "complete_mid_batch", "complete_across_activations",
             "first_complete_across_activations", "none_values", "none_values_final", "interned_keys", "numeric_text_order",
             "final_eof_many_keys", "epochs"}
    assert want <= set(golden["cases"])
    assert set(golden["digests"]) == {str(s) for s in ko.SEEDS}


@pytest.mark.parametrize("name", CASE_NAMES)
def test_hand_built_case(golden, name):
    case = golden["cases"][name]
    assert ko.run_oracle(case) == case["rows"]


@pytest.mark.parametrize("seed", ko.SEEDS)
def test_seeded_digests(golden, seed):
    assert rows_digest(ko.run_oracle(ko.seeded_case(seed))) == golden["digests"][str(seed)]


def test_seeded_streams_cover_every_mode():
    """Across the seeds: every insert x emit mode x side count, with and without interned keys."""
    shapes = {}
    for s in ko.SEEDS:
        c = ko.seeded_case(s)
        interned = any(ko.key_id(k, {}) >= 1 << 63 for b in c["steps"] for _e, its in b for k, _s, _v in its)
        shapes.setdefault((c["insert_mode"], c["emit_mode"], c["sides"]), set()).add(interned)
    assert len(shapes) == 36
    assert all(v == {True, False} for v in shapes.values())


def test_releases_every_handle_once():
    """The oracle releases every handle exactly once over a run, in the call after which no list holds it."""
    for s in ko.SEEDS:
        case = ko.seeded_case(s)
        rel = []
        ko.run_oracle(case, rel)
        flat = [v for r in rel for v in r]
        n = sum(len(its) for b in case["steps"] for _e, its in b)
        assert sorted(flat) == list(range(n)), s


def _join_flow(n_sides, insert_mode, emit_mode):
    from bytewax_b200.dataflow import Dataflow
    from bytewax_b200.testing import TestingSource
    import bytewax_b200.operators as op

    flow = Dataflow("kj")
    sides = [op.key_on(f"k{i}", op.input(f"in{i}", flow, TestingSource([1])), lambda _x: "ALL") for i in range(n_sides)]
    op.join("join", *sides, insert_mode=insert_mode, emit_mode=emit_mode)
    return flow


def _plan(flow):
    from bytewax_b200.engine import _core_steps

    steps = [st for st in _core_steps(flow) if type(st).__name__ == "stateful_batch"]
    assert len(steps) == 1
    return getattr(steps[0].builder, "_gpu_plan", None)


@pytest.mark.parametrize("insert_mode", ko.INSERTS)
@pytest.mark.parametrize("emit_mode", ko.EMITS)
@pytest.mark.parametrize("sides", [1, 2, 3, 4, 5])
def test_plan_per_join(insert_mode, emit_mode, sides):
    """Two-sided first / last keeps K6's plan; 5 sides has none; every other join with 1 to 4 sides carries K15's."""
    from bytewax_b200.operators import GpuJoinPlan, GpuKeyJoinPlan

    plan = _plan(_join_flow(sides, insert_mode, emit_mode))
    if sides == 2 and insert_mode in ("first", "last"):
        assert plan == GpuJoinPlan(insert_mode, emit_mode)
    elif sides == 5:
        assert plan is None
    else:
        assert plan == GpuKeyJoinPlan(insert_mode, emit_mode, sides)


def _run_reference_example(inp_l, inp_r, insert_mode=None, emit_mode=None):
    """pytests/operators/test_join.py's `_build_join_dataflow` on the host engine."""
    from bytewax_b200.dataflow import Dataflow
    from bytewax_b200.testing import TestingSink, TestingSource, run_main
    import bytewax_b200.operators as op

    out = []
    flow = Dataflow("test_df")
    lefts = op.key_on("key_l", op.input("inp_l", flow, TestingSource(inp_l)), lambda _: "ALL")
    rights = op.key_on("key_r", op.input("inp_r", flow, TestingSource(inp_r)), lambda _: "ALL")
    kw = {} if insert_mode is None else dict(insert_mode=insert_mode, emit_mode=emit_mode)
    joined = op.join("join", lefts, rights, **kw)
    op.output("out", op.key_rm("unkey", joined), TestingSink(out))
    run_main(flow)
    return out


@pytest.mark.parametrize("inp_l, inp_r, insert_mode, emit_mode, want", [
    ([1], [2], "last", "complete", [(1, 2)]),
    ([1], [2], None, None, [(1, 2)]),
    ([1], [2, 3], "first", "final", [(1, 2)]),
    ([1], [2, 3], "last", "final", [(1, 3)]),
    ([1], [2, 3], "last", "running", [(1, None), (1, 2), (1, 3)]),
    ([1, 2], [3, 4], "product", "final", [(1, 3), (1, 4), (2, 3), (2, 4)]),
])
def test_host_engine_reference_examples(inp_l, inp_r, insert_mode, emit_mode, want):
    """pytests/operators/test_join.py's dataflow examples on the host engine."""
    assert _run_reference_example(inp_l, inp_r, insert_mode, emit_mode) == want


def test_join_state_astuples():
    """pytests/operators/test_join.py::test_join_state_astuples against the oracle's product."""
    o = ko.KeyJoinOracle("product", "final", 3)
    o.apply([0, 0, 0, 0], [0, 0, 2, 2], [1, 2, 3, 4])
    rows, _rel = o.eof()
    assert [t for _k, t in rows] == [(1, None, 3), (1, None, 4), (2, None, 3), (2, None, 4)]
