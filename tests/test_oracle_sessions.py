"""The session restatement (tests/session_oracle.py) against rows of the reference's own, unmodified session windower
(tests/golden/session_cases.json, made by tools/gen_session_golden.py) and the expected lists of the reference's tests."""

import json
import math
import os

import pytest

from oracle.streams import rows_digest
from tests import session_oracle as so

S, A = so.S, so.A


@pytest.fixture(scope="module")
def golden(golden_dir):
    with open(os.path.join(golden_dir, "session_cases.json")) as f:
        return json.load(f)


def _same(a, b):
    """Row lists equal, NaN == NaN and -0.0 != 0.0 (the float bits matter)."""
    if isinstance(a, float) and isinstance(b, float):
        return (math.isnan(a) and math.isnan(b)) or (a == b and math.copysign(1, a) == math.copysign(1, b))
    if isinstance(a, list) and isinstance(b, list):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return type(a) is type(b) and a == b


with open(os.path.join(os.path.dirname(__file__), "golden", "session_cases.json")) as _f:
    CASE_NAMES = sorted(json.load(_f)["cases"])


def test_case_count(golden):
    assert len(golden["cases"]) >= 25


@pytest.mark.parametrize("name", CASE_NAMES)
def test_hand_built_case(golden, name):
    case = golden["cases"][name]
    assert _same(so.run_sessions(case["spec"], case["steps"]), case["acts"])


MERGE_CASES = {"three_way_merge": [[0, [1, 2]]], "chained_merges_survivor_merged_later": [[4, [0]]],
               "merged_close_same_activation": [[0, [1]], [2, [3]]], "f64_sum_merge_order": [[0, [1, 2]], [3, [4]]],
               "first_by_id_merge_into_earlier": [[1, [0]]]}


@pytest.mark.parametrize("name", sorted(MERGE_CASES))
def test_merge_cases_really_merge(golden, name):
    """The cases named for merges carry the merged ids their names promise (direct merges only)."""
    acts = golden["cases"][name]["acts"]
    assert [[r[1], r[3][2]] for act in acts for r in act if r[2] == "M" and r[3][2]] == MERGE_CASES[name]
    if name == "chained_merges_survivor_merged_later":  # every value of sessions 0..4 ends in session 4
        assert [[r[1], r[3]] for act in acts for r in act if r[2] == "E"] == [[4, 511], [5, 512]]


@pytest.mark.parametrize("seed", list(so.SEEDED))
def test_seeded_digests(golden, seed):
    spec, steps = so.seeded_steps(seed, moving=seed % 3 != 0)
    got = so.run_sessions(spec, steps)
    want = golden["seeded"][f"seed_{seed}"]
    assert [len(a) for a in got] == want["rows"]
    assert rows_digest(got) == want["sha256"]


def test_seeded_streams_merge_and_late(golden):
    merges = lates = 0
    for seed in so.SEEDED:
        spec, steps = so.seeded_steps(seed, moving=seed % 3 != 0)
        for act in so.run_sessions(spec, steps):
            merges += sum(len(r[3][2]) for r in act if r[2] == "M")
            lates += sum(r[2] == "L" for r in act)
    assert merges > 100 and lates > 100


def test_reference_test_expectations(golden):
    cases = golden["cases"]

    def down(name):
        return [[r[0], r[1], r[3]] for act in so.run_sessions(cases[name]["spec"], cases[name]["steps"]) for r in act if r[2] == "E"]

    # pytests/operators/windowing/test_fold_window.py:136-140 (list lengths) and test_session_windower.py:293
    assert down("ref_fold_window_session") == [[0, 0, 2], [0, 1, 4], [0, 2, 1]]
    assert down("ref_session_with_system_clock") == [[0, 0, 10]]


def _windower(gap_s, opens):
    w = so.SessionWindower(gap_s * S)
    for o in opens:
        w.max_key += 1
        w.sessions[w.max_key] = [A + o * S, A + o * S, set()]
    return w


def test_session_windower_reference_cases():
    # pytests/operators/windowing/test_session_windower.py:19-265, restated on integer microseconds
    w = so.SessionWindower(10 * S)
    assert w.open_for(A) == 0 and w.sessions[0] == [A, A, set()]
    assert w.open_for(A + 10 * S) == 0 and w.sessions[0] == [A, A + 10 * S, set()]  # exact gap extends
    assert w.open_for(A - 10 * S) == 0 and w.sessions[0] == [A - 10 * S, A + 10 * S, set()]
    w = so.SessionWindower(10 * S)
    w.open_for(A)
    w.open_for(A + 20 * S)
    assert w.open_for(A + 10 * S) == 0
    assert w.merged() == [(1, 0)] and w.sessions == {0: [A, A + 20 * S, {1}]}
    w = _windower(10, (0, 20))
    w._find_merges()
    assert w.merge_queue == []
    w = _windower(10, (0, 5))
    w._find_merges()
    assert w.merge_queue == [(1, 0)] and w.sessions == {0: [A, A + 5 * S, {1}]}
    w = _windower(10, (0, 5, 10))
    w._find_merges()
    assert w.merge_queue == [(1, 0), (2, 0)] and w.sessions == {0: [A, A + 10 * S, {1, 2}]}
    w = _windower(10, (0, 20, 25, 40))
    w._find_merges()
    assert w.merge_queue == [(2, 1)]
    assert w.sessions == {0: [A, A, set()], 1: [A + 20 * S, A + 25 * S, {2}], 3: [A + 40 * S, A + 40 * S, set()]}


def test_merged_ids_are_direct_only():
    # B (2) absorbs C (3); then A (0) absorbs B: A holds B's id, not C's (windowing.py:707)
    w = _windower(5, (0, 20, 30))
    assert w.open_for(A + 25 * S) == 1  # 20..25, then 25 is within 5 s of 30: 2 merges into 1
    assert w.sessions[1][2] == {2}
    assert w.open_for(A + 5 * S) == 0  # 0..5; 1 opens at 20: no merge
    assert w.open_for(A + 15 * S) == 1  # 1 opens at 15, within 5 s of 0's close at 5? no: 10 s; extend only
    assert w.open_for(A + 10 * S) == 0  # 0 closes at 10, within 5 s of 15: 1 merges into 0
    assert w.sessions == {0: [A, A + 30 * S, {1}]}
