"""The `join_window` restatement (tests/join_window_oracle.py) against rows of the reference's own, unmodified
`_WindowLogic` + `_SlidingWindowerLogic` + `_JoinWindowLogic` (tests/golden/join_window_cases.json, made by
tools/gen_join_window_golden.py), and the handle-release rule the device follows."""

import json
import os

import pytest

from oracle.streams import rows_digest
from tests import join_window_oracle as jo

S, A = jo.S, jo.A
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "join_window_cases.json")

with open(GOLDEN) as _f:
    CASE_NAMES = sorted(json.load(_f)["cases"])


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_case_list(golden):
    want = {"guide_walkthrough_tumbling", "first_complete_refills", "last_final_overwrites", "running_every_value",
            "sliding_indivisible_offset", "negative_window_ids", "late_sliding_all_windows", "close_first_opened_not_id_order",
            "ordered_ties_stable", "ordered_queue_across_activations", "ordered_notify_wakes_queue_head",
            "wait_forever_flush_at_eof", "discard_resets_watermark", "one_side", "four_sides_partial", "system_clock_moving_now",
            "near_utc_max"}
    assert want <= set(golden["cases"])


@pytest.mark.parametrize("name", CASE_NAMES)
def test_hand_built_case(golden, name):
    case = golden["cases"][name]
    acts, _ = jo.run_join_window(case["spec"], case["steps"])
    assert acts == case["acts"]


@pytest.mark.parametrize("seed", list(jo.SEEDED))
def test_seeded_digests(golden, seed):
    spec, steps = jo.seeded_steps(seed, moving=seed % 3 != 0)
    acts, _ = jo.run_join_window(spec, steps)
    want = golden["seeded"][f"seed_{seed}"]
    assert [len(a) for a in acts] == want["rows"]
    assert rows_digest(acts) == want["sha256"]


def test_seeded_streams_cover_every_mode():
    combos, lates, emits = set(), 0, 0
    for seed in jo.SEEDED:
        spec, steps = jo.seeded_steps(seed, moving=seed % 3 != 0)
        combos.add((spec["insert_mode"], spec["emit_mode"], spec["ordered"]))
        acts, _ = jo.run_join_window(spec, steps)
        lates += sum(r[2] == "L" for a in acts for r in a)
        emits += sum(r[2] == "E" for a in acts for r in a)
    assert len(combos) == 12 and lates > 100 and emits > 1000


def test_guide_walkthrough_rows(golden):
    # docs/guide/concepts/joins.md:630-634: ('456', (8328, (Hive, None))), ('123', (8328, (Bee, bee@))), ('456', (8329, (None, hive@)))
    acts = golden["cases"]["guide_walkthrough_tumbling"]["acts"]
    assert [[r[0], r[1], r[3]] for a in acts for r in a if r[2] == "E"] == [[456, 8328, [1, None]], [123, 8328, [0, 2]],
                                                                            [456, 8329, [None, 3]]]


@pytest.mark.parametrize("seed", list(jo.SEEDED))
def test_every_handle_released_once(seed):
    """Each input handle is released exactly once, by EOF at the latest, and never while a row still needs it later."""
    spec, steps = jo.seeded_steps(seed, moving=seed % 3 != 0)
    acts, released = jo.run_join_window(spec, steps)
    flat = [h for r in released for h in r]
    inputs = [v for st in steps if st[0] == "batch" for v in st[5]]
    assert sorted(flat) == sorted(inputs)
    gone = set()
    for act, rel in zip(acts, released):
        for r in act:
            vals = r[3] if r[2] == "E" else ([r[3][1]] if r[2] == "L" else [])
            assert not gone.intersection(v for v in vals if v is not None)
        gone.update(rel)


def test_sliding_release_waits_for_the_last_window():
    spec = dict(insert_mode="first", emit_mode="final", ordered=False, sides=1, length_us=6 * S, offset_us=2 * S, align_us=A,
                wait_us=0)
    # the value sits in windows [A-4s, A+2s), [A-2s, A+4s), [A, A+6s): released only when the last of them closes
    steps = [["batch", A, [1], [A], [0], [10]], ["batch", A, [1], [A + 2 * S], [0], [11]], ["batch", A, [1], [A + 4 * S], [0], [12]],
             ["batch", A, [1], [A + 6 * S], [0], [13]]]
    _, released = jo.run_join_window(spec, steps)
    # `first` keeps 10 in all three; 11, 12 and 13 each open a window of their own
    assert released == [[], [], [], [10], [11, 12, 13]]
