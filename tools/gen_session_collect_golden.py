"""Generate ``tests/golden/session_collect_cases.json`` from the UNMODIFIED reference `collect_window` over
`SessionWindower`.

TEST INFRASTRUCTURE ONLY.  Needs a bytewax v0.21.1 source checkout, named by $BYTEWAX_SRC:

    python tools/gen_session_collect_golden.py

Every case builds a real reference flow (``win.collect_window`` into list, set or dict over an ``EventClock`` and a
``SessionWindower``), pulls the ``stateful_batch`` step's builder out of the step tree, and drives the reference's own
``_WindowLogic`` + ``_SessionWindowerLogic`` + ``_FoldWindowLogic`` with the collect callbacks through
``tests.session_collect_oracle.drive`` (the engine rules of src/operators.rs:755-806, :808-858, :862-894).

Steps carry distinct int handles; the value a case plays for handle h is h (list), ``set_value(h)`` (set) or
``dict_value(h)`` (dict: keys repeat, so merges overwrite).  Hand-built cases store their rows in full for each
``into``, with the number of merges; every case named for a merge is checked to merge, and enough merged set cases are
checked to iterate differently under a flat replay of their values that a flat rebuild fails the tests.  The seeded
streams of ``tests/session_collect_oracle.py`` store the SHA-256 of their rows per ``into``.  Int hashes are not
randomised, so the stored set orders hold in every process.  The file holds data only.
"""

import json
import os
import sys
from datetime import datetime, timedelta, timezone

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refstub  # noqa: E402
from oracle.streams import rows_digest  # noqa: E402
from tests import session_collect_oracle as sc  # noqa: E402

win = refstub.load()
import bytewax.operators as op  # noqa: E402  (the reference's)
from bytewax.dataflow import Dataflow  # noqa: E402
from bytewax.testing import TestingSource  # noqa: E402

EPOCH = datetime(1970, 1, 1, tzinfo=timezone.utc)
S, A, F = sc.S, sc.A, sc.WAIT_FOREVER
UTC_MAX = 253_402_300_799_999_999


def dt(t: int) -> datetime:
    return EPOCH + timedelta(microseconds=t)


def us(d: datetime) -> int:
    delta = d - EPOCH
    return (delta.days * 86400 + delta.seconds) * 1_000_000 + delta.microseconds


def run_reference(spec, steps, into):
    now = [dt(steps[0][1])]
    builder = sc.builder_of(win, op, Dataflow, TestingSource, refstub.find_stateful_batch, spec, steps, into, now, dt)
    return sc.drive(builder, steps, now, us, dt, into)


class Steps:
    """Golden steps; every value is a fresh int (its handle)."""

    def __init__(self, now=A + 10**6 * S):
        self.steps, self.n, self.now = [], 0, now

    def batch(self, *items, now=None):
        """``items``: ``(key, ts)``."""
        if now is not None:
            self.now = now
        self.steps.append(["batch", self.now, [k for k, _ in items], [t for _, t in items], list(range(self.n, self.n + len(items)))])
        self.n += len(items)
        return self

    def notify(self, now):
        self.now = now
        self.steps.append(["notify", now])
        return self


def spec_(ordered=False, gap=10 * S, wait=F):
    return dict(ordered=ordered, gap_us=gap, wait_us=wait)


def main():
    cases = {}
    set_flat_differs = []

    def add(name, spec, st, merges=False):
        for into in sc.INTOS:
            acts, n_merges = run_reference(spec, st.steps, into)
            assert (n_merges > 0) == merges, (name, into, n_merges)  # a case named for a merge must merge; the others not
            cases[f"{name}/{into}"] = dict(spec=spec, into=into, steps=st.steps, acts=acts, merges=n_merges)
            if into == "set":  # does a flat replay of some merged session's values iterate differently?
                oacts, _ = sc.run_session_collect(spec, st.steps)
                for r in (r for a in oacts for r in a if r[2] == "E" and r[3][1]):
                    vo = sc.value_fn("set")
                    if list(sc.container("set", r[3][0], r[3][1], vo)) != list(sc.flat("set", r[3][0], vo)):
                        set_flat_differs.append(name)
                        break

    # --- opening, extending before and after -------------------------------------------------------------------------------
    add("open_extend_before_after", spec_(), Steps().batch((1, A + 5 * S), (1, A), (1, A + 12 * S), (1, A + 2 * S)))
    # --- a bridging value merges two sessions (one flush), several values on each side -----------------------------------------
    add("bridge_merges_two", spec_(), Steps().batch(*[(1, A + i) for i in range(5)], *[(1, A + 20 * S + i) for i in range(6)],
                                                    (1, A + 10 * S), (1, A + 5)), merges=True)
    # --- a chain in one flush: the bridge at A+30 merges session 2 into 1, the one at A+10 then 1 into 0 -------------------
    add("chain_one_flush", spec_(), Steps().batch(*[(1, A + i) for i in range(4)], *[(1, A + 20 * S + i) for i in range(4)],
                                                  *[(1, A + 40 * S + i) for i in range(4)], (1, A + 30 * S), (1, A + 10 * S), (1, A + 7)),
        merges=True)
    # --- a merge across flushes, with values before and after it ---------------------------------------------------------------
    add("merge_across_flushes", spec_(), Steps().batch(*[(2, A + i) for i in range(5)], *[(2, A + 20 * S + i) for i in range(5)])
        .batch((2, A + 10 * S), (2, A + 9)).batch(*[(2, A + 25 * S + i) for i in range(4)]), merges=True)
    # --- a value played into a session its own open_for just merged away ---------------------------------------------------
    add("value_in_merged_away_session", spec_(), Steps().batch((4, A + 20 * S), (4, A + 20 * S + 1), (4, A), (4, A + 1), (4, A + 10 * S),
                                                               (4, A + 11 * S)), merges=True)
    # --- gap 0 and equal timestamps ------------------------------------------------------------------------------------------
    add("gap_zero_equal_ts", spec_(gap=0, wait=0), Steps().batch((1, A), (1, A), (1, A + 1)).batch((1, A + 1), (1, A + 5)))
    # --- late rows -----------------------------------------------------------------------------------------------------------
    add("late_rows", spec_(gap=S, wait=0), Steps().batch((3, A + 10 * S), (3, A), (5, A + 10 * S)).batch((3, A + 2 * S), (5, A + 30 * S)))
    # --- a moving clock: notify phases close what the drifted watermark allows, in both orders ------------------------------
    for ordered in (False, True):
        add(f"moving_clock_notify_{'ordered' if ordered else 'unordered'}", spec_(ordered=ordered, gap=2 * S, wait=S),
            Steps(now=A).batch((7, A), (8, A + S), (7, A + S // 2), now=A).notify(A + 2 * S).notify(A + 4 * S)
            .batch((7, A + 5 * S), (8, A + 3 * S), now=A + 6 * S).notify(A + 20 * S))
    # queue[0] (ts A+8) is not the smallest queued ts (A+5): the notify wakes at A+8 once `now` drifts the watermark
    add("ordered_notify_wakes_queue_head", spec_(ordered=True, gap=20 * S, wait=10 * S),
        Steps(now=A).batch((4, A + 8 * S), (4, A + 5 * S), (4, A + 12 * S), now=A).notify(A + 4 * S).notify(A + 6 * S)
        .notify(A + 8 * S).notify(A + 9 * S).notify(A + 60 * S))
    # --- wait forever: nothing closes before EOF -----------------------------------------------------------------------------
    add("wait_forever_flush_at_eof", spec_(ordered=True, gap=S, wait=F),
        Steps().batch((1, A + 9 * S), (1, A + S), (1, A + 5 * S)).batch((1, A), (2, A + 3 * S), (1, A + 2 * S)))
    add("wait_forever_merge_at_eof", spec_(gap=3 * S, wait=F),
        Steps().batch(*[(1, A + 2 * i * S) for i in range(0, 12, 2)]).batch(*[(1, A + 2 * i * S) for i in range(1, 12, 2)]), merges=True)
    # --- EOF with a session close near UTC_MAX - gap ------------------------------------------------------------------------
    add("eof_near_utc_max", spec_(ordered=True, gap=2 * S, wait=0),
        Steps().batch((9, UTC_MAX - S), (10, UTC_MAX - 3 * S), (11, UTC_MAX - 2 * S)))

    # enough merged set cases iterate differently under a flat replay that a flat rebuild fails the tests
    assert len(set(set_flat_differs)) >= 3, set_flat_differs

    seeded = {}
    for seed in sc.SEEDED:
        spec, steps = sc.seeded_steps(seed, moving=seed % 3 != 0)
        for into in sc.INTOS:
            acts, n_merges = run_reference(spec, steps, into)
            assert not (spec["ordered"] and n_merges), seed  # ordered mode never merges
            seeded[f"seed_{seed}/{into}"] = dict(sha256=rows_digest(acts), rows=[len(a) for a in acts], merges=n_merges)
    path = os.path.join(ROOT, "tests", "golden", "session_collect_cases.json")
    with open(path, "w") as f:
        json.dump(dict(cases=cases, seeded=seeded, set_flat_differs=sorted(set(set_flat_differs))), f, separators=(",", ":"))
    print("wrote", path, os.path.getsize(path), "bytes,", len(cases), "cases,", len(seeded), "seeded streams; sets that differ"
          " from a flat replay:", sorted(set(set_flat_differs)))


if __name__ == "__main__":
    main()
