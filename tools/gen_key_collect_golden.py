"""Generate ``tests/golden/key_collect_cases.json`` from the UNMODIFIED reference `_CollectLogic`.

TEST INFRASTRUCTURE ONLY.  Needs a bytewax v0.21.1 source checkout, named by $BYTEWAX_SRC:

    python tools/gen_key_collect_golden.py

Every key's logic is the reference's `_StatefulLogic` (pysrc/bytewax/operators/__init__.py:1025-1062) around its
`_CollectLogic` + `_CollectState` (:1106-1145), built with a stepping `now_getter` as pytests/operators/test_collect.py
does.  They run under the engine rules, restated here with the reference's datetimes: per activation the epochs with
items plus the previous activation's epoch, ascending (src/operators.rs:698-707); per epoch `on_batch` per key in
ascending key order, a logic that reports itself complete discarded (:755-806), then every key whose `notify_at()` is
<= now notified in key order (:808-858); EOF after the last activation (:862-894).

Cases use ``tests/key_collect_oracle.py``'s format.  Hand-built cases store their rows in full; the seeded streams of
``key_collect_oracle.seeded_case`` store the SHA-256 of their rows.  The file holds data only.
"""

import json
import os
import sys
from datetime import datetime, timedelta, timezone

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refstub  # noqa: E402
from oracle.streams import rows_digest  # noqa: E402
from tests import key_collect_oracle as ko  # noqa: E402

refstub.load()
import bytewax.operators as op  # noqa: E402  (the reference's)

S, T0, UTC_MAX = ko.S, ko.T0, ko.UTC_MAX
EPOCH = datetime(1970, 1, 1, tzinfo=timezone.utc)


def dt(t: int) -> datetime:
    return EPOCH + timedelta(microseconds=t)


def run_reference(case):
    now = [None]
    timeout = timedelta(microseconds=case["timeout_us"])

    def builder(resume_state):
        return op._CollectLogic("collect", lambda: now[0], timeout, case["max_size"], op._CollectState())

    logics, sched, acts, last_out = {}, {}, [], 0
    for now_us, batches in case["steps"]:
        now[0] = dt(now_us)
        ready = {}
        for epoch, items in batches:
            ready.setdefault(epoch, []).extend(items)
        epochs = sorted(set(ready) | ({last_out} if last_out else set()))
        act = []
        acts.append(act)
        for e in epochs:
            grouped = {}
            for k, v in ready.get(e, []):
                grouped.setdefault(k, []).append(v)
            out = []
            try:
                for k in sorted(grouped):
                    logic = logics.setdefault(k, op._StatefulLogic(None, builder))
                    emit, done = logic.on_batch(grouped[k])
                    out.extend([k, list(w)] for w in emit)
                    if done:
                        del logics[k]
                        sched.pop(k, None)
            except OverflowError:
                act.append(["raises", "OverflowError"])
                return acts
            for k in sorted(grouped):
                if k in logics:
                    sched[k] = logics[k].notify_at()
            if grouped:
                act.append(["B", e, out])
            out = []
            for k in sorted(k for k, at in sched.items() if at <= now[0]):
                emit, done = logics[k].on_notify()
                out.extend([k, list(w)] for w in emit)
                del sched[k]
                assert done
                del logics[k]
            act.append(["N", e, out])
        if epochs:
            last_out = epochs[-1]
        act[:] = [c for c in act if c[2]]
    out = []
    for k in sorted(logics):
        emit, _done = logics[k].on_eof()
        out.extend([k, list(w)] for w in emit)
    acts.append([c for c in [["E", None, out]] if c[2]])
    return acts


def one(now, epoch, *items):
    return [now, [[epoch, [list(i) for i in items]]]]


def ones(key, values):
    return [[key, v] for v in values]


def cases():
    c = {}
    # pytests/operators/test_collect.py: ten items of one key, max_size 3, a timeout that never comes
    c["test_collect"] = dict(max_size=3, timeout_us=10 * S, steps=[[T0, [[1, ones("ALL", range(10))]]]])
    # the docstring example (:1167-1204): a / b alternating, max_size 2, timeout 1 s
    c["docstring"] = dict(max_size=2, timeout_us=S, steps=[[T0, [[1, [["ab"[i % 2], i + 1] for i in range(8)]]]]])
    for m, name in ((1, "max_size_1"), (0, "max_size_0"), (-3, "max_size_negative")):
        c[name] = dict(max_size=m, timeout_us=S, steps=[[T0, [[1, ones("k", range(5)) + ones("j", range(5, 7))]]],
                                                        [T0 + S // 2, [[2, ones("k", [7])]]]])
    c["exact_multiples"] = dict(max_size=4, timeout_us=0, steps=[[T0, [[1, ones("a", range(8)) + ones("b", range(8, 12))]]],
                                                                 [T0 + S, [[2, ones("a", range(12, 16))]]]])
    c["many_lists_one_batch"] = dict(max_size=3, timeout_us=5 * S, steps=[[T0, [[1, ones("7", range(3, 20))]]]])
    c["carry_across_activations"] = dict(max_size=5, timeout_us=100 * S, steps=[
        [T0 + i * S, [[i + 1, ones("k", range(3 * i, 3 * i + 3)) + ones("m", [100 + i])]]] for i in range(6)])
    c["timeout_zero_same_activation"] = dict(max_size=10, timeout_us=0, steps=[
        [T0, [[1, ones("a", [1, 2]) + ones("b", [3])]]], [T0 + S, [[2, ones("a", [4])]]]])
    c["timeout_negative_same_activation"] = dict(max_size=10, timeout_us=-S, steps=[
        [T0, [[1, ones("a", [1, 2])]]], [T0, [[1, ones("a", [3])]]]])
    c["timeout_at_later_notify"] = dict(max_size=10, timeout_us=3 * S, steps=[
        [T0, [[1, ones("a", [1, 2]) + ones("b", [3])]]], [T0 + S, []], [T0 + 2 * S, [[2, ones("b", [4])]]],
        [T0 + 3 * S, []], [T0 + 4 * S, []], [T0 + 5 * S, []], [T0 + 9 * S, []]])
    # a key whose timeout came due receives items: with the epoch advancing the previous epoch's notify fires first;
    # with the same epoch the items join the overdue list and the new timeout decides
    due = [[T0, [[1, ones("a", [1, 2])]]]]
    c["due_key_epoch_advances"] = dict(max_size=10, timeout_us=S, steps=due + [[T0 + 2 * S, [[2, ones("a", [3])]]]])
    c["due_key_same_epoch"] = dict(max_size=10, timeout_us=S, steps=due + [[T0 + 2 * S, [[1, ones("a", [3])]]], [T0 + 4 * S, []]])
    c["due_key_same_epoch_timeout_zero"] = dict(max_size=10, timeout_us=0, steps=[
        [T0, [[1, ones("a", [1])]]], [T0 + S, [[1, ones("a", [2])]]], [T0 + S, [[1, ones("a", [3])]]]])
    c["reopened_after_timeout"] = dict(max_size=3, timeout_us=S, steps=[
        [T0, [[1, ones("a", [1, 2])]]], [T0 + 2 * S, []], [T0 + 3 * S, [[2, ones("a", [3, 4, 5, 6])]]], [T0 + 3 * S, []]])
    c["eof"] = dict(max_size=100, timeout_us=10**6 * S, steps=[[T0, [[1, [[k, i] for i, k in enumerate("zyxabc" * 3)]]]]])
    c["numeric_text_order"] = dict(max_size=2, timeout_us=S, steps=[
        [T0, [[1, [[k, i] for i, k in enumerate(["10", "9", "100", "2", "19", "1", "0", "10", "9", "18446744073709551615",
                                                  "9223372036854775807", "9223372036854775808", "1", "2"])]]]],
        [T0 + 5 * S, []]])
    c["interned_keys"] = dict(max_size=2, timeout_us=S, steps=[
        [T0, [[1, [[k, i] for i, k in enumerate(["b", "", "a", "007", "10", "9", "a", "é", "b", "-1", "007", " "])]]]],
        [T0 + 5 * S, [[2, [["Z", 20], ["9", 21], ["", 22]]]]]])
    # timeout_at exactly datetime.max, then one microsecond past it
    c["timeout_at_utc_max"] = dict(max_size=3, timeout_us=UTC_MAX - T0, steps=[[T0, [[1, ones("a", [1, 2])]]], [T0 + S, []]])
    c["timeout_at_past_utc_max"] = dict(max_size=3, timeout_us=UTC_MAX - T0, steps=[
        [T0, [[1, ones("a", [1])]]], [T0 + 1, [[2, ones("a", [2])]]]])
    c["overflow_first_batch"] = dict(max_size=3, timeout_us=UTC_MAX - T0 + 1, steps=[[T0, [[1, ones("a", [1])]]]])
    c["max_size_past_u64"] = dict(max_size=2**70, timeout_us=10 * S, steps=[[T0, [[1, ones("a", range(50))]]]])
    return c


def main():
    out = {"cases": {}, "digests": {}}
    for name, case in cases().items():
        want = run_reference(case)
        assert ko.run_oracle(case) == want, name
        out["cases"][name] = dict(case, rows=want)
    for seed in ko.SEEDS:
        case = ko.seeded_case(seed)
        want = run_reference(case)
        assert ko.run_oracle(case) == want, seed
        out["digests"][str(seed)] = rows_digest(want)
    path = os.path.join(ROOT, "tests", "golden", "key_collect_cases.json")
    with open(path, "w") as f:
        json.dump(out, f, separators=(",", ":"))
        f.write("\n")
    print(f"{len(out['cases'])} cases, {len(out['digests'])} digests -> {path}")


if __name__ == "__main__":
    main()
