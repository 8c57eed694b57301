"""Generate ``tests/golden/key_join_cases.json`` from the UNMODIFIED reference `_JoinLogic`.

TEST INFRASTRUCTURE ONLY.  Needs a bytewax v0.21.1 source checkout, named by $BYTEWAX_SRC:

    python tools/gen_key_join_golden.py

Every key's logic is the reference's `_StatefulLogic` (pysrc/bytewax/operators/__init__.py:1025-1062) around its
`_JoinLogic` + `_JoinState` (:2076-2190), built as `op.join` builds it.  They run under the engine rules, restated here:
per activation the epochs with items, ascending (src/operators.rs:698-707); per epoch `on_batch` per key in ascending
key order with the key's `(side, value)` items in arrival order, a logic that reports itself complete discarded
(:755-806); EOF after the last activation, `on_eof` per key in key order (:862-894).  The join has no clock, so no
notify phase runs.

Cases use ``tests/key_join_oracle.py``'s format.  Hand-built cases store their rows in full; the seeded streams of
``key_join_oracle.seeded_case`` store the SHA-256 of their rows.  The file holds data only.
"""

import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refstub  # noqa: E402
from oracle.streams import rows_digest  # noqa: E402
from tests import key_join_oracle as ko  # noqa: E402

refstub.load()
import bytewax.operators as op  # noqa: E402  (the reference's)


def run_reference(case):
    def builder(resume_state):
        return op._JoinLogic(case["insert_mode"], case["emit_mode"], op._JoinState.for_side_count(case["sides"]))

    logics, acts = {}, []
    for batches in case["steps"]:
        ready = {}
        for epoch, items in batches:
            ready.setdefault(epoch, []).extend(items)
        act = []
        acts.append(act)
        for e in sorted(ready):
            grouped = {}
            for k, s, v in ready[e]:
                grouped.setdefault(k, []).append((s, v))
            out = []
            for k in sorted(grouped):
                logic = logics.setdefault(k, op._StatefulLogic(None, builder))
                emit, done = logic.on_batch(grouped[k])
                out.extend([k, list(t)] for t in emit)
                if done:
                    del logics[k]
            if grouped:
                act.append(["B", e, out])
        act[:] = [c for c in act if c[2]]
    out = []
    for k in sorted(logics):
        emit, _done = logics[k].on_eof()
        out.extend([k, list(t)] for t in emit)
    acts.append([c for c in [["E", None, out]] if c[2]])
    return acts


def one(epoch, *items):
    """One activation of one batch."""
    return [[epoch, [list(i) for i in items]]]


def cases():
    c = {}
    # every insert x emit mode x side count: two keys, values on every side, a side repeated, a side left empty
    for ins in ko.INSERTS:
        for em in ko.EMITS:
            for n in range(1, 5):
                items = [["a", 0, 1], ["b", n - 1, 2], ["a", n - 1, 3], ["a", 0, 4], ["b", 0, 5]]
                items += [["a", s, 10 + s] for s in range(1, n)] + [["a", 0, 20], ["b", n - 1, 21]]
                c[f"{ins}_{em}_{n}"] = dict(insert_mode=ins, emit_mode=em, sides=n, steps=[
                    one(1, *items[:4]), one(2, *items[4:]), one(2, ["c", 0, 30])])
    # the reference's own examples (pytests/operators/test_join.py) as items
    c["test_join_product_final"] = dict(insert_mode="product", emit_mode="final", sides=2, steps=[
        one(1, ["ALL", 0, 1], ["ALL", 0, 2], ["ALL", 1, 3], ["ALL", 1, 4])])
    c["test_join_last_running"] = dict(insert_mode="last", emit_mode="running", sides=2, steps=[
        one(1, ["ALL", 0, 1], ["ALL", 1, 2], ["ALL", 1, 3])])
    # a complete generation that ends mid-batch: the key's next items start from empty lists in the same batch
    c["complete_mid_batch"] = dict(insert_mode="product", emit_mode="complete", sides=3, steps=[
        one(1, ["k", 0, 1], ["k", 0, 2], ["k", 1, 3], ["k", 2, 4], ["k", 2, 5], ["k", 0, 6], ["k", 1, 7], ["k", 2, 8], ["k", 1, 9])])
    # a complete generation that spans activations, then a second one
    c["complete_across_activations"] = dict(insert_mode="product", emit_mode="complete", sides=2, steps=[
        one(1, ["k", 0, 1], ["j", 1, 2]), one(2, ["k", 0, 3]), one(3, ["k", 1, 4], ["k", 1, 5], ["j", 0, 6]),
        one(4, ["k", 1, 7], ["k", 0, 8])])
    c["first_complete_across_activations"] = dict(insert_mode="first", emit_mode="complete", sides=3, steps=[
        one(1, ["k", 0, 1], ["k", 0, 2]), one(2, ["k", 1, 3], ["k", 1, 4]), one(3, ["k", 0, 5], ["k", 2, 6], ["k", 2, 7])])
    # None values next to empty sides
    c["none_values"] = dict(insert_mode="product", emit_mode="running", sides=3, steps=[
        one(1, ["k", 0, None], ["k", 2, None], ["k", 0, 1], ["m", 1, None])])
    c["none_values_final"] = dict(insert_mode="last", emit_mode="final", sides=4, steps=[
        one(1, ["k", 1, None], ["k", 3, 0], ["m", 0, None]), one(2, ["k", 3, None])])
    # non-numeric keys, which the engine interns and re-sorts
    c["interned_keys"] = dict(insert_mode="product", emit_mode="running", sides=2, steps=[
        one(1, *[[k, i % 2, i] for i, k in enumerate(["b", "", "a", "007", "10", "9", "a", "é", "b", "-1", "007", " "])]),
        one(2, ["Z", 0, 20], ["9", 1, 21], ["", 1, 22])])
    c["numeric_text_order"] = dict(insert_mode="last", emit_mode="complete", sides=2, steps=[
        one(1, *[[k, i % 2, i] for i, k in enumerate(["10", "9", "100", "2", "19", "1", "0", "10", "9", "18446744073709551615",
                                                      "9223372036854775807", "9223372036854775808", "1", "2", "100", "19"])])])
    # final EOF over many keys, in ascending key-string order
    c["final_eof_many_keys"] = dict(insert_mode="product", emit_mode="final", sides=2, steps=[
        one(1, *[[str(k), k % 2, k] for k in range(0, 300, 7)]), one(2, *[[str(k), (k + 1) % 2, 1000 + k] for k in range(0, 300, 11)])])
    # epochs that stand still across activations and two epochs in one activation
    c["epochs"] = dict(insert_mode="product", emit_mode="running", sides=2, steps=[
        [[3, [["k", 0, 1]]], [2, [["k", 1, 2]]]], one(3, ["k", 1, 3]), [[3, [["k", 0, 4]]], [3, [["j", 1, 5]]]]])
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
    path = os.path.join(ROOT, "tests", "golden", "key_join_cases.json")
    with open(path, "w") as f:
        json.dump(out, f, separators=(",", ":"))
        f.write("\n")
    print(f"{len(out['cases'])} cases, {len(out['digests'])} digests -> {path}")


if __name__ == "__main__":
    main()
