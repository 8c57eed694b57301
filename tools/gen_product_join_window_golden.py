"""Generate ``tests/golden/product_join_window_cases.json`` from the UNMODIFIED reference
`join_window(insert_mode="product")`.

TEST INFRASTRUCTURE ONLY.  Needs a bytewax v0.21.1 source checkout, named by $BYTEWAX_SRC:

    python tools/gen_product_join_window_golden.py

Every case builds a real reference flow (``win.join_window(..., insert_mode="product")`` over an ``EventClock`` and a
``TumblingWindower`` or ``SlidingWindower``) and drives the reference's own ``_WindowLogic`` + ``_SlidingWindowerLogic``
+ ``_JoinWindowLogic`` under the engine's activation rules, exactly as ``tools/gen_join_window_golden.py`` does (its
``run_reference`` is used as is).  Values are distinct ints, so they double as the handles the device joins.  Hand-built
cases store their rows in full; the seeded streams of ``tests/product_join_window_oracle.py`` (``seeded_steps``) store
the SHA-256 of their rows.  The file holds data only.
"""

import json
import os
import sys
from datetime import datetime, timezone

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import gen_join_window_golden as gj  # noqa: E402  (loads the reference)
from oracle.streams import rows_digest  # noqa: E402
from tests import product_join_window_oracle as po  # noqa: E402

S, A = po.S, po.A
UTC_MAX = gj.UTC_MAX
FOREVER = po.WAIT_FOREVER


def spec_(emit="final", ordered=True, sides=2, length=10 * S, offset=None, align=A, wait=0):
    return gj.spec_("product", emit, ordered, sides, length, offset, align, wait)


def main():
    cases = {}

    def add(name, spec, st, check=None, cite=None):
        acts = gj.run_reference(spec, st.steps)
        if check is not None:
            assert check(acts), (name, acts)
        cases[name] = dict(spec=spec, steps=st.steps, acts=acts, cite=cite)

    def tags(acts, tag):
        return [r for act in acts for r in act if r[2] == tag]

    Steps = gj.Steps
    H = 3600 * S
    # docs/guide/concepts/joins.md:641-728: Bee's name and two emails in one 1 h window; the product gives two rows
    g0 = gj.us(datetime(2023, 12, 14, tzinfo=timezone.utc))
    add("guide_bee_product", spec_(length=H, align=gj.us(datetime(2023, 1, 1, tzinfo=timezone.utc))),
        Steps().batch((123, g0, 0), (123, g0 + 15 * 60 * S, 1)).batch((123, g0 + 30 * 60 * S, 1)),
        check=lambda a: [r[3] for r in tags(a, "E")] == [[0, 1], [0, 2]], cite="docs/guide/concepts/joins.md:641-728")
    # --- emit modes -------------------------------------------------------------------------------------------------------
    add("final_side_empty_at_close", spec_("final", sides=3, wait=S),
        Steps().batch((1, A, 0), (1, A + 1, 0), (1, A + 2, 2), (1, A + 3, 2), (1, A + 4, 2)).batch((1, A + 30 * S, 1)),
        check=lambda a: [r[3] for r in tags(a, "E")][:6] == [[0, None, 2], [0, None, 3], [0, None, 4], [1, None, 2],
                                                               [1, None, 3], [1, None, 4]])
    add("complete_refills_and_reemits", spec_("complete", wait=FOREVER),
        Steps().batch((1, A, 0), (1, A + 1, 0), (1, A + 2, 1), (1, A + 3, 1), (1, A + 4, 0), (1, A + 5, 1), (1, A + 6, 0)),
        check=lambda a: [r[3] for r in tags(a, "E")] == [[0, 2], [1, 2], [4, 3], [6, 5]])
    add("complete_nothing_at_close_after_clear", spec_("complete", ordered=False, wait=S),
        Steps().batch((1, A, 0), (1, A + 1, 1)).batch((1, A + 30 * S, 0)),
        check=lambda a: len(tags(a, "E")) == 1 and [r[1] for r in tags(a, "M")] == [0, 3])
    add("running_empty_sides", spec_("running", sides=3, wait=2 * S),
        Steps().batch((1, A, 1), (1, A + 1, 1), (1, A + 2, 0), (1, A + 3, 2)).batch((1, A + 20 * S, 1)))
    add("running_unordered_growth", spec_("running", ordered=False, sides=2, wait=S),
        Steps().batch((2, A, 0), (2, A + 1, 1), (2, A + 2, 0), (2, A + 3, 1)).batch((2, A + 4, 0), (3, A, 1)).batch((2, A + 40 * S, 0)))
    # --- side counts --------------------------------------------------------------------------------------------------------
    add("one_side", spec_("final", ordered=False, sides=1, length=3 * S, wait=S),
        Steps().batch((1, A, 0), (1, A + 1, 0), (2, A + S, 0)).batch((1, A + 10 * S, 0)))
    add("one_side_complete", spec_("complete", ordered=True, sides=1, length=3 * S, wait=S),
        Steps().batch((1, A, 0), (1, A + 1, 0)).batch((1, A + 10 * S, 0)))
    add("four_sides_with_gaps", spec_("final", ordered=True, sides=4, wait=S),
        Steps().batch((1, A, 3), (1, A + S, 1), (1, A + 2 * S, 3), (2, A, 0), (2, A + 1, 2), (2, A + 2, 2), (2, A + 3, 1))
        .batch((1, A + 50 * S, 0)))
    add("four_sides_running", spec_("running", ordered=False, sides=4, length=5 * S, wait=2 * S),
        Steps().batch((1, A, 0), (1, A + 1, 1), (1, A + 2, 2), (1, A + 3, 3), (1, A + 4, 0), (1, A + 5, 3)).batch((1, A + 20 * S, 2)))
    # --- sliding windows --------------------------------------------------------------------------------------------------
    # complete: window 1 clears value 0 (its first full product) while window 0 still holds it, and later closes with it
    add("sliding_clear_while_lower_window_holds", spec_("complete", ordered=False, sides=2, length=4 * S, offset=2 * S, wait=FOREVER),
        Steps().batch((1, A + 3 * S, 0)).batch((1, A + 4 * S + 1, 1)).batch((1, A + S, 1)).batch((1, A + 5 * S, 0)),
        check=lambda a: [[r[1], r[3]] for r in tags(a, "E")][:2] == [[1, [0, 1]], [0, [0, 2]]])
    add("sliding_final_overlap", spec_("final", ordered=True, sides=2, length=7 * S, offset=3 * S, align=A + 1, wait=S),
        Steps().batch((1, A, 0), (1, A + 4 * S, 1), (1, A + 5 * S, 1), (1, A + 9 * S, 0)).batch((1, A + 30 * S, 1)))
    add("late_sliding_all_windows", spec_("running", sides=2, length=6 * S, offset=2 * S, wait=0),
        Steps().batch((5, A + 20 * S, 0)).batch((5, A + 11 * S, 1), (5, A + 19 * S, 0), (5, A + 21 * S, 1)),
        check=lambda a: len(tags(a, "L")) == 6)
    # --- ordered mode, clocks -----------------------------------------------------------------------------------------------
    add("ordered_out_of_order_ts", spec_("running", ordered=True, sides=2, wait=5 * S),
        Steps().batch((1, A + 3 * S, 0), (1, A + S, 1), (1, A + S, 0), (1, A + 3 * S, 1), (1, A + 2 * S, 0), (1, A + 9 * S, 0))
        .batch((1, A + 30 * S, 1)))
    add("ordered_notify_wakes_queue_head", spec_("final", ordered=True, sides=2, length=20 * S, wait=10 * S),
        Steps(now=A).batch((4, A + 8 * S, 0), (4, A + 5 * S, 1), (4, A + 12 * S, 1), (4, A + 6 * S, 0), now=A)
        .notify(A + 4 * S).notify(A + 8 * S).notify(A + 9 * S).notify(A + 30 * S))
    add("moving_clock_notifies", spec_("complete", ordered=False, sides=2, length=4 * S, wait=2 * S),
        Steps(now=A + S).batch((7, A + S, 0), (8, A + S, 1), (7, A + S + 5, 0), now=A + S).batch((7, A + 2 * S, 1), now=A + 21 * S)
        .batch((8, A + 25 * S, 0), now=A + 22 * S).notify(A + 40 * S))
    add("wait_forever_flush_at_eof", spec_("final", ordered=True, sides=3, length=4 * S, wait=FOREVER),
        Steps().batch((1, A + 9 * S, 2), (1, A + 1 * S, 0), (1, A + 5 * S, 1)).batch((1, A, 1), (2, A + 3 * S, 0), (1, A + 2 * S, 2)),
        check=lambda a: not any(a[:-1]) and len(tags(a, "M")) == 4)
    sc = Steps(now=A)
    for i, k in enumerate((1, 2, 1, 1, 2, 1)):
        now = A + i * 3 * S
        sc.batch((k, now, i % 2), (k, now, (i + 1) % 2), (k, now, 0), now=now)
        if i % 2:
            sc.notify(now + 2 * S)
    add("system_clock_moving_now", spec_("running", ordered=True, sides=2, length=5 * S, wait=0), sc.notify(A + 60 * S))
    add("near_utc_max", spec_("final", ordered=True, sides=2, length=10 * S, align=0, wait=0),
        Steps().batch((1, UTC_MAX - 25 * S, 0), (1, UTC_MAX - 24 * S, 1), (2, UTC_MAX - 12 * S, 1))
        .batch((1, UTC_MAX - 19 * S - 1, 1), (2, UTC_MAX - 11 * S, 0), (2, UTC_MAX - 11 * S + 1, 0)))
    add("discard_resets_watermark", spec_("final", ordered=False, sides=2, length=5 * S, wait=0),
        Steps(now=A).batch((1, A + 20 * S, 0), now=A).notify(A + 10 * S).batch((1, A + 2 * S, 1), now=A + 10 * S)
        .batch((1, A + 1 * S, 0)).notify(A + 30 * S).batch((1, A, 0), now=A + 30 * S))
    keys = [0, 2**64 - 1, 2**63] + [10**k - 1 for k in range(1, 20)] + [10**k for k in range(1, 20)]
    add("digit_boundary_keys", spec_("running", ordered=False, sides=2, length=S, wait=0),
        Steps().batch(*[(k, A + (i % 3) * S, i % 2) for i, k in enumerate(keys)]).batch(*[(k, A + 5 * S, 1) for k in keys[::-1]]))

    seeded = {}
    for seed in po.SEEDED:
        spec, steps = po.seeded_steps(seed, moving=seed % 3 != 0)
        acts = gj.run_reference(spec, steps)
        seeded[f"seed_{seed}"] = dict(sha256=rows_digest(acts), rows=[len(a) for a in acts])
    path = os.path.join(ROOT, "tests", "golden", "product_join_window_cases.json")
    with open(path, "w") as f:
        json.dump(dict(cases=cases, seeded=seeded), f, separators=(",", ":"))
    print("wrote", path, os.path.getsize(path), "bytes,", len(cases), "cases,", len(seeded), "seeded streams")


if __name__ == "__main__":
    main()
