"""CPU restatement of `collect_window` on integer microseconds.  TEST INFRASTRUCTURE ONLY.

What the CUDA windowed collect (``bw_collect``, csrc/bw_collect.cuh) replaces, restated in plain Python over value
HANDLES (paths relative to the bytewax v0.21.1 source tree):

* ``collect_window``       -> pysrc/bytewax/operators/windowing.py:1436-1576, callbacks :1356-1384
* ``_FoldWindowLogic``     -> windowing.py:1046-1190 with the collect folder: a window's state is its values in play order
* the clock, windower, queue, ordered flush and close are `join_window`'s (``tests/join_window_oracle.JoinWindowLogic``,
  which this module reuses with one unlabelled side)
* engine                   -> src/operators.rs:755-806 (ascending key string per activation, discard of empty logics),
                              :808-858 (notify), :862-894 (EOF)

Steps use ``tests/join_window_oracle.py``'s format with every side 0.  ``tools/gen_collect_window_golden.py`` drives the
reference's own classes and writes ``tests/golden/collect_window_cases.json``; ``tests/test_oracle_collect_window.py``
checks this restatement against it.  Rows are ``[key, window_id, tag, payload]`` in the order the reference's logic
returns them: ``E`` carries the window's values in play order, ``L`` the value, ``M`` ``[open_us, close_us]``.

``run_collect_window`` also reports the handles each call RELEASES: those no window and no queue entry of their key
holds after the call, among the ones held before it and the ones the call received (``bw_collect_rows.released``).
"""

from __future__ import annotations

from typing import Dict, List

from oracle.pyoracle import key_str
from tests.join_window_oracle import A, S, WAIT_FOREVER, JoinWindowLogic

__all__ = ["A", "S", "WAIT_FOREVER", "CollectWindowLogic", "run_collect_window", "seeded_spec", "seeded_steps", "SEEDED"]


class CollectWindowLogic(JoinWindowLogic):
    """``_WindowLogic`` over a sliding windower with the collect folder per window, for one key: the join window's
    steps with an empty starting state (no sides) that every value appends to, and its list emitted at close."""

    def __init__(self, spec: dict, now_us: int):
        super().__init__(dict(spec, insert_mode=None, emit_mode="final", sides=0), now_us)

    def _on_value(self, st: List[int], side: int, value) -> List[list]:
        st.append(value)  # `_collect_list_folder` (windowing.py:1341-1344)
        return []

    def on_batch(self, items) -> List[list]:
        events = super().on_batch(items)
        return [[w, t, p[1]] if t == "L" else [w, t, p] for w, t, p in events]


def run_collect_window(spec: dict, steps, eof: bool = True):
    """``spec``: ordered, length_us, offset_us, align_us, wait_us.  ``steps``: ``["batch", now_us, keys, ts, sides, values]``
    (one activation, ``now_getter() == now_us``; sides ignored) or ``["notify", now_us]``.  Values must be distinct ints
    (the handles).  Returns ``(acts, released)``: the rows of every step (then EOF), and per step the sorted handles it
    released."""
    logics: Dict[str, CollectWindowLogic] = {}
    ids: Dict[str, int] = {}
    acts, released = [], []
    held: set = set()

    def finish(ks, lg, rows, events):
        rows.extend([ids[ks], wid, tag, payload] for wid, tag, payload in events)
        if lg.is_empty():
            del logics[ks]  # src/operators.rs:796-799: the clock state goes too

    def settle(rows, incoming):
        nonlocal held
        now_held = set().union(*(lg.held() for lg in logics.values())) if logics else set()
        released.append(sorted((held | incoming) - now_held))
        held = now_held
        acts.append(rows)

    for step in steps:
        now = step[1]
        for lg in logics.values():
            lg.clock.now_us = now
        rows, incoming = [], set()
        if step[0] == "batch":
            grouped: Dict[str, list] = {}
            for k, t, v in zip(step[2], step[3], step[5]):
                ks = key_str(k)
                ids[ks] = int(k)
                grouped.setdefault(ks, []).append((0, v, int(t)))
                incoming.add(v)
            for ks in sorted(grouped):  # BTreeMap order, src/operators.rs:758-767
                lg = logics.get(ks)
                if lg is None:
                    lg = logics[ks] = CollectWindowLogic(spec, now)
                finish(ks, lg, rows, lg.on_batch(grouped[ks]))
        else:
            for ks in sorted(logics):
                at = logics[ks].notify_at()
                if at is not None and at <= now:
                    lg = logics[ks]
                    finish(ks, lg, rows, lg.on_notify())
        settle(rows, incoming)
    if eof:
        rows = []
        for ks in sorted(logics):
            lg = logics[ks]
            finish(ks, lg, rows, lg.on_eof())
        settle(rows, set())
    return acts, released


def seeded_spec(seed: int) -> dict:
    ordered = seed % 2 == 0
    length, offset = ((4 * S, 4 * S), (6 * S, 2 * S), (5 * S, 3 * S), (3 * S, 3 * S))[(seed // 2) % 4]
    wait = (0, S, 3 * S, WAIT_FOREVER)[(seed // 8) % 4]
    align = A + (seed % 7) * 333_333
    return dict(ordered=ordered, length_us=length, offset_us=offset, align_us=align, wait_us=wait)


def seeded_steps(seed: int, n_steps: int = 30, n_keys: int = 6, moving: bool = True):
    """A seeded stream of activations and notify steps, as ``join_window_oracle.seeded_steps`` with one side: keys
    0..n_keys, timestamps jittered by +-4 s around a base that moves forward 1 s per activation, one item in ten up to
    30 s behind.  ``moving``: the system clock steps forward and some steps are notify phases."""
    import random

    rnd = random.Random(9000 + seed)
    spec = seeded_spec(seed)
    now, base, steps, nxt = A + 50 * S, A, [], 0
    for _ in range(n_steps):
        if moving:
            now += rnd.randint(0, 3 * S)
        if moving and rnd.random() < 0.25:
            steps.append(["notify", now])
            continue
        n = rnd.randint(1, 25)
        keys = [rnd.randint(0, n_keys) for _ in range(n)]
        ts = [base + rnd.randint(-4 * S, 4 * S) - (rnd.randint(5 * S, 30 * S) if rnd.random() < 0.1 else 0) for _ in range(n)]
        steps.append(["batch", now, keys, ts, [0] * n, list(range(nxt, nxt + n))])
        nxt += n
        base += S
    return spec, steps


SEEDED = range(32)
