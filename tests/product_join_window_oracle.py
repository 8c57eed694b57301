"""CPU restatement of `join_window(insert_mode="product")` on integer microseconds.  TEST INFRASTRUCTURE ONLY.

What the CUDA windowed product join (``bw_pjwin``, csrc/bw_pjwin.cuh) replaces, restated in plain Python over value
HANDLES (paths relative to the bytewax v0.21.1 source tree).  Everything but the join state is the first / last
join's (``tests/join_window_oracle.py``): the late test, the queue, ordered play, ``open_for`` in ascending id, the close
in first-opened order, notify, EOF and the discard of an empty logic.  The join state is ``_JoinState``
(pysrc/bytewax/operators/__init__.py:2072-2120) with ``add_val``: one list per side, ``astuples`` is
``itertools.product`` of the lists with one None for an empty side, ``clear`` empties every list.

``tools/gen_product_join_window_golden.py`` drives the reference's own classes and writes
``tests/golden/product_join_window_cases.json``; ``tests/test_oracle_product_join_window.py`` checks this restatement
against it.  Rows are ``[key, window_id, tag, payload]`` as in ``join_window_oracle``.

``run_product_join_window`` also reports the handles each call RELEASES: those that no window list and no queue entry of
their key holds after the call, among the ones held before it and the ones the call received.
"""

from __future__ import annotations

import itertools
from typing import Dict, List

from oracle.pyoracle import key_str
from tests.join_window_oracle import A, S, WAIT_FOREVER, JoinWindowLogic  # noqa: F401

EMITS = ("complete", "final", "running")


def product_rows(st: List[list]) -> List[list]:
    """``_JoinState.astuples``: the product of the side lists, the last side fastest, an empty side giving one None."""
    return [list(t) for t in itertools.product(*(vals if vals else [None] for vals in st))]


class ProductJoinWindowLogic(JoinWindowLogic):
    """``_WindowLogic`` over a sliding windower and ``_JoinWindowLogic(insert_mode="product")`` per window, for one key.
    A window's state is one list of values per side."""

    def _on_value(self, st, side, value):
        # windowing.py:1866-1876 with `add_val`
        st[side].append(value)
        if self.emit_mode == "complete" and all(st):
            rows = product_rows(st)
            for vals in st:
                vals.clear()
            return rows
        if self.emit_mode == "running":
            return product_rows(st)
        return []

    def _flush(self, watermark):
        # the first / last join's flush with list states: `setdefault` opens a window with empty lists, and a
        # `final` close emits the whole product
        if self.ordered:
            due = [e for e in self.queue if e[1] <= watermark]
            self.queue = [e for e in self.queue if not (e[1] <= watermark)]
            due.sort(key=lambda e: e[1])  # stable
        else:
            due, self.queue = self.queue, []
        events = []
        for (side, value), ts in due:
            for wid in self.windower.open_for(ts):
                st = self.states.setdefault(wid, [[] for _ in range(self.sides)])
                events.extend([wid, "E", row] for row in self._on_value(st, side, value))
        for wid, meta in self.windower.close_for(watermark):
            st = self.states.pop(wid)
            if self.emit_mode == "final":
                events.extend([wid, "E", row] for row in product_rows(st))
            events.append([wid, "M", [meta[0], meta[1]]])
        return events

    def held(self) -> set:
        out = {v for st in self.states.values() for vals in st for v in vals}
        out.update(e[0][1] for e in self.queue)
        return out


def run_product_join_window(spec: dict, steps, eof: bool = True):
    """``spec``: emit_mode, ordered, sides, length_us, offset_us, align_us, wait_us.  ``steps``: ``["batch", now_us,
    keys, ts, sides, values]`` (one activation, ``now_getter() == now_us``) or ``["notify", now_us]`` (every key whose
    ``notify_at()`` has come, src/operators.rs:808-858).  Values must be distinct ints (the handles).

    Returns ``(acts, released)``: the rows of every step (then EOF), and per step the sorted handles it released."""
    logics: Dict[str, ProductJoinWindowLogic] = {}
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
            for k, t, sd, v in zip(step[2], step[3], step[4], step[5]):
                ks = key_str(k)
                ids[ks] = int(k)
                grouped.setdefault(ks, []).append((int(sd), v, int(t)))
                incoming.add(v)
            for ks in sorted(grouped):  # BTreeMap order, src/operators.rs:758-767
                lg = logics.get(ks)
                if lg is None:
                    lg = logics[ks] = ProductJoinWindowLogic(dict(spec, insert_mode="product"), now)
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
    emit_mode = EMITS[seed % 3]
    ordered = (seed // 3) % 2 == 0
    sides = 1 + (seed // 2) % 4
    length, offset = ((4 * S, 4 * S), (6 * S, 2 * S), (5 * S, 3 * S), (3 * S, 3 * S))[(seed // 5) % 4]
    wait = (0, S, 3 * S, WAIT_FOREVER)[(seed // 7) % 4]
    align = A + (seed % 7) * 333_333
    return dict(insert_mode="product", emit_mode=emit_mode, ordered=ordered, sides=sides, length_us=length, offset_us=offset,
                align_us=align, wait_us=wait)


def seeded_steps(seed: int, n_steps: int = 24, n_keys: int = 5, moving: bool = True):
    """A seeded stream as ``join_window_oracle.seeded_steps``, with the product spec of ``seeded_spec`` and fewer items
    per activation, so that products stay small."""
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
        n = rnd.randint(1, 12)
        keys = [rnd.randint(0, n_keys) for _ in range(n)]
        ts = [base + rnd.randint(-4 * S, 4 * S) - (rnd.randint(5 * S, 30 * S) if rnd.random() < 0.1 else 0) for _ in range(n)]
        sides = [rnd.randrange(spec["sides"]) for _ in range(n)]
        steps.append(["batch", now, keys, ts, sides, list(range(nxt, nxt + n))])
        nxt += n
        base += S
    return spec, steps


SEEDED = range(48)
