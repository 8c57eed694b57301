"""CPU restatement of `join_window(insert_mode="product")` over session windows, on integer microseconds.
TEST INFRASTRUCTURE ONLY.

What the CUDA session product join (``bw_spjwin``, csrc/bw_spjwin.cuh) replaces, restated in plain Python over value
HANDLES (paths relative to the bytewax v0.21.1 source tree).  Everything but the join state is the first / last session
join's (``tests/session_join_oracle.py``): the late test, the queue, ordered play, ``open_for`` with its merges, the
merge queue, the close in id order, notify, EOF, and session state that is never discarded.  The join state is
``_JoinState`` (pysrc/bytewax/operators/__init__.py:2072-2120) with ``add_val``: one list per side; ``on_merge``
(windowing.py:1879-1891) does ``self.state += original.state`` (``__iadd__``, :2106-2112: per side the survivor's list,
then the merged-away session's); ``astuples`` is ``itertools.product`` of the lists with one None for an empty side.

``tools/gen_session_product_join_golden.py`` drives the reference's own classes and writes
``tests/golden/session_product_join_cases.json``; ``tests/test_oracle_session_product_join.py`` checks this restatement
against it.  Rows are ``[key, window_id, tag, payload]`` as in ``session_join_oracle``, one ``E`` row per tuple.

``run_session_product_join`` also reports the handles each call RELEASES: those that no session list and no queue entry
of their key holds after the call, among the ones held before it and the ones the call received.
"""

from __future__ import annotations

from typing import Dict, List, Optional

from oracle.pyoracle import key_str
from tests.product_join_window_oracle import EMITS, product_rows
from tests.session_join_oracle import A, S, WAIT_FOREVER, SessionJoinLogic  # noqa: F401


class SessionProductJoinLogic(SessionJoinLogic):
    """``_WindowLogic`` over a session windower and ``_JoinWindowLogic(insert_mode="product")`` per session, for one key.
    A session's state is one list of values per side."""

    def _check_emit(self, st: List[list]) -> List[list]:
        if self.emit_mode == "complete" and all(st):
            rows = product_rows(st)
            for vals in st:
                vals.clear()  # _JoinState.clear
            return rows
        if self.emit_mode == "running":
            return product_rows(st)
        return []

    def _on_value(self, st, side, value):
        st[side].append(value)  # add_val, windowing.py:1866-1876
        return self._check_emit(st)

    def _on_merge(self, into, orig):
        for s in range(self.sides):  # self.state += original.state
            into[s].extend(orig[s])
        return self._check_emit(into)

    def _flush(self, watermark: int) -> List[list]:
        # the first / last session join's flush with list states: `setdefault` opens a session with empty lists, and a
        # `final` close emits the whole product
        if self.ordered:
            due = [e for e in self.queue if e[1] <= watermark]
            self.queue = [e for e in self.queue if not (e[1] <= watermark)]
            due.sort(key=lambda e: e[1])  # stable
        else:
            due, self.queue = self.queue, []
        events = []
        for (side, value), ts in due:  # _handle_inserts, windowing.py:1064-1077
            wid = self.windower.open_for(ts)
            st = self.states.setdefault(wid, [[] for _ in range(self.sides)])
            events.extend([wid, "E", row] for row in self._on_value(st, side, value))
        for orig, into in self.windower.merged():  # _handle_merged, windowing.py:1079-1085
            self.merges += 1
            events.extend([into, "E", row] for row in self._on_merge(self.states[into], self.states.pop(orig)))
        for wid, meta in self.windower.close_for(watermark):  # _handle_closed, windowing.py:1087-1093
            st = self.states.pop(wid)
            if self.emit_mode == "final":
                events.extend([wid, "E", row] for row in product_rows(st))
            events.append([wid, "M", [meta[0], meta[1], sorted(meta[2])]])
        return events

    def held(self) -> set:
        out = {v for st in self.states.values() for vals in st for v in vals}
        out.update(e[0][1] for e in self.queue)
        return out


def run_session_product_join(spec: dict, steps, eof: bool = True, stats: Optional[dict] = None):
    """``spec``: emit_mode, ordered, sides, gap_us, wait_us.  ``steps``: ``["batch", now_us, keys, ts, sides, values]``
    (one activation, ``now_getter() == now_us``) or ``["notify", now_us]`` (every key whose ``notify_at()`` has come,
    src/operators.rs:808-858).  Values must be distinct ints (the handles).  ``stats``: gets ``merges``.

    Returns ``(acts, released)``: the rows of every step (then EOF), and per step the sorted handles it released."""
    logics: Dict[str, SessionProductJoinLogic] = {}  # never discarded (windowing.py:798-806)
    ids: Dict[str, int] = {}
    acts, released = [], []
    held: set = set()
    spec = dict(spec, insert_mode="product")

    def rows_of(ks, events):
        return [[ids[ks], wid, tag, payload] for wid, tag, payload in events]

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
                    lg = logics[ks] = SessionProductJoinLogic(spec, now)
                rows.extend(rows_of(ks, lg.on_batch(grouped[ks])))
        else:
            for ks in sorted(logics):
                at = logics[ks].notify_at()
                if at is not None and at <= now:
                    rows.extend(rows_of(ks, logics[ks].on_notify()))
        settle(rows, incoming)
    if eof:
        rows = []
        for ks in sorted(logics):
            rows.extend(rows_of(ks, logics[ks].on_eof()))
        settle(rows, set())
    if stats is not None:
        stats["merges"] = sum(lg.merges for lg in logics.values())
    return acts, released


def seeded_spec(seed: int) -> dict:
    emit_mode = EMITS[seed % 3]
    ordered = (seed // 3) % 2 == 0
    sides = 1 + (seed // 2) % 4
    gap = (0, S, 2 * S, 4 * S)[(seed // 5) % 4]
    wait = (0, S, 3 * S, WAIT_FOREVER)[(seed // 7) % 4]
    if gap == 0 and wait == WAIT_FOREVER:  # nothing would close before EOF: a key would need too many sessions
        wait = 3 * S
    return dict(insert_mode="product", emit_mode=emit_mode, ordered=ordered, sides=sides, gap_us=gap, wait_us=wait)


def seeded_steps(seed: int, n_steps: int = 24, n_keys: int = 5, moving: bool = True):
    """A seeded stream as ``session_join_oracle.seeded_steps``, with the product spec of ``seeded_spec`` and fewer items
    per activation, so that products stay small: keys 0..n_keys, timestamps jittered by +-4 s around a base that moves
    forward 1 s per activation, one item in ten up to 30 s behind.  ``moving``: the system clock steps forward and some
    steps are notify phases; otherwise it is frozen."""
    import random

    rnd = random.Random(16000 + seed)
    spec = seeded_spec(seed)
    now, base, steps, nxt = A + 50 * S, A, [], 0
    for _ in range(n_steps):
        if moving:
            now += rnd.randint(0, 3 * S)
        if moving and rnd.random() < 0.25:
            steps.append(["notify", now])
            continue
        n = rnd.randint(1, 10)
        keys = [rnd.randint(0, n_keys) for _ in range(n)]
        ts = [base + rnd.randint(-4 * S, 4 * S) - (rnd.randint(5 * S, 30 * S) if rnd.random() < 0.1 else 0) for _ in range(n)]
        sides = [rnd.randrange(spec["sides"]) for _ in range(n)]
        steps.append(["batch", now, keys, ts, sides, list(range(nxt, nxt + n))])
        nxt += n
        base += S
    return spec, steps


SEEDED = range(48)
