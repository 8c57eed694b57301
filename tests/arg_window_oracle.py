"""CPU restatement of `max_window` / `min_window` with a ``by=`` projection, on integer microseconds.  TEST
INFRASTRUCTURE ONLY.

What the CUDA windowed arg-max / arg-min (``bw_argwin``, csrc/bw_argwin.cuh) replaces, restated in plain Python over
item HANDLES (paths relative to the bytewax v0.21.1 source tree):

* ``max_window`` / ``min_window`` -> pysrc/bytewax/operators/windowing.py:2145-2236: ``reduce_window(partial(max, key=by))``
* ``reduce_window``        -> windowing.py:2268-2285: ``fold_window(ordered=False)``, the first value seeds the state
* ``_FoldWindowLogic``     -> windowing.py:1692-1714: folder and merger are both ``max(acc, v, key=by)``
* the clock, windower, queue, inserts, merges and close are `join_window`'s (``tests/join_window_oracle.JoinWindowLogic``
  for tumbling / sliding windows, ``tests/session_join_oracle.SessionJoinLogic`` for sessions), which this module reuses
  with one side whose state is the pick
* engine                   -> src/operators.rs:755-806, :808-858 (notify), :862-894 (EOF)

Steps are ``["batch", now_us, keys, ts, bys, handles]`` or ``["notify", now_us]``; ``bys[i]`` is ``by`` of item i (an
int or a float).  ``tools/gen_arg_window_golden.py`` drives the reference's own classes and writes
``tests/golden/arg_window_cases.json`` (floats as ``float.hex``, so NaN and -0.0 survive JSON);
``tests/test_oracle_arg_window.py`` checks this restatement against it.  Rows are ``[key, window_id, tag, payload]`` in
the order the reference's logic returns them: ``E`` carries the pick's handle, ``L`` the late item's handle, ``M``
``[open_us, close_us]`` (sessions: ``[open_us, close_us, sorted merged ids]``).

``run_arg_window`` also reports the handles each call RELEASES (``bw_argwin_rows.released``): those no window holds
after the call, among the ones held before it and the ones the call received.
"""

from __future__ import annotations

import math
from typing import Dict, List, Optional

from oracle.pyoracle import key_str
from tests.join_window_oracle import A, S, WAIT_FOREVER, JoinWindowLogic
from tests.session_join_oracle import SessionJoinLogic

__all__ = ["A", "S", "WAIT_FOREVER", "run_arg_window", "seeded_spec", "seeded_steps", "SEEDED", "enc", "dec"]


def enc(b):
    """A by-value as JSON: ints as they are, floats as ``float.hex`` strings."""
    return b.hex() if isinstance(b, float) else b


def dec(b):
    return float.fromhex(b) if isinstance(b, str) else b


class _Pick:
    """The compare-insert of ``max(acc, v, key=by)`` on a one-side state ``[handle]``."""

    def _better(self, h: int, pick: Optional[int]) -> bool:
        if pick is None:
            return True  # shim_folder: the first value seeds the state
        a, b = self.by[h], self.by[pick]
        return a > b if self.extreme == "max" else a < b  # Python's comparison: NaN never wins, ties keep the pick

    def _on_value(self, st: List[Optional[int]], side: int, value) -> List[list]:
        if self._better(value, st[0]):
            st[0] = value
        return []

    def _on_merge(self, into: List[Optional[int]], orig: List[Optional[int]]) -> List[list]:
        # `into.state = max(into.state, orig.state, key=by)` (windowing.py:1700-1705)
        if orig[0] is not None and into[0] is not None and self._better(orig[0], into[0]):
            into[0] = orig[0]
        return []


class ArgWindowLogic(_Pick, JoinWindowLogic):
    """``_WindowLogic`` over a sliding windower with the arg-max / arg-min fold per window, for one key."""

    def __init__(self, spec: dict, now_us: int, by: dict):
        super().__init__(dict(spec, insert_mode=None, emit_mode="final", ordered=False, sides=1), now_us)
        self.extreme, self.by = spec["extreme"], by


class SessionArgWindowLogic(_Pick, SessionJoinLogic):
    """``_WindowLogic`` over a session windower with the arg-max / arg-min fold per session, for one key."""

    def __init__(self, spec: dict, now_us: int, by: dict):
        super().__init__(dict(spec, insert_mode=None, emit_mode="final", ordered=False, sides=1), now_us)
        self.extreme, self.by = spec["extreme"], by


def _events(events) -> List[list]:
    # E [pick] -> pick; L [side, handle] -> handle
    return [[w, t, p[0] if t == "E" else p[1] if t == "L" else p] for w, t, p in events]


def run_arg_window(spec: dict, steps, eof: bool = True):
    """``spec``: extreme, wait_us, and either gap_us (sessions) or length_us, offset_us, align_us.  Handles must be
    distinct ints.  Returns ``(acts, released)``: the rows of every step (then EOF), and per step the sorted handles it
    released."""
    session = "gap_us" in spec
    logics: Dict[str, object] = {}
    ids: Dict[str, int] = {}
    by: Dict[int, object] = {}
    acts, released = [], []
    held: set = set()

    def finish(ks, lg, rows, events):
        rows.extend([ids[ks], w, t, p] for w, t, p in _events(events))
        if not session and lg.is_empty():
            del logics[ks]  # src/operators.rs:796-799: the clock state goes too (sessions are never discarded)

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
            for k, t, b, h in zip(step[2], step[3], step[4], step[5]):
                ks = key_str(k)
                ids[ks] = int(k)
                by[h] = dec(b)
                grouped.setdefault(ks, []).append((0, h, int(t)))
                incoming.add(h)
            for ks in sorted(grouped):  # BTreeMap order, src/operators.rs:758-767
                lg = logics.get(ks)
                if lg is None:
                    lg = logics[ks] = (SessionArgWindowLogic if session else ArgWindowLogic)(spec, now, by)
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


WINDOWERS = ("tumbling", "sliding", "session")


def seeded_spec(seed: int) -> dict:
    kind = WINDOWERS[seed % 3]
    spec = dict(extreme=("max", "min")[(seed // 3) % 2], wait_us=(0, S, 3 * S, WAIT_FOREVER)[(seed // 6) % 4])
    if kind == "session":
        spec["gap_us"] = (0, S, 2 * S)[(seed // 2) % 3]
        if spec["wait_us"] == WAIT_FOREVER and spec["gap_us"] == 0:  # nothing would close before EOF
            spec["wait_us"] = 3 * S
    else:
        shapes = ((4 * S, 4 * S), (3 * S, 3 * S)) if kind == "tumbling" else ((6 * S, 2 * S), (5 * S, 3 * S))
        length, offset = shapes[seed % 2]
        spec.update(length_us=length, offset_us=offset, align_us=A + (seed % 7) * 333_333)
    return spec


def by_values(rnd, n: int, f64: bool) -> list:
    """By-values with many ties; f64 adds NaN, +-0.0, +-inf and subnormals."""
    if not f64:
        return [rnd.choice((rnd.randint(-5, 5), rnd.randint(-(1 << 63), (1 << 63) - 1))) for _ in range(n)]
    special = (math.nan, 0.0, -0.0, math.inf, -math.inf, 5e-324, -5e-324)
    return [rnd.choice(special) if rnd.random() < 0.15 else float(rnd.randint(-5, 5)) / 2 for _ in range(n)]


def seeded_steps(seed: int, n_steps: int = 30, n_keys: int = 6, moving: bool = True, f64: Optional[bool] = None,
                 max_items: int = 25):
    """A seeded stream of activations and notify steps, as ``join_window_oracle.seeded_steps``: keys 0..n_keys,
    1..max_items items per activation, timestamps jittered by +-4 s around a base that moves forward 1 s per activation,
    one item in ten up to 30 s behind.  Handles are running integers.  ``f64``: float by-values (default: odd seeds // 12)."""
    import random

    rnd = random.Random(13000 + seed)
    spec = seeded_spec(seed)
    f64 = (seed // 12) % 2 == 1 if f64 is None else f64
    now, base, steps, nxt = A + 50 * S, A, [], 0
    for _ in range(n_steps):
        if moving:
            now += rnd.randint(0, 3 * S)
        if moving and rnd.random() < 0.25:
            steps.append(["notify", now])
            continue
        n = rnd.randint(1, max_items)
        keys = [rnd.randint(0, n_keys) for _ in range(n)]
        ts = [base + rnd.randint(-4 * S, 4 * S) - (rnd.randint(5 * S, 30 * S) if rnd.random() < 0.1 else 0) for _ in range(n)]
        steps.append(["batch", now, keys, ts, [enc(b) for b in by_values(rnd, n, f64)], list(range(nxt, nxt + n))])
        nxt += n
        base += S
    return spec, steps


SEEDED = range(48)
