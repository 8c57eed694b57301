"""K15 restated: the keyed `op.join` on integer key ids and value handles.  TEST INFRASTRUCTURE ONLY.

`KeyJoinOracle` has the interface of `bytewax_b200.gpu.KeyJoin` (apply / advance / eof) with rows as ``[(key_id,
(handle or None, ...)), ...]`` and the handles each call released.  It restates `_JoinLogic` + `_JoinState`
(pysrc/bytewax/operators/__init__.py:2076-2190) under `_StatefulLogic.on_batch` (:1030-1042): per key one list per
side; "product" appends, "last" replaces the list with [value], "first" sets it only while it is empty; "complete" emits
the product once every side is non-empty and discards the key's lists, "running" emits after every item, "final" at
EOF for every key with a logic.  A product is `itertools.product` of the lists, an empty side giving one None.  Each
call's rows are in ascending key-string order, a key's emissions in item order.  A call RELEASES the handles that no
list holds after it, among those held before it and those it received.

`run_engine` drives any such object the way the engine's `_GpuKeyJoinStep` does (bytewax_b200/engine.py): per
activation the epochs with items, ascending, each one batch (keys interned as the engine does); EOF after the last
activation.  A case is ``{"insert_mode", "emit_mode", "sides", "steps": [[[epoch, [[key, side, value], ...]], ...],
...]}``: one list of batches per activation; the values are any JSON values.  The result per activation is a list of
chunks ``[tag, epoch, rows]`` (tag B: a batch's rows, E: EOF's; empty chunks left out) with rows ``[key_str, [value or
None, ...]]``.
"""

import itertools
import random

INSERTS = ("first", "last", "product")
EMITS = ("complete", "final", "running")


class KeyJoinOracle:
    def __init__(self, insert_mode: str, emit_mode: str, sides: int):
        self.insert_mode, self.emit_mode, self.sides = insert_mode, emit_mode, sides
        self.lists = {}  # key id -> one list of handles per side, while the key has a logic
        self.rows = []
        self.released = []

    def _held(self) -> set:
        return {h for st in self.lists.values() for vals in st for h in vals}

    def _emit(self, k, st):
        for t in itertools.product(*(vals if vals else [None] for vals in st)):
            self.rows.append((k, t))

    def apply(self, keys, sides, handles, epoch=None):
        before = self._held() | {int(h) for h in handles}
        seg = {}
        for k, s, h in zip(keys, sides, handles):
            seg.setdefault(int(k), []).append((int(s), int(h)))
        for k in sorted(seg, key=str):
            for side, h in seg[k]:
                st = self.lists.setdefault(k, [[] for _ in range(self.sides)])
                if self.insert_mode == "first" and not st[side]:
                    st[side] = [h]
                elif self.insert_mode == "last":
                    st[side] = [h]
                elif self.insert_mode == "product":
                    st[side].append(h)
                if self.emit_mode == "complete" and all(st):
                    self._emit(k, st)
                    del self.lists[k]
                elif self.emit_mode == "running":
                    self._emit(k, st)
        self.released.extend(sorted(before - self._held()))

    def advance(self):
        rows, released = self.rows, sorted(self.released)
        self.rows, self.released = [], []
        return rows, released

    def eof(self):
        before = self._held()
        for k in sorted(self.lists, key=str):
            if self.emit_mode == "final":
                self._emit(k, self.lists[k])
        self.lists = {}
        self.released.extend(sorted(before))
        return self.advance()


def key_id(k: str, interned: dict) -> int:
    """The engine's key ids (`_GpuWindowStep._key_id`): canonical decimal text below 2^63 is the number, every other key
    is interned from 2^63 up."""
    if k.isascii() and k.isdigit() and (k == "0" or k[0] != "0") and len(k) < 20 and int(k) < (1 << 63):
        return int(k)
    if k not in interned:
        interned[k] = (1 << 63) + len(interned)
    return interned[k]


def run_engine(case, dev, releases=None) -> list:
    """``dev``'s rows per activation as the engine hands them on; ``releases``, if a list, gets per call (each batch, then
    EOF) the sorted values whose handles the call released."""
    interned, names, values = {}, {}, {}
    acts, last_epoch, nxt = [], 0, 0

    def rows(out):
        got, rel = out
        r = [[names.get(k, str(k)), [None if h is None else values[h] for h in t]] for k, t in got]
        if interned:  # interned keys: restore ascending key-string order; stable
            r.sort(key=lambda x: x[0])
        if releases is not None:
            releases.append(sorted(rel))
        return r

    for batches in case["steps"]:
        ready = {}
        for epoch, items in batches:
            ready.setdefault(epoch, []).extend(items)
        act = []
        acts.append(act)
        for e in sorted(ready):
            items = ready[e]
            if not items:
                continue
            keys = [key_id(k, interned) for k, _s, _v in items]
            for (k, _s, _v), i in zip(items, keys):
                names[i] = k
            handles = list(range(nxt, nxt + len(items)))
            for h, (_k, _s, v) in zip(handles, items):
                values[h] = v
            nxt += len(items)
            last_epoch = max(e, last_epoch)
            dev.apply(keys, [s for _k, s, _v in items], handles, last_epoch)
            act.append(["B", e, rows(dev.advance())])
        act[:] = [c for c in act if c[2]]
    acts.append([c for c in [["E", None, rows(dev.eof())]] if c[2]])
    return acts


def run_oracle(case, releases=None) -> list:
    return run_engine(case, KeyJoinOracle(case["insert_mode"], case["emit_mode"], case["sides"]), releases)


def seeded_case(seed: int, n_keys: int = 8, steps: int = 8, per_step: int = 24) -> dict:
    """A multi-key stream for every insert x emit mode x side count across the seeds: numeric keys whose text order
    differs from their numeric order, interned keys in one of the two seeds of each mode and side count, epochs that
    advance or stand still, few items per key and side in "product" mode so that products stay small."""
    rnd = random.Random(seed)
    insert_mode, emit_mode, sides = INSERTS[seed % 3], EMITS[(seed // 3) % 3], 1 + (seed // 9) % 4
    keys = [str(rnd.randrange(0, 10 ** rnd.randrange(1, 8))) for _ in range(n_keys)]
    if (seed + seed // 36) % 2:
        keys[: n_keys // 3] = [rnd.choice(["", "a", "b", "007", "x" * 3, "-1", "é"]) + str(i) for i in range(n_keys // 3)]
    if insert_mode == "product" and emit_mode != "complete":
        per_step = max(2, per_step // (2 * sides))
    epoch, value, out = 1, 0, []
    for _ in range(steps):
        batches = []
        for _b in range(rnd.choice([1, 1, 2])):
            epoch += rnd.choice([0, 1, 1])
            items = []
            for _i in range(rnd.randrange(1, per_step + 1)):
                items.append([rnd.choice(keys), rnd.randrange(sides), value])
                value += 1
            batches.append([epoch, items])
        out.append(batches)
    return {"insert_mode": insert_mode, "emit_mode": emit_mode, "sides": sides, "steps": out}


SEEDS = list(range(72))
