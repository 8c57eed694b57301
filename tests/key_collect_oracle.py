"""K13 restated: the keyed `collect(step_id, up, timeout, max_size)` on integer key ids, microseconds and handles.

`KeyCollectOracle` has the interface of `bytewax_b200.gpu.KeyCollect` (apply / advance / eof) with rows as
``[(key_id, [handle, ...]), ...]``: per key a list and a timeout; every item appends and sets the timeout to the call's
``timeout_at_us``; a list that reaches max_size leaves as a row and the key starts over; advance(now) emits every list
whose timeout is <= now, eof every list, each call's rows in ascending key-string order.

`run_engine` drives any such object the way the engine's `_GpuCollectStep` does (bytewax_b200/engine.py): per
activation the epochs with items plus the previous activation's epoch, ascending; per epoch first the batch (keys
interned as the engine does, ``timeout_at = now + timeout``), then the notify phase at the activation's ``now``; EOF
after the last activation.  A case is ``{"max_size", "timeout_us", "steps": [[now_us, [[epoch, [[key, value], ...]],
...]], ...]}``; values are distinct ints, so they double as handles.  The result per activation is a list of chunks
``[tag, epoch, rows]`` (tag B: a batch's rows, N: a notify phase's, E: EOF's; empty chunks left out) with rows
``[key_str, [value, ...]]``; a `now + timeout` outside the range of `datetime` ends the run with ``["raises",
"OverflowError"]``, as the reference's `_CollectLogic.on_item` raises it.
"""

import random
from datetime import datetime, timedelta, timezone

S = 1_000_000
EPOCH = datetime(1970, 1, 1, tzinfo=timezone.utc)
UTC_MAX = 253_402_300_799_999_999
T0 = 1_700_000_000 * S


class KeyCollectOracle:
    def __init__(self, max_size: int):
        self.M = max(1, min(max_size, 2**64 - 1))
        self.carry = {}  # key id -> [handles, timeout_at_us]
        self.rows = []

    def apply(self, keys, handles, epoch=None, timeout_at_us=0):
        seg = {}
        for k, h in zip(keys, handles):
            seg.setdefault(int(k), []).append(int(h))
        for k in sorted(seg, key=str):
            acc = self.carry.pop(k, [[], None])[0]
            for h in seg[k]:
                acc.append(h)
                if len(acc) >= self.M:
                    self.rows.append((k, acc))
                    acc = []
            if acc:
                self.carry[k] = [acc, timeout_at_us]

    def _emit(self, keys):
        for k in sorted(keys, key=str):
            self.rows.append((k, self.carry.pop(k)[0]))

    def advance(self, now_us=0):
        if now_us > 0:
            self._emit([k for k, (_acc, at) in self.carry.items() if at <= now_us])
        rows, self.rows = self.rows, []
        return rows

    def eof(self):
        self._emit(list(self.carry))
        return self.advance()


def key_id(k: str, interned: dict) -> int:
    """The engine's key ids (`_GpuWindowStep._key_id`): canonical decimal text below 2^63 is the number, every other key
    is interned from 2^63 up."""
    if k.isascii() and k.isdigit() and (k == "0" or k[0] != "0") and len(k) < 20 and int(k) < (1 << 63):
        return int(k)
    if k not in interned:
        interned[k] = (1 << 63) + len(interned)
    return interned[k]


def timeout_at_us(now_us: int, timeout_us: int) -> int:
    """`now_getter() + timeout` in microseconds; OverflowError where the reference's datetime arithmetic raises it."""
    d = EPOCH + timedelta(microseconds=now_us) + timedelta(microseconds=timeout_us)
    d -= EPOCH
    return (d.days * 86400 + d.seconds) * 1_000_000 + d.microseconds


def run_engine(case, dev) -> list:
    interned: dict = {}
    names: dict = {}
    acts, last_out, last_epoch = [], 0, 0

    def rows(out):
        r = [[names.get(k, str(k)), list(hs)] for k, hs in out]
        if interned:  # interned keys: restore ascending key-string order; stable
            r.sort(key=lambda x: x[0])
        return r

    for now, batches in case["steps"]:
        ready = {}
        for epoch, items in batches:
            ready.setdefault(epoch, []).extend(items)
        epochs = sorted(set(ready) | ({last_out} if last_out else set()))
        act = []
        acts.append(act)
        for e in epochs:
            items = ready.get(e)
            if items:
                keys = [key_id(k, interned) for k, _v in items]
                for k, i in zip((k for k, _v in items), keys):
                    names[i] = k
                try:
                    at = timeout_at_us(now, case["timeout_us"])
                except OverflowError:
                    act.append(["raises", "OverflowError"])
                    return acts
                last_epoch = max(e, last_epoch)
                dev.apply(keys, [v for _k, v in items], last_epoch, at)
                act.append(["B", e, rows(dev.advance())])
            act.append(["N", e, rows(dev.advance(now))])
        if epochs:
            last_out = epochs[-1]
        act[:] = [c for c in act if c[2]]
    acts.append([c for c in [["E", None, rows(dev.eof())]] if c[2]])
    return acts


def run_oracle(case) -> list:
    return run_engine(case, KeyCollectOracle(case["max_size"]))


def seeded_case(seed: int, n_keys: int = 12, steps: int = 10, per_step: int = 40) -> dict:
    """A multi-key stream under a moving clock: numeric keys whose text order differs from their numeric order, interned
    keys when ``seed`` is odd, a max_size and a timeout drawn from edge values, epochs that advance or stand still."""
    rnd = random.Random(seed)
    keys = [str(rnd.randrange(0, 10 ** rnd.randrange(1, 8))) for _ in range(n_keys)]
    if seed % 2:
        keys[: n_keys // 3] = [rnd.choice(["", "a", "b", "007", "x" * 3, "-1", "é"]) + str(i) for i in range(n_keys // 3)]
    max_size = [1, 2, 3, 5, 16, 0, -3, 2**70][seed % 8]
    timeout = [0, -S, S, 3 * S, 10 * S, 10**6 * S][seed % 6]
    now, epoch, value, out = T0, 1, 0, []
    for _ in range(steps):
        now += rnd.choice([0, 0, S // 2, S, 2 * S, 7 * S])
        batches = []
        for _b in range(rnd.choice([0, 1, 1, 2])):
            epoch += rnd.choice([0, 1, 1])
            items = []
            for _i in range(rnd.randrange(1, per_step + 1)):
                items.append([rnd.choice(keys), value])
                value += 1
            batches.append([epoch, items])
        out.append([now, batches])
    return {"max_size": max_size, "timeout_us": timeout, "steps": out}


SEEDS = list(range(40))
