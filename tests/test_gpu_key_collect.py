"""K13: the keyed `collect` on the device (`bw_kcollect_*`) against the reference's own `_CollectLogic`.  -m gpu.

Rows are compared exactly, in the order the device emits them: the goldens of tests/golden/key_collect_cases.json (made
by the reference's `_StatefulLogic` + `_CollectLogic` under the engine's activation rules,
tools/gen_key_collect_golden.py), the SHA-256 digests of its seeded streams, and `tests/key_collect_oracle` on larger
streams."""

import json
import os

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle.streams import rows_digest
from tests import key_collect_oracle as ko

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first

S = ko.S
SENTINEL = 2**64 - 1
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "key_collect_cases.json")

with open(GOLDEN) as _f:
    CASE_NAMES = sorted(json.load(_f)["cases"])


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


class Device:
    """`gpu.KeyCollect` with the oracle's interface; ``handle_of`` maps a value to the handle the device carries."""

    def __init__(self, ctx, max_size, handle_of=None, **kw):
        from bytewax_b200 import gpu

        kw.setdefault("capacity_hint", 1 << 12)
        kw.setdefault("max_batch_rows", 1 << 16)
        self.c = gpu.KeyCollect(ctx, max(1, min(max_size, SENTINEL)), **kw)
        self.fwd = handle_of or (lambda v: v)
        self.back = {}

    def apply(self, keys, values, epoch, at):
        hs = [self.fwd(v) for v in values]
        self.back.update(zip(hs, values))
        self.c.apply(np.array(keys, dtype=np.uint64), np.array(hs, dtype=np.uint64), epoch, at)

    def rows(self, out):
        return [(k, [self.back.pop(h) for h in hs]) for k, hs in zip(out.key.tolist(), out.lists())]

    def advance(self, now_us=0):
        return self.rows(self.c.advance(now_us))

    def eof(self):
        return self.rows(self.c.eof())


def run_device(ctx, case, **kw):
    d = Device(ctx, case["max_size"], **kw)
    try:
        acts = ko.run_engine(case, d)
        assert not d.back or acts[-1][-1][0] == "raises", "a handle never came back"
        return acts
    finally:
        d.c.close()


@pytest.mark.parametrize("name", CASE_NAMES)
def test_golden_case(ctx, golden, name):
    case = golden["cases"][name]
    assert run_device(ctx, case) == case["rows"]


@pytest.mark.parametrize("seed", ko.SEEDS)
def test_seeded_digests(ctx, golden, seed):
    assert rows_digest(run_device(ctx, ko.seeded_case(seed))) == golden["digests"][str(seed)]


@pytest.mark.parametrize("name", ["docstring", "many_lists_one_batch", "interned_keys", "carry_across_activations"])
def test_any_u64_is_a_handle(ctx, golden, name):
    """Handles 0, 2^64-1 and random bit patterns travel unchanged."""
    case = golden["cases"][name]
    rnd = np.random.default_rng(7)
    values = sorted({v for _now, batches in case["steps"] for _e, items in batches for _k, v in items})
    bits = [0, SENTINEL] + [int(x) for x in rnd.integers(0, 2**64, len(values), dtype=np.uint64)]
    table = dict(zip(values, bits))
    assert run_device(ctx, case, handle_of=table.__getitem__) == case["rows"]


@pytest.mark.parametrize("n_keys, seed", [(1000, 1), (10_000, 2), (100_000, 3), (100_000, 4)])
def test_random_streams_match_oracle(ctx, n_keys, seed):
    case = ko.seeded_case(seed, n_keys=n_keys, steps=8, per_step=60_000)
    assert run_device(ctx, case, capacity_hint=n_keys, max_batch_rows=1 << 17) == ko.run_oracle(case)


@pytest.mark.parametrize("max_size", [7, 10**6 - 1])
def test_hot_key(ctx, max_size):
    """10^6 items of one key in one call, and 10^6 more in the next: lists placed by the whole grid."""
    from bytewax_b200 import gpu

    n = 10**6
    c = gpu.KeyCollect(ctx, max_size, max_batch_rows=n)
    try:
        got = []
        for b in range(2):
            c.apply(np.full(n, 42, np.uint64), np.arange(b * n, (b + 1) * n, dtype=np.uint64), b + 1, ko.T0)
            got += c.advance().lists()
        got += c.eof().lists()
    finally:
        c.close()
    flat = list(range(2 * n))
    assert got == [flat[i:i + max_size] for i in range(0, 2 * n, max_size)]


def test_list_fills_across_many_calls(ctx):
    from bytewax_b200 import gpu

    c = gpu.KeyCollect(ctx, 10**6, max_batch_rows=1 << 17)
    try:
        got = []
        for b in range(25):  # 25 * 100 000 items of key 5 and one of key 6 per call
            keys = np.full(100_001, 5, np.uint64)
            keys[b * 4000] = 6
            c.apply(keys, np.arange(b * 100_001, (b + 1) * 100_001, dtype=np.uint64), b + 1, ko.T0)
            got += list(zip(*(lambda r: (r.key.tolist(), r.lists()))(c.advance())))
        got += list(zip(*(lambda r: (r.key.tolist(), r.lists()))(c.eof())))
    finally:
        c.close()
    five = [h for h in range(25 * 100_001) if (h % 100_001) != (h // 100_001) * 4000]
    six = [h for h in range(25 * 100_001) if (h % 100_001) == (h // 100_001) * 4000]
    assert got == [(5, five[:10**6]), (5, five[10**6:2 * 10**6]), (5, five[2 * 10**6:]), (6, six)]


def test_carry_store_growth_and_compaction(ctx):
    """Carried handles pass the store's starting size (one batch) many times over, then most leave by timeout so the
    store compacts: the rows equal those of a store sized up front, and the oracle's."""
    steps = []
    now, v = ko.T0, 0
    for b in range(30):
        items = [[str((v + i) % 5000), v + i] for i in range(1000)]
        v += 1000
        steps.append([now + b * S, [[b + 1, items]]])
    steps.append([now + 200 * S, []])  # every carry times out
    for b in range(10):
        items = [[str((v + i) % 300), v + i] for i in range(1000)]
        v += 1000
        steps.append([now + (300 + b) * S, [[40 + b, items]]])
    case = {"max_size": 8, "timeout_us": 100 * S, "steps": steps}
    want = ko.run_oracle(case)
    assert run_device(ctx, case, max_batch_rows=1000) == run_device(ctx, case, max_batch_rows=1 << 16) == want


def test_apply_device_equals_apply(ctx):
    from bytewax_b200 import gpu

    case = ko.seeded_case(11, n_keys=3000, steps=6, per_step=20_000)
    want = run_device(ctx, case, max_batch_rows=1 << 16)

    class OnDevice(Device):
        def apply(self, keys, values, epoch, at):
            self.back.update(zip(values, values))
            d = lambda a: torch.tensor(np.array(a, dtype=np.uint64).view(np.int64), device="cuda")  # noqa: E731
            dk, dh = d(keys), d(values)
            self.c.apply_device(dk.data_ptr(), dh.data_ptr(), len(keys), epoch, at)
            self.keep = (dk, dh)  # valid until the next call

    dev = OnDevice(ctx, case["max_size"], max_batch_rows=1 << 16)
    try:
        assert ko.run_engine(case, dev) == want
    finally:
        dev.c.close()


# ---------------------------------------------------------------------------
# capacity and spec edges
# ---------------------------------------------------------------------------


def _expect_capacity(fn, what):
    with pytest.raises(N.BwError) as ei:
        fn()
    assert ei.value.status == 3 and what in str(ei.value), str(ei.value)


def _refused(c):
    with pytest.raises(N.BwError) as ei:
        c.advance()
    assert ei.value.status == 5


def test_key_table_exactly_full(ctx):
    from bytewax_b200 import gpu

    c = gpu.KeyCollect(ctx, 2, capacity_hint=16)  # 1024 slots, plus the alias slot of key 2^64-1
    try:
        keys = np.array(list(range(1, 1024)) + [10**19, SENTINEL], dtype=np.uint64)
        c.apply(keys, np.arange(keys.size), 1, ko.T0)
        assert c.advance().key.size == 0
        c.apply(keys, np.arange(keys.size) + 5000, 2, ko.T0)  # every key fills its list
        out = c.advance()
        assert out.key.size == 1025 and sorted(map(tuple, out.lists())) == [(i, i + 5000) for i in range(1025)]
        _expect_capacity(lambda: c.apply(np.array([2000, 2001], np.uint64), np.array([1, 2]), 3, ko.T0), "key table full")
        _refused(c)
    finally:
        c.close()


def test_emit_buffer_exactly_full(ctx):
    from bytewax_b200 import gpu

    c = gpu.KeyCollect(ctx, 3, max_emit_rows=10)
    try:
        c.apply(np.array([1] * 15 + [2] * 12, np.uint64), np.arange(27), 1, ko.T0)  # 5 + 4 lists
        c.apply(np.array([3], np.uint64), np.array([27]), 2, ko.T0)
        assert c.advance(ko.T0).key.tolist() == [1] * 5 + [2] * 4 + [3]  # and key 3's carry times out: 10 rows
    finally:
        c.close()
    c = gpu.KeyCollect(ctx, 3, max_emit_rows=10)
    try:
        c.apply(np.array([1] * 15 + [2] * 15, np.uint64), np.arange(30), 1, ko.T0)
        assert c.advance().key.size == 10
        c.apply(np.array([1] * 2 + [2] * 2 + [3] * 2, np.uint64), np.arange(6), 2, ko.T0)
        c.advance()
        _expect_capacity(lambda: c.apply(np.array([7] * 33, np.uint64), np.arange(33), 3, ko.T0), "max_emit_rows")
        _refused(c)
    finally:
        c.close()
    c = gpu.KeyCollect(ctx, 3, max_emit_rows=10)
    try:
        c.apply(np.arange(11, dtype=np.uint64), np.arange(11), 1, ko.T0)
        _expect_capacity(lambda: c.advance(ko.T0), "max_emit_rows")  # 11 carries time out at once
        _refused(c)
    finally:
        c.close()


def test_spec_errors(ctx):
    from bytewax_b200 import gpu

    for kw in (dict(max_size=0), dict(max_size=1, max_batch_rows=0), dict(max_size=1, max_emit_rows=1 << 31),
               dict(max_size=1, capacity_hint=1 << 30)):
        with pytest.raises(N.BwError) as ei:
            gpu.KeyCollect(ctx, **kw)
        assert ei.value.status == 4, kw
    c = gpu.KeyCollect(ctx, 2, max_batch_rows=4)
    try:
        with pytest.raises(N.BwError) as ei:
            c.apply(np.arange(5, dtype=np.uint64), np.arange(5), 1, 0)
        assert ei.value.status == 4
        c.apply(np.arange(4, dtype=np.uint64), np.arange(4), 2, 0)
        with pytest.raises(N.BwError) as ei:
            c.apply(np.arange(4, dtype=np.uint64), np.arange(4), 1, 0)
        assert ei.value.status == 5 and "epochs" in str(ei.value)
    finally:
        c.close()
    ctxs = gpu.Context.loopback_world(2)
    try:
        with pytest.raises(N.BwError) as ei:
            gpu.KeyCollect(ctxs[0], 3)
        assert ei.value.status == 4 and "one GPU" in str(ei.value)
    finally:
        for x in ctxs:
            x.close()


def test_create_destroy_returns_memory(ctx):
    from bytewax_b200 import gpu

    def cycle():
        c = gpu.KeyCollect(ctx, 64, capacity_hint=1 << 16, max_batch_rows=4096)
        rnd = np.random.default_rng(1)
        for b in range(8):  # the store and staging buffers grow past their starting size
            c.apply(rnd.integers(0, 50, 4096).astype(np.uint64), np.arange(4096) + 4096 * b, b + 1, ko.T0 + b)
            c.advance()
        c.advance(ko.T0 + 3)
        c.eof()
        c.close()

    def free():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info()[0]

    cycle()
    before = free()
    for _ in range(3):
        cycle()
    assert before - free() < (32 << 20)
