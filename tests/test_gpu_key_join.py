"""K15: the keyed `op.join` on the device (`bw_kjoin_*`) against the reference.  -m gpu.

Rows are compared exactly, in the order the device emits them: the goldens of tests/golden/key_join_cases.json (made by
the reference's own `_StatefulLogic` + `_JoinLogic`), the SHA-256 digests of its seeded streams, and
`tests/key_join_oracle` on larger streams -- including the call in which each handle is released."""

import json
import os
import random
import time

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle.streams import rows_digest
from tests import key_join_oracle as ko

pytestmark = pytest.mark.gpu
CAPACITY, SPEC, STATE = 3, 4, 5  # BW_ERR_CAPACITY, BW_ERR_SPEC, BW_ERR_STATE
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "key_join_cases.json")
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
    """`gpu.KeyJoin` with the oracle's interface: rows ``[(key_id, tuple)]`` and the sorted released handles."""

    def __init__(self, ctx, insert_mode, emit_mode, sides, **kw):
        from bytewax_b200 import gpu

        self.j = gpu.KeyJoin(ctx, insert_mode, emit_mode, sides, **kw)

    def apply(self, keys, sides, handles, epoch=None):
        self.j.apply(np.array(keys, np.uint64), np.array(sides, np.uint8), np.array(handles, np.uint64), epoch)

    @staticmethod
    def _out(out):
        return list(zip(out.key.tolist(), out.tuples())), sorted(out.released.tolist())

    def advance(self):
        return self._out(self.j.advance())

    def eof(self):
        return self._out(self.j.eof())

    def close(self):
        self.j.close()


def run_device(ctx, case, **kw):
    """A case through the device as the engine drives it: ``(acts, releases)``."""
    d = Device(ctx, case["insert_mode"], case["emit_mode"], case["sides"], **kw)
    try:
        rel = []
        acts = ko.run_engine(case, d, rel)
    finally:
        d.close()
    return acts, rel


def run_oracle(case):
    rel = []
    return ko.run_oracle(case, rel), rel


@pytest.mark.parametrize("name", CASE_NAMES)
def test_golden_case(ctx, golden, name):
    case = golden["cases"][name]
    acts, rel = run_device(ctx, case)
    assert acts == case["rows"]
    assert rel == run_oracle(case)[1]


def test_golden_seeded_digests(ctx, golden):
    for seed in ko.SEEDS:
        case = ko.seeded_case(seed)
        acts, rel = run_device(ctx, case)
        assert rows_digest(acts) == golden["digests"][str(seed)], seed
        assert rel == run_oracle(case)[1], seed


def _stream(seed, insert_mode, emit_mode, sides, n_keys, n_steps, per_step):
    rnd = random.Random(seed)
    steps, value = [], 0
    for i in range(n_steps):
        items = []
        for _ in range(per_step):
            items.append([str(rnd.randrange(n_keys)), rnd.randrange(sides), value])
            value += 1
        steps.append([[i + 1, items]])
    return dict(insert_mode=insert_mode, emit_mode=emit_mode, sides=sides, steps=steps)


@pytest.mark.parametrize("sides", [1, 2, 3, 4])
@pytest.mark.parametrize("emit", ko.EMITS)
@pytest.mark.parametrize("insert", ko.INSERTS)
def test_streams_match_oracle(ctx, insert, emit, sides):
    i = (ko.INSERTS.index(insert) + ko.EMITS.index(emit) + sides) % 3
    n_keys = (1000, 10_000, 100_000)[i]
    # product lists that never empty stay short, so the products stay small
    per_step = n_keys // 2 if insert == "product" and emit != "complete" else 2 * n_keys
    case = _stream(1000 + 100 * i + 10 * ko.EMITS.index(emit) + sides, insert, emit, sides, n_keys, 4, per_step)
    got = run_device(ctx, case, capacity_hint=n_keys, max_batch_rows=per_step, max_emit_rows=1 << 22)
    want = run_oracle(case)
    assert got[0] == want[0]
    assert got[1] == want[1]
    assert sum(len(c[2]) for a in want[0] for c in a) > 100


def test_handles_zero_and_max(ctx):
    top = 2**64 - 1
    for ins, em in (("product", "final"), ("last", "running"), ("first", "complete")):
        d = Device(ctx, ins, em, 3)
        o = ko.KeyJoinOracle(ins, em, 3)
        try:
            for dev in (d, o):
                dev.apply([5, 5, 5, 6], [0, 2, 1, 1], [0, top, top - 1, 1], 1)
            assert d.advance() == o.advance()
            for dev in (d, o):
                dev.apply([5, 6, top], [1, 0, 2], [2, top - 2, 3], 2)
            assert d.advance() == o.advance()
            assert d.eof() == o.eof()
        finally:
            d.close()


def test_one_key_2048_by_2048_final(ctx):
    """One key, 2^11 values per side: 2^22 rows at EOF in itertools.product order."""
    from bytewax_b200 import gpu

    n = 2048
    j = gpu.KeyJoin(ctx, "product", "final", 2, max_batch_rows=2 * n, max_product_rows=1 << 22)
    try:
        rnd = np.random.default_rng(5)
        sides = rnd.permutation(np.repeat(np.arange(2, dtype=np.uint8), n))
        vals = rnd.permutation(np.arange(2 * n, dtype=np.uint64) + np.uint64(2**63))
        j.apply(np.full(2 * n, 7, np.uint64), sides, vals)
        assert j.advance().key.size == 0
        out = j.eof()
        l0, l1 = vals[sides == 0], vals[sides == 1]
        assert out.key.size == n * n
        assert np.array_equal(out.handles[:, 0], np.repeat(l0, n))
        assert np.array_equal(out.handles[:, 1], np.tile(l1, n))
        assert (out.mask == 3).all() and (out.key == 7).all()
        assert sorted(out.released.tolist()) == sorted(vals.tolist())
    finally:
        j.close()


def test_four_sides_near_2_pow_22(ctx):
    from bytewax_b200 import gpu

    lens = [45, 45, 45, 46]  # 4_191_750 rows from one key
    j = gpu.KeyJoin(ctx, "product", "final", 4, max_product_rows=1 << 22)
    try:
        rnd = np.random.default_rng(11)
        sides = np.concatenate([np.full(n, s, np.uint8) for s, n in enumerate(lens)])
        sides = sides[rnd.permutation(sides.size)]
        vals = rnd.integers(0, 2**63, sides.size, dtype=np.int64).astype(np.uint64)
        half = sides.size // 2  # two activations: the lists span calls
        j.apply(np.full(half, 3, np.uint64), sides[:half], vals[:half])
        j.apply(np.full(sides.size - half, 3, np.uint64), sides[half:], vals[half:])
        out = j.eof()
        lists = [vals[sides == s] for s in range(4)]
        it = np.indices(lens).reshape(4, -1)  # itertools.product order: the last side fastest
        assert out.key.size == int(np.prod(lens))
        for s in range(4):
            assert np.array_equal(out.handles[:, s], lists[s][it[s]])
        assert (out.mask == 15).all()
    finally:
        j.close()


@pytest.mark.parametrize("insert, emit", [("product", "complete"), ("last", "running")])
def test_hot_key_million_items(ctx, insert, emit):
    """One key with 10^6 items in one activation: one thread walks them.  Prints the time of apply + advance."""
    n = 10**6
    rnd = random.Random(17)
    items = [["42", rnd.randrange(2), i] for i in range(n)]
    d = Device(ctx, insert, emit, 2, max_batch_rows=n, max_emit_rows=n, max_product_rows=1 << 22)
    try:
        t0 = time.perf_counter()
        d.apply([42] * n, [it[1] for it in items], list(range(n)), 1)
        rows, rel = d.advance()
        dt = time.perf_counter() - t0
        d.apply([42, 42], [0, 1], [n, n + 1], 2)
        rows2, rel2 = d.advance()
        rows3, rel3 = d.eof()
    finally:
        d.close()
    print(f"hot key, {insert} {emit}: 10^6 items, apply + advance {dt * 1e3:.1f} ms (host columns included)")
    o = ko.KeyJoinOracle(insert, emit, 2)
    o.apply([42] * n, [it[1] for it in items], list(range(n)), 1)
    assert (rows, rel) == o.advance()
    o.apply([42, 42], [0, 1], [n, n + 1], 2)
    assert (rows2, rel2) == o.advance()
    assert (rows3, rel3) == o.eof()
    assert len(rows) > n // 4


def test_max_product_rows_exactly_and_one_past(ctx):
    keys, sides = [1] * 7, [0, 0, 0, 1, 1, 1, 1]
    for limit, ok in ((12, True), (11, False)):
        d = Device(ctx, "product", "final", 2, max_product_rows=limit)
        try:
            d.apply(keys, sides, list(range(7)), 1)
            if ok:
                assert len(d.eof()[0]) == 12
                continue
            with pytest.raises(N.BwError) as e:
                d.eof()
            assert e.value.status == CAPACITY and "max_product_rows" in str(e.value)
            with pytest.raises(N.BwError) as e:
                d.apply(keys, sides, list(range(7, 14)), 2)
            assert e.value.status == STATE
        finally:
            d.close()


def test_emit_buffer_exactly_full_and_one_past(ctx):
    for n, ok in ((16, True), (17, False)):
        d = Device(ctx, "last", "running", 3, max_emit_rows=16)
        try:
            def run():
                d.apply(list(range(n)), [0] * n, list(range(n)), 1)
                return d.advance()

            if ok:
                assert len(run()[0]) == 16
                continue
            with pytest.raises(N.BwError) as e:
                run()
            assert e.value.status == CAPACITY and "max_emit_rows" in str(e.value)
            with pytest.raises(N.BwError) as e:
                d.apply([1], [0], [99], 2)
            assert e.value.status == STATE
        finally:
            d.close()


def test_key_table_exactly_full_and_one_past(ctx):
    d = Device(ctx, "product", "final", 1, capacity_hint=1)  # 1024 slots + the alias slot
    try:
        d.apply(list(range(1024)), [0] * 1024, list(range(1024)), 1)
        assert d.advance() == ([], [])
        d.apply(list(range(1024)), [0] * 1024, list(range(1024, 2048)), 2)  # keys already seen keep their slots
        assert d.advance() == ([], [])
        with pytest.raises(N.BwError) as e:
            d.apply([5000], [0], [9999], 3)
            d.advance()
        assert e.value.status == CAPACITY and "key table full" in str(e.value)
        with pytest.raises(N.BwError) as e:
            d.advance()
        assert e.value.status == STATE
    finally:
        d.close()


def test_store_growth_and_compaction_under_live_running_key(ctx):
    """Many keys' complete generations die and are compacted away, many times over, while key 1 keeps a running product
    list that grows across every call: each of its emissions must still name the right handles."""
    rnd = random.Random(3)
    d = Device(ctx, "product", "running", 2, max_batch_rows=64)
    o = ko.KeyJoinOracle("product", "running", 2)
    # a second join in complete mode churns the store of its own
    c = Device(ctx, "last", "complete", 3, max_batch_rows=64)
    oc = ko.KeyJoinOracle("last", "complete", 3)
    nxt = 0
    try:
        for i in range(60):
            keys = [1] + [2 + rnd.randrange(50) for _ in range(40)]
            sides = [rnd.randrange(2) if i % 3 else 0] + [rnd.randrange(2) for _ in range(40)]
            hs = list(range(nxt, nxt + 41))
            nxt += 41
            if i % 2:  # key 1 only on odd calls: its list is live across the others' compactions
                for dev in (d, o):
                    dev.apply(keys, sides, hs, i)
            else:
                for dev in (d, o):
                    dev.apply(keys[1:], sides[1:], hs[1:], i)
            assert d.advance() == o.advance(), i
            cs = [rnd.randrange(3) for _ in range(41)]
            for dev in (c, oc):
                dev.apply(keys, cs, hs, i)
            assert c.advance() == oc.advance(), i
        assert d.eof() == o.eof()
        assert c.eof() == oc.eof()
    finally:
        d.close()
        c.close()


def test_apply_device_matches_apply(ctx):
    case = _stream(77, "product", "complete", 3, 300, 10, 500)
    want = run_device(ctx, case)
    from bytewax_b200 import gpu

    j = gpu.KeyJoin(ctx, "product", "complete", 3)
    acts = []
    try:
        for batches in case["steps"]:
            (epoch, items), = batches
            keys = np.array([int(k) for k, _s, _v in items], np.uint64)
            cols = [torch.tensor(keys.view(np.int64), device="cuda"),
                    torch.tensor(np.array([s for _k, s, _v in items], np.uint8), device="cuda"),
                    torch.tensor(np.array([v for _k, _s, v in items], np.uint64).view(np.int64), device="cuda")]
            torch.cuda.synchronize()
            j.apply_device(*(c.data_ptr() for c in cols), len(items), epoch)
            out = j.advance()
            acts.append((list(zip(out.key.tolist(), out.tuples())), sorted(out.released.tolist())))
        out = j.eof()
        acts.append((list(zip(out.key.tolist(), out.tuples())), sorted(out.released.tolist())))
    finally:
        j.close()
    rows = [[[str(k), list(t)] for k, t in r] for r, _rel in acts]
    assert [[c for a in want[0][i] for c in a[2]] for i in range(len(acts))] == rows
    assert [rel for _r, rel in acts] == want[1]


def test_bad_device_side_is_a_spec_error(ctx):
    from bytewax_b200 import gpu

    j = gpu.KeyJoin(ctx, "product", "final", 2)
    try:
        keys = torch.zeros(2, dtype=torch.int64, device="cuda")
        sides = torch.tensor([0, 2], dtype=torch.uint8, device="cuda")
        j.apply_device(keys.data_ptr(), sides.data_ptr(), keys.data_ptr(), 2)
        with pytest.raises(N.BwError) as e:
            j.advance()
        assert e.value.status == SPEC and "not below sides" in str(e.value)
    finally:
        j.close()


def test_spec_errors(ctx):
    from bytewax_b200 import gpu

    for kw in (dict(sides=0), dict(sides=5), dict(insert_mode="bogus"), dict(emit_mode="bogus"), dict(max_emit_rows=1 << 31),
               dict(max_batch_rows=0), dict(max_batch_rows=1 << 31), dict(capacity_hint=1 << 30)):
        with pytest.raises(N.BwError) as e:
            gpu.KeyJoin(ctx, **kw)
        assert e.value.status == SPEC, kw
    j = gpu.KeyJoin(ctx, "last", "running", 3)
    try:  # a host side column is checked before anything runs
        with pytest.raises(N.BwError) as e:
            j.apply(np.array([1], np.uint64), np.array([3], np.uint8), np.array([1], np.uint64))
        assert e.value.status == SPEC
        with pytest.raises(N.BwError) as e:
            n = (1 << 20) + 1  # one past max_batch_rows
            j.apply(np.zeros(n, np.uint64), np.zeros(n, np.uint8), np.zeros(n, np.uint64))
        assert e.value.status == SPEC
    finally:
        j.close()
    ctxs = gpu.Context.loopback_world(2)
    try:
        with pytest.raises(N.BwError) as e:
            gpu.KeyJoin(ctxs[0])
        assert e.value.status == SPEC and "one GPU" in str(e.value)
    finally:
        for c in ctxs:
            c.close()


def test_memory_returned_on_destroy(ctx):
    case = _stream(9, "product", "running", 2, 2000, 6, 4000)
    run_device(ctx, case)  # warm the allocator's pools
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        run_device(ctx, case)
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < (64 << 20)
