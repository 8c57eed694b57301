"""K14: `join_window(insert_mode="product")` on the device (`bw_pjwin_*`) against the reference.  -m gpu.

Rows are compared exactly, in the order the device emits them: the goldens of tests/golden/product_join_window_cases.json
(made by the reference's own `_WindowLogic` + `_SlidingWindowerLogic` + `_JoinWindowLogic`), the SHA-256 digests of its
seeded streams, and `tests/product_join_window_oracle.run_product_join_window` on larger streams -- including the call in
which each handle is released."""

import json
import os
import random

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle.streams import rows_digest
from tests import product_join_window_oracle as po

pytestmark = pytest.mark.gpu
CAPACITY, SPEC, STATE = 3, 4, 5  # BW_ERR_CAPACITY, BW_ERR_SPEC, BW_ERR_STATE
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first

S, A = po.S, po.A
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "product_join_window_cases.json")
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


def _join(ctx, spec, **kw):
    from bytewax_b200 import gpu

    wait = spec["wait_us"]
    kw.setdefault("max_windows_per_key", 64)
    return gpu.ProductJoinWindow(ctx, spec["emit_mode"], spec["ordered"], spec["sides"], spec["length_us"], spec["offset_us"],
                                 spec["align_us"], None if wait == po.WAIT_FOREVER else wait, **kw)


def _groups(keys, what):
    """Runs of equal keys, checked to come in ascending key-string order, each key once."""
    runs = []
    for i, k in enumerate(keys):
        if runs and runs[-1][0] == k:
            runs[-1][1].append(i)
        else:
            runs.append((k, [i]))
    text = [str(k) for k, _ in runs]
    assert text == sorted(text) and len(set(text)) == len(text), f"{what} rows not in ascending key-string order"
    return dict(runs)


def _rows(out, bounds, batch, final):
    """Device rows of one call as the reference's row list.  Per key: late rows, then down rows, then meta rows; with
    emit mode final every down row is a close-time row, and each closed window's run of rows precedes its meta row."""
    lk, lw, lr = out.late_key.tolist(), out.late_window_id.tolist(), out.late_row.tolist()
    dk, dw, dt = out.down_key.tolist(), out.down_window_id.tolist(), out.tuples()
    mk, mw = out.meta_key.tolist(), out.meta_window_id.tolist()
    gl, gd, gm = _groups(lk, "late"), _groups(dk, "down"), _groups(mk, "meta")
    rows = []
    for k in sorted(set(gl) | set(gd) | set(gm), key=str):
        for i in gl.get(k, []):
            rows.append([k, lw[i], "L", [batch["sides"][lr[i]], batch["vals"][lr[i]]]])
        di, mi = gd.get(k, []), gm.get(k, [])
        if not final:
            rows.extend([k, dw[i], "E", list(dt[i])] for i in di)
            rows.extend([k, mw[i], "M", list(bounds(mw[i]))] for i in mi)
            continue
        at = 0
        for i in mi:
            while at < len(di) and dw[di[at]] == mw[i]:
                rows.append([k, dw[di[at]], "E", list(dt[di[at]])])
                at += 1
            rows.append([k, mw[i], "M", list(bounds(mw[i]))])
        assert at == len(di), "a final row without its window's meta row"
    return rows


def run_device(ctx, spec, steps, eof=True, **kw):
    """Every step through the device, one advance per step: ``(acts, released)`` as the oracle returns them."""
    j = _join(ctx, spec, **kw)
    final = spec["emit_mode"] == "final"
    acts, released = [], []
    try:
        for st in steps:
            if st[0] == "batch":
                _, now, keys, ts, sides, vals = st
                j.apply(np.array(keys, np.uint64), np.array(sides, np.uint8), np.array(vals, np.uint64), np.array(ts, np.int64),
                        system_now_us=now)
                out = j.advance()
                batch = dict(sides=sides, vals=vals)
            else:
                out = j.advance(system_now_us=st[1])
                batch = None
            acts.append(_rows(out, j.window_bounds, batch, final))
            released.append(sorted(out.released.tolist()))
        if eof:
            out = j.eof()
            acts.append(_rows(out, j.window_bounds, None, final))
            released.append(sorted(out.released.tolist()))
    finally:
        j.close()
    return acts, released


@pytest.mark.parametrize("name", CASE_NAMES)
def test_golden_case(ctx, golden, name):
    case = golden["cases"][name]
    acts, released = run_device(ctx, case["spec"], case["steps"])
    assert acts == case["acts"]
    assert released == po.run_product_join_window(case["spec"], case["steps"])[1]


def test_golden_seeded_digests(ctx, golden):
    for seed in po.SEEDED:
        spec, steps = po.seeded_steps(seed, moving=seed % 3 != 0)
        acts, released = run_device(ctx, spec, steps)
        want = golden["seeded"][f"seed_{seed}"]
        assert rows_digest(acts) == want["sha256"], seed
        assert released == po.run_product_join_window(spec, steps)[1], seed


def _stream(seed, spec, n_keys, n_steps, per_step, moving=True):
    rnd = random.Random(seed)
    now, base, steps, nxt = A + 50 * S, A, [], 0
    for _ in range(n_steps):
        if moving:
            now += rnd.randint(0, 2 * S)
        if moving and rnd.random() < 0.2:
            steps.append(["notify", now])
            continue
        keys = [rnd.randrange(n_keys) for _ in range(per_step)]
        ts = [base + rnd.randint(-3 * S, 3 * S) - (rnd.randint(5 * S, 20 * S) if rnd.random() < 0.05 else 0) for _ in range(per_step)]
        sides = [rnd.randrange(spec["sides"]) for _ in range(per_step)]
        steps.append(["batch", now, keys, ts, sides, list(range(nxt, nxt + per_step))])
        nxt += per_step
        base += S
    return steps


@pytest.mark.parametrize("emit", ["complete", "final", "running"])
@pytest.mark.parametrize("ordered", [True, False])
@pytest.mark.parametrize("sliding", [False, True])
def test_streams_match_oracle(ctx, emit, ordered, sliding):
    i = ["complete", "final", "running"].index(emit)
    n_keys = (1000, 10_000, 100_000)[i]
    spec = dict(emit_mode=emit, ordered=ordered, sides=1 + (i + ordered + sliding) % 4, length_us=4 * S,
                offset_us=2 * S if sliding else 4 * S, align_us=A, wait_us=S)
    steps = _stream(100 + i * 4 + ordered * 2 + sliding, spec, n_keys, 8, max(n_keys // 4, 3000))
    want = po.run_product_join_window(spec, steps)
    got = run_device(ctx, spec, steps, capacity_hint=n_keys)
    assert got[0] == want[0]
    assert got[1] == want[1]
    assert sum(len(a) for a in want[0]) > 1000


def test_hot_window_2048_by_2048(ctx):
    """One key, one window, 2^11 values per side: 2^22 rows in itertools.product order."""
    n = 2048
    spec = dict(emit_mode="final", ordered=False, sides=2, length_us=10 * S, offset_us=10 * S, align_us=A, wait_us=S)
    j = _join(ctx, spec, max_batch_rows=2 * n, max_product_rows=1 << 22)
    try:
        rnd = np.random.default_rng(5)
        sides = rnd.permutation(np.repeat(np.arange(2, dtype=np.uint8), n))
        vals = rnd.permutation(np.arange(2 * n, dtype=np.uint64) + np.uint64(2**63))
        ts = A + np.arange(2 * n, dtype=np.int64)
        j.apply(np.full(2 * n, 7, np.uint64), sides, vals, ts)
        assert j.advance().down_key.size == 0
        out = j.eof()
        l0, l1 = vals[sides == 0], vals[sides == 1]
        assert out.down_key.size == n * n
        assert np.array_equal(out.down_handles[:, 0], np.repeat(l0, n))
        assert np.array_equal(out.down_handles[:, 1], np.tile(l1, n))
        assert (out.down_mask == 3).all() and (out.down_window_id == 0).all() and (out.down_key == 7).all()
        assert sorted(out.released.tolist()) == sorted(vals.tolist())
    finally:
        j.close()


def test_four_sides_near_2_pow_22(ctx):
    lens = [45, 45, 45, 46]  # 4_191_750 rows from one window
    spec = dict(emit_mode="final", ordered=True, sides=4, length_us=10 * S, offset_us=10 * S, align_us=A, wait_us=S)
    j = _join(ctx, spec, max_product_rows=1 << 22)
    try:
        rnd = np.random.default_rng(11)
        sides = np.concatenate([np.full(n, s, np.uint8) for s, n in enumerate(lens)])
        sides = sides[rnd.permutation(sides.size)]  # arrival order interleaves the sides; ts ties keep it
        vals = rnd.integers(0, 2**63, sides.size, dtype=np.int64).astype(np.uint64)
        j.apply(np.full(sides.size, 3, np.uint64), sides, vals, np.full(sides.size, A, np.int64), system_now_us=A)
        out = j.eof()
        lists = [vals[sides == s] for s in range(4)]
        it = np.indices(lens).reshape(4, -1)  # itertools.product order: the last side fastest
        assert out.down_key.size == int(np.prod(lens))
        for s in range(4):
            assert np.array_equal(out.down_handles[:, s], lists[s][it[s]])
        assert (out.down_mask == 15).all()
    finally:
        j.close()


def test_max_product_rows_exactly_and_one_past(ctx):
    spec = dict(emit_mode="final", ordered=False, sides=2, length_us=10 * S, offset_us=10 * S, align_us=A, wait_us=S)
    keys, sides = np.full(7, 1, np.uint64), np.array([0, 0, 0, 1, 1, 1, 1], np.uint8)
    for limit, ok in ((12, True), (11, False)):
        j = _join(ctx, spec, max_product_rows=limit)
        try:
            j.apply(keys, sides, np.arange(7, dtype=np.uint64), np.full(7, A, np.int64))
            if ok:
                assert j.eof().down_key.size == 12
                continue
            with pytest.raises(N.BwError) as e:
                j.eof()
            assert e.value.status == CAPACITY and "max_product_rows" in str(e.value)
            with pytest.raises(N.BwError) as e:
                j.apply(keys, sides, np.arange(7, 14, dtype=np.uint64), np.full(7, A, np.int64))
            assert e.value.status == STATE
        finally:
            j.close()


def test_emit_buffer_exactly_full_and_one_past(ctx):
    spec = dict(emit_mode="running", ordered=False, sides=2, length_us=10 * S, offset_us=10 * S, align_us=A, wait_us=po.WAIT_FOREVER)
    for n, ok in ((16, True), (17, False)):
        j = _join(ctx, spec, max_emit_rows=16)
        try:
            def run():
                j.apply(np.arange(n, dtype=np.uint64), np.zeros(n, np.uint8), np.arange(n, dtype=np.uint64), np.full(n, A, np.int64))
                return j.advance()

            if ok:
                assert run().down_key.size == 16
            else:
                with pytest.raises(N.BwError) as e:
                    run()
                assert e.value.status == CAPACITY and "max_emit_rows" in str(e.value)
        finally:
            j.close()


def test_key_table_exactly_full_and_one_past(ctx):
    spec = dict(emit_mode="final", ordered=False, sides=1, length_us=10 * S, offset_us=10 * S, align_us=A, wait_us=po.WAIT_FOREVER)
    j = _join(ctx, spec, capacity_hint=1)  # 1024 slots + the alias slot
    try:
        j.apply(np.arange(1024, dtype=np.uint64), np.zeros(1024, np.uint8), np.arange(1024, dtype=np.uint64), np.full(1024, A, np.int64))
        assert j.advance().down_key.size == 0
        with pytest.raises(N.BwError) as e:
            j.apply(np.array([5000], np.uint64), np.zeros(1, np.uint8), np.array([9999], np.uint64), np.array([A], np.int64))
            j.advance()
        assert e.value.status == CAPACITY and "key table full" in str(e.value)
    finally:
        j.close()


def test_window_list_exactly_full_and_one_past(ctx):
    spec = dict(emit_mode="final", ordered=False, sides=2, length_us=S, offset_us=S, align_us=A, wait_us=po.WAIT_FOREVER)
    for n, ok in ((4, True), (5, False)):
        j = _join(ctx, spec, max_windows_per_key=4)
        try:
            def run():
                j.apply(np.zeros(n, np.uint64), np.zeros(n, np.uint8), np.arange(n, dtype=np.uint64), A + S * np.arange(n, dtype=np.int64))
                return j.eof()

            if ok:
                assert run().meta_key.size == 4
            else:
                with pytest.raises(N.BwError) as e:
                    run()
                assert e.value.status == CAPACITY and "max_windows_per_key" in str(e.value)
        finally:
            j.close()


def test_store_compaction_during_live_running_windows(ctx):
    """Short windows of many keys close and their entries are compacted away, many times over, while key 1 keeps one
    running window open and growing: every one of its emissions must still name the right handles."""
    spec = dict(emit_mode="running", ordered=False, sides=2, length_us=2 * S, offset_us=2 * S, align_us=A, wait_us=S)
    rnd = random.Random(3)
    steps, nxt = [], 0
    for i in range(40):
        k = [1] + [2 + rnd.randrange(50) for _ in range(30)]
        ts = [A + 5000 * S + i + 1] + [A + (1000 + i * 3 + rnd.randrange(3)) * S for _ in range(30)]
        sd = [rnd.randrange(2) for _ in range(31)]
        steps.append(["batch", A, k, ts, sd, list(range(nxt, nxt + 31))])
        nxt += 31
    want = po.run_product_join_window(spec, steps)
    got = run_device(ctx, spec, steps, max_batch_rows=64)
    assert got == want
    assert sum(len(r[3]) > 0 for a in want[0] for r in a if r[0] == 1 and r[2] == "E") > 300


def test_apply_device_matches_apply(ctx):
    spec = dict(emit_mode="complete", ordered=True, sides=3, length_us=4 * S, offset_us=2 * S, align_us=A, wait_us=S)
    steps = _stream(77, spec, 300, 10, 500, moving=False)
    want = run_device(ctx, spec, steps)
    j = _join(ctx, spec)
    acts, released = [], []
    try:
        for st in steps:
            _, now, keys, ts, sides, vals = st
            cols = [torch.tensor(np.array(keys, np.uint64).view(np.int64), device="cuda"),
                    torch.tensor(np.array(sides, np.uint8), device="cuda"),
                    torch.tensor(np.array(vals, np.uint64).view(np.int64), device="cuda"),
                    torch.tensor(np.array(ts, np.int64), device="cuda")]
            torch.cuda.synchronize()
            j.apply_device(*(c.data_ptr() for c in cols), len(keys), system_now_us=now)
            out = j.advance()
            acts.append(_rows(out, j.window_bounds, dict(sides=sides, vals=vals), False))
            released.append(sorted(out.released.tolist()))
        out = j.eof()
        acts.append(_rows(out, j.window_bounds, None, False))
        released.append(sorted(out.released.tolist()))
    finally:
        j.close()
    assert (acts, released) == want


def test_bad_device_side_is_a_spec_error(ctx):
    spec = dict(emit_mode="final", ordered=True, sides=2, length_us=S, offset_us=S, align_us=A, wait_us=0)
    j = _join(ctx, spec)
    try:
        keys = torch.zeros(2, dtype=torch.int64, device="cuda")
        sides = torch.tensor([0, 2], dtype=torch.uint8, device="cuda")
        ts = torch.full((2,), A, dtype=torch.int64, device="cuda")
        j.apply_device(keys.data_ptr(), sides.data_ptr(), keys.data_ptr(), ts.data_ptr(), 2)
        with pytest.raises(N.BwError) as e:
            j.advance()
        assert e.value.status == SPEC
    finally:
        j.close()


def test_spec_errors(ctx):
    from bytewax_b200 import gpu

    base = dict(emit_mode="final", ordered=True, sides=2, length_us=S, offset_us=S, align_us=A, wait_us=0)
    for bad in (dict(sides=0), dict(sides=5), dict(emit_mode="bogus"), dict(offset_us=2 * S), dict(length_us=0), dict(wait_us=-1)):
        with pytest.raises(N.BwError) as e:
            _join(ctx, dict(base, **bad))
        assert e.value.status == SPEC, bad
    for kw in (dict(max_windows_per_key=0), dict(max_windows_per_key=65), dict(max_emit_rows=1 << 31), dict(max_batch_rows=0)):
        with pytest.raises(N.BwError) as e:
            _join(ctx, base, **kw)
        assert e.value.status == SPEC, kw
    j = _join(ctx, base)
    try:  # a host side column is checked before anything runs
        with pytest.raises(N.BwError) as e:
            j.apply(np.array([1], np.uint64), np.array([2], np.uint8), np.array([1], np.uint64), np.array([A], np.int64))
        assert e.value.status == SPEC
    finally:
        j.close()
    ctxs = gpu.Context.loopback_world(2)
    try:
        with pytest.raises(N.BwError) as e:
            gpu.ProductJoinWindow(ctxs[0])
        assert e.value.status == SPEC and "one GPU" in str(e.value)
    finally:
        for c in ctxs:
            c.close()
    with pytest.raises(N.BwError):  # bw_jwin keeps refusing product
        gpu.JoinWindow(ctx, insert_mode="product")


def test_memory_returned_on_destroy(ctx):
    spec = dict(emit_mode="running", ordered=True, sides=2, length_us=4 * S, offset_us=2 * S, align_us=A, wait_us=S)
    steps = _stream(9, spec, 2000, 6, 4000, moving=False)
    run_device(ctx, spec, steps)  # warm the allocator's pools
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        run_device(ctx, spec, steps)
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < (64 << 20)
