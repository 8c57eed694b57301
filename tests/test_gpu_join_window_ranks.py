"""K8, the windowed join, sharded by key over W ranks: threads of one process on a loopback world (include/bwgpu.h,
bw_loopback_create), whose partition kernels, peer stores into the owners' receive regions and barriers are the ones an
NCCL world runs.  -m gpu.

Each rank applies its own rows per call; each row goes to rank `po.dest_rank(key, W)`, which joins what arrived in
(source rank, source order).  The rows of all ranks of one call, the down, meta and late columns each stably sorted by
key string, must equal what a world-1 join returns for the rank-major concatenation of every rank's columns: the
reference's rows (tests/golden/join_window_cases.json, `jo.run_join_window`) and a world-1 `JoinWindow`.  A late row
(rank r, row i) of an activation is world-1 row offset_r + i.  Handles are the rows' values in the stream, so joined
tuples compare directly; every handle is released exactly once over all ranks, on the owner of its key."""

import ctypes as C
import json
import os

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle import pyoracle as po  # checker only
from oracle.streams import rows_digest
from tests import join_window_oracle as jo
from tests.test_gpu_join_ranks import no_errors, run_ranks
from tests.test_gpu_join_window import _rows
from tests.test_gpu_session_ranks import _errors_fast, _owned_by, _status, contiguous, interleaved, random_split

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first
CAPACITY, SPEC, STATE = 3, 4, 5  # BW_ERR_CAPACITY, BW_ERR_SPEC, BW_ERR_STATE
S, A = jo.S, jo.A
SENTINEL = 2**64 - 1
WORLDS = [2, 3, 4]
SMALL = dict(capacity_hint=64, max_emit_rows=4096, max_late_rows=4096, max_queued_rows=4096)

with open(os.path.join(os.path.dirname(__file__), "golden", "join_window_cases.json")) as _f:
    GOLDEN = json.load(_f)


def _join(ctx, spec, shard=True, **kw):
    from bytewax_b200 import gpu

    wait = spec["wait_us"]
    kw.setdefault("max_windows_per_key", 64)
    return gpu.JoinWindow(ctx, spec["insert_mode"], spec["emit_mode"], spec["ordered"], spec["sides"], spec["length_us"],
                          spec["offset_us"], spec["align_us"], None if wait == jo.WAIT_FOREVER else wait, shard_by_key=shard, **kw)


def _cols(step, idx=None):
    """keys, sides, handles, ts of a batch step (rows `idx` of it)."""
    _, _, keys, ts, sides, vals = step
    cols = (np.array(keys, np.uint64), np.array(sides, np.uint8), np.array(vals, np.uint64), np.array(ts, np.int64))
    return cols if idx is None else tuple(c[idx] for c in cols)


def _apply(j, cols, epoch, now, device):
    if not device:
        j.apply(*cols, epoch=epoch, system_now_us=now)
        return
    d = [torch.from_numpy(c.view(np.int64) if c.dtype == np.uint64 else c).cuda() for c in cols]
    torch.cuda.synchronize()  # the join reads them on its own stream
    j.apply_device(*(t.data_ptr() for t in d), cols[0].size, epoch=epoch, system_now_us=now)


def single_rank(world):
    """Every row of a batch on one rank, cycling through the ranks."""
    return lambda i, n: [np.arange(n) if r == i % world else np.zeros(0, np.int64) for r in range(world)]


SPLITS = ["contiguous", "interleaved", "random", "single"]


def _split(how, world, seed):
    return dict(contiguous=lambda: contiguous(world, seed), interleaved=lambda: interleaved(world),
                random=lambda: random_split(world, seed), single=lambda: single_rank(world))[how]()


# ---- the drivers ------------------------------------------------------------------------------------------------------


def plan(steps, world, split):
    """Per step: the per-rank index arrays of a batch (None for notify) and the rank-major concatenation's steps."""
    parts, cat = [], []
    for i, step in enumerate(steps):
        if step[0] != "batch":
            parts.append(None)
            cat.append(step)
            continue
        p = split(i, len(step[2]))
        order = np.concatenate(p).astype(np.int64)
        assert sorted(order.tolist()) == list(range(len(step[2])))
        parts.append(p)
        cat.append(["batch", step[1]] + [[step[c][j] for j in order.tolist()] for c in (2, 3, 4, 5)])
    return parts, cat


def run_world(world, spec, steps, parts, device=False, **kw):
    """Every rank plays every step with its slice, then EOF.  Per rank: its JoinWindowRows per call."""

    def body(r, ctx, keep):
        j = _join(ctx, spec, **kw)
        keep.append(j)
        out = []
        for i, step in enumerate(steps):
            if step[0] == "batch":
                _apply(j, _cols(step, parts[i][r]), i + 1, step[1], device)
                out.append(j.advance())
            else:
                out.append(j.advance(system_now_us=step[1]))
        out.append(j.eof())
        return out

    results, errors = run_ranks(world, body)
    no_errors(errors)
    return results


def run_one(spec, steps, **kw):
    """A world-1 join (created without shard_by_key) fed `steps`: its JoinWindowRows per call."""
    from bytewax_b200 import gpu

    ctx = gpu.Context(0)
    j = _join(ctx, spec, shard=False, **kw)
    out = []
    try:
        for i, step in enumerate(steps):
            if step[0] == "batch":
                j.apply(*_cols(step), epoch=i + 1, system_now_us=step[1])
                out.append(j.advance())
            else:
                out.append(j.advance(system_now_us=step[1]))
        out.append(j.eof())
    finally:
        j.close()
        ctx.close()
    return out


def merge(outs, world, offsets):
    """Every rank's JoinWindowRows of one call as one world-1 JoinWindowRows: the down, meta and late columns
    concatenated and each stably sorted by key string, late rows renamed to rows of the rank-major concatenation
    (offsets[r] rows come before rank r's), the released handles sorted.  Checks that each rank returned only keys it
    owns."""
    from bytewax_b200 import gpu

    for r, o in enumerate(outs):
        keys = np.unique(np.concatenate([o.down_key, o.meta_key, o.late_key])).tolist()
        assert all(po.dest_rank(k, world) == r for k in keys), r
        assert o.late_rank.size == o.late_key.size and (o.late_rank < world).all()  # the source rank, not the owner

    def cat(name):
        return np.concatenate([getattr(o, name) for o in outs])

    dk, mk, lk = cat("down_key"), cat("meta_key"), cat("late_key")
    do, mo, lo = (np.argsort(k.astype(str), kind="stable") for k in (dk, mk, lk))
    rank, row = cat("late_rank"), cat("late_row")
    base = np.array(offsets or [0] * world, np.uint64)[rank.astype(np.int64)]
    return gpu.JoinWindowRows(dk[do], cat("down_window_id")[do], cat("down_handles")[do], cat("down_mask")[do], cat("down_epoch")[do],
                              mk[mo], cat("meta_window_id")[mo], cat("meta_epoch")[mo], lk[lo], cat("late_window_id")[lo],
                              cat("late_epoch")[lo], cat("late_activation")[lo], (base + row)[lo], np.zeros(lk.size, np.uint64),
                              np.sort(cat("released")))


def merged_calls(results, world, cat, parts):
    """Per call (each step of the rank-major concatenation `cat`, then EOF): the merged JoinWindowRows."""
    out = []
    for i in range(len(cat) + 1):
        offsets = None
        if i < len(cat) and cat[i][0] == "batch":
            sizes = [len(p) for p in parts[i]]
            offsets = [sum(sizes[:r]) for r in range(world)]
        m = merge([results[r][i] for r in range(world)], world, offsets)
        if offsets is None:
            assert m.late_key.size == 0
        out.append(m)
    return out


def ref_rows(spec, cat, merged):
    """The merged calls as the reference's row lists (tests/test_gpu_join_window._rows), and their released handles."""
    bounds = lambda w: (spec["align_us"] + spec["offset_us"] * w, spec["align_us"] + spec["offset_us"] * w + spec["length_us"])  # noqa: E731
    final = spec["emit_mode"] == "final"
    rows, rel, n_act = [], [], 0
    for i, m in enumerate(merged):
        step = cat[i] if i < len(cat) else None
        if step is not None and step[0] == "batch":
            rows.append(_rows(m, bounds, dict(act=n_act, sides=step[4], vals=step[5], final=final)))
            n_act += 1
        else:
            rows.append(_rows(m, bounds, dict(act=None, final=final)))
        rel.append(m.released.tolist())
    return rows, rel


def same_rows(a, b):
    """Two JoinWindowRows equal column for column (the down handles of the sides that are set), releases as sets."""
    for c in ("down_key", "down_window_id", "down_mask", "down_epoch", "meta_key", "meta_window_id", "meta_epoch", "late_key",
              "late_window_id", "late_epoch", "late_activation", "late_row"):
        assert np.array_equal(getattr(a, c), getattr(b, c)), c
    assert a.tuples() == b.tuples()
    assert sorted(a.released.tolist()) == sorted(b.released.tolist())


def check_handles(results, world, steps):
    """Every input handle is released exactly once over all ranks and calls, by the owner of its key."""
    key_of = {int(v): int(k) for st in steps if st[0] == "batch" for k, v in zip(st[2], st[5])}
    seen = []
    for r in range(world):
        for o in results[r]:
            hs = o.released.tolist()
            assert all(po.dest_rank(key_of[h], world) == r for h in hs), r
            seen += hs
    assert sorted(seen) == sorted(key_of)


def check_world(world, spec, steps, how, seed, want_rows=None, want_digest=None, device=False, **kw):
    """One stream under one split at one world size, against the oracle (or the goldens, when the concatenation is the
    stream itself) and a world-1 join of the concatenation."""
    parts, cat = plan(steps, world, _split(how, world, seed))
    results = run_world(world, spec, steps, parts, device=device, **kw)
    got = merged_calls(results, world, cat, parts)
    rows, rel = ref_rows(spec, cat, got)
    oracle_rows, oracle_rel = jo.run_join_window(spec, cat)
    if cat == steps and want_rows is not None:
        assert rows == want_rows, (world, how)
    if cat == steps and want_digest is not None:
        assert [len(a) for a in rows] == want_digest["rows"] and rows_digest(rows) == want_digest["sha256"], (world, how)
    assert rows == oracle_rows, (world, how)
    assert rel == oracle_rel, (world, how)
    one = run_one(spec, cat, **kw)
    assert len(one) == len(got)
    for m, o in zip(got, one):
        assert (o.late_rank == 0).all()
        same_rows(m, o)
    check_handles(results, world, steps)
    return got


# ---- the reference's rows ---------------------------------------------------------------------------------------------


@pytest.mark.parametrize("how", SPLITS)
@pytest.mark.parametrize("name", sorted(GOLDEN["cases"]))
def test_golden_case_ranks(name, how):
    case = GOLDEN["cases"][name]
    for world in WORLDS:
        for seed in range(3 if how == "contiguous" else 1):  # each batch of the case meets each kind of contiguous cut
            check_world(world, case["spec"], case["steps"], how, seed, want_rows=case["acts"], max_batch_rows=64, **SMALL)


@pytest.mark.parametrize("seed", list(jo.SEEDED))
def test_seeded_digests_ranks(seed):
    """Every seeded spec (insert and emit modes, 1-4 sides, ordered or not, tumbling or sliding, a moving clock with
    notify steps) under every kind of split, at a world size that cycles with the seed."""
    spec, steps = jo.seeded_steps(seed, moving=seed % 3 != 0)
    world = WORLDS[seed % 3]
    for how in SPLITS:
        check_world(world, spec, steps, how, seed, want_digest=GOLDEN["seeded"][f"seed_{seed}"], max_batch_rows=32, **SMALL)


def _big_stream(seed, n_act, rows, n_keys, sides, moving=True):
    rnd = np.random.default_rng(seed)
    steps, base, now, nxt = [], A, A + 100 * S, 0
    for b in range(n_act):
        keys = rnd.integers(0, n_keys, rows).astype(np.uint64)
        keys[rnd.random(rows) < 0.002] = SENTINEL
        keys[rnd.random(rows) < 0.002] = 0
        ts = base + rnd.integers(-4 * S, 4 * S, rows) - np.where(rnd.random(rows) < 0.05, rnd.integers(5 * S, 30 * S, rows), 0)
        if moving:
            now += int(rnd.integers(0, 2 * S))
        steps.append(["batch", now, keys.tolist(), ts.tolist(), rnd.integers(0, sides, rows).tolist(), list(range(nxt, nxt + rows))])
        nxt += rows
        if moving and b % 2:
            now += 3 * S
            steps.append(["notify", now])
        base += 3 * S
    return steps


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("how", ["interleaved", "random"])
@pytest.mark.parametrize("ins,emit,ordered,sliding", [("first", "complete", True, False), ("last", "final", False, True),
                                                      ("last", "running", True, True), ("first", "final", True, False)])
def test_larger_streams(device, world, how, ins, emit, ordered, sliding):
    """Four activations of 3000 rows over 500 keys, with notify steps, host or device columns: merged rows == the
    oracle == a world-1 JoinWindow over the rank-major concatenation; every handle released once, on its key's owner."""
    spec = dict(insert_mode=ins, emit_mode=emit, ordered=ordered, sides=3, length_us=4 * S, offset_us=2 * S if sliding else 4 * S,
                align_us=A + 123_457, wait_us=S)
    steps = _big_stream(world * 10 + len(ins + emit), 4, 3000, 500, 3)
    got = check_world(world, spec, steps, how, 1, device=device, capacity_hint=1 << 12, max_batch_rows=3000, max_queued_rows=1 << 15,
                      max_emit_rows=1 << 15, max_late_rows=1 << 14)
    assert sum(m.late_key.size for m in got) > 200 and sum(m.down_key.size + m.meta_key.size for m in got) > 500


def test_late_rows_name_their_source():
    """Late rows, one per rank, named (activation, rank, row in that rank's columns)."""
    world = 3
    spec = dict(insert_mode="last", emit_mode="final", ordered=False, sides=1, length_us=S, offset_us=S, align_us=A, wait_us=0)
    keys = [1, 2, 3, 4, 5, 6]
    first = ["batch", A + 60 * S, keys, [A + 50 * S] * 6, [0] * 6, list(range(6))]  # every key's watermark reaches A + 50 s
    # rank r holds rows [2r, 2r + 1] of the second batch: the second row of each rank is late
    second = ["batch", A + 61 * S, keys, [A + 51 * S, A, A + 52 * S, A + S, A + 53 * S, A + 2 * S], [0] * 6, list(range(6, 12))]
    steps = [first, second]
    parts, _ = plan(steps, world, lambda i, n: [np.arange(2 * r, 2 * r + 2) for r in range(world)])
    results = run_world(world, spec, steps, parts, max_batch_rows=8)
    late = sorted((k, int(a), int(rk), int(rw)) for o in (results[r][1] for r in range(world))
                  for k, a, rk, rw in zip(o.late_key.tolist(), o.late_activation, o.late_rank, o.late_row))
    assert late == [(2, 1, 0, 1), (4, 1, 1, 1), (6, 1, 2, 1)]
    one = run_one(spec, steps, max_batch_rows=8)[1]
    assert sorted(zip(one.late_key.tolist(), one.late_row.tolist())) == [(2, 1), (4, 3), (6, 5)]
    assert (one.late_rank == 0).all()


def test_world_one_late_rank_is_zero():
    """On one GPU late_rank is all zeros, for K8 and for K14 (bw_pjwin_*, which shares the rows struct)."""
    from bytewax_b200 import gpu

    spec = dict(insert_mode="first", emit_mode="final", ordered=True, sides=2, length_us=4 * S, offset_us=2 * S, align_us=A, wait_us=S)
    steps = _big_stream(3, 4, 3000, 200, 2)
    lates = [m.late_key.size for m in run_one(spec, steps, max_batch_rows=4096)]
    assert sum(lates) > 100
    ctx = gpu.Context(0)
    j = gpu.ProductJoinWindow(ctx, "final", True, 2, 4 * S, 2 * S, A, S, capacity_hint=1 << 10, max_batch_rows=4096)
    try:
        n = 0
        for i, step in enumerate(steps):
            if step[0] == "batch":
                j.apply(*_cols(step), epoch=i + 1, system_now_us=step[1])
                out = j.advance()
            else:
                out = j.advance(system_now_us=step[1])
            assert out.late_rank.size == out.late_key.size and (out.late_rank == 0).all()
            n += out.late_key.size
        assert n > 100
    finally:
        j.close()
        ctx.close()


@pytest.mark.parametrize("ordered", [False, True])
def test_scale_four_ranks(ordered):
    """2^20 rows per rank over 10^5 keys at W = 4, against a world-1 join of the concatenation, column for column, and
    every handle released once over the ranks, on its key's owner."""
    world, rows, n_keys = 4, 1 << 20, 100_000
    spec = dict(insert_mode="last", emit_mode="final", ordered=ordered, sides=2, length_us=4 * S, offset_us=4 * S, align_us=A, wait_us=S)
    rnd = np.random.default_rng(20)
    steps = []
    for a in range(2):  # 10 s of event time each, 20 s apart
        n = rows * world
        keys = rnd.integers(0, n_keys, n).astype(np.uint64)
        ts = A + a * 20 * S + np.arange(n, dtype=np.int64) * (10 * S) // n + rnd.integers(-S, S + 1, n)
        steps.append(["batch", A + 100 * S, keys, ts, rnd.integers(0, 2, n).astype(np.uint8), np.arange(a * n, (a + 1) * n, dtype=np.uint64)])
    kw = dict(capacity_hint=n_keys, max_emit_rows=1 << 20, max_late_rows=1 << 21, max_queued_rows=1 << 23, max_windows_per_key=16)

    def cols(step, sl=slice(None)):
        return step[2][sl], step[4][sl], step[5][sl], step[3][sl]

    def body(r, ctx, keep):
        j = _join(ctx, spec, max_batch_rows=rows, **kw)
        keep.append(j)
        out = []
        for a, step in enumerate(steps):
            j.apply(*cols(step, slice(r * rows, (r + 1) * rows)), epoch=a + 1, system_now_us=step[1])
            out.append(j.advance())
        out.append(j.eof())
        return out

    results, errors = run_ranks(world, body)
    no_errors(errors)
    from bytewax_b200 import gpu

    ctx = gpu.Context(0)
    j = _join(ctx, spec, shard=False, max_batch_rows=rows * world, **kw)
    one = []
    for a, step in enumerate(steps):
        j.apply(*cols(step), epoch=a + 1, system_now_us=step[1])
        one.append(j.advance())
    one.append(j.eof())
    j.close()
    ctx.close()
    down = late = 0
    for i in range(len(steps) + 1):
        m = merge([results[r][i] for r in range(world)], world, [r * rows for r in range(world)] if i < len(steps) else None)
        same_rows(m, one[i])
        down, late = down + m.down_key.size, late + m.late_key.size
    assert down > n_keys and late > 1000
    key_of = np.concatenate([s[2] for s in steps]).astype(np.int64)  # handle h is row h of the stream
    owner_of = np.array([po.dest_rank(k, world) for k in range(n_keys)])
    seen = []
    for r in range(world):
        for o in results[r]:
            hs = o.released.astype(np.int64)
            assert (owner_of[key_of[hs]] == r).all(), r
            seen.append(hs)
    assert np.array_equal(np.sort(np.concatenate(seen)), np.arange(key_of.size))


# ---- errors: every rank returns, none waits out a barrier -----------------------------------------------------------


SPEC0 = dict(insert_mode="last", emit_mode="running", ordered=True, sides=2, length_us=4 * S, offset_us=2 * S, align_us=A, wait_us=S)


@pytest.mark.parametrize("what", ["epoch", "now"])
def test_ranks_disagree(what):
    """Ranks that pass different epochs, or different system times, to one call: BW_ERR_STATE on every rank."""
    world = 3

    def body(r, ctx, keep):
        j = _join(ctx, SPEC0, capacity_hint=64, max_batch_rows=64)
        keep.append(j)
        j.apply(np.array([r, r + 1], np.uint64), np.zeros(2, np.uint8), np.array([2 * r, 2 * r + 1], np.uint64), np.array([A, A], np.int64),
                epoch=5, system_now_us=A)
        epoch, now = (6 if r == 2 else 7, A) if what == "epoch" else (6, A + (r == 1))
        j.apply(np.array([r], np.uint64), np.zeros(1, np.uint8), np.array([10 + r], np.uint64), np.array([A], np.int64), epoch=epoch,
                system_now_us=now)
        return "no error"

    results, errors = _errors_fast(world, body)
    assert [_status(e) for e in errors] == [STATE] * world, (results, errors)


@pytest.mark.parametrize("bad", [0, 1, 2])
@pytest.mark.parametrize("what", ["rows", "null", "side", "decreasing"])
def test_refused_call_plays_nothing(what, bad):
    """One rank's call cannot go ahead (too many rows, a NULL column, a host side >= sides, a decreasing epoch): that
    rank gets its own error, every other rank BW_ERR_STATE, no rank plays the call, and the join goes on as if it had
    not been made."""
    world, B = 3, 16
    spec = dict(SPEC0, emit_mode="final")
    steps = _big_stream(5, 3, 30, 20, 2)
    parts, cat = plan(steps, world, interleaved(world))

    def body(r, ctx, keep):
        j = _join(ctx, spec, max_batch_rows=B)
        keep.append(j)
        out, err = [], None
        for i, step in enumerate(steps):
            if i == 1:  # the refused call, between two good ones
                try:
                    if r == bad and what == "rows":
                        j.apply(np.zeros(B + 1, np.uint64), np.zeros(B + 1, np.uint8), np.arange(B + 1) + 10**6, np.full(B + 1, A, np.int64),
                                epoch=2, system_now_us=step[1])
                    elif r == bad and what == "null":
                        j.apply_device(0, 0, 0, 0, 4, epoch=2, system_now_us=step[1])
                    elif r == bad and what == "side":
                        k, s, h, t = _cols(step, parts[i][r])
                        j.apply(k, np.full(k.size, 2, np.uint8), h + 10**6, t, epoch=2, system_now_us=step[1])
                    else:
                        k, s, h, t = _cols(step, parts[i][r])
                        j.apply(k, s, h + 10**6, t, epoch=0 if (r == bad and what == "decreasing") else 2, system_now_us=step[1])
                except N.BwError as ex:
                    err = ex.status
                out.append(j.advance())
            if step[0] == "batch":
                j.apply(*_cols(step, parts[i][r]), epoch=i + 1, system_now_us=step[1])
                out.append(j.advance())
            else:
                out.append(j.advance(system_now_us=step[1]))
        out.append(j.eof())
        return err, out

    results, errors = _errors_fast(world, body)
    no_errors(errors)
    want_bad = STATE if what == "decreasing" else SPEC
    assert [e for e, _ in results] == [STATE if r != bad else want_bad for r in range(world)]
    assert all(o.down_key.size == 0 and o.late_key.size == 0 and o.released.size == 0 for _, out in results for o in [out[1]])
    outs = [[o for k, o in enumerate(out) if k != 1] for _, out in results]
    rows, rel = ref_rows(spec, cat, merged_calls(outs, world, cat, parts))
    assert (rows, rel) == jo.run_join_window(spec, cat)
    check_handles(outs, world, steps)


def _full(what, owner, world):
    """The spec, per-rank arguments and rows of one call that overfills `what` on rank `owner`."""
    base = dict(insert_mode="last", emit_mode="final", ordered=False, sides=2, length_us=10 * S, offset_us=10 * S, align_us=A, wait_us=0)
    if what == "key table":  # 1024 slots at capacity_hint 16, and one more key (2^64-1 has its own slot)
        keys, ts, kw = _owned_by(owner, world, 1025, start=10), [A] * 1025, dict(capacity_hint=16)
    elif what == "window list":  # each item opens 3 windows; items 2 s apart need 5, a key may hold 4
        base.update(length_us=6 * S, offset_us=2 * S, wait_us=jo.WAIT_FOREVER)
        keys, ts, kw = _owned_by(owner, world, 1) * 3, [A, A + 2 * S, A + 4 * S], dict(max_windows_per_key=4)
    elif what == "queue":  # nothing is due with wait forever: 11 entries, 10 may queue
        base.update(ordered=True, wait_us=jo.WAIT_FOREVER)
        keys, ts, kw = _owned_by(owner, world, 11), [A] * 11, dict(max_queued_rows=10)
    else:  # emit buffer: 11 running rows, 10 may wait for advance
        base.update(emit_mode="running")
        keys, ts, kw = _owned_by(owner, world, 11), [A + 5 * S] * 11, dict(max_emit_rows=10)
    n = len(keys)
    step = ["batch", A, keys, ts, [i % 2 for i in range(n)], list(range(n))]
    return base, step, kw


OWNERS = [(world, owner) for world in WORLDS for owner in range(world)]


@pytest.mark.parametrize("world,owner", OWNERS)
@pytest.mark.parametrize("what", ["key table", "window list", "queue", "emit buffer"])
def test_owner_capacity(what, world, owner):
    """An owner's key table, a key's window list, the owner's queue or its emit buffer fills up in one call: that rank's
    apply gets BW_ERR_CAPACITY, every other rank goes on; in the next call the owner refuses (its join has failed), so
    every rank gets BW_ERR_STATE."""
    spec, step, kw = _full(what, owner, world)
    parts = [np.arange(r, len(step[2]), world) for r in range(world)]

    def body(r, ctx, keep):
        j = _join(ctx, spec, max_batch_rows=1024, **kw)
        keep.append(j)
        st = []
        for epoch in (1, 2):
            try:
                j.apply(*_cols(step, parts[r] if epoch == 1 else np.zeros(0, np.int64)), epoch=epoch, system_now_us=A)
                st.append(0)
            except N.BwError as ex:
                st.append(ex.status)
        return st

    results, errors = _errors_fast(world, body)
    no_errors(errors)
    assert results == [[CAPACITY, STATE] if r == owner else [0, STATE] for r in range(world)], results


@pytest.mark.parametrize("world,owner", OWNERS)
@pytest.mark.parametrize("what", ["emit buffer", "side"])
def test_owner_device_error(what, world, owner):
    """apply_device: an owner's full emit buffer, or a device side >= sides it received, fails that owner's next call
    (BW_ERR_CAPACITY / BW_ERR_SPEC, found by the call's opening drain); every other rank gets BW_ERR_STATE there, and
    every rank after it."""
    spec, step, kw = _full("emit buffer", owner, world)
    if what == "side":
        step = step[:4] + [[5] + step[4][1:], step[5]]  # row 0, owned by `owner`, sent from rank 0
        kw = {}
    parts = [np.arange(r, len(step[2]), world) for r in range(world)]

    def body(r, ctx, keep):
        j = _join(ctx, spec, max_batch_rows=1024, **kw)
        keep.append(j)
        st = []
        for epoch in (1, 2, 3):
            try:
                _apply(j, _cols(step, parts[r] if epoch == 1 else np.zeros(0, np.int64)), epoch, A, True)
                st.append(0)
            except N.BwError as ex:
                st.append(ex.status)
        return st

    results, errors = _errors_fast(world, body)
    no_errors(errors)
    want = CAPACITY if what == "emit buffer" else SPEC
    assert results == [[0, want, STATE] if r == owner else [0, STATE, STATE] for r in range(world)], results


@pytest.mark.parametrize("world,owner", OWNERS)
def test_owner_late_buffer(world, owner):
    """A sliding join whose owner's late buffer (4 rows) overflows in the middle of a late item's rows, while the slots
    that item would take still hold an earlier call's late rows from rank 1: the owner's apply gets BW_ERR_CAPACITY,
    every other rank goes on, and every rank's next apply gets BW_ERR_STATE.

    Windows of 5 s every 2 s from A: an item at A + k s belongs to 3 windows for even k and 2 for odd k.  Call 1 sets the
    key's watermark to A + 50 s.  Call 2 (rows from rank 1): late items at A + 1 s and A + 3 s, 2 + 2 rows, fill the
    buffer exactly, and the advance hands them out, named by rank 1.  Call 3 (rows from rank 0): late items at A and
    A + 1 s want 3 + 2 rows; the second does not fit, so slot 3 is not written this call."""
    spec = dict(insert_mode="last", emit_mode="final", ordered=False, sides=2, length_us=5 * S, offset_us=2 * S, align_us=A, wait_us=0)
    key = _owned_by(owner, world, 1)[0]
    calls = [(0, [A + 50 * S]), (1, [A + S, A + 3 * S]), (0, [A, A + S]), (0, [])]  # (the rank that sends, its rows' ts)

    def body(r, ctx, keep):
        j = _join(ctx, spec, max_batch_rows=16, max_late_rows=4)
        keep.append(j)
        st, late = [], []
        for c, (src, ts) in enumerate(calls):
            n = len(ts) if r == src else 0
            try:
                j.apply(np.full(n, key, np.uint64), np.zeros(n, np.uint8), np.arange(n, dtype=np.uint64) + 10 * c,
                        np.array(ts[:n], np.int64), epoch=c + 1, system_now_us=A)
                st.append(0)
                out = j.advance()
                late.append(sorted(zip(out.late_rank.tolist(), out.late_row.tolist())))
            except N.BwError as ex:
                st.append(ex.status)
        return st, late

    results, errors = _errors_fast(world, body)
    no_errors(errors)
    assert [st for st, _ in results] == [[0, 0, CAPACITY, STATE] if r == owner else [0, 0, 0, STATE] for r in range(world)], results
    assert results[owner][1][1] == [(1, 0), (1, 0), (1, 1), (1, 1)], results[owner][1]


def test_sharding_is_opt_in():
    """Without shard_by_key every rank of a world of 2 gets BW_ERR_SPEC at create, at once (no collective is entered);
    with it every rank creates the join.  On one rank the flag changes nothing."""
    from bytewax_b200 import gpu

    def body(r, ctx, keep):
        with pytest.raises(N.BwError) as ei:
            gpu.JoinWindow(ctx, max_batch_rows=1024, **SMALL)
        assert ei.value.status == SPEC and "one GPU" in str(ei.value)
        keep.append(gpu.JoinWindow(ctx, max_batch_rows=1024, shard_by_key=True, **SMALL))
        return r

    results, errors = _errors_fast(2, body)
    no_errors(errors)
    assert results == [0, 1]
    spec, steps = jo.seeded_steps(7)
    from bytewax_b200 import gpu

    ctx = gpu.Context(0)
    try:
        flagged, plain = _join(ctx, spec, shard=True, **SMALL), _join(ctx, spec, shard=False, **SMALL)
        for i, step in enumerate(steps):
            outs = []
            for j in (flagged, plain):
                if step[0] == "batch":
                    j.apply(*_cols(step), epoch=i + 1, system_now_us=step[1])
                    outs.append(j.advance())
                else:
                    outs.append(j.advance(system_now_us=step[1]))
            same_rows(*outs)
        same_rows(flagged.eof(), plain.eof())
        flagged.close()
        plain.close()
    finally:
        ctx.close()


def _raw_spec(size, shard):
    s = N.BwJwinSpec()
    s.struct_size = size
    s.insert_mode, s.emit_mode, s.ordered, s.sides, s.max_windows_per_key = 1, 1, 1, 2, 4
    s.length_us, s.offset_us, s.align_us = S, S, A
    s.capacity_hint, s.max_queued_rows, s.max_batch_rows, s.max_emit_rows, s.max_late_rows = 64, 64, 64, 64, 64
    s.shard_by_key = shard
    return s


def test_spec_without_shard_field():
    """A spec whose struct_size ends before shard_by_key (built against the header without it) reads the flag as 0: it
    creates a world-1 join, and on a world of 2 it is refused even though the memory past it holds 1.  A spec of any
    other size is BW_ERR_SPEC."""
    from bytewax_b200 import gpu

    short = N.BwJwinSpec.shard_by_key.offset
    ctx = gpu.Context(0)
    try:
        for size, ok in ((short, True), (C.sizeof(N.BwJwinSpec), True), (C.sizeof(N.BwJwinSpec) - 4, False)):
            h = C.c_void_p()
            st = ctx.lib.bw_jwin_create(ctx.h, C.byref(_raw_spec(size, 1)), C.byref(h))
            assert (st == 0) == ok, size
            if st == 0:
                ctx.lib.bw_jwin_destroy(h)
    finally:
        ctx.close()

    def body(r, ctx, keep):
        h = C.c_void_p()
        return ctx.lib.bw_jwin_create(ctx.h, C.byref(_raw_spec(short, 1)), C.byref(h))

    results, errors = _errors_fast(2, body)
    no_errors(errors)
    assert results == [SPEC, SPEC]


@pytest.mark.parametrize("world,rows", [(2, 1 << 30), (3, 715_827_883), (4, 1 << 29), (8, 1 << 28)])
def test_batch_limit(world, rows):
    """max_batch_rows x world reaching 2^31 is BW_ERR_SPEC at create, on every rank."""
    assert rows * world >= 2**31 and (rows - 1) * world < 2**31

    def body(r, ctx, keep):
        keep.append(_join(ctx, SPEC0, max_batch_rows=rows))

    _, errors = _errors_fast(world, body)
    assert [_status(e) for e in errors] == [SPEC] * world, errors


@pytest.mark.parametrize("world", WORLDS)
def test_queue_limit(world):
    """max_queued_rows + world x max_batch_rows reaching 2^31 is BW_ERR_SPEC at create, on every rank, though
    max_queued_rows + max_batch_rows stays below it."""
    rows = 1 << 24
    queued = 2**31 - world * rows
    assert queued + rows < 2**31

    def body(r, ctx, keep):
        keep.append(_join(ctx, SPEC0, max_batch_rows=rows, max_queued_rows=queued))

    _, errors = _errors_fast(world, body)
    assert [_status(e) for e in errors] == [SPEC] * world, errors
    assert all("max_queued_rows" in str(e) for e in errors)


def test_memory_returned_on_destroy():
    """Create, use and destroy a W = 2 join three times: device memory comes back (regions, mappings, scratch, pools)."""
    spec = dict(SPEC0, emit_mode="final")
    steps = _big_stream(3, 3, 2000, 300, 2)
    parts, _ = plan(steps, 2, interleaved(2))

    def cycle():
        run_world(2, spec, steps, parts, capacity_hint=1 << 14, max_batch_rows=1 << 16, max_queued_rows=1 << 17, max_windows_per_key=16)

    cycle()  # warm the allocator's pools
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        cycle()
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < (64 << 20)
