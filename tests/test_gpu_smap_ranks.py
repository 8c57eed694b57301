"""K5, the z-score `stateful_map`, sharded by key over W ranks: threads of one process on a loopback world (include/bwgpu.h,
bw_loopback_create), whose partition kernels, peer stores into the owners' receive regions and return sections, and
barriers are the ones an NCCL world runs.  -m gpu.

Each rank applies its own rows per call; each row goes to rank `po.dest_rank(key, W)`, which maps what arrived in
(source rank, source order) and stores each row's mu, sigma and flag back at the row's index on its source rank.  Every
rank's outputs of one call, concatenated rank-major, must equal bit for bit what a world-1 `ZScoreMap` and the correctly
rounded twin of the reference mapper (`po.run_zscore(..., correctly_rounded=True)`) return for the rank-major
concatenation of every rank's rows."""

import ctypes as C

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle import pyoracle as po  # checker only
from tests.test_gpu_join_ranks import no_errors, run_ranks
from tests.test_gpu_lifecycle import check_no_growth
from tests.test_gpu_session_ranks import _errors_fast, _owned_by, _status, contiguous, interleaved, random_split

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")  # before libbwgpu: torch loads its own NCCL first
CAPACITY, SPEC, STATE = 3, 4, 5  # BW_ERR_CAPACITY, BW_ERR_SPEC, BW_ERR_STATE
SENTINEL = 2**64 - 1  # the key table's empty marker; the key itself lives in the alias slot `cap`
WORLDS = [2, 3, 4]
THRESHOLD = 2.0


def _np_val(dtype):
    return np.float32 if dtype == "f32" else np.float64


def _map(ctx, window, dtype, **kw):
    from bytewax_b200 import gpu

    return gpu.ZScoreMap(ctx, window, THRESHOLD, dtype, shard_by_key=True, **kw)


def stream(seed, n_acts, rows, n_keys, dtype, edge=False):
    """Zipf keys over 1..n_keys (a few hot keys whose rings carry across calls, many cold ones), values mixing small
    integers (sigma 0, exact means) and spread floats (flags)."""
    rnd = np.random.default_rng(seed)
    out = []
    for _ in range(n_acts):
        keys = np.minimum(rnd.zipf(1.3, rows), n_keys).astype(np.uint64)
        if edge:
            keys[rnd.random(rows) < 0.02] = 0
            keys[rnd.random(rows) < 0.02] = SENTINEL
        vals = np.where(rnd.random(rows) < 0.3, rnd.integers(-3, 4, rows), rnd.normal(0.0, 10.0, rows))
        out.append((keys, vals.astype(_np_val(dtype))))
    return out


def plan(batches, world, split):
    """Per activation: the per-rank index arrays, and the rank-major concatenation's (keys, vals)."""
    parts, cat = [], []
    for a, (k, v) in enumerate(batches):
        p = split(a, len(k))
        order = np.concatenate(p).astype(np.int64)
        assert sorted(order.tolist()) == list(range(len(k)))
        parts.append(p)
        cat.append((k[order], v[order]))
    return parts, cat


def run_world(world, batches, parts, window, dtype, **kw):
    """Every rank applies its slice of every activation.  Per rank, per activation: (mu, sigma, flag)."""

    def body(r, ctx, keep):
        m = _map(ctx, window, dtype, **kw)
        keep.append(m)
        return [m.apply(k[parts[a][r]], v[parts[a][r]]) for a, (k, v) in enumerate(batches)]

    results, errors = run_ranks(world, body)
    no_errors(errors)
    return results


def merged(results, world, a):
    return tuple(np.concatenate([results[r][a][c] for r in range(world)]) for c in range(3))


def run_one(cat, window, dtype, **kw):
    """A world-1 map over the activations `cat`."""
    from bytewax_b200 import gpu

    ctx = gpu.Context(0)
    m = gpu.ZScoreMap(ctx, window, THRESHOLD, dtype, max_batch_rows=max(len(k) for k, _ in cat) + 1, **kw)
    try:
        return [m.apply(k, v) for k, v in cat]
    finally:
        m.close()
        ctx.close()


def twin(cat, window):
    out = []
    for rows in po.run_zscore([(k.tolist(), v.astype(np.float64).tolist()) for k, v in cat], window, THRESHOLD, correctly_rounded=True):
        out.append(tuple(np.array([row[c] for row in rows], dtype=bool if c == 2 else np.float64) for c in range(3)))
    return out


def same(got, want, what=""):
    for c, name in enumerate(("mu", "sigma")):
        g, w = np.asarray(got[c], np.float64), np.asarray(want[c], np.float64)
        bad = np.flatnonzero(g.view(np.uint64) != w.view(np.uint64))
        assert bad.size == 0, (what, name, bad[:4].tolist(), g[bad[:4]].tolist(), w[bad[:4]].tolist())
    assert np.array_equal(np.asarray(got[2], bool), np.asarray(want[2], bool)), (what, "flag")


def check_world(world, batches, parts, cat, window, dtype, **kw):
    results = run_world(world, batches, parts, window, dtype, **kw)
    one, tw = run_one(cat, window, dtype), twin(cat, window)
    for a in range(len(batches)):
        for r in range(world):
            assert results[r][a][0].size == len(parts[a][r])
        got = merged(results, world, a)
        same(got, one[a], ("world 1", a))
        same(got, tw[a], ("twin", a))
    return results


def one_rank(world):
    """Every row of every activation on the last rank; the others pass none."""
    return lambda a, n: [np.arange(0) for _ in range(world - 1)] + [np.arange(n)]


SPLITS = {"contiguous": lambda w, seed: contiguous(w, seed), "interleaved": lambda w, seed: interleaved(w),
          "random": lambda w, seed: random_split(w, seed), "one_rank": lambda w, seed: one_rank(w)}


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("how", sorted(SPLITS))
@pytest.mark.parametrize("dtype,window", [("f32", 10), ("f64", 1), ("f64", 10), ("f32", 32), ("f64", 32)])
def test_matches_one_rank_and_twin(world, how, dtype, window):
    """Several activations (rings carry across calls); contiguous splits cycle through even cuts, every row on one
    rank and cuts that leave ranks empty."""
    seed = 11 * world + window
    batches = stream(seed, 4, 3000, 400, dtype)
    parts, cat = plan(batches, world, SPLITS[how](world, seed))
    check_world(world, batches, parts, cat, window, dtype, capacity_hint=512, max_batch_rows=3000)


def test_edge_keys_on_different_owners():
    """Keys 0 and 2^64-1 (the alias slot) land on different owners at W = 2 and map like any other key."""
    world = 2
    assert po.dest_rank(0, world) != po.dest_rank(SENTINEL, world)
    batches = stream(3, 3, 2000, 100, "f64", edge=True)
    parts, cat = plan(batches, world, random_split(world, 3))
    check_world(world, batches, parts, cat, 10, "f64", capacity_hint=128, max_batch_rows=2000)
    assert all((k == 0).sum() > 10 and (k == SENTINEL).sum() > 10 for k, _ in batches)


@pytest.mark.parametrize("dtype", ["f32", "f64"])
def test_apply_device_matches_apply(dtype):
    """apply_device (device columns in and out) gives the results apply gives, on every rank."""
    world, window = 3, 10
    batches = stream(9, 3, 2500, 300, dtype)
    parts, _ = plan(batches, world, random_split(world, 9))
    want = run_world(world, batches, parts, window, dtype, capacity_hint=512, max_batch_rows=2500)
    dev = "cuda:0"

    def body(r, ctx, keep):
        m = _map(ctx, window, dtype, capacity_hint=512, max_batch_rows=2500)
        keep.append(m)
        out = []
        for a, (k, v) in enumerate(batches):
            idx = parts[a][r]
            n = len(idx)
            dk = torch.from_numpy(np.ascontiguousarray(k[idx]).view(np.int64)).to(dev)
            dv = torch.from_numpy(np.ascontiguousarray(v[idx])).to(dev)
            mu = torch.empty(n, dtype=torch.float64, device=dev)
            sg = torch.empty(n, dtype=torch.float64, device=dev)
            fl = torch.empty(n, dtype=torch.uint8, device=dev)
            torch.cuda.synchronize()
            m.apply_device(dk.data_ptr(), dv.data_ptr(), n, mu.data_ptr(), sg.data_ptr(), fl.data_ptr())
            m.sync()
            out.append((mu.cpu().numpy(), sg.cpu().numpy(), fl.cpu().numpy().astype(bool)))
        return out

    results, errors = run_ranks(world, body)
    no_errors(errors)
    for r in range(world):
        for a in range(len(batches)):
            same(results[r][a], want[r][a], (r, a))


# ---- errors: every rank returns, none waits out a barrier -----------------------------------------------------------


@pytest.mark.parametrize("what", ["rows", "null"])
def test_refused_call_maps_nothing(what):
    """One rank's call cannot go ahead (too many rows, a NULL column), each rank in turn: that rank gets BW_ERR_SPEC,
    every other rank BW_ERR_STATE, no rank maps the call, and the map goes on as if it had not been made."""
    world, B, window = 3, 64, 4
    batches = stream(5, 3, 150, 20, "f64")
    parts, cat = plan(batches, world, interleaved(world))
    want = run_one(cat, window, "f64")
    for bad in range(world):

        def body(r, ctx, keep):
            m = _map(ctx, window, "f64", capacity_hint=64, max_batch_rows=B)
            keep.append(m)
            out, err = [], None
            for a, (k, v) in enumerate(batches):
                if a == 1:  # the refused call, between two good ones
                    try:
                        if r == bad and what == "rows":
                            m.apply(np.zeros(B + 1, np.uint64), np.zeros(B + 1, np.float64))
                        elif r == bad:
                            m.apply_device(0, 0, 4, 0, 0, 0)
                        else:
                            m.apply(k[parts[a][r]], v[parts[a][r]])
                    except N.BwError as ex:
                        err = ex.status
                out.append(m.apply(k[parts[a][r]], v[parts[a][r]]))
            return err, out

        results, errors = _errors_fast(world, body)
        no_errors(errors)
        assert [e for e, _ in results] == [SPEC if r == bad else STATE for r in range(world)], bad
        outs = [out for _, out in results]
        for a in range(len(batches)):
            same(merged(outs, world, a), want[a], (bad, a))


def test_owner_capacity():
    """An owner's key table (1024 slots at capacity_hint 16) fills up: the call fails on every rank, the owner with
    BW_ERR_CAPACITY and the other with BW_ERR_STATE; every later call, with rows or without, is BW_ERR_STATE on every rank,
    and sync re-reports."""
    world, owner = 2, 0
    keys = np.array(_owned_by(owner, world, 1025, start=10), np.uint64)  # one more than the table holds
    parts = [np.arange(r, len(keys), world) for r in range(world)]

    def body(r, ctx, keep):
        m = _map(ctx, 4, "f64", capacity_hint=16, max_batch_rows=1024)
        keep.append(m)
        st = []
        for idx in (parts[r], parts[r][:5], parts[r][:0]):
            try:
                m.apply(keys[idx], np.ones(len(idx)))
                st.append(0)
            except N.BwError as ex:
                st.append(ex.status)
        try:
            m.sync()
            st.append(0)
        except N.BwError as ex:
            st.append(ex.status)
        return st

    results, errors = _errors_fast(world, body)
    no_errors(errors)
    assert results[owner] == [CAPACITY, STATE, STATE, CAPACITY], results
    assert results[1 - owner] == [STATE, STATE, STATE, STATE], results


# ---- the opt-in ------------------------------------------------------------------------------------------------------


def _shared_key_batches(world):
    """Per rank, activations over the same 30 keys: a rank-local map and a sharded one give different results."""
    return [stream(40 + r, 3, 400, 30, "f64") for r in range(world)]


def test_without_flag_each_rank_is_local():
    """Without shard_by_key a map on a world of 2 is rank-local: each rank equals a world-1 map over its own rows."""
    from bytewax_b200 import gpu

    world, window = 2, 10
    per_rank = _shared_key_batches(world)

    def body(r, ctx, keep):
        m = gpu.ZScoreMap(ctx, window, THRESHOLD, "f64", capacity_hint=64, max_batch_rows=400)
        keep.append(m)
        return [m.apply(k, v) for k, v in per_rank[r]]

    results, errors = _errors_fast(world, body)
    no_errors(errors)
    for r in range(world):
        for a, (got, one, tw) in enumerate(zip(results[r], run_one(per_rank[r], window, "f64"), twin(per_rank[r], window))):
            same(got, one, (r, a))
            same(got, tw, (r, a))
    cat = [tuple(np.concatenate([per_rank[r][a][c] for r in range(world)]) for c in range(2)) for a in range(3)]
    sharded = twin(cat, window)
    assert any(not np.array_equal(merged(results, world, a)[0], sharded[a][0]) for a in range(3))


def test_short_spec_reads_flag_as_zero():
    """A spec whose struct_size ends before shard_by_key (built against the header without it) creates a rank-local map
    on a world of 2 whatever the bytes after it hold; a spec of any other size is BW_ERR_SPEC."""
    world, window = 2, 10
    per_rank = _shared_key_batches(world)

    def body(r, ctx, keep):
        lib = ctx.lib
        s = N.BwSmapSpec()
        s.window, s.val_dtype, s.threshold, s.capacity_hint, s.max_batch_rows = window, N.VAL["f64"], THRESHOLD, 64, 400
        s.shard_by_key = 1
        s.struct_size = C.sizeof(N.BwSmapSpec) - 4
        h = C.c_void_p()
        assert lib.bw_smap_create(ctx.h, C.byref(s), C.byref(h)) == SPEC
        s.struct_size = N.BwSmapSpec.shard_by_key.offset
        assert lib.bw_smap_create(ctx.h, C.byref(s), C.byref(h)) == 0
        out = []
        try:
            for k, v in per_rank[r]:
                n = len(k)
                mu, sg, fl = np.empty(n), np.empty(n), np.empty(n, np.uint8)
                vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
                N.check(lib.bw_smap_apply(h, vp(k), vp(v), n, vp(mu), vp(sg), vp(fl)), ctx.h)
                out.append((mu, sg, fl.astype(bool)))
        finally:
            lib.bw_smap_destroy(h)
        return out

    results, errors = _errors_fast(world, body)
    no_errors(errors)
    for r in range(world):
        for a, (got, tw) in enumerate(zip(results[r], twin(per_rank[r], window))):
            same(got, tw, (r, a))


@pytest.mark.parametrize("world,rows", [(2, 1 << 30), (3, 715_827_883), (4, 1 << 29), (8, 1 << 28)])
def test_batch_limit(world, rows):
    """max_batch_rows x world reaching 2^31 is BW_ERR_SPEC at create, on every rank, before any collective."""
    assert rows * world >= 2**31 and (rows - 1) * world < 2**31

    def body(r, ctx, keep):
        keep.append(_map(ctx, 10, "f32", max_batch_rows=rows))

    _, errors = _errors_fast(world, body)
    assert [_status(e) for e in errors] == [SPEC] * world, errors


# ---- scale and memory -------------------------------------------------------------------------------------------------


def test_scale_c2_shape_four_ranks():
    """The C2 shape (Zipf-1.1 keys over 1e5 values, f32, window 10) at 2^20 rows per rank and W = 4, two activations,
    against a world-1 map of the concatenation, bit for bit."""
    world, rows, n_keys, window = 4, 1 << 20, 100_000, 10
    rnd = np.random.default_rng(2)
    batches = [(np.minimum(rnd.zipf(1.1, rows * world), n_keys).astype(np.uint64), rnd.normal(0.0, 1.0, rows * world).astype(np.float32))
               for _ in range(2)]
    parts = [[np.arange(r * rows, (r + 1) * rows) for r in range(world)]] * 2
    results = run_world(world, batches, parts, window, "f32", capacity_hint=n_keys, max_batch_rows=rows)
    one = run_one(batches, window, "f32", capacity_hint=n_keys)
    for a in range(2):
        same(merged(results, world, a), one[a], a)
    assert sum(int(o[2].sum()) for o in one) > 1000


def test_memory_returned_on_destroy():
    """Create, use and destroy a W = 2 sharded map: device memory comes back (regions, mappings, scratch)."""
    batches = stream(3, 2, 4000, 500, "f32")
    parts, _ = plan(batches, 2, interleaved(2))
    check_no_growth(lambda: run_world(2, batches, parts, 10, "f32", capacity_hint=1 << 14, max_batch_rows=1 << 16))
