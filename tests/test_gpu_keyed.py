"""K5 (stateful_map z-score detector, config C2) and K6 (keyed join, config C4) against the oracle.  -m gpu."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import pyoracle as po  # noqa: E402  (checker only)


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


def _zipf_keys(n, ranks, seed):
    # inverse-CDF Zipf(1.1) over `ranks` ranks from splitmix64 uniforms (SURVEY.md 8d, config C2)
    w = 1.0 / np.arange(1, ranks + 1) ** 1.1
    cdf = np.cumsum(w) / w.sum()
    u = np.array([po.splitmix64(seed ^ i) / 2.0**64 for i in range(n)])
    return np.searchsorted(cdf, u).astype(np.uint64)


@pytest.mark.parametrize("dtype", ["f32", "f64"])
def test_zscore_map_matches_oracle(ctx, dtype):
    from bytewax_b200 import gpu

    n, nb = 6000, 5
    keys = _zipf_keys(n * nb, 300, 0xC2)
    vals = np.array([po.splitmix64(0xF1 ^ i) % 10 for i in range(n * nb)], dtype=np.float32 if dtype == "f32" else np.float64)
    if dtype == "f64":
        vals = vals + np.array([po.splitmix64(0xAB ^ i) % 1000 for i in range(n * nb)]) / 1000.0
    m = gpu.ZScoreMap(ctx, 10, 2.0, dtype, capacity_hint=1024, max_batch_rows=1 << 14)
    batches = [(keys[b * n:(b + 1) * n], vals[b * n:(b + 1) * n]) for b in range(nb)]
    lists = [(k.tolist(), v.astype(np.float64).tolist()) for k, v in batches]
    want = po.run_zscore(lists)
    twin = po.run_zscore(lists, correctly_rounded=True)  # the device's arithmetic: bit for bit
    near_threshold = 0
    for (k, v), w, t in zip(batches, want, twin):
        mu, sigma, flag = m.apply(k, v)
        tm, ts, tf = (np.array([r[i] for r in t]) for i in range(3))
        assert np.array_equal(mu.view(np.uint64), tm.view(np.uint64))
        assert np.array_equal(sigma.view(np.uint64), ts.view(np.uint64))
        assert np.array_equal(flag, tf)
        # the reference's own arithmetic: the same means, sigma within one ulp (libm pow), the same flags here
        wm = np.array([r[0] for r in w])
        ws = np.array([r[1] for r in w])
        wf = np.array([r[2] for r in w])
        assert np.array_equal(mu.view(np.uint64), wm.view(np.uint64))
        assert (np.abs(sigma - ws) <= np.spacing(sigma)).all()
        diff = np.nonzero(flag != wf)[0]
        near_threshold += len(diff)
    assert near_threshold == 0  # no z within a few ulp of 2 in this set
    m.close()


def test_zscore_single_hot_key_and_sentinel_key(ctx):
    from bytewax_b200 import gpu

    vals = np.array([float(po.splitmix64(i) % 10) for i in range(5000)], dtype=np.float32)
    keys = np.full(5000, 2**64 - 1, dtype=np.uint64)
    m = gpu.ZScoreMap(ctx, 10, 2.0, "f32", capacity_hint=16, max_batch_rows=4096)
    got = []
    for lo in (0, 4096):
        mu, sigma, flag = m.apply(keys[lo:lo + 4096], vals[lo:lo + 4096])
        got += list(zip(mu.tolist(), sigma.tolist(), flag.tolist()))
    want = po.run_zscore([(keys.tolist(), vals.astype(np.float64).tolist())])[0]
    twin = po.run_zscore([(keys.tolist(), vals.astype(np.float64).tolist())], correctly_rounded=True)[0]
    assert [g[2] for g in got] == [w[2] for w in want] == [t[2] for t in twin]
    assert np.array_equal(np.array([g[0] for g in got]).view(np.uint64), np.array([t[0] for t in twin]).view(np.uint64))
    assert np.array_equal(np.array([g[1] for g in got]).view(np.uint64), np.array([t[1] for t in twin]).view(np.uint64))
    assert [g[0] for g in got] == [w[0] for w in want]
    m.close()


@pytest.mark.parametrize("insert_mode", ["first", "last"])
@pytest.mark.parametrize("emit_mode", ["complete", "running", "final"])
def test_join_matches_oracle(ctx, insert_mode, emit_mode):
    from bytewax_b200 import gpu

    rnd = np.random.default_rng(11)
    batches = []
    for b in range(5):
        n = 4000
        keys = rnd.integers(0, 1500, n).astype(np.uint64) * 48271
        sides = rnd.integers(0, 2, n).astype(np.uint8)
        vals = rnd.integers(0, 2**40, n).astype(np.uint64)
        batches.append((keys, sides, vals))
    want = po.run_join([(k.tolist(), s.tolist(), v.tolist()) for k, s, v in batches], insert_mode, emit_mode)
    j = gpu.KeyedJoin(ctx, insert_mode, emit_mode, capacity_hint=4096, max_batch_rows=1 << 13, max_emit_rows=1 << 16)
    for i, (k, s, v) in enumerate(batches):
        j.apply(k, s, v)
        rows, _ = j.advance()
        assert rows == want[i], (insert_mode, emit_mode, i)
    rows, _ = j.eof()
    assert rows == want[-1]
    j.close()


def test_join_c4_shape_permutations(ctx):
    """C4 shape scaled down: two permutations of [0, N), default modes -> N rows (key, (l, r)), exact multiset;
    single advance over all activations keeps per-activation grouping."""
    from bytewax_b200 import gpu

    N_ = 200_000
    rnd = np.random.default_rng(4)
    left, right = rnd.permutation(N_).astype(np.uint64), rnd.permutation(N_).astype(np.uint64)
    keys = np.concatenate([left, right])
    sides = np.concatenate([np.zeros(N_, np.uint8), np.ones(N_, np.uint8)])
    vals = np.concatenate([left * 3 + 1, right * 7 + 2]).astype(np.uint64)
    order = rnd.permutation(2 * N_)  # interleave the two streams arbitrarily
    keys, sides, vals = keys[order], sides[order], vals[order]
    j = gpu.KeyedJoin(ctx, "last", "complete", capacity_hint=N_, max_batch_rows=1 << 17, max_emit_rows=1 << 18)
    B = 1 << 17
    for lo in range(0, 2 * N_, B):
        j.apply(keys[lo:lo + B], sides[lo:lo + B], vals[lo:lo + B])
    rows, epoch = j.advance()
    assert len(rows) == N_
    assert sorted(rows) == [(k, 3 * k + 1, 7 * k + 2) for k in range(N_)]
    assert (np.diff(epoch.astype(np.int64)) >= 0).all()
    rows, _ = j.eof()
    assert rows == []
    j.close()
