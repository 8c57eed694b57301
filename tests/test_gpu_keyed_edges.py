"""K5 (z-score map) and K6 (keyed join) at the edges of their inputs and tables.  -m gpu.

K5 is compared bit for bit with the correctly rounded twin of the reference mapper (`po.run_zscore(...,
correctly_rounded=True)`), and with the reference's own arithmetic where the two must agree: the means, and every flag
the twin does not predict to differ.  K6 is compared row for row, in order, with `po.run_join` in all six modes."""

import random

import numpy as np
import pytest

from bytewax_b200 import _native as N
from oracle import pyoracle as po  # checker only
from oracle import streams

pytestmark = pytest.mark.gpu

SENTINEL = 2**64 - 1  # the key tables' empty marker; the key itself lives in the alias slot `cap`


@pytest.fixture(scope="module")
def ctx():
    from bytewax_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.close()


# ---------------------------------------------------------------------------
# K5
# ---------------------------------------------------------------------------


def _same_bits(a, b):
    """Bitwise equality of two f64 arrays, where any NaN equals any NaN (the device's default NaN has other bits than the
    host's, and the host propagates NaN payloads)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return (a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))


def _distinct_keys(rnd, n):
    """n distinct keys drawn from 1 .. 2^64-2."""
    keys = {}
    while len(keys) < n:
        keys.setdefault(rnd.randrange(1, SENTINEL))
    return list(keys)


def _cols(rows):
    return tuple(np.array([r[i] for r in rows], dtype=(bool if i == 2 else np.float64)) for i in range(3))


def _zscore_run(m, batches, window, threshold, dtype):
    """Apply each activation (keys, vals) to `m`.  Every row must equal the twin bit for bit; the mean must equal the
    reference's; a flag may differ from the reference's only where the twin's does.  Returns those rows (batch, index)."""
    vt = np.float32 if dtype == "f32" else np.float64
    host = [(np.asarray(k, np.uint64), np.asarray(v, vt)) for k, v in batches]
    lists = [(k.tolist(), v.astype(np.float64).tolist()) for k, v in host]
    twin = po.run_zscore(lists, window, threshold, correctly_rounded=True)
    ref = po.run_zscore(lists, window, threshold)
    flips = []
    for b, ((k, v), tw, rf) in enumerate(zip(host, twin, ref)):
        mu, sigma, flag = m.apply(k, v)
        tm, ts, tf = _cols(tw)
        rm, _rs, rfl = _cols(rf)
        for name, got, want in (("mu", mu, tm), ("sigma", sigma, ts)):
            bad = np.nonzero(~_same_bits(got, want))[0]
            assert bad.size == 0, (name, b, bad[:4].tolist(), got[bad[:4]].tolist(), want[bad[:4]].tolist())
        bad = np.nonzero(flag != tf)[0]
        assert bad.size == 0, ("flag", b, bad[:4].tolist(), v[bad[:4]].tolist())
        assert _same_bits(mu, rm).all(), b
        assert np.array_equal(np.nonzero(flag != rfl)[0], np.nonzero(tf != rfl)[0]), b
        flips += [(b, int(i)) for i in np.nonzero(flag != rfl)[0]]
    return flips


def _interleave(rnd, rows):
    """(keys, vals) of the (key, value) rows in a random order that keeps every key's own order."""
    per = {}
    for k, v in rows:
        per.setdefault(k, []).append(v)
    order = [k for k, _ in rows]
    rnd.shuffle(order)
    return order, [per[k].pop(0) for k in order]


def _tie_rows(key0, threshold):
    """Fresh keys whose third value lies exactly at z == threshold, one ulp above it, and at mean 0 (suppressed):
    after 0, 2 the mean is 1 and sigma is 1."""
    t = threshold
    seqs = [[0.0, 2.0, 1.0 + t], [2.0, 0.0, 1.0 - t], [0.0, 2.0, float(np.nextafter(1.0 + t, 9.0))], [-1.0, 1.0, 5.0],
            [1.0, -1.0, -7.0, 0.0]]
    return [(key0 + i, v) for i, s in enumerate(seqs) for v in s]


@pytest.mark.parametrize("threshold", [0.5, 2.0, 3.0])
@pytest.mark.parametrize("dtype", ["f32", "f64"])
@pytest.mark.parametrize("window", [1, 2, 10, 31, 32])
def test_zscore_value_families_bitwise(ctx, window, dtype, threshold):
    """Every value family (small integers, three decimals, magnitudes to 1e150, +-1e16 against O(1), subnormals, signed
    zeros, inf and NaN), one family per key, keys 0 and 2^64-1 among them, over activations of 1 to max_batch_rows rows;
    plus exact ties at the threshold and windows of mean 0."""
    from bytewax_b200 import gpu

    rnd = random.Random(f"k5-{window}-{dtype}-{threshold}")
    fams = streams.ZSCORE_FAMILIES + ("nonfinite",)
    keyset = [0, SENTINEL] + [rnd.randrange(1, SENTINEL) for _ in range(26)]
    fam_of = {k: fams[i % len(fams)] for i, k in enumerate(keyset)}
    mbr = 2048
    m = gpu.ZScoreMap(ctx, window, threshold, dtype, capacity_hint=64, max_batch_rows=mbr)
    batches = []
    for b, n in enumerate([1, 30, 1500, 1, mbr, 700]):
        ties = _tie_rows(1000 + 10 * b, threshold) if n > 100 else []
        ks = [rnd.choice(keyset) for _ in range(n - len(ties))]
        batches.append(_interleave(rnd, [(k, streams.zscore_value(fam_of[k], rnd, dtype == "f32")) for k in ks] + ties))
    assert len(batches[4][0]) == mbr
    _zscore_run(m, batches, window, threshold, dtype)
    m.close()


def test_zscore_nonfinite_values(ctx):
    """An inf after a finite window is flagged; while it is in the window mu is inf, sigma NaN and no flag is raised."""
    from bytewax_b200 import gpu

    m = gpu.ZScoreMap(ctx, 3, 2.0, "f64", capacity_hint=16, max_batch_rows=64)
    vals = [1.0, 2.0, 3.0, np.inf, 1.0, 2.0, 3.0, 1.0, -np.inf, np.nan, 5.0, 5.0, 6.0, 5.0, 100.0]
    keys = [5] * len(vals)
    _zscore_run(m, [(keys[:5], vals[:5]), (keys[5:], vals[5:])], 3, 2.0, "f64")
    m.close()
    # what the rows above were compared with
    twin = po.run_zscore([(keys, vals)], 3, 2.0, correctly_rounded=True)[0]
    assert twin[3][2] is True and np.isinf(twin[3][0]) and np.isnan(twin[3][1])
    assert [r[2] for r in twin[4:7]] == [False] * 3 and np.isfinite(twin[6][0])
    assert twin[14][2] is True


@pytest.mark.parametrize("dtype", ["f32", "f64"])
@pytest.mark.parametrize("window", [1, 2, 10, 31, 32])
def test_zscore_ring_across_activations(ctx, window, dtype):
    """One key per (ring state, count): W-1, W, W+1 and 2W+3 items in one activation after an empty, a partly filled
    and a full ring; a key absent for several activations that returns; an activation of one row (every term from the
    ring) and one of exactly max_batch_rows rows."""
    from bytewax_b200 import gpu

    W = window
    rnd = random.Random(f"ring-{W}-{dtype}")
    mbr = 1024
    m = gpu.ZScoreMap(ctx, W, 2.0, dtype, capacity_hint=64, max_batch_rows=mbr)
    prior = {"empty": 0, "partial": W // 2, "full": W + 3}
    counts = [W - 1, W, W + 1, 2 * W + 3]
    cases = [(st, c) for st in prior for c in counts]
    key_of = {case: 7 + 13 * i for i, case in enumerate(cases)}
    val = lambda: streams.zscore_value(rnd.choice(("dec3", "int", "mix1e16")), rnd, dtype == "f32")  # noqa: E731
    shuffled = lambda rows: _interleave(rnd, rows)  # noqa: E731
    absent = 99
    batches = [
        shuffled([(key_of[(st, c)], val()) for (st, c) in cases for _ in range(prior[st])] + [(absent, val()) for _ in range(W + 1)]),
        shuffled([(key_of[(st, c)], val()) for (st, c) in cases for _ in range(c)] + [(absent, val()) for _ in range(2)]),
        ([key_of[("full", W)]], [val()]),  # one row: all of its window comes from the ring
    ]
    ks = [rnd.choice(list(key_of.values())) for _ in range(mbr)]
    batches.append((ks, [val() for _ in ks]))  # exactly max_batch_rows rows
    batches.append(([], []))
    batches.append(shuffled([(absent, val()) for _ in range(3)] + [(key_of[("partial", W + 1)], val()) for _ in range(2)]))
    _zscore_run(m, batches, W, 2.0, dtype)
    m.close()


def test_zscore_flip_sequence_is_the_one_predicted_difference(ctx):
    """The reference flags the last value of this key's sequence, correctly rounded arithmetic does not; the device gives
    the twin's answer, split over two activations (the first terms come from the ring)."""
    from bytewax_b200 import gpu

    seq = streams.ZSCORE_FLIP
    rnd = random.Random(3)
    other = [rnd.randrange(1, 50) for _ in range(40)]
    keys = [2**63] * 6 + other[:20], [2**63] * 5 + other[20:]
    vals = seq[:6] + [round(rnd.uniform(0, 10), 3) for _ in range(20)], seq[6:] + [round(rnd.uniform(0, 10), 3) for _ in range(20)]
    m = gpu.ZScoreMap(ctx, 10, 2.0, "f64", capacity_hint=16, max_batch_rows=64)
    flips = _zscore_run(m, list(zip(keys, vals)), 10, 2.0, "f64")
    assert (1, 4) in flips
    assert po.run_zscore([([1] * len(seq), seq)])[0][-1][2] is True
    m.close()


def test_zscore_key_table_exactly_full(ctx):
    """cap = max(1024, 2 * capacity_hint) distinct keys plus the sentinel key fit; one key more is BW_ERR_CAPACITY."""
    from bytewax_b200 import gpu

    rnd = random.Random(17)
    cap = 1024
    m = gpu.ZScoreMap(ctx, 4, 2.0, "f64", capacity_hint=16, max_batch_rows=4096)
    keys = [0] + _distinct_keys(rnd, cap - 1) + [SENTINEL]
    b1 = keys + [rnd.choice(keys) for _ in range(1000)]
    rnd.shuffle(b1)
    b2 = [rnd.choice(keys) for _ in range(3000)]
    batches = [(b, [round(rnd.uniform(-5, 5), 3) for _ in b]) for b in (b1, b2)]
    _zscore_run(m, batches, 4, 2.0, "f64")
    new = next(k for k in range(1, 1 << 20) if k not in set(keys))
    with pytest.raises(N.BwError) as e:
        m.apply(np.array([new], np.uint64), np.array([1.0]))
    assert e.value.status == 3  # BW_ERR_CAPACITY
    m.close()


def test_zscore_spec_limits(ctx):
    """max_batch_rows + 1 rows is BW_ERR_SPEC; windows 0 and 33 are refused at create (1..32 are accepted)."""
    from bytewax_b200 import gpu

    m = gpu.ZScoreMap(ctx, 32, 2.0, "f32", capacity_hint=16, max_batch_rows=100)
    with pytest.raises(N.BwError) as e:
        m.apply(np.zeros(101, np.uint64), np.zeros(101, np.float32))
    assert e.value.status == 4  # BW_ERR_SPEC
    mu, _, _ = m.apply(np.zeros(100, np.uint64), np.ones(100, np.float32))
    assert (mu == 1.0).all()
    m.close()
    for w in (0, 33):
        with pytest.raises(N.BwError) as e:
            gpu.ZScoreMap(ctx, w, 2.0, "f64", capacity_hint=16, max_batch_rows=16)
        assert e.value.status == 4


# ---------------------------------------------------------------------------
# K6
# ---------------------------------------------------------------------------

MODES = [(im, em) for im in ("first", "last") for em in ("complete", "running", "final")]

# keys whose decimal text orders differently from their value, at every digit-count boundary (k_sortkey), the 20-digit
# keys (ordered by their 20th digit), 2^63, the sentinel and 0
EDGE_KEYS = sorted({0, 9, 10, 2**63, SENTINEL} | {10**k - 1 for k in range(1, 20)} | {10**k for k in range(1, 20)}
                   | {10**19 + d for d in range(10)})
HANDLES = [0, 2**63, 2**64 - 1, 1]


def _join_items(rnd, keys, n):
    ks = [rnd.choice(keys) for _ in range(n)]
    return ks, [rnd.randrange(2) for _ in ks], [rnd.choice(HANDLES) if rnd.random() < 0.5 else rnd.randrange(2**64) for _ in ks]


def _arrays(k, s, v):
    return np.array(k, np.uint64), np.array(s, np.uint8), np.array(v, np.uint64)


def _join_run(j, acts, im, em):
    """One `apply` + `advance` per activation, then `eof`; every row list must equal the oracle's, in order."""
    want = po.run_join(acts, im, em)
    for i, a in enumerate(acts):
        j.apply(*_arrays(*a))
        rows, _ = j.advance()
        assert rows == want[i], (im, em, i)
    rows, _ = j.eof()
    assert rows == want[-1], (im, em, "eof")
    return want


@pytest.mark.parametrize("im,em", MODES)
def test_join_key_text_order_and_handles(ctx, im, em):
    """Keys at every digit-count boundary, 10^19 .. 10^19+9, 2^63, 2^64-1 and 0, and handles 0, 2^63 and 2^64-1 (only the
    mask says None): first all in one activation in shuffled order, then across several."""
    from bytewax_b200 import gpu

    rnd = random.Random(f"join-order-{im}-{em}")
    first = [k for k in EDGE_KEYS for _ in range(3)]
    rnd.shuffle(first)
    acts = [(first, [rnd.randrange(2) for _ in first], [rnd.choice(HANDLES) for _ in first])]
    acts += [_join_items(rnd, EDGE_KEYS, n) for n in (1, 40, 200, 7)]
    j = gpu.KeyedJoin(ctx, im, em, capacity_hint=64, max_batch_rows=1024, max_emit_rows=1024)
    want = _join_run(j, acts, im, em)
    if em == "final":
        assert [r[0] for r in want[-1]] == sorted(EDGE_KEYS, key=str)  # every key holds state at the end
    j.close()

    # a single activation holding only the sentinel key, and one holding only 20-digit keys
    j = gpu.KeyedJoin(ctx, im, em, capacity_hint=16, max_batch_rows=64, max_emit_rows=1024)
    twenty = [10**19 + d for d in range(10)]
    rnd.shuffle(twenty)
    _join_run(j, [([SENTINEL] * 3, [0, 1, 0], [2**64 - 1, 0, 2**63]), (twenty, [0] * 10, list(range(10)))], im, em)
    j.close()


@pytest.mark.parametrize("im,em", MODES)
def test_join_hot_key_serial(ctx, im, em):
    """One key with 100 000 items of mostly alternating sides in one activation, walked by one thread: complete mode
    discards and restarts many times inside the activation."""
    from bytewax_b200 import gpu

    rnd = random.Random(f"hot-{im}-{em}")
    n = 100_000
    hot = 10**19 + 3
    keys = [hot if rnd.random() < 0.98 else rnd.choice(EDGE_KEYS) for _ in range(n)]
    sides, s = [], 0
    for _ in range(n):
        s ^= 1 if rnd.random() < 0.9 else 0
        sides.append(s)
    vals = [rnd.randrange(2**64) for _ in range(n)]
    j = gpu.KeyedJoin(ctx, im, em, capacity_hint=64, max_batch_rows=1 << 17, max_emit_rows=1 << 17)
    _join_run(j, [(keys, sides, vals), _join_items(rnd, [hot], 5)], im, em)
    j.close()


@pytest.mark.parametrize("im,em", MODES)
def test_join_epochs_and_empty_calls(ctx, im, em):
    """Three applies (and an empty one) with one epoch, then one advance: one activation's order (key string, then
    arrival across the calls).  Then epochs with gaps in one advance, an advance with nothing pending, eof after an
    advance and eof twice.  A decreasing epoch is BW_ERR_STATE."""
    from bytewax_b200 import gpu

    rnd = random.Random(f"epochs-{im}-{em}")
    keys = EDGE_KEYS[:20] + [12, 123, 1234]
    j = gpu.KeyedJoin(ctx, im, em, capacity_hint=64, max_batch_rows=256, max_emit_rows=1024)
    parts = [_join_items(rnd, keys, n) for n in (60, 0, 50, 70)]
    one = tuple(sum((list(p[c]) for p in parts), []) for c in range(3))
    gapped = [_join_items(rnd, keys, n) for n in (30, 40, 25)]
    want = po.run_join([one] + gapped, im, em)

    for p in parts:
        j.apply(*_arrays(*p), epoch=5)
    rows, epoch = j.advance()
    assert rows == want[0] and (epoch == 5).all()

    for a, e in zip(gapped, (7, 9, 1009)):
        j.apply(*_arrays(*a), epoch=e)
    rows, epoch = j.advance()
    assert rows == want[1] + want[2] + want[3]
    assert epoch.tolist() == [7] * len(want[1]) + [9] * len(want[2]) + [1009] * len(want[3])

    rows, epoch = j.advance()  # nothing pending
    assert rows == [] and epoch.size == 0
    rows, _ = j.eof()
    assert rows == want[4]
    rows, _ = j.eof()
    assert rows == []
    j.close()

    j = gpu.KeyedJoin(ctx, im, em, capacity_hint=64, max_batch_rows=256, max_emit_rows=1024)
    j.apply(*_arrays(*parts[0]), epoch=5)
    with pytest.raises(N.BwError) as e:
        j.apply(*_arrays(*parts[2]), epoch=4)
    assert e.value.status == 5  # BW_ERR_STATE
    j.close()


def _exact_rows(em, n, key0):
    """Items on which mode `em` emits exactly n rows (at advance, or at eof for final)."""
    keys = [key0 + i for i in range(n)]
    if em == "running":
        return keys, [i & 1 for i in range(n)], list(range(n))
    if em == "complete":
        return keys + keys, [0] * n + [1] * n, list(range(2 * n))
    return keys, [0] * n, list(range(n))


@pytest.mark.parametrize("im,em", MODES)
def test_join_emit_buffer_exactly_full(ctx, im, em):
    """max_emit_rows (below the 1024 rows the buffers hold at least) rows pass; one more is BW_ERR_CAPACITY."""
    from bytewax_b200 import gpu

    M = 700
    items = _exact_rows(em, M, 10**18)
    want = po.run_join([items], im, em)
    assert sum(map(len, want)) == M
    j = gpu.KeyedJoin(ctx, im, em, capacity_hint=2048, max_batch_rows=4096, max_emit_rows=M)
    _join_run(j, [items], im, em)
    j.close()

    items = _exact_rows(em, M + 1, 10**18)
    j = gpu.KeyedJoin(ctx, im, em, capacity_hint=2048, max_batch_rows=4096, max_emit_rows=M)
    with pytest.raises(N.BwError) as e:
        j.apply(*_arrays(*items))
        j.advance()
        j.eof()
    assert e.value.status == 3  # BW_ERR_CAPACITY
    j.close()


@pytest.mark.parametrize("im,em", MODES)
def test_join_key_table_exactly_full(ctx, im, em):
    """cap = max(1024, 2 * capacity_hint) distinct keys plus the sentinel key fit; one key more is BW_ERR_CAPACITY."""
    from bytewax_b200 import gpu

    rnd = random.Random(f"join-full-{im}-{em}")
    cap = 1024
    keys = [0] + _distinct_keys(rnd, cap - 1) + [SENTINEL]
    a1 = keys + [rnd.choice(keys) for _ in range(500)]
    rnd.shuffle(a1)
    acts = [(a1, [rnd.randrange(2) for _ in a1], [rnd.randrange(2**64) for _ in a1]), _join_items(rnd, keys, 800)]
    j = gpu.KeyedJoin(ctx, im, em, capacity_hint=16, max_batch_rows=2048, max_emit_rows=4096)
    _join_run(j, acts, im, em)
    new = next(k for k in range(1, 1 << 20) if k not in set(keys))
    with pytest.raises(N.BwError) as e:
        j.apply(*_arrays([new], [0], [1]))
        j.advance()
    assert e.value.status == 3  # BW_ERR_CAPACITY
    j.close()
