"""The streams of tests/keyed_limits_streams.py reach the per-key limits they are named for, as measured by the
instrumented oracles, at every M the GPU tests use.  CPU only."""

import pytest

from tests import keyed_limits_streams as ks
from tests import session_join_oracle as sj
from tests import session_oracle as so


def _k7(clock, steps):
    spec, st = ks.for_kernel("k7", clock, steps, reduction="sum", val_dtype="f64")
    return ks.measure("k7", spec, st)[1]


def _k9(clock, steps):
    spec, st = ks.for_kernel("k9", clock, steps, ordered=False)
    return ks.measure("k9", spec, st)


@pytest.mark.parametrize("M", ks.MS)
def test_fill_holds_exactly_M(M):
    b = ks.session_builders(M)
    for name in ("fill_one_call", "fill_gap0", "fill_spread"):
        logs = _k7(*b[name])
        assert ks.peak(logs, "records") == M and ks.first_overflow(logs, M) is None, name
    for name, step in (("fill_over", 0), ("fill_over_spread", 2)):
        logs = _k7(*b[name])
        assert ks.peak(logs, "records") == M + 1 and ks.first_overflow(logs, M) == step, name


@pytest.mark.parametrize("M", ks.MS)
@pytest.mark.parametrize("order", ks.ORDERS)
def test_collapse_merges_M_minus_1_in_one_call(M, order):
    logs = _k7(*ks.session_builders(M)[f"collapse_{order}"])
    hot = max(ks.calls(logs), key=lambda c: c.merges)
    assert hot.merges == M - 1 and hot.dead == M - 1 >= 31 and hot.records == M
    assert ks.first_overflow(logs, M) is None
    if order == "asc":
        assert ks.peak(logs, "mids") == M - 1


@pytest.mark.parametrize("M", ks.MS)
def test_collapse_fills_the_merged_ids(M):
    b = ks.session_builders(M)
    logs = _k7(*b["collapse_extra1"])
    assert ks.peak(logs, "mids") == M and ks.first_overflow(logs, M) is None
    logs = _k7(*b["collapse_extra2"])
    assert ks.peak(logs, "mids") == M + 1 and ks.peak(logs, "records") <= M and ks.first_overflow(logs, M) == 3


@pytest.mark.parametrize("M", ks.MS)
def test_records_not_live(M):
    """Live sessions stay within M, but the merged-away record still holds its slot: the new session is the M + 1st."""
    b = ks.session_builders(M)
    logs = _k7(*b["records_not_live"])
    c = [c for c in ks.calls(logs) if c.step == 1 and c.merges][0]
    assert c.records == M + 1 and c.records - c.merges == M and ks.first_overflow(logs, M) == 1  # live: M at most
    logs = _k7(*b["records_not_live_below"])
    assert ks.peak(logs, "records") == M and ks.peak(logs, "merges") == 1 and ks.first_overflow(logs, M) is None


@pytest.mark.parametrize("M", ks.MS)
def test_many_keys(M):
    logs = _k7(*ks.session_builders(M)["many_keys"])
    assert ks.first_overflow(logs, M) is None and ks.peak(logs, "records") == M
    assert sum(c.merges for c in ks.calls(logs)) > 500 and ks.peak(logs, "dead") >= M - 2
    assert all(max(c.records for c in log) >= M - 31 for log in logs)
    if M >= 63:
        assert sum(max(c.records for c in log) >= 33 for log in logs) > 100
    _, steps = ks.session_builders(M)["many_keys"]
    rows = so.run_sessions(*ks.for_kernel("k7", *ks.session_builders(M)["many_keys"], reduction="count"))
    assert any(r[2] == "L" for a in rows for r in a) and any(s[0] == "notify" for s in steps)
    assert any(r[2] == "M" for a, s in zip(rows, steps) if s[0] == "notify" for r in a)


def test_open_ties_never_reach_the_sort():
    """Two live sessions never share an open when ``_find_merges`` sorts them: every session is created or extended only
    where no live session lies within gap, and each sort merges the ones that come within gap, so live sessions stay
    more than gap apart.  The sort's tie rule (stable, by id) is therefore never exercised -- on every builder here, and
    on the seeded streams of the session kernels."""
    streams = [b for M in ks.MS for b in ks.session_builders(M).values()]
    for clock, steps in streams:
        assert ks.peak(_k7(clock, steps), "tie") == -1
    for seed in so.SEEDED:
        spec, steps = so.seeded_steps(seed)
        assert ks.peak(ks.measure("k7", spec, steps)[1], "tie") == -1
    for seed in sj.SEEDED:
        spec, steps = sj.seeded_steps(seed)
        assert ks.peak(ks.measure("k10", spec, steps)[1], "tie") == -1


@pytest.mark.parametrize("M", ks.MS)
def test_window_builders(M):
    b = ks.window_builders(M)
    for name in ("tumbling_desc", "tumbling_random", "tumbling_reopen", "sliding_full", "many_keys"):
        (acts, _), logs = _k9(*b[name])
        assert ks.peak(logs, "open") == M and ks.first_overflow(logs, M) is None, name
        closing = [sum(r[2] == "M" for r in a) for a in acts]
        assert sum(x > 0 for x in closing) >= (2 if name.startswith("sliding") else 3), (name, closing)  # closed in slices
    for name in ("tumbling_over", "sliding_over"):
        _, logs = _k9(*b[name])
        assert ks.peak(logs, "open") == M + 1 and ks.first_overflow(logs, M) == 0, name
    _, logs = _k9(*b["sliding_full"])
    assert ks.peak(logs, "values") >= 6 and all(c.open in (0, M) for c in ks.calls(logs) if c.step == 0)


@pytest.mark.parametrize("M", ks.MS)
def test_window_cells_reused(M):
    """K9's lowest-free-cell rule: windows opened in descending id order put the oldest windows on the highest cells,
    so the windows opened after the first close take cells up to M - 1 again."""
    _, logs = _k9(*ks.window_builders(M)["tumbling_reopen"])
    assert ks.peak(logs, "cell") == M - 1 and ks.peak(logs, "reuse") == M - 1
    if M > 32:
        assert ks.peak(logs, "reuse") >= 32


@pytest.mark.parametrize("M", ks.MS)
def test_window_many_keys(M):
    """300 keys, each opening M - 31 .. M windows in one call: every key's walk is long, and at M = 64 all of them hold
    33 or more windows at once (300 keys give the grid as many hot walks as 500 would here, at 60 % of the cost)."""
    (acts, _), logs = _k9(*ks.window_builders(M)["many_keys"])
    assert ks.peak(logs, "open") == M and ks.first_overflow(logs, M) is None
    assert len(logs) >= 300 and all(max(c.open for c in log) >= M - 31 for log in logs[:300])
    if M >= 63:
        assert sum(max(c.open for c in log) >= 33 for log in logs) > 100
    assert any(r[2] == "L" for a in acts for r in a)


@pytest.mark.parametrize("M", ks.MS)
def test_capacity_is_the_peak(M):
    """``first_overflow`` passes a stream at exactly its peak and fails it one below, at the call that reaches it."""
    for clock, steps in list(ks.session_builders(M).values()) + list(ks.window_builders(M).values()):
        logs = _k7(clock, steps) if "gap_us" in clock else _k9(clock, steps)[1]
        top = max(c.peak() for c in ks.calls(logs))
        assert ks.first_overflow(logs, top) is None
        assert ks.first_overflow(logs, top - 1) == min(c.step for c in ks.calls(logs) if c.peak() == top)
