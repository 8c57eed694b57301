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


def _spec(kernel, clock, steps, emit_mode="final", sides=2):
    """K12: unordered; K14 / K16: unordered, ``emit_mode`` over ``sides`` sides."""
    if kernel == "k12":
        return ks.for_kernel("k12", clock, steps, ordered=False)
    return ks.for_kernel(kernel, clock, steps, emit_mode=emit_mode, ordered=False, sides=sides)


def _k12(clock, steps):
    return ks.measure("k12", *_spec("k12", clock, steps))


def _k14(clock, steps, **kw):
    return ks.measure("k14", *_spec("k14", clock, steps, **kw))


def _k16(clock, steps, **kw):
    return ks.measure("k16", *_spec("k16", clock, steps, **kw))


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
    """``first_overflow`` passes a stream at exactly its peak and fails it one below, at the call that reaches it: for
    K7 and K9's measurements, and for K12's (which also counts merge intervals), K14's and K16's."""
    runs = []
    for clock, steps in ks.session_builders(M).values():
        runs += [(None, _k7(clock, steps)), ("k12", _k12(clock, steps)[1]), ("k16", _k16(clock, steps)[1])]
    for clock, steps in ks.window_builders(M).values():
        runs += [(None, _k9(clock, steps)[1]), ("k14", _k14(clock, steps)[1])]
    for kernel, logs in runs:
        fields = ks.counted(kernel)
        top = max(c.peak(fields) for c in ks.calls(logs))
        assert ks.first_overflow(logs, top, kernel) is None
        assert ks.first_overflow(logs, top - 1, kernel) == min(c.step for c in ks.calls(logs) if c.peak(fields) == top)


# ---------------------------------------------------------------------------
# K12 (session collect), K14 (product join over windows), K16 (product join over sessions)
# ---------------------------------------------------------------------------


@pytest.mark.parametrize("M", ks.MS)
def test_collapse_desc_fills_the_intervals(M):
    """A descending collapse chains M - 1 merges into session 0: M - 1 intervals on one merged id.  One more merge
    makes K12's intervals exactly M, two more M + 1 -- while records and merged ids stay within M, so only K12 fails."""
    b = ks.session_builders(M)
    logs = _k12(*b["collapse_desc"])[1]
    assert ks.peak(logs, "ivs") == M - 1 and ks.peak(logs, "mids") == 1
    for name, ivs, fail in (("collapse_desc_extra1", M, None), ("collapse_desc_extra2", M + 1, 3)):
        logs = _k12(*b[name])[1]
        assert ks.peak(logs, "ivs") == ivs and ks.peak(logs, "mids") <= 3 and ks.peak(logs, "records") == M, name
        assert ks.first_overflow(logs, M, "k12") == fail and ks.first_overflow(logs, M) is None, name
        for logs in (_k7(*b[name]), _k16(*b[name])[1]):
            assert ks.first_overflow(logs, M) is None and ks.peak(logs, "mids") < M, name
    logs = _k12(*b["collapse_extra2"])[1]  # ascending: intervals and merged ids grow together
    assert ks.peak(logs, "ivs") == ks.peak(logs, "mids") == M + 1 and ks.first_overflow(logs, M, "k12") == 3


@pytest.mark.parametrize("M", ks.MS)
@pytest.mark.parametrize("order", ks.ORDERS)
def test_collapse_chains_in_k12_and_k16(M, order):
    """Every collapse order gives K12 and K16 M - 1 merges in one call, with M records held; K12's intervals are the
    merges (each merge adds one, whatever the chain)."""
    b = ks.session_builders(M)[f"collapse_{order}"]
    for kernel, logs in (("k12", _k12(*b)[1]), ("k16", _k16(*b)[1])):
        hot = max(ks.calls(logs), key=lambda c: c.merges)
        assert hot.merges == M - 1 and hot.dead == M - 1 and hot.records == M, kernel
        assert ks.first_overflow(logs, M, kernel) is None, kernel
    assert ks.peak(_k12(*b)[1], "ivs") == M - 1


def _held_after_clear(acts, released):
    """Values a ``complete`` emission cleared from one window that are released in a later call: another window still
    held them."""
    rel_at = {h: i for i, r in enumerate(released) for h in r}
    return {h for i, a in enumerate(acts) for r in a if r[2] == "E" for h in r[3] if h is not None and rel_at[h] > i}


@pytest.mark.parametrize("M", ks.MS)
def test_sliding_creep(M):
    """Every value goes into M windows; the key holds M open windows in every call, and each new window takes the cell
    the closed one left (up to cell M - 1); under ``complete`` with 2 - 4 sides, clears free values in some of their
    windows while others still hold them."""
    clock, steps = ks.window_builders(M)["sliding_creep"]
    for sides in (1, 2, 3, 4):
        (acts, released), logs = _k14(clock, steps, emit_mode="complete", sides=sides)
        assert ks.peak(logs, "wins") == M and ks.peak(logs, "open") == M and ks.first_overflow(logs, M) is None
        assert ks.peak(logs, "cell") == M - 1 and ks.peak(logs, "reuse") >= 7
        hot = [c for c in max(logs, key=len) if c.step < len(steps)]  # (the light key's logic wakes once, at EOF)
        assert len(hot) == len(steps) and all(c.open == M for c in hot if steps[c.step][0] == "batch"), [c.open for c in hot]
        if sides > 1:
            assert len(_held_after_clear(acts, released)) >= 3, sides
    closing = [sum(r[2] == "M" and r[0] == 7 for r in a) for a in acts]
    assert closing[1:-1:2] == [1] * (len(steps) // 2) and not any(closing[:-1:2])  # each notify closes the hot key's lowest window


@pytest.mark.parametrize("M", ks.MS)
def test_k14_window_builders(M):
    """K14 counts open windows as K9 does: the same builders reach M (and M + 1 on the ``*_over`` ones)."""
    b = ks.window_builders(M)
    for name in sorted(b):
        logs9, logs14 = _k9(*b[name])[1], _k14(*b[name])[1]
        assert ks.peak(logs14, "open") == ks.peak(logs9, "open") in (M, M + 1), name
        assert ks.first_overflow(logs14, M) == ks.first_overflow(logs9, M), name


@pytest.mark.parametrize("kernel", ["k12", "k14", "k16"])
def test_instrumentation_changes_nothing(kernel):
    """The instrumented oracle returns what the plain one does -- rows and released handles -- on every builder at
    M = 64 and on seeded streams."""
    streams = list(ks.session_builders(64).values()) if kernel != "k14" else list(ks.window_builders(64).values())
    for clock, steps in streams:
        spec, st = _spec(kernel, clock, steps)
        assert ks.measure(kernel, spec, st)[0] == ks.RUNNERS[kernel](spec, st)
    mod = {"k12": ks.sc, "k14": ks.po, "k16": ks.sp}[kernel]
    for seed in list(mod.SEEDED)[:12]:
        spec, st = mod.seeded_steps(seed)
        assert ks.measure(kernel, spec, st)[0] == ks.RUNNERS[kernel](spec, st), seed
