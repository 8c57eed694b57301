"""The `*_final` operators with the CUDA path enabled (run_main(..., gpu=True)) against the host engine, row for row and
type for type, and the rule that keeps ints and floats apart on the numeric fold steps.  The gpu-marked tests need an
H100 (-m gpu); the first-batch rule is checked without a device."""

import math
import operator
from datetime import datetime, timedelta, timezone

import numpy as np
import pytest

import bytewax_b200.engine as E
import bytewax_b200.operators as op
import bytewax_b200.operators.windowing as win
from bytewax_b200 import gpu as gpu_mod
from bytewax_b200.dataflow import Dataflow
from bytewax_b200.errors import BytewaxRuntimeError
from bytewax_b200.operators.windowing import ZERO_TD, EventClock, TumblingWindower
from bytewax_b200.testing import TestingSink, TestingSource, run_main
from oracle import exact

ALIGN = datetime(2022, 1, 1, tzinfo=timezone.utc)
FROZEN = datetime(2030, 1, 1, tzinfo=timezone.utc)
BIG = 2**53


@pytest.fixture
def device_calls(monkeypatch):
    """Counts the activations the device folded (`WindowFold.ingest`), to check that the CUDA path really ran."""
    calls = []
    orig = gpu_mod.WindowFold.ingest

    def ingest(self, *a, **k):
        calls.append(len(a[0]))
        return orig(self, *a, **k)

    monkeypatch.setattr(gpu_mod.WindowFold, "ingest", ingest)
    return calls


FINALS = {
    "sum": lambda s: op.reduce_final("r", s, operator.add),
    "max": lambda s: op.max_final("r", s),
    "min": lambda s: op.min_final("r", s),
}


def _final_flow(sources, make):
    """Every source is its own input, merged: each activation hands the fold one pre-reduced item per source and key."""
    out = []
    flow = Dataflow("df")
    ins = [op.input(f"in{i}", flow, src) for i, src in enumerate(sources)]
    s = ins[0] if len(ins) == 1 else op.merge("m", *ins)
    op.output("out", make(s), TestingSink(out))
    return flow, out


def _window_flow(source, reducer):
    out = []
    flow = Dataflow("df")
    s = op.input("in", flow, source)
    clock = EventClock(lambda v: ALIGN, ZERO_TD, now_getter=lambda: FROZEN)
    wo = win.reduce_window("w", s, clock, TumblingWindower(timedelta(seconds=10), ALIGN), reducer)
    op.output("out", wo.down, TestingSink(out))
    return flow, out


def _both(build):
    outs = []
    for gpu in (False, True):
        flow, out = build()
        run_main(flow, gpu=gpu)
        outs.append(out)
    return outs


def _typed(rows):
    return [(k, v, type(v)) for k, v in rows]


def _items(rnd, keys, n, floats):
    ks = rnd.choice(keys, n).tolist()
    if floats:
        vs = (rnd.normal(0, 1e3, n) * 10.0 ** rnd.integers(-3, 7, n)).tolist()
    else:
        vs = rnd.integers(-10**12, 10**12, n).tolist()
    return list(zip(ks, vs))


# ---------------------------------------------------------------------------- ints, floats, several items per key


@pytest.mark.gpu
@pytest.mark.parametrize("floats", [False, True])
@pytest.mark.parametrize("red", ["count", "sum", "max", "min"])
def test_final_ops_match_host(device_calls, red, floats):
    """Three merged sources in batches of 20 over 5 keys: every call of the fold gets several pre-reduced items of a key.
    Ints, max and min: the host's rows exactly, types included; float sums: within the exact bound of their values."""
    rnd = np.random.default_rng(1 + floats)
    keys = np.array([f"k{i}" for i in range(5)])
    parts = [_items(rnd, keys, 500, floats) for _ in range(3)]
    make = (lambda s: op.count_final("c", s, lambda kv: kv[0])) if red == "count" else FINALS[red]
    host, gpu = _both(lambda: _final_flow([TestingSource(p, batch_size=20) for p in parts], make))
    assert device_calls and max(device_calls) > len(keys)  # several items of a key in one call
    assert [k for k, _ in gpu] == sorted({k for p in parts for k, _ in p})
    if red == "sum" and floats:
        want = {}
        for k, v in (kv for p in parts for kv in p):
            want.setdefault(k, []).append(v)
        for (k, g), (hk, h) in zip(gpu, host):
            e = exact._reduce("sum", "f64", want[k])
            assert hk == k and type(g) is float and type(h) is float
            assert abs(g - e.fsum) <= e.bound() and abs(h - e.fsum) <= e.bound(), k
    else:
        assert _typed(gpu) == _typed(host)


# ---------------------------------------------------------------------------- ints and floats do not mix


def _cause(flow):
    with pytest.raises(BytewaxRuntimeError) as ei:
        run_main(flow, gpu=True)
    cause = ei.value.__cause__
    msg = str(cause)
    assert isinstance(cause, TypeError) and "stateful_batch'" in msg and ("mid-stream" in msg or "mixing" in msg), cause
    return cause


MIXED = [("max", [BIG + 1, float(BIG)], BIG + 1), ("sum", [BIG, 1, 1, 0.5], 9007199254740994.0)]


@pytest.mark.gpu
@pytest.mark.parametrize("red,vals,want", MIXED)
def test_mixed_first_batch_runs_on_host_final(device_calls, red, vals, want):
    """`max_final` over 2^53 + 1 and 2.0^53, `reduce_final(add)` over 2^53, 1, 1, 0.5 in the fold's first call: a
    float64 column would give 2.0^53 for both, so the step runs on the host logic and gives the host's value and type."""
    host, gpu = _both(lambda: _final_flow([TestingSource([("a", v)]) for v in vals], FINALS[red]))
    assert gpu == [("a", want)] and _typed(gpu) == _typed(host)
    assert not device_calls


@pytest.mark.gpu
@pytest.mark.parametrize("red,vals,want", MIXED)
def test_mixed_first_batch_runs_on_host_window(device_calls, red, vals, want):
    reducer = {"max": max, "sum": operator.add}[red]
    host, gpu = _both(lambda: _window_flow(TestingSource([("a", v) for v in vals], batch_size=len(vals)), reducer))
    assert gpu == [("a", (0, want))] and [type(v) for _k, (_w, v) in gpu] == [type(want)] and gpu == host
    assert not device_calls


LATER = [[BIG + 1, float(BIG)], [float(BIG), BIG + 1], [BIG, 1, 1, 0.5], [0.5, 1.0, BIG, 1]]


@pytest.mark.gpu
@pytest.mark.parametrize("vals", LATER, ids=["int-float", "float-int", "int-mix", "float-mix"])
def test_mixed_later_batch_raises_final(device_calls, vals):
    """After the fold's first call fixed the kind, a value of the other kind raises a TypeError naming the step, in both
    directions (a float after ints, an int after floats)."""
    red = "max" if len(vals) == 2 else "sum"
    flow, _ = _final_flow([TestingSource([("a", v) for v in vals], batch_size=1)], FINALS[red])
    _cause(flow)
    assert device_calls


@pytest.mark.gpu
@pytest.mark.parametrize("vals", LATER, ids=["int-float", "float-int", "int-mix", "float-mix"])
def test_mixed_later_batch_raises_window(device_calls, vals):
    reducer = max if len(vals) == 2 else operator.add
    flow, _ = _window_flow(TestingSource([("a", v) for v in vals], batch_size=1 if len(vals) == 2 else 2), reducer)
    _cause(flow)
    assert device_calls


@pytest.mark.gpu
def test_sum_of_negative_zero_alone(device_calls):
    """A float sum whose only value is -0.0: the device's sum starts from its identity +0.0 and gives +0.0, the host keeps
    the first value, -0.0.  They compare equal (DESIGN.md section 10)."""
    host, gpu = _both(lambda: _final_flow([TestingSource([("a", -0.0), ("b", 1.5)])], FINALS["sum"]))
    assert gpu == host == [("a", 0.0), ("b", 1.5)] and device_calls
    assert math.copysign(1.0, host[0][1]) < 0 and math.copysign(1.0, gpu[0][1]) > 0


# ---------------------------------------------------------------------------- keys


KEYS = ["0", "9", "10", "9223372036854775807", "9223372036854775808", "18446744073709551615", "007", "+1", "-1", "1.0",
        "٣", "²", "1٣", "a", "B", "zz", "", "10a"]


@pytest.mark.gpu
@pytest.mark.parametrize("red", ["count", "sum", "max", "min"])
def test_string_keys(device_calls, red):
    """Keys that are canonical decimal ids below 2^63 and keys interned from 2^63 up (2^63 and above, leading zeros,
    signs, other scripts' digits, letters, the empty key): `_key_id` and the re-sort give the host's keys and order."""
    rnd = np.random.default_rng(4)
    items = [(KEYS[i], int(v)) for i, v in zip(rnd.integers(0, len(KEYS), 600), rnd.integers(-1000, 1000, 600))]
    make = (lambda s: op.count_final("c", s, lambda kv: kv[0])) if red == "count" else FINALS[red]
    host, gpu = _both(lambda: _final_flow([TestingSource(items, batch_size=50)], make))
    assert _typed(gpu) == _typed(host) and [k for k, _ in gpu] == sorted(KEYS) and device_calls


# ---------------------------------------------------------------------------- without a device


def test_first_batch_rule_needs_no_fold():
    """The numeric fold steps refuse a batch that mixes int and float values before any fold exists (`_GpuPlanUnfit`:
    the engine runs the step on the host logic); once a fold exists, a mix or a change of kind is a TypeError naming the
    step.  No device is touched."""
    clock = EventClock(lambda v: ALIGN, ZERO_TD, now_getter=lambda: FROZEN)

    def steps():
        yield E._gpu_step_for("s", op.GpuFinalPlan("max"))
        yield E._gpu_step_for("s", win.GpuFoldPlan("sum", clock, TumblingWindower(timedelta(seconds=10), ALIGN), False, lambda v: v))

    for step in steps():
        assert isinstance(step, (E._GpuFinalStep, E._GpuWindowStep))
        for vals in ([BIG + 1, float(BIG)], [float(BIG), BIG + 1], [BIG, 1, 1, 0.5]):
            with pytest.raises(E._GpuPlanUnfit):
                step.on_epoch(1, [("a", v) for v in vals])
            assert step.fold is None
    for step in steps():
        step.fold = object()  # (as if the device fold existed: no longer the first batch)
        for float_vals, vals in ((False, [1.5]), (True, [1]), (False, [1, 2.5]), (True, [2.5, 1])):
            step.float_vals = float_vals
            with pytest.raises(TypeError, match="'s'"):
                step.on_epoch(2, [("a", v) for v in vals])


def test_interned_keys_map_back():
    """Every key string maps back from its id, the empty key included (its id is interned like any non-numeric key)."""
    step = E._gpu_step_for("s", op.GpuFinalPlan("sum"))
    for k in KEYS:
        assert step._key_str(step._key_id(k)) == k
