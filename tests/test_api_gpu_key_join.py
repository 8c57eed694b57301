"""`op.join` flows with the CUDA path enabled (run_main(..., gpu=True)): the recogniser hands two-sided first / last joins
to K6 (`bw_join_*`) and every other join with 1 to 4 sides to K15 (`bw_kjoin_*`); the rows must equal the host
engine's, with arbitrary Python values.  -m gpu."""

import random

import pytest

pytestmark = pytest.mark.gpu

import bytewax_b200.operators as op  # noqa: E402
from bytewax_b200 import engine  # noqa: E402
from bytewax_b200.dataflow import Dataflow  # noqa: E402
from bytewax_b200.testing import TestingSink, TestingSource, run_main  # noqa: E402

INSERTS = ("first", "last", "product")
EMITS = ("complete", "final", "running")


def _values(seed, n, n_keys):
    """Items ``(key, value)``: dicts, None, tuples, strings; a few keys that are not canonical numbers."""
    rnd = random.Random(seed)
    keys = [str(k) for k in range(n_keys)] + ["", "a", "007", "é"]
    out = []
    for i in range(n):
        v = rnd.choice([{"i": i}, None, (i, "x"), f"s{i}", i, [i]])
        out.append((rnd.choice(keys), v))
    return out


def _flow(side_items, insert_mode, emit_mode, batch_size=7):
    out = []
    flow = Dataflow("df")
    sides = []
    for i, items in enumerate(side_items):
        s = op.input(f"in{i}", flow, TestingSource(items, batch_size=batch_size))
        sides.append(op.map_value(f"val{i}", op.key_on(f"key{i}", s, lambda kv: kv[0]), lambda kv: kv[1]))
    joined = op.join("join", *sides, insert_mode=insert_mode, emit_mode=emit_mode)
    op.output("out", joined, TestingSink(out))
    return flow, out


@pytest.fixture
def steps_run(monkeypatch):
    """Records which device step ran each activation of a join: K6's `_GpuJoinStep` or K15's `_GpuKeyJoinStep`."""
    ran = []
    for cls, name in ((engine._GpuJoinStep, "KeyedJoin"), (engine._GpuKeyJoinStep, "KeyJoin")):
        orig = cls.on_epoch

        def on_epoch(self, epoch, items, orig=orig, name=name, cls=cls):
            rows = orig(self, epoch, items)
            dev = getattr(self, "join", None) or getattr(self, "jwin", None)
            assert type(dev).__name__ == name
            ran.append(cls.__name__)
            return rows

        monkeypatch.setattr(cls, "on_epoch", on_epoch)
    spied = []
    orig_for = engine._gpu_step_for

    def step_for(step_id, plan):
        st = orig_for(step_id, plan)
        spied.append(type(st).__name__)
        return st

    monkeypatch.setattr(engine, "_gpu_step_for", step_for)
    return ran, spied


def _both(side_items, insert_mode, emit_mode, workers=1):
    outs = []
    for gpu in (False, True):
        flow, out = _flow(side_items, insert_mode, emit_mode)
        engine._Run(flow, workers, None, gpu).run() if workers > 1 else run_main(flow, gpu=gpu)
        outs.append(out)
    return outs


@pytest.mark.parametrize("sides", [1, 2, 3, 4])
@pytest.mark.parametrize("emit", EMITS)
@pytest.mark.parametrize("insert", INSERTS)
def test_matches_host_engine(steps_run, insert, emit, sides):
    ran, spied = steps_run
    n = 60 if insert == "product" and emit != "complete" else 400
    side_items = [_values(100 * sides + 10 * INSERTS.index(insert) + EMITS.index(emit) + s, n // sides, 6) for s in range(sides)]
    host, gpu = _both(side_items, insert, emit)
    assert gpu == host
    assert host
    want = "_GpuJoinStep" if sides == 2 and insert in ("first", "last") else "_GpuKeyJoinStep"
    assert spied == [want] and ran and set(ran) == {want}


@pytest.mark.parametrize("insert, emit", [("product", "final"), ("last", "running"), ("first", "complete"), ("product", "complete")])
def test_two_workers_match_host_engine(steps_run, insert, emit):
    ran, _spied = steps_run
    side_items = [_values(7 + s, 150, 20) for s in range(3)]
    host, gpu = _both(side_items, insert, emit, workers=2)
    # two workers interleave their rows: each key's rows, in order, are the host engine's on the same two workers
    per_key = lambda rows: {k: [v for kk, v in rows if kk == k] for k, _ in rows}  # noqa: E731
    assert per_key(gpu) == per_key(host) and len(gpu) == len(host) and host
    assert ran and set(ran) == {"_GpuKeyJoinStep"}


def test_five_sides_stay_on_the_host(steps_run):
    ran, spied = steps_run
    side_items = [_values(50 + s, 20, 3) for s in range(5)]
    host, gpu = _both(side_items, "product", "final")
    assert gpu == host and host
    assert not ran and not spied
