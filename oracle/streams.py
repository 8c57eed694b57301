"""Seeded input streams of the golden cases, and the digest their expected rows are stored under.  TEST INFRASTRUCTURE
ONLY; needs nothing outside the repository (oracle/gen_golden.py, which runs the reference, imports it from here)."""

import hashlib
import json
import random

ALIGN_US = 1_640_995_200_000_000  # 2022-01-01T00:00:00Z


def spec_(reduction="count", length_us=10_000_000, offset_us=None, wait_us=0, ordered=False, align_us=ALIGN_US):
    return dict(
        reduction=reduction, length_us=length_us, offset_us=offset_us, wait_us=wait_us, ordered=ordered, align_us=align_us
    )


def gen_random(seed, n, n_keys, span_us, jitter_us, batch_sizes, fval=False, start_us=ALIGN_US, key_base=0):
    rnd = random.Random(seed)
    keys, ts, vals = [], [], []
    for i in range(n):
        base = start_us + (i * span_us) // n
        t = base + rnd.randint(-jitter_us, jitter_us) if jitter_us else base
        keys.append(key_base + rnd.randrange(n_keys))
        ts.append(t)
        vals.append(round(rnd.uniform(-100, 100), 3) if fval else rnd.randint(-1000, 1000))
    batches, i, b = [], 0, 0
    while i < n:
        sz = batch_sizes[b % len(batch_sizes)]
        batches.append([keys[i : i + sz], ts[i : i + sz], vals[i : i + sz]])
        i += sz
        b += 1
    return batches


def live_cases():
    """(name, spec, batches) of the two differential sweeps: 6 specs at seeds 30-35, 48 at seeds 100-147 (all five
    reductions, tumbling / sliding with divisible and indivisible offsets, waits from 0 to beyond the data span, ordered and
    unordered, timestamps on both sides of align_to, bursts of late items)."""
    S = 10**6
    for seed in range(30, 36):
        spec = spec_(["count", "sum", "min", "max"][seed % 4], 10 * S, [None, 5 * S, 3 * S][seed % 3], wait_us=(seed % 4) * S,
                     ordered=bool(seed % 2) and (seed % 4) < 2)
        yield f"random_{seed}", spec, gen_random(seed, 400, 7, 50 * S, 4 * S, [17, 60])
    for seed in range(100, 148):
        red = ["count", "sum", "min", "max", "mean"][seed % 5]
        length = [10 * S, 7 * S, 60 * S, 1 * S][seed % 4]
        offset = [None, length // 2 or None, 3 * S if 3 * S < length else None][seed % 3]
        wait = [0, S, 4 * S, 500 * S][(seed // 3) % 4]
        ordered = bool((seed // 5) % 2) and red in ("count", "sum", "mean")  # max/min_window are always unordered (windowing.py:2189, 2236)
        spec = spec_(red, length, offset, wait_us=wait, ordered=ordered)
        yield f"sweep_{seed}", spec, gen_random(seed, 300, 5, 40 * S, [0, 2 * S, 9 * S][seed % 3], [11, 50, 7], start_us=ALIGN_US - 15 * S)


def rows_digest(acts):
    """SHA-256 of the canonical JSON of per-activation rows [[key, window_id, tag, payload], ...]."""
    return hashlib.sha256(json.dumps(acts, separators=(",", ":")).encode()).hexdigest()


SNAPSHOT_CASES = [("count", 10, None, 0), ("sum", 10, None, 3), ("sum", 10, 5, 2), ("max", 12, 4, 1)]


def snapshot_case(red, length, offset, wait):
    """(spec, batches, cut) of a snapshot / resume case of tests/test_snapshot_rows.py: 12 activations of keys 1..9, some
    items up to 8 s late, lengths in seconds; the state is taken after activation `cut`."""
    S = 10**6
    spec = spec_(red, length * S, offset * S if offset else None, wait * S, False)
    rnd = random.Random(f"{red}-{length}")
    batches, t = [], ALIGN_US
    for _ in range(12):
        n = rnd.randint(20, 60)
        keys = [rnd.randint(1, 9) for _ in range(n)]
        ts = [t + rnd.randint(0, 6 * S) - (rnd.randint(0, 8 * S) if rnd.random() < 0.2 else 0) for _ in range(n)]
        t += 5 * S
        batches.append((keys, ts, [rnd.randint(-20, 20) for _ in range(n)]))
    return spec, batches, 6


def key_items(batches, key):
    """{arrival sequence (batch << 32 | index): (ts, value)} of `key`'s items, in arrival order."""
    return {bi << 32 | i: (t, v) for bi, (keys, ts, vals) in enumerate(batches) for i, (k, t, v) in enumerate(zip(keys, ts, vals)) if k == key}


def drive(logics, builder, chunk, unwrap, seq0, accepted=None, max_ts=None):
    """Run activations through per-key window logics the way the engine does (ascending key string, discard on done).
    Returns the (key, window, tag, payload) rows; with `accepted` / `max_ts` also records, per key, the items that were
    not late ((batch << 32 | index, ts, value)) and the newest accepted timestamp, forgetting them when the key is discarded."""
    rows = []
    for bi, (keys, ts, vals) in enumerate(chunk):
        grouped = {}
        for i, (k, tt, v) in enumerate(zip(keys, ts, vals)):
            grouped.setdefault(str(k), []).append((str(k), v, tt, (seq0 + bi) << 32 | i))
        for ks in sorted(grouped):
            logic = logics.get(ks)
            if logic is None:
                logic = logics[ks] = builder(None)
            events, done = logic.on_batch([(k, v, tt) for k, v, tt, _s in grouped[ks]])
            events = list(events)
            late_vals = [p[1] for _w, tag, p in events if tag == "L"]
            for k, v, tt, sq in grouped[ks]:
                if accepted is not None:
                    if late_vals and v in late_vals and any(p[2] == tt for _w, tag, p in events if tag == "L"):
                        continue
                    accepted.setdefault(int(ks), []).append((sq, tt, v))
                    max_ts[int(ks)] = max(max_ts.get(int(ks), -(1 << 63)), tt)
            rows.extend((ks, w, tag, (unwrap(p) if tag == "E" else None)) for w, tag, p in events if tag != "M")
            if done:
                del logics[ks]
                if accepted is not None:  # the key's state is gone with its logic (discard resets the watermark)
                    accepted.pop(int(ks), None)
                    max_ts.pop(int(ks), None)
    return rows
