"""Timing of the session-window fold (K7, `bw_session_*`) on one GPU.

Workload: session `count_window`, gap 2 s, EventClock wait 1 s, frozen system clock, `max_sessions_per_key` 64 (a key
whose session keeps extending across activations holds the id of every session merged into it).  Each activation holds 2^24 rows
over 10^6 keys drawn uniformly (seeded), and covers the next 10 s of event time: row i of activation a is stamped
a * 10 s + i * 10 s / 2^24, plus a uniform jitter of +-1 s.  The columns are generated on the device before timing and
fed through `bw_session_apply_device`.  Two warm-up activations, then K timed ones, each ended by a device synchronise;
the rows of each activation are collected (`bw_session_advance`, not timed) before the next.  EOF closes the rest.

Conservation is checked at the end: the counts of every closed session plus the late rows must equal the rows ingested.

    python tools/bench_sessions.py [--steps K] [--warmup W]

Prints one JSON line: events/s over the timed activations, sessions closed, merges, late rows, and the card's name and
power limit as `nvidia-smi --query-gpu` reports them during the same run.
"""

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402  (before libbwgpu: torch loads its own NCCL first)

from bytewax_b200 import gpu  # noqa: E402

ROWS = 1 << 24
KEYS = 1_000_000
S = 1_000_000
A = 1_640_995_200_000_000


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as ex:  # noqa: BLE001 - reported, not fatal
        return f"unknown ({ex})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    ctx = gpu.Context(0)
    sess = gpu.SessionFold(ctx, "count", 2 * S, 1 * S, capacity_hint=KEYS, max_batch_rows=ROWS, max_emit_rows=ROWS,
                           max_late_rows=ROWS, max_sessions_per_key=64)
    g = torch.Generator(device="cuda").manual_seed(7)
    keys = torch.randint(0, KEYS, (ROWS,), device="cuda", generator=g, dtype=torch.int64)
    offs = torch.arange(ROWS, device="cuda", dtype=torch.int64) * (10 * S) // ROWS
    jitter = torch.randint(-S, S + 1, (ROWS,), device="cuda", generator=g, dtype=torch.int64)
    ts = torch.empty(ROWS, device="cuda", dtype=torch.int64)
    closed = counted = merges = lates = 0
    times = []

    def collect(rows):
        nonlocal closed, counted, merges, lates
        closed += rows.closed_key.size
        counted += int(rows.closed_acc.sum())
        merges += rows.merged_ids.size
        lates += rows.late_key.size

    t_adv = 0.0
    for a in range(args.warmup + args.steps):
        torch.add(offs, jitter, out=ts)
        ts.add_(A + a * 10 * S)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sess.apply_device(keys.data_ptr(), None, ts.data_ptr(), ROWS, epoch=a + 1)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        if a >= args.warmup:
            times.append(t1 - t0)
        collect(sess.advance())
        t_adv += time.perf_counter() - t1
    collect(sess.eof())
    sess.close()
    ctx.close()
    ingested = ROWS * (args.warmup + args.steps)
    ok = counted + lates == ingested
    name, power = card()
    res = {
        "workload": "session count_window, gap 2 s, wait 1 s, 2^24 rows x 10^6 keys per activation, 10 s event time, +-1 s jitter",
        "events_per_s": ROWS * len(times) / sum(times),
        "activation_ms_median": sorted(times)[len(times) // 2] * 1e3,
        "advance_ms_mean": t_adv / (args.warmup + args.steps) * 1e3,
        "timed_activations": len(times),
        "rows_ingested": ingested,
        "sessions_closed": closed,
        "merges": merges,
        "late_rows": lates,
        "conservation_ok": ok,
        "gpu": name,
        "power_limit": power,
    }
    print(json.dumps(res))
    if not ok:
        print(f"conservation failed: closed counts {counted} + late rows {lates} != rows ingested {ingested}", file=sys.stderr)
        sys.exit(1)


if __name__ == "__main__":
    main()
