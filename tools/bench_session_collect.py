"""Timing of the collect within session windows (K12, `bw_scwin_*`) on one GPU.

Workload: `collect_window` over `SessionWindower` gap 2 s, EventClock wait 1 s, frozen system clock; once with
`ordered=True` (values played in timestamp order once the watermark passes them) and once with `ordered=False`
(sessions merge).  `max_sessions_per_key` is 64.  Each activation holds 2^24 rows over 10^6 keys drawn uniformly
(seeded) and covers the next 10 s of event time: row i of activation a is stamped a * 10 s + i * 10 s / 2^24, plus a
uniform jitter of +-1 s, and carries handle a * 2^24 + i.  The columns are generated on the device before timing and
fed through `bw_scwin_apply_device`.  Two warm-up activations, then K timed ones, each ended by a device synchronise;
the rows of each activation are collected (`bw_scwin_advance`, not timed) before the next.  EOF closes the rest.
The workload is K10's (tools/bench_session_join.py) and K9's (tools/bench_collect_window.py), so the three compare.

Conservation is checked at the end, on the device:
- every input handle is released exactly once;
- each handle in a list belongs to the row's key, and its ts lies in the session's [open, close];
- no handle is in two lists, and none of them is a late item's;
- list entries plus late rows equal the rows ingested.

    python tools/bench_session_collect.py [--steps K] [--warmup W]

Prints one JSON line per order: events/s over the timed activations, the median activation time, closed sessions,
merged ids, merge intervals, emitted handles, and the card's name and power limit as `nvidia-smi --query-gpu` reports
them during the same run.
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
SPAN = 10 * S
GAP = 2 * S


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as ex:  # noqa: BLE001 - reported, not fatal
        return f"unknown ({ex})", "unknown"


def run(ordered, steps, warmup):
    ctx = gpu.Context(0)
    j = gpu.SessionCollectWindow(ctx, ordered, GAP, S, capacity_hint=KEYS, max_sessions_per_key=64,
                                 max_queued_rows=ROWS if ordered else 0, max_batch_rows=ROWS, max_emit_rows=ROWS, max_late_rows=ROWS)
    n_act = warmup + steps
    g = torch.Generator(device="cuda").manual_seed(7)
    keys = torch.randint(0, KEYS, (ROWS,), device="cuda", generator=g, dtype=torch.int64)
    offs = torch.arange(ROWS, device="cuda", dtype=torch.int64) * SPAN // ROWS
    jitter = torch.randint(-S, S + 1, (ROWS,), device="cuda", generator=g, dtype=torch.int64)
    base_ts = offs + jitter  # handle h: key keys[h % ROWS], ts base_ts[h % ROWS] + A + (h // ROWS) * 10 s
    ts = torch.empty(ROWS, device="cuda", dtype=torch.int64)
    handles = torch.empty(ROWS, device="cuda", dtype=torch.int64)
    released = torch.zeros(ROWS * n_act, device="cuda", dtype=torch.int32)
    in_rows = torch.zeros(ROWS * n_act, device="cuda", dtype=torch.int32)  # list entries (+1 each) and late rows (+1)
    down = lates = merges = intervals = emitted = 0
    bad = 0
    times = []

    def collect(out):
        nonlocal down, lates, merges, intervals, emitted, bad
        down += out.down_key.size
        lates += out.late_key.size
        merges += int(out.merged_off[-1])
        intervals += int(out.merge_off[-1])
        emitted += out.handle.size
        if out.released.size:
            released.index_add_(0, torch.from_numpy(out.released.astype("int64")).cuda(), torch.ones(out.released.size, device="cuda", dtype=torch.int32))
        if out.late_key.size:
            h = torch.from_numpy((out.late_activation * ROWS + out.late_row).astype("int64")).cuda()
            in_rows.index_add_(0, h, torch.ones(h.numel(), device="cuda", dtype=torch.int32))
            bad += int((keys[h % ROWS] != torch.from_numpy(out.late_key.astype("int64")).cuda()).sum())
        if out.handle.size:
            cnt = torch.from_numpy(out.down_offset[1:].astype("int64") - out.down_offset[:-1].astype("int64")).cuda()
            k = torch.repeat_interleave(torch.from_numpy(out.down_key.astype("int64")).cuda(), cnt)
            lo = torch.repeat_interleave(torch.from_numpy(out.open_us).cuda(), cnt)
            hi = torch.repeat_interleave(torch.from_numpy(out.close_us).cuda(), cnt)
            h = torch.from_numpy(out.handle.astype("int64")).cuda()
            t = base_ts[h % ROWS] + A + (h // ROWS) * SPAN
            bad += int(((keys[h % ROWS] != k) | (t < lo) | (t > hi)).sum())
            in_rows.index_add_(0, h, torch.ones(h.numel(), device="cuda", dtype=torch.int32))

    for a in range(n_act):
        torch.add(base_ts, A + a * SPAN, out=ts)
        torch.add(torch.arange(ROWS, device="cuda", dtype=torch.int64), a * ROWS, out=handles)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        j.apply_device(keys.data_ptr(), handles.data_ptr(), ts.data_ptr(), ROWS, epoch=a + 1)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        if a >= warmup:
            times.append(t1 - t0)
        collect(j.advance())
    collect(j.eof())
    j.close()
    ctx.close()
    released_once = bool((released == 1).all())
    rows_once = bool((in_rows == 1).all())
    ok = released_once and rows_once and bad == 0 and emitted + lates == ROWS * n_act
    times.sort()
    return {
        "workload": f"collect_window list, session gap 2 s, wait 1 s, ordered={ordered}, 2^24 rows x 10^6 keys per activation",
        "events_per_s": ROWS * len(times) / sum(times),
        "activation_ms_median": times[len(times) // 2] * 1e3,
        "activation_ms_min": times[0] * 1e3,
        "activation_ms_max": times[-1] * 1e3,
        "timed_activations": len(times),
        "rows_ingested": ROWS * n_act,
        "closed_sessions": down,
        "merged_ids": merges,
        "merge_intervals": intervals,
        "emitted_handles": emitted,
        "late_rows": lates,
        "every_handle_released_once": released_once,
        "every_handle_in_one_row": rows_once,
        "lists_match_sessions": bad == 0,
        "conservation_ok": ok,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    name, power = card()
    ok = True
    for ordered in (True, False):
        res = run(ordered, args.steps, args.warmup)
        res.update(gpu=name, power_limit=power)
        print(json.dumps(res), flush=True)
        ok = ok and res["conservation_ok"]
    if not ok:
        print("conservation failed", file=sys.stderr)
        sys.exit(1)


if __name__ == "__main__":
    main()
