"""Timing of the windowed collect (K9, `bw_collect_*`) on one GPU.

Workload: `collect_window` over 10 s tumbling windows, EventClock wait 1 s, frozen system clock; once with
`ordered=True` (values played in timestamp order once the watermark passes them), once with `ordered=False`, and once
unordered over 60 s / 10 s sliding windows (six entries per row).  Each activation holds 2^24 rows over 10^6 keys drawn
uniformly (seeded) and covers the next 10 s of event time: row i of activation a is stamped a * 10 s + i * 10 s / 2^24,
plus a uniform jitter of +-1 s.  Row i of activation a carries handle a * 2^24 + i.  The columns are generated on the
device before timing and fed through `bw_collect_apply_device`.  Two warm-up activations, then K timed ones, each
ended by a device synchronise; the rows of each activation are collected (`bw_collect_advance`, not timed) before the
next.  EOF flushes the rest.

Conservation is checked at the end, on the device: every input handle is released exactly once; every handle of a
list belongs to the list's key and window; the summed list lengths equal the on-time rows times their windows (with
aligned windows every row has length / offset of them, so lists + late rows == rows x windows per row).

    python tools/bench_collect_window.py [--steps K] [--warmup W]

Prints one JSON line per configuration: events/s over the timed activations, the median activation time, handles
emitted per second (list entries of the timed activations over their time), and the card's name and power limit as
`nvidia-smi --query-gpu` reports them during the same run.
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
STEP = 10 * S  # event time covered by one activation


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as ex:  # noqa: BLE001 - reported, not fatal
        return f"unknown ({ex})", "unknown"


def run(ordered, length, steps, warmup):
    offset = 10 * S
    per_row = length // offset
    ctx = gpu.Context(0)
    c = gpu.CollectWindow(ctx, ordered, length, offset, A, S, capacity_hint=KEYS, max_windows_per_key=8,
                          max_queued_rows=ROWS if ordered else 0, max_batch_rows=ROWS, max_emit_rows=ROWS, max_late_rows=ROWS * per_row)
    n_act = warmup + steps
    g = torch.Generator(device="cuda").manual_seed(7)
    keys = torch.randint(0, KEYS, (ROWS,), device="cuda", generator=g, dtype=torch.int64)
    offs = torch.arange(ROWS, device="cuda", dtype=torch.int64) * STEP // ROWS
    jitter = torch.randint(-S, S + 1, (ROWS,), device="cuda", generator=g, dtype=torch.int64)
    base_ts = offs + jitter  # handle h: key keys[h % ROWS], ts base_ts[h % ROWS] + A + (h // ROWS) * 10 s
    ts = torch.empty(ROWS, device="cuda", dtype=torch.int64)
    handles = torch.empty(ROWS, device="cuda", dtype=torch.int64)
    seen = torch.zeros(ROWS * n_act, device="cuda", dtype=torch.int32)
    lists = entries = lates = bad = 0
    timed_entries = 0
    times = []

    def collect(out, timed):
        nonlocal lists, entries, lates, bad, timed_entries
        lists += out.down_key.size
        entries += out.handle.size
        timed_entries += out.handle.size if timed else 0
        lates += out.late_key.size
        if out.released.size:
            seen.index_add_(0, torch.from_numpy(out.released.astype("int64")).cuda(), torch.ones(out.released.size, device="cuda", dtype=torch.int32))
        if out.handle.size:
            off = torch.from_numpy(out.down_offset.astype("int64")).cuda()
            row = torch.repeat_interleave(torch.arange(out.down_key.size, device="cuda"), off[1:] - off[:-1])
            k = torch.from_numpy(out.down_key.astype("int64")).cuda()[row]
            w = torch.from_numpy(out.down_window_id).cuda()[row]
            h = torch.from_numpy(out.handle.astype("int64")).cuda()
            t = base_ts[h % ROWS] + (h // ROWS) * STEP  # (relative to A == align)
            opn = w * offset
            bad += int(((keys[h % ROWS] != k) | (t < opn) | (t >= opn + length)).sum())

    for a in range(n_act):
        torch.add(base_ts, A + a * STEP, out=ts)
        torch.add(torch.arange(ROWS, device="cuda", dtype=torch.int64), a * ROWS, out=handles)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        c.apply_device(keys.data_ptr(), handles.data_ptr(), ts.data_ptr(), ROWS, epoch=a + 1)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        if a >= warmup:
            times.append(t1 - t0)
        collect(c.advance(), a >= warmup)
    collect(c.eof(), False)
    c.close()
    ctx.close()
    released_once = bool((seen == 1).all())
    counted = entries + lates == ROWS * n_act * per_row
    ok = released_once and bad == 0 and counted
    times.sort()
    shape = "tumbling 10 s" if length == offset else f"sliding {length // S} s / {offset // S} s"
    return {
        "workload": f"collect_window, {shape}, wait 1 s, ordered={ordered}, 2^24 rows x 10^6 keys per activation",
        "events_per_s": ROWS * len(times) / sum(times),
        "activation_ms_median": times[len(times) // 2] * 1e3,
        "handles_emitted_per_s": timed_entries / sum(times),
        "timed_activations": len(times),
        "rows_ingested": ROWS * n_act,
        "lists": lists,
        "list_entries": entries,
        "late_rows": lates,
        "every_handle_released_once": released_once,
        "lists_match_windows": bad == 0,
        "entries_plus_late_rows_equal_rows_times_windows": counted,
        "conservation_ok": ok,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    name, power = card()
    ok = True
    for ordered, length in ((True, 10 * S), (False, 10 * S), (False, 60 * S)):
        res = run(ordered, length, args.steps, args.warmup)
        res.update(gpu=name, power_limit=power)
        print(json.dumps(res), flush=True)
        ok = ok and res["conservation_ok"]
    if not ok:
        print("conservation failed", file=sys.stderr)
        sys.exit(1)


if __name__ == "__main__":
    main()
