"""Timing of the windowed join (K8, `bw_jwin_*`) on one GPU.

Workload: `join_window` of 2 sides, insert mode last, emit mode final, 10 s tumbling windows, EventClock wait 1 s,
frozen system clock; once with `ordered=True` (values played in timestamp order once the watermark passes them) and
once with `ordered=False`.  Each activation holds 2^24 rows over 10^6 keys drawn uniformly (seeded), each on a random
side, and covers the next 10 s of event time: row i of activation a is stamped a * 10 s + i * 10 s / 2^24, plus a
uniform jitter of +-1 s.  Row i of activation a carries handle a * 2^24 + i.  The columns are generated on the device
before timing and fed through `bw_jwin_apply_device`.  Two warm-up activations, then K timed ones, each ended by a
device synchronise; the rows of each activation are collected (`bw_jwin_advance`, not timed) before the next.  EOF
flushes the rest.

Conservation is checked at the end, on the device: every input handle is released exactly once; every down row's
handles belong to the row's key and window; there is one down row per closed window.

    python tools/bench_join_window.py [--steps K] [--warmup W]

Prints one JSON line per order: events/s over the timed activations, the median activation time, rows, and the card's
name and power limit as `nvidia-smi --query-gpu` reports them during the same run.
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
LENGTH = 10 * S


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
    j = gpu.JoinWindow(ctx, "last", "final", ordered, 2, LENGTH, None, A, S, capacity_hint=KEYS, max_windows_per_key=8,
                       max_queued_rows=ROWS if ordered else 0, max_batch_rows=ROWS, max_emit_rows=ROWS, max_late_rows=ROWS)
    n_act = warmup + steps
    g = torch.Generator(device="cuda").manual_seed(7)
    keys = torch.randint(0, KEYS, (ROWS,), device="cuda", generator=g, dtype=torch.int64)
    sides = torch.randint(0, 2, (ROWS,), device="cuda", generator=g, dtype=torch.uint8)
    offs = torch.arange(ROWS, device="cuda", dtype=torch.int64) * LENGTH // ROWS
    jitter = torch.randint(-S, S + 1, (ROWS,), device="cuda", generator=g, dtype=torch.int64)
    base_ts = offs + jitter  # handle h: key keys[h % ROWS], ts base_ts[h % ROWS] + A + (h // ROWS) * 10 s
    ts = torch.empty(ROWS, device="cuda", dtype=torch.int64)
    handles = torch.empty(ROWS, device="cuda", dtype=torch.int64)
    seen = torch.zeros(ROWS * n_act, device="cuda", dtype=torch.int32)
    down = meta = lates = 0
    bad_rows = 0
    times = []

    def collect(out):
        nonlocal down, meta, lates, bad_rows
        down += out.down_key.size
        meta += out.meta_key.size
        lates += out.late_key.size
        if out.released.size:
            seen.index_add_(0, torch.from_numpy(out.released.astype("int64")).cuda(), torch.ones(out.released.size, device="cuda", dtype=torch.int32))
        if out.down_key.size:
            k = torch.from_numpy(out.down_key.astype("int64")).cuda()
            w = torch.from_numpy(out.down_window_id).cuda()
            for s in range(2):
                m = torch.from_numpy((out.down_mask >> s & 1).astype(bool)).cuda()
                h = torch.from_numpy(out.down_handles[:, s].astype("int64")).cuda()[m]
                t = base_ts[h % ROWS] + (h // ROWS) * LENGTH
                bad_rows += int(((keys[h % ROWS] != k[m]) | (torch.div(t, LENGTH, rounding_mode="floor") != w[m])).sum())

    for a in range(n_act):
        torch.add(base_ts, A + a * LENGTH, out=ts)
        torch.add(torch.arange(ROWS, device="cuda", dtype=torch.int64), a * ROWS, out=handles)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        j.apply_device(keys.data_ptr(), sides.data_ptr(), handles.data_ptr(), ts.data_ptr(), ROWS, epoch=a + 1)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        if a >= warmup:
            times.append(t1 - t0)
        collect(j.advance())
    collect(j.eof())
    j.close()
    ctx.close()
    released_once = bool((seen == 1).all())
    ok = released_once and bad_rows == 0 and down == meta
    times.sort()
    return {
        "workload": f"join_window last/final, 2 sides, tumbling 10 s, wait 1 s, ordered={ordered}, 2^24 rows x 10^6 keys per activation",
        "events_per_s": ROWS * len(times) / sum(times),
        "activation_ms_median": times[len(times) // 2] * 1e3,
        "timed_activations": len(times),
        "rows_ingested": ROWS * n_act,
        "down_rows": down,
        "meta_rows": meta,
        "late_rows": lates,
        "every_handle_released_once": released_once,
        "rows_match_windows": bad_rows == 0,
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
