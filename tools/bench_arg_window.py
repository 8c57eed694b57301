"""Timing of the windowed arg-max (K11, `bw_argwin_*`) on one GPU.

Workload: `max_window(..., by=)` over 10 s tumbling windows, 60 s / 10 s sliding windows (six windows per row) and
session windows with a 2 s gap; EventClock wait 1 s, frozen system clock.  Each activation holds 2^24 rows over 10^6
keys drawn uniformly (seeded) and covers the next 10 s of event time: row i of activation a is stamped a * 10 s +
i * 10 s / 2^24, plus a uniform jitter of +-1 s, carries handle a * 2^24 + i, and a by-value in -500..499 (many ties),
i64.  Sessions may number 64 per key: a key whose session keeps extending across activations holds the id of every
session merged into it.  The columns are generated on the device before timing and fed through
`bw_argwin_apply_device`.  Two warm-up activations, then K timed ones, each ended by a device synchronise; the rows of
each activation are collected (`bw_argwin_advance`, not timed) before the next.  EOF closes the rest.

Checked at the end: on the device, every input handle is released exactly once; on 64 sampled keys, with numpy, every
closed row's pick is an on-time item of its key inside the window whose by-value is the window's best, and for
tumbling and sliding windows the FIRST such item in arrival order.  (A session merge keeps the survivor's pick on a
tie, which may have arrived later than the merged-away session's.)

    python tools/bench_arg_window.py [--steps K] [--warmup W]

Prints one JSON line per configuration: events/s over the timed activations, the median activation time, and the card's
name and power limit as `nvidia-smi --query-gpu` reports them during the same run.
"""

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402  (before libbwgpu: torch loads its own NCCL first)

from bytewax_b200 import gpu  # noqa: E402

ROWS = 1 << 24
KEYS = 1_000_000
S = 1_000_000
A = 1_640_995_200_000_000
STEP = 10 * S  # event time covered by one activation
WAIT = S
SAMPLED = 64


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as ex:  # noqa: BLE001 - reported, not fatal
        return f"unknown ({ex})", "unknown"


def check_sampled(kind, sk_rows, closed, n_act, base_ts, by_of):
    """Per sampled key: replay the late test (frozen clock: late iff ts < max earlier ts - wait) and check each closed
    row's pick against its window's on-time items.  Returns the number of bad rows and of rows checked."""
    bad = checked = 0
    for k, rows in sk_rows.items():
        h = np.concatenate([a * ROWS + rows for a in range(n_act)])
        ts = base_ts[rows % ROWS][None, :].repeat(n_act, 0).reshape(-1) + np.repeat(np.arange(n_act) * STEP, len(rows))
        b = by_of(h)
        prev_max = np.maximum.accumulate(np.concatenate([[np.iinfo(np.int64).min + WAIT], ts[:-1]]))
        ontime = ts >= prev_max - WAIT
        for wid, pick, opn, cls in closed.get(k, []):
            inside = ontime & (ts >= opn) & ((ts <= cls) if kind == "session" else (ts < cls))
            if not inside.any():
                bad += 1
                continue
            best = b[inside].max()
            cand = h[inside][b[inside] == best]
            ok = pick in set(cand.tolist()) if kind == "session" else pick == int(cand[0])
            bad += not ok
            checked += 1
    return bad, checked


def run(kind, steps, warmup):
    length = 60 * S if kind == "sliding" else 10 * S
    per_row = 6 if kind == "sliding" else 1
    ctx = gpu.Context(0)
    common = dict(wait_us=WAIT, capacity_hint=KEYS, max_batch_rows=ROWS, max_emit_rows=ROWS, max_late_rows=ROWS * per_row)
    if kind == "session":
        a = gpu.ArgWindow(ctx, "max", "i64", gap_us=2 * S, max_windows_per_key=64, **common)
    else:
        a = gpu.ArgWindow(ctx, "max", "i64", length, 10 * S, 0, max_windows_per_key=8, **common)
    n_act = warmup + steps
    g = torch.Generator(device="cuda").manual_seed(7)
    keys = torch.randint(0, KEYS, (ROWS,), device="cuda", generator=g, dtype=torch.int64)
    offs = torch.arange(ROWS, device="cuda", dtype=torch.int64) * STEP // ROWS
    jitter = torch.randint(-S, S + 1, (ROWS,), device="cuda", generator=g, dtype=torch.int64)
    base_ts = offs + jitter  # handle h: key keys[h % ROWS], ts base_ts[h % ROWS] + A + (h // ROWS) * 10 s
    base_by = torch.randint(-500, 500, (ROWS,), device="cuda", generator=g, dtype=torch.int64)  # by: base_by[h % ROWS] ^ (h // ROWS)
    ts = torch.empty(ROWS, device="cuda", dtype=torch.int64)
    by = torch.empty(ROWS, device="cuda", dtype=torch.int64)
    handles = torch.empty(ROWS, device="cuda", dtype=torch.int64)
    seen = torch.zeros(ROWS * n_act, device="cuda", dtype=torch.int32)
    keys_np = keys.cpu().numpy()
    sampled = np.unique(keys_np)[:: max(1, len(np.unique(keys_np)) // SAMPLED)][:SAMPLED]
    sk_rows = {int(k): np.nonzero(keys_np == k)[0] for k in sampled}
    closed = {}
    n_closed = n_late = n_merged = 0
    times = []

    def collect(out):
        nonlocal n_closed, n_late, n_merged
        n_closed += out.closed_key.size
        n_late += out.late_key.size
        n_merged += out.merged_ids.size
        if out.released.size:
            seen.index_add_(0, torch.from_numpy(out.released.astype("int64")).cuda(), torch.ones(out.released.size, device="cuda", dtype=torch.int32))
        for i in np.nonzero(np.isin(out.closed_key, sampled.astype(np.uint64)))[0].tolist():
            closed.setdefault(int(out.closed_key[i]), []).append(
                (int(out.closed_window_id[i]), int(out.closed_handle[i]), int(out.closed_open_us[i]) - A, int(out.closed_close_us[i]) - A))

    for act in range(n_act):
        torch.add(base_ts, A + act * STEP, out=ts)
        torch.bitwise_xor(base_by, act, out=by)
        torch.add(torch.arange(ROWS, device="cuda", dtype=torch.int64), act * ROWS, out=handles)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        a.apply_device(keys.data_ptr(), handles.data_ptr(), by.data_ptr(), ts.data_ptr(), ROWS, epoch=act + 1)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        if act >= warmup:
            times.append(t1 - t0)
        collect(a.advance())
    collect(a.eof())
    a.close()
    ctx.close()
    released_once = bool((seen == 1).all())
    base_by_np = base_by.cpu().numpy()
    bad, checked = check_sampled(kind, sk_rows, closed, n_act, base_ts.cpu().numpy(),
                                 lambda h: base_by_np[h % ROWS] ^ (h // ROWS))
    ok = released_once and bad == 0 and checked > 0
    times.sort()
    shape = {"tumbling": "tumbling 10 s", "sliding": "sliding 60 s / 10 s", "session": "session gap 2 s"}[kind]
    return {
        "workload": f"max_window(by=), {shape}, wait 1 s, i64 by-values, 2^24 rows x 10^6 keys per activation",
        "events_per_s": ROWS * len(times) / sum(times),
        "activation_ms_median": times[len(times) // 2] * 1e3,
        "timed_activations": len(times),
        "rows_ingested": ROWS * n_act,
        "closed_rows": n_closed,
        "late_rows": n_late,
        "merged_ids": n_merged,
        "every_handle_released_once": released_once,
        "sampled_rows_checked": checked,
        "sampled_picks_are_first_best": bad == 0,
        "conservation_ok": ok,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    name, power = card()
    ok = True
    for kind in ("tumbling", "sliding", "session"):
        res = run(kind, args.steps, args.warmup)
        res.update(gpu=name, power_limit=power)
        print(json.dumps(res), flush=True)
        ok = ok and res["conservation_ok"]
    if not ok:
        print("conservation failed", file=sys.stderr)
        sys.exit(1)


if __name__ == "__main__":
    main()
