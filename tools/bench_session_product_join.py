"""Timing of the windowed product join over session windows (K16, `bw_spjwin_*`) on one GPU, with K10 (`bw_sjwin_*`,
insert mode last) on the same stream for reference.

Workload: `join_window` of 2 sides, emit mode final, `SessionWindower` gap 2 s, EventClock wait 1 s, frozen system
clock; once with `ordered=True` and once with `ordered=False` (sessions merge).  `max_sessions_per_key` is 64.  Each
activation holds `--rows` rows (default 2^22) over 10^6 keys drawn uniformly (seeded), each on a random side, and covers
the next 10 s of event time: row i of activation a is stamped a * 10 s + i * 10 s / rows, plus a uniform jitter of
+-1 s; it carries handle a * rows + i.  (At 2^24 rows per activation a key's values lie 0.6 s apart on average, well
inside the gap, so its sessions rarely close and each closing session's product runs to hundreds of rows, which the
advance copies to the host; the default of 2^22 keeps that within host memory.  2^24 has not been measured.)  The
columns are generated on the device before timing and fed through `bw_spjwin_apply_device`.  Timed: one activation, apply_device then advance (host copies of the rows
included), each ended by a device synchronise; two warm-up activations, then K timed ones; median reported.  EOF closes
the rest.

Conservation, checked at the end on the device:
- every input handle is released exactly once;
- the final rows come as one run per closed session, in the order of the meta rows;
- each handle in a down row belongs to the row's key, and its ts lies in the session's [open, close];
- no handle is in two sessions, and none of them is a late item's; every input is a late row or in one session;
- the down rows equal the sum, over the closed sessions, of prod_s max(1, n_s), n_s the session's values on side s.

    python tools/bench_session_product_join.py [--steps K] [--warmup W] [--rows N]

Prints one JSON line per order and join, with the card's name and power limit as `nvidia-smi --query-gpu` reports them
during the same run.
"""

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402  (before libbwgpu: torch loads its own NCCL first)

from bytewax_b200 import gpu  # noqa: E402

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


def cu(a, dt="int64"):
    return torch.from_numpy(np.ascontiguousarray(a).astype(dt)).cuda()


def run(product, ordered, rows, steps, warmup):
    ctx = gpu.Context(0)
    kw = dict(capacity_hint=KEYS, max_sessions_per_key=64, max_queued_rows=rows if ordered else 0, max_batch_rows=rows,
              max_emit_rows=max(rows, KEYS), max_late_rows=rows)
    if product:
        j = gpu.SessionProductJoinWindow(ctx, "final", ordered, 2, GAP, S, max_product_rows=1 << 28, **kw)
    else:
        j = gpu.SessionJoinWindow(ctx, "last", "final", ordered, 2, GAP, S, **kw)
    n_act = warmup + steps
    g = torch.Generator(device="cuda").manual_seed(7)
    keys = torch.randint(0, KEYS, (rows,), device="cuda", generator=g, dtype=torch.int64)
    sides = torch.randint(0, 2, (rows,), device="cuda", generator=g, dtype=torch.uint8)
    offs = torch.arange(rows, device="cuda", dtype=torch.int64) * SPAN // rows
    jitter = torch.randint(-S, S + 1, (rows,), device="cuda", generator=g, dtype=torch.int64)
    base_ts = offs + jitter  # handle h: key keys[h % rows], side sides[h % rows], ts base_ts[h % rows] + A + (h // rows) * 10 s
    ts = torch.empty(rows, device="cuda", dtype=torch.int64)
    handles = torch.empty(rows, device="cuda", dtype=torch.int64)
    total = rows * n_act
    released = torch.zeros(total, device="cuda", dtype=torch.int32)
    late = torch.zeros(total, device="cuda", dtype=torch.int32)
    session = torch.full((total,), -1, device="cuda", dtype=torch.int64)  # the closed session a handle's rows name
    n_sess = 0
    down = meta = lates = merges = bad = 0
    prods = []  # per closed session: its down rows
    sess_sides = []  # per closed session: (n_0, n_1), counted from the handles its rows name
    times = []

    def collect(out):
        nonlocal down, meta, lates, merges, bad, n_sess
        nd, nm = out.down_key.size, out.meta_key.size
        down += nd
        meta += nm
        lates += out.late_key.size
        merges += int(out.merged_off[-1]) if nm else 0
        if out.released.size:
            released.index_add_(0, cu(out.released), torch.ones(out.released.size, device="cuda", dtype=torch.int32))
        if out.late_key.size:
            h = cu(out.late_activation * rows + out.late_row)
            late.index_add_(0, h, torch.ones(h.numel(), device="cuda", dtype=torch.int32))
            bad += int((keys[h % rows] != cu(out.late_key)).sum())
        if not nd and not nm:
            return
        k, w = cu(out.down_key), cu(out.down_window_id)
        new = torch.ones(nd, device="cuda", dtype=torch.bool)
        new[1:] = (k[1:] != k[:-1]) | (w[1:] != w[:-1])
        run_id = torch.cumsum(new.to(torch.int64), 0) - 1  # each down row's closed session, in meta order
        starts = torch.nonzero(new).flatten()
        if starts.numel() != nm or (k[starts] != cu(out.meta_key)).any() or (w[starts] != cu(out.meta_window_id)).any():
            bad += 1  # final rows not one run per closed session in meta order
            return
        if not product:
            run_id = torch.arange(nd, device="cuda", dtype=torch.int64)
        lo, hi = cu(out.meta_open_us)[run_id], cu(out.meta_close_us)[run_id]
        counts = torch.bincount(run_id, minlength=nm)
        n = torch.zeros((nm, 2), device="cuda", dtype=torch.int64)
        for s in range(2):
            m = cu((out.down_mask >> s & 1).astype(bool), "bool")
            h = cu(out.down_handles[:, s])[m]
            r = run_id[m]
            t = base_ts[h % rows] + A + (h // rows) * SPAN
            bad += int(((keys[h % rows] != k[m]) | (t < lo[m]) | (t > hi[m]) | (sides[h % rows] != s)).sum())
            # distinct handles per session: a handle names one session only
            uh, inv = torch.unique(h, return_inverse=True)
            first = torch.full((uh.numel(),), -1, device="cuda", dtype=torch.int64)
            first.scatter_reduce_(0, inv, r, reduce="amax", include_self=True)
            lowest = torch.full((uh.numel(),), 1 << 62, device="cuda", dtype=torch.int64)
            lowest.scatter_reduce_(0, inv, r, reduce="amin", include_self=True)
            bad += int((first != lowest).sum()) + int((session[uh] >= 0).sum())
            session[uh] = first + n_sess
            n[:, s] = torch.bincount(first, minlength=nm)
        prods.append(counts)
        sess_sides.append(n)
        n_sess += nm

    for a in range(n_act):
        torch.add(base_ts, A + a * SPAN, out=ts)
        torch.add(torch.arange(rows, device="cuda", dtype=torch.int64), a * rows, out=handles)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        j.apply_device(keys.data_ptr(), sides.data_ptr(), handles.data_ptr(), ts.data_ptr(), rows, epoch=a + 1)
        out = j.advance()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        if a >= warmup:
            times.append(t1 - t0)
        collect(out)
    collect(j.eof())
    j.close()
    ctx.close()
    released_once = bool((released == 1).all())
    in_session = session >= 0
    placed_once = bool(((late == 1) ^ in_session).all()) if product else True
    ok = released_once and bad == 0
    res = {
        "workload": f"join_window {'product' if product else 'last'}/final, 2 sides, session gap 2 s, wait 1 s, ordered={ordered}, "
                    f"{rows} rows x 10^6 keys per activation",
        "activation_ms_median": sorted(times)[len(times) // 2] * 1e3,
        "events_per_s": rows * len(times) / sum(times),
        "timed_activations": len(times),
        "rows_ingested": total,
        "down_rows": down,
        "meta_rows": meta,
        "merged_ids": merges,
        "late_rows": lates,
        "every_handle_released_once": released_once,
        "rows_match_sessions": bad == 0,
    }
    if product:
        n = torch.cat(sess_sides) if sess_sides else torch.zeros((0, 2), device="cuda", dtype=torch.int64)
        want = int(n.clamp(min=1).prod(1).sum())
        got = int(torch.cat(prods).sum()) if prods else 0
        res.update(down_rows_expected=want, every_input_late_or_in_one_session=placed_once)
        ok = ok and placed_once and want == got == down
    res["conservation_ok"] = ok
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rows", type=int, default=1 << 22)
    args = ap.parse_args()
    name, power = card()
    ok = True
    for ordered in (False, True):
        for product in (True, False):
            res = run(product, ordered, args.rows, args.steps, args.warmup)
            res.update(gpu=name, power_limit=power)
            print(json.dumps(res), flush=True)
            ok = ok and res["conservation_ok"]
    if not ok:
        print("conservation failed", file=sys.stderr)
        sys.exit(1)


if __name__ == "__main__":
    main()
