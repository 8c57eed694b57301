"""Creating and destroying folds gives back all the device memory they took.

Free memory is read with torch.cuda.mem_get_info(): the library allocates with the CUDA runtime directly, so torch's
caching allocator does not see it.  Each case runs one warm-up cycle (module loading, lazily set kernel attributes),
then N measured cycles, and compares free memory after them with free memory after the warm-up.  The reading is
device-wide: another process allocating on the same GPU at the same moment can disturb it."""
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
# imported before libbwgpu is loaded: torch must load its own NCCL before the library loads the system one
torch = pytest.importorskip("torch")

A = 1_640_995_200_000_000
S = 1_000_000
CYCLES = 3
TOL = 32 << 20


def free_bytes():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def check_no_growth(cycle):
    cycle()
    before = free_bytes()
    for _ in range(CYCLES):
        cycle()
    after = free_bytes()
    assert before - after < TOL, f"{(before - after) / 2**20:.1f} MiB less free device memory after {CYCLES} cycles"


def loopback_cycle():
    """A world of two ranks on the streaming path: each fold shares a receive region of 2 sides x W x 128 segments x
    8192 partials x 32 B = 128 MiB with its peer."""
    from bytewax_b200 import _native as N, gpu

    world, n = 2, 1 << 14
    ctxs = gpu.Context.loopback_world(world)
    folds, errors = [None] * world, [None] * world

    def rank_main(r):
        try:
            fold = gpu.WindowFold(ctxs[r], "sum", 10 * S, None, A, 0, val_dtype="i64", capacity_hint=1 << 18,
                                  max_batch_rows=n, max_emit_rows=1 << 20, exchange=N.XCHG_P2P)
            folds[r] = fold
            rnd = np.random.default_rng(r)
            for b in range(3):
                ts = A + (b * world + r) * 10 * S + (np.arange(n) * 10 * S) // n
                fold.ingest(rnd.integers(0, 5000, n).astype(np.uint64), rnd.integers(-100, 100, n), ts)
            fold.advance()
            fold.eof()
            assert fold.stats().combined_folds == 3
        except BaseException as ex:  # noqa: BLE001 - reported by the main thread
            errors[r] = ex

    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for f in folds:  # every rank is done with its peer's memory
        if f is not None:
            f.close()
    for c in ctxs:
        c.close()
    for ex in errors:
        if ex is not None:
            raise ex


def single_fold_cycle():
    """One fold through every resource it makes on demand: ingest slots and stages, the side-stream flush of closed
    epochs, the late-row split, the sort path, a snapshot, the timing events and the generator's event."""
    from bytewax_b200 import gpu

    ctx = gpu.Context(0)
    n = 1 << 16
    fold = gpu.WindowFold(ctx, "sum", 1 * S, None, A, 2 * S, val_dtype="i64", capacity_hint=1 << 14, max_batch_rows=n,
                          max_emit_rows=1 << 20, max_late_rows=1 << 18)
    rnd = np.random.default_rng(7)
    keys = lambda: rnd.integers(0, 3000, n).astype(np.uint64)  # noqa: E731
    vals = lambda: rnd.integers(-1000, 1000, n)  # noqa: E731
    t = A
    for _ in range(4):  # in order, several windows per activation: rows of closed epochs flushed on the side stream
        fold.ingest(keys(), vals(), t + (np.arange(n) * 4 * S) // n)
        t += 4 * S
    ts = t + (np.arange(n) * 4 * S) // n
    ts[rnd.random(n) < 0.005] -= 30 * S  # a few stragglers: the late-row split
    fold.ingest(keys(), vals(), ts)
    t += 4 * S
    fold.ingest(keys(), vals(), t + rnd.integers(-100 * S, 4 * S, n))  # mostly late: the sort path
    t += 4 * S
    fold.advance()
    fold.snapshot()
    fold.time_begin()
    fold.ingest(keys(), vals(), t + (np.arange(n) * 4 * S) // n)
    fold.time_end()
    d_keys, d_vals = ctx.dev_alloc(n * 8), ctx.dev_alloc(n * 8)
    fold.gen_c1(d_keys, d_vals, 0, n, 1000)
    fold.sync()
    ctx.dev_free(d_keys)
    ctx.dev_free(d_vals)
    fold.eof()
    st = fold.stats()
    assert st.split_batches >= 1 and st.slow_batches >= 1, (st.split_batches, st.slow_batches)
    fold.close()
    ctx.close()


def test_loopback_folds_release_receive_regions(monkeypatch):
    monkeypatch.setenv("BW_STREAM", "1")
    check_no_growth(loopback_cycle)


def test_fold_releases_lazily_made_resources(monkeypatch):
    monkeypatch.setenv("BW_STREAM", "1")
    check_no_growth(single_fold_cycle)
