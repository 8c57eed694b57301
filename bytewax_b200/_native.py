"""ctypes binding of ``libbwgpu.so`` (the C ABI declared in ``include/bwgpu.h``).

This is the thin layer the reference's PyO3 module ``bytewax._bytewax``
(src/lib.rs:24-32) occupies: Python on top, native engine below.  There is no
CPU fallback: if the shared library is missing or no H100 is visible, every
entry point fails loudly.
"""

from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.environ.get("BWGPU_LIB") or os.path.join(HERE, "libbwgpu.so")
CSRC = os.path.join(HERE, "csrc")

BW_OK = 0
STATUS_NAMES = {
    0: "BW_OK", 1: "BW_ERR_CUDA", 2: "BW_ERR_NCCL", 3: "BW_ERR_CAPACITY", 4: "BW_ERR_SPEC",
    5: "BW_ERR_STATE", 6: "BW_ERR_RANGE", 7: "BW_ERR_NOMEM",
}
BW_WAIT_FOREVER = (1 << 63) - 1
RED = {"count": 0, "sum": 1, "min": 2, "max": 3, "mean": 4}
VAL = {"u64": 0, "i64": 1, "f32": 2, "f64": 3}
TS_COLUMN, TS_FROM_VALUE, TS_NONE = 0, 1, 2
ORDER_REFERENCE, ORDER_NONE = 0, 1
XCHG_P2P, XCHG_NCCL = 0, 1


class BwFoldSpec(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("reduction", C.c_int32), ("val_dtype", C.c_int32), ("ts_source", C.c_int32),
        ("length_us", C.c_int64), ("offset_us", C.c_int64), ("align_to_us", C.c_int64), ("wait_us", C.c_int64),
        ("ordered", C.c_int32), ("emit_order", C.c_int32), ("exchange", C.c_int32), ("ring_slots", C.c_int32),
        ("capacity_hint", C.c_uint64), ("max_batch_rows", C.c_uint64), ("max_emit_rows", C.c_uint64),
        ("max_late_rows", C.c_uint64),
    ]


class BwBatch(C.Structure):
    _fields_ = [
        ("keys", C.POINTER(C.c_uint64)), ("vals", C.c_void_p), ("ts_us", C.POINTER(C.c_int64)),
        ("capacity", C.c_uint64), ("slot", C.c_uint32), ("reserved", C.c_uint32),
    ]


class BwEmit(C.Structure):
    _fields_ = [
        ("n_closed", C.c_uint64), ("closed_key", C.POINTER(C.c_uint64)), ("closed_window_id", C.POINTER(C.c_int64)),
        ("closed_acc", C.POINTER(C.c_uint64)), ("closed_count", C.POINTER(C.c_uint64)),
        ("closed_epoch", C.POINTER(C.c_uint64)),
        ("n_late", C.c_uint64), ("late_key", C.POINTER(C.c_uint64)), ("late_window_id", C.POINTER(C.c_int64)),
        ("late_val", C.POINTER(C.c_uint64)), ("late_ts_us", C.POINTER(C.c_int64)), ("late_epoch", C.POINTER(C.c_uint64)),
    ]


class BwStats(C.Structure):
    _fields_ = [
        ("kernel_launches", C.c_uint64), ("rows_ingested", C.c_uint64), ("rows_received", C.c_uint64),
        ("slow_batches", C.c_uint64), ("live_keys", C.c_uint64), ("table_capacity", C.c_uint64),
        ("pane_nodes_used", C.c_uint64), ("last_fold_ms", C.c_float), ("sum_fold_ms", C.c_float),
        ("fold_launches", C.c_uint64), ("fold_rows", C.c_uint64), ("combined_folds", C.c_uint64),
        ("sum_scatter_ms", C.c_float), ("sum_verdict_ms", C.c_float), ("scatter_launches", C.c_uint64),
        ("split_batches", C.c_uint64), ("timed_folds", C.c_uint64), ("scatter_spill_rows", C.c_uint64),
    ]


class BwSnapshot(C.Structure):
    _fields_ = [("n", C.c_uint64), ("key", C.POINTER(C.c_uint64)), ("pane_id", C.POINTER(C.c_int64)), ("acc", C.POINTER(C.c_uint64)),
                ("count", C.POINTER(C.c_uint64)), ("open_seq", C.POINTER(C.c_uint64)), ("max_ts_us", C.POINTER(C.c_int64)),
                ("closed_upto", C.POINTER(C.c_int64)), ("batch_no", C.c_uint64), ("gmax_ts_us", C.c_int64), ("last_epoch", C.c_uint64)]


class BwSmapSpec(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("window", C.c_int32), ("val_dtype", C.c_int32), ("reserved", C.c_int32),
                ("threshold", C.c_double), ("capacity_hint", C.c_uint64), ("max_batch_rows", C.c_uint64)]


class BwJoinSpec(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("insert_mode", C.c_int32), ("emit_mode", C.c_int32), ("reserved", C.c_int32),
                ("capacity_hint", C.c_uint64), ("max_batch_rows", C.c_uint64), ("max_emit_rows", C.c_uint64)]


class BwJoinRows(C.Structure):
    _fields_ = [("n", C.c_uint64), ("key", C.POINTER(C.c_uint64)), ("left", C.POINTER(C.c_uint64)), ("right", C.POINTER(C.c_uint64)),
                ("mask", C.POINTER(C.c_uint64)), ("epoch", C.POINTER(C.c_uint64))]


class BwSessionSpec(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("reduction", C.c_int32), ("val_dtype", C.c_int32), ("max_sessions_per_key", C.c_int32),
                ("gap_us", C.c_int64), ("wait_us", C.c_int64), ("capacity_hint", C.c_uint64), ("max_batch_rows", C.c_uint64),
                ("max_emit_rows", C.c_uint64), ("max_late_rows", C.c_uint64)]


class BwSessionRows(C.Structure):
    _fields_ = [("n_closed", C.c_uint64), ("closed_key", C.POINTER(C.c_uint64)), ("closed_window_id", C.POINTER(C.c_int64)),
                ("closed_acc", C.POINTER(C.c_uint64)), ("closed_open_us", C.POINTER(C.c_int64)),
                ("closed_close_us", C.POINTER(C.c_int64)), ("closed_epoch", C.POINTER(C.c_uint64)),
                ("merged_off", C.POINTER(C.c_uint64)), ("merged_ids", C.POINTER(C.c_int64)),
                ("n_late", C.c_uint64), ("late_key", C.POINTER(C.c_uint64)), ("late_epoch", C.POINTER(C.c_uint64)),
                ("late_activation", C.POINTER(C.c_uint64)), ("late_row", C.POINTER(C.c_uint64))]


class BwJwinSpec(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("insert_mode", C.c_int32), ("emit_mode", C.c_int32), ("ordered", C.c_int32),
                ("sides", C.c_int32), ("max_windows_per_key", C.c_int32), ("length_us", C.c_int64), ("offset_us", C.c_int64),
                ("align_us", C.c_int64), ("wait_us", C.c_int64), ("capacity_hint", C.c_uint64), ("max_queued_rows", C.c_uint64),
                ("max_batch_rows", C.c_uint64), ("max_emit_rows", C.c_uint64), ("max_late_rows", C.c_uint64)]


class BwJwinRows(C.Structure):
    _fields_ = [("n_down", C.c_uint64), ("down_key", C.POINTER(C.c_uint64)), ("down_window_id", C.POINTER(C.c_int64)),
                ("down_handle", C.POINTER(C.c_uint64) * 4), ("down_mask", C.POINTER(C.c_uint64)), ("down_epoch", C.POINTER(C.c_uint64)),
                ("n_meta", C.c_uint64), ("meta_key", C.POINTER(C.c_uint64)), ("meta_window_id", C.POINTER(C.c_int64)),
                ("meta_epoch", C.POINTER(C.c_uint64)),
                ("n_late", C.c_uint64), ("late_key", C.POINTER(C.c_uint64)), ("late_window_id", C.POINTER(C.c_int64)),
                ("late_epoch", C.POINTER(C.c_uint64)), ("late_activation", C.POINTER(C.c_uint64)), ("late_row", C.POINTER(C.c_uint64)),
                ("n_released", C.c_uint64), ("released", C.POINTER(C.c_uint64))]


class BwCollectSpec(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("ordered", C.c_int32), ("max_windows_per_key", C.c_int32), ("pad", C.c_int32),
                ("length_us", C.c_int64), ("offset_us", C.c_int64), ("align_us", C.c_int64), ("wait_us", C.c_int64),
                ("capacity_hint", C.c_uint64), ("max_queued_rows", C.c_uint64), ("max_batch_rows", C.c_uint64),
                ("max_emit_rows", C.c_uint64), ("max_late_rows", C.c_uint64)]


class BwCollectRows(C.Structure):
    _fields_ = [("n_down", C.c_uint64), ("down_key", C.POINTER(C.c_uint64)), ("down_window_id", C.POINTER(C.c_int64)),
                ("down_epoch", C.POINTER(C.c_uint64)), ("down_offset", C.POINTER(C.c_uint64)), ("handle", C.POINTER(C.c_uint64)),
                ("n_late", C.c_uint64), ("late_key", C.POINTER(C.c_uint64)), ("late_window_id", C.POINTER(C.c_int64)),
                ("late_epoch", C.POINTER(C.c_uint64)), ("late_activation", C.POINTER(C.c_uint64)), ("late_row", C.POINTER(C.c_uint64)),
                ("n_released", C.c_uint64), ("released", C.POINTER(C.c_uint64))]


class BwSjwinSpec(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("insert_mode", C.c_int32), ("emit_mode", C.c_int32), ("ordered", C.c_int32),
                ("sides", C.c_int32), ("max_sessions_per_key", C.c_int32), ("gap_us", C.c_int64), ("wait_us", C.c_int64),
                ("capacity_hint", C.c_uint64), ("max_queued_rows", C.c_uint64), ("max_batch_rows", C.c_uint64),
                ("max_emit_rows", C.c_uint64), ("max_late_rows", C.c_uint64)]


class BwSjwinRows(C.Structure):
    _fields_ = [("n_down", C.c_uint64), ("down_key", C.POINTER(C.c_uint64)), ("down_window_id", C.POINTER(C.c_int64)),
                ("down_handle", C.POINTER(C.c_uint64) * 4), ("down_mask", C.POINTER(C.c_uint64)), ("down_epoch", C.POINTER(C.c_uint64)),
                ("n_meta", C.c_uint64), ("meta_key", C.POINTER(C.c_uint64)), ("meta_window_id", C.POINTER(C.c_int64)),
                ("meta_open_us", C.POINTER(C.c_int64)), ("meta_close_us", C.POINTER(C.c_int64)), ("meta_epoch", C.POINTER(C.c_uint64)),
                ("merged_off", C.POINTER(C.c_uint64)), ("merged_ids", C.POINTER(C.c_int64)),
                ("n_late", C.c_uint64), ("late_key", C.POINTER(C.c_uint64)), ("late_epoch", C.POINTER(C.c_uint64)),
                ("late_activation", C.POINTER(C.c_uint64)), ("late_row", C.POINTER(C.c_uint64)),
                ("n_released", C.c_uint64), ("released", C.POINTER(C.c_uint64))]


# every symbol include/bwgpu.h declares: (restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    "bw_abi_version": (C.c_uint32, []),
    "bw_last_error": (C.c_char_p, [_P]),
    "bw_last_global_error": (C.c_char_p, []),
    "bw_route": (C.c_uint32, [C.c_uint64, C.c_uint32]),
    "bw_nccl_unique_id": (C.c_int32, [_P]),
    "bw_ctx_create": (C.c_int32, [C.c_int, C.c_int, C.c_int, _P, C.POINTER(_P)]),
    "bw_ctx_destroy": (None, [_P]),
    "bw_loopback_create": (C.c_int32, [C.c_int, C.POINTER(_P)]),
    "bw_loopback_destroy": (None, [_P]),
    "bw_ctx_create_loopback": (C.c_int32, [C.c_int, C.c_int, _P, C.POINTER(_P)]),
    "bw_fold_create": (C.c_int32, [_P, C.POINTER(BwFoldSpec), C.POINTER(_P)]),
    "bw_fold_destroy": (None, [_P]),
    "bw_ingest_acquire": (C.c_int32, [_P, C.c_uint64, C.POINTER(BwBatch)]),
    "bw_ingest_commit": (C.c_int32, [_P, C.POINTER(BwBatch), C.c_uint64, C.c_uint64]),
    "bw_ingest_device": (C.c_int32, [_P, _P, _P, _P, C.c_uint64, C.c_uint64]),
    "bw_fold_set_system_now": (C.c_int32, [_P, C.c_int64]),
    "bw_advance": (C.c_int32, [_P, C.c_uint64, C.c_int64, C.POINTER(BwEmit)]),
    "bw_eof": (C.c_int32, [_P, C.POINTER(BwEmit)]),
    "bw_snapshot_take": (C.c_int32, [_P, C.POINTER(BwSnapshot)]),
    "bw_snapshot_load": (C.c_int32, [_P, C.POINTER(BwSnapshot)]),
    "bw_window_bounds": (None, [C.POINTER(BwFoldSpec), C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "bw_fold_stats": (C.c_int32, [_P, C.POINTER(BwStats)]),
    "bw_fold_reset_timers": (C.c_int32, [_P]),
    "bw_fold_sync": (C.c_int32, [_P]),
    "bw_fold_stream": (_P, [_P]),
    "bw_fold_time_begin": (C.c_int32, [_P]),
    "bw_fold_time_end": (C.c_int32, [_P, C.POINTER(C.c_float)]),
    "bw_gen_c1": (C.c_int32, [_P, _P, _P, C.c_uint64, C.c_uint64, C.c_uint64]),
    "bw_smap_create": (C.c_int32, [_P, C.POINTER(BwSmapSpec), C.POINTER(_P)]),
    "bw_smap_destroy": (None, [_P]),
    "bw_smap_apply": (C.c_int32, [_P, _P, _P, C.c_uint64, _P, _P, _P]),
    "bw_smap_apply_device": (C.c_int32, [_P, _P, _P, C.c_uint64, _P, _P, _P]),
    "bw_smap_sync": (C.c_int32, [_P]),
    "bw_join_create": (C.c_int32, [_P, C.POINTER(BwJoinSpec), C.POINTER(_P)]),
    "bw_join_destroy": (None, [_P]),
    "bw_join_apply": (C.c_int32, [_P, _P, _P, _P, C.c_uint64, C.c_uint64]),
    "bw_join_advance": (C.c_int32, [_P, C.POINTER(BwJoinRows)]),
    "bw_join_eof": (C.c_int32, [_P, C.POINTER(BwJoinRows)]),
    "bw_session_create": (C.c_int32, [_P, C.POINTER(BwSessionSpec), C.POINTER(_P)]),
    "bw_session_destroy": (None, [_P]),
    "bw_session_apply": (C.c_int32, [_P, _P, _P, _P, C.c_uint64, C.c_uint64, C.c_int64]),
    "bw_session_apply_device": (C.c_int32, [_P, _P, _P, _P, C.c_uint64, C.c_uint64, C.c_int64]),
    "bw_session_advance": (C.c_int32, [_P, C.c_int64, C.POINTER(BwSessionRows)]),
    "bw_session_eof": (C.c_int32, [_P, C.POINTER(BwSessionRows)]),
    "bw_jwin_create": (C.c_int32, [_P, C.POINTER(BwJwinSpec), C.POINTER(_P)]),
    "bw_jwin_destroy": (None, [_P]),
    "bw_jwin_apply": (C.c_int32, [_P, _P, _P, _P, _P, C.c_uint64, C.c_uint64, C.c_int64]),
    "bw_jwin_apply_device": (C.c_int32, [_P, _P, _P, _P, _P, C.c_uint64, C.c_uint64, C.c_int64]),
    "bw_jwin_advance": (C.c_int32, [_P, C.c_int64, C.POINTER(BwJwinRows)]),
    "bw_jwin_eof": (C.c_int32, [_P, C.POINTER(BwJwinRows)]),
    "bw_collect_create": (C.c_int32, [_P, C.POINTER(BwCollectSpec), C.POINTER(_P)]),
    "bw_collect_destroy": (None, [_P]),
    "bw_collect_apply": (C.c_int32, [_P, _P, _P, _P, C.c_uint64, C.c_uint64, C.c_int64]),
    "bw_collect_apply_device": (C.c_int32, [_P, _P, _P, _P, C.c_uint64, C.c_uint64, C.c_int64]),
    "bw_collect_advance": (C.c_int32, [_P, C.c_int64, C.POINTER(BwCollectRows)]),
    "bw_collect_eof": (C.c_int32, [_P, C.POINTER(BwCollectRows)]),
    "bw_sjwin_create": (C.c_int32, [_P, C.POINTER(BwSjwinSpec), C.POINTER(_P)]),
    "bw_sjwin_destroy": (None, [_P]),
    "bw_sjwin_apply": (C.c_int32, [_P, _P, _P, _P, _P, C.c_uint64, C.c_uint64, C.c_int64]),
    "bw_sjwin_apply_device": (C.c_int32, [_P, _P, _P, _P, _P, C.c_uint64, C.c_uint64, C.c_int64]),
    "bw_sjwin_advance": (C.c_int32, [_P, C.c_int64, C.POINTER(BwSjwinRows)]),
    "bw_sjwin_eof": (C.c_int32, [_P, C.POINTER(BwSjwinRows)]),
    "bw_dev_alloc": (C.c_int32, [_P, C.c_uint64, C.POINTER(_P)]),
    "bw_dev_free": (C.c_int32, [_P, _P]),
    "bw_host_alloc": (C.c_int32, [_P, C.c_uint64, C.POINTER(_P)]),
    "bw_host_free": (C.c_int32, [_P, _P]),
    "bw_memcpy": (C.c_int32, [_P, _P, _P, C.c_uint64, C.c_int]),
    "bw_flush_l2": (C.c_int32, [_P]),
}

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-shared",
    "-Xcompiler", "-fPIC",
]


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile ``csrc/bwgpu.cu`` for sm_90a into ``libbwgpu.so`` (in-tree)."""
    srcs = [os.path.join(CSRC, n) for n in sorted(os.listdir(CSRC))]
    srcs.append(os.path.join(ROOT, "include", "bwgpu.h"))
    if not force and os.path.exists(LIB_PATH):
        lib_m = os.path.getmtime(LIB_PATH)
        if all(os.path.getmtime(s) <= lib_m for s in srcs):
            return LIB_PATH
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, *NVCC_FLAGS, "-o", LIB_PATH, os.path.join(CSRC, "bwgpu.cu"), "-lnccl"]
    if verbose:
        print(" ".join(cmd), file=sys.stderr)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    return LIB_PATH


_lib = None


def load():
    """dlopen libbwgpu.so and type every symbol.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback for the GPU path)"
        )
    lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.bw_abi_version() != 1:
        raise RuntimeError("libbwgpu ABI version mismatch")
    _lib = lib
    return lib


class BwError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"{STATUS_NAMES.get(status, status)}: {msg}")
        self.status = status


def check(status: int, ctx=None):
    if status != BW_OK:
        lib = load()
        msg = lib.bw_last_error(ctx) if ctx else lib.bw_last_global_error()
        raise BwError(status, (msg or b"").decode(errors="replace"))
