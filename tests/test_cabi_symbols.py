"""The C-ABI library builds for sm_90a, loads, and exports every symbol include/bwgpu.h declares.
No compute is called here (no GPU in this tier)."""

import ctypes as C
import os
import re
import subprocess

import pytest

from bytewax_b200 import _native as N
from oracle import pyoracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    N.build()
    return N.load()


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "bwgpu.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(bw_[a-z0-9_]+)\s*\(", src)))


def test_every_declared_symbol_is_exported_and_bound(lib):
    declared = _declared_symbols()
    assert len(declared) >= 25
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in bwgpu.h but not exported"
        assert name in N.SYMBOLS, f"{name} declared in bwgpu.h but not bound in _native.py"
    for name in N.SYMBOLS:
        assert name in declared, f"{name} bound but not declared in bwgpu.h"


def test_library_is_sm90a_only():
    out = subprocess.run(["cuobjdump", "-lelf", N.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs


def test_abi_version_and_struct_sizes(lib):
    assert lib.bw_abi_version() == 1
    assert C.sizeof(N.BwFoldSpec) == 96
    assert C.sizeof(N.BwBatch) == 40


def test_route_matches_oracle(lib):
    for world in (1, 2, 3, 4, 8):
        for key in [0, 1, 2, 999_999, 2**63, 2**64 - 1] + [po.splitmix64(i) for i in range(200)]:
            assert lib.bw_route(key, world) == po.dest_rank(key, world)
    # the hash spreads keys evenly
    counts = [0] * 8
    for i in range(8000):
        counts[lib.bw_route(i, 8)] += 1
    assert min(counts) > 800


def test_window_bounds_match_windower(lib):
    # WindowMetadata(open, close): windowing.py:620-623
    s = N.BwFoldSpec()
    s.length_us, s.offset_us, s.align_to_us = 10_000_000, 5_000_000, 1_640_995_200_000_000
    o, c = C.c_int64(), C.c_int64()
    for wid in (-3, -1, 0, 1, 7):
        lib.bw_window_bounds(C.byref(s), wid, C.byref(o), C.byref(c))
        assert (o.value, c.value) == po.SlidingWindower(s.length_us, s.offset_us, s.align_to_us).metadata_for(wid)


def test_no_gpu_fails_loudly(lib):
    """Without a device the product path must error, not fall back."""
    import ctypes

    try:
        import torch

        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    h = ctypes.c_void_p()
    st = lib.bw_ctx_create(0, 0, 1, None, ctypes.byref(h))
    if has_gpu:
        assert st == 0
        lib.bw_ctx_destroy(h)
    else:
        assert st == 1  # BW_ERR_CUDA
        assert b"CUDA device" in lib.bw_last_global_error()
        from bytewax_b200 import gpu

        with pytest.raises(N.BwError):
            gpu.Context(0)
