"""Every CUDA resource of the host library has one owner.

bwgpu.cu makes and releases device memory, pinned host memory, events and streams only inside its `Owner` type: the fold,
the smap and the join each hold one, so destroying an object, or a create that fails halfway, frees all of it.  A few
entry points manage memory the caller or the context holds and are named here."""

import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "bytewax_b200", "csrc", "bwgpu.cu")

RAW = re.compile(r"\b(cudaMalloc\w*|cudaHostAlloc|cudaFree\w*|cudaEventCreate\w*|cudaEventDestroy|cudaStreamCreate\w*"
                 r"|cudaStreamDestroy)\s*\(")
# memory the caller owns (bw_dev_*, bw_host_*), the context's L2-flush buffer, and the snapshot load's staging copy
ALLOWED = ["bw_dev_alloc", "bw_dev_free", "bw_host_alloc", "bw_host_free", "bw_ctx_destroy", "bw_flush_l2",
           "bw_snapshot_load"]


def _source():
    src = open(SRC).read()
    # blank out comments, keeping offsets and line numbers
    return re.sub(r"//[^\n]*|/\*.*?\*/", lambda m: re.sub(r"[^\n]", " ", m.group(0)), src, flags=re.S)


def _body(src, header):
    """(start, end) of the first definition whose header matches, up to its closing brace."""
    m = re.search(header, src, flags=re.M)
    assert m, f"no definition matching {header!r} in bwgpu.cu"
    depth, i = 0, src.index("{", m.end() - 1)
    for j in range(i, len(src)):
        depth += {"{": 1, "}": -1}.get(src[j], 0)
        if depth == 0:
            return m.start(), j + 1
    raise AssertionError(f"unbalanced braces after {header!r}")


def _spans(src):
    spans = {"Owner": _body(src, r"^class Owner\b[^;{]*\{")}
    for name in ALLOWED:
        spans[name] = _body(src, rf"^[\w*\s]+\b{name}\([^;{{]*\)\s*\{{")
    return spans


def test_raw_cuda_resource_calls_only_in_owner():
    src = _source()
    spans = _spans(src)
    inside = lambda pos: any(a <= pos < b for a, b in spans.values())  # noqa: E731
    stray = [f"line {src.count(chr(10), 0, m.start()) + 1}: {m.group(1)}" for m in RAW.finditer(src) if not inside(m.start())]
    assert not stray, "raw CUDA allocation / release outside Owner:\n" + "\n".join(stray)


def test_owner_makes_and_releases_every_kind():
    src = _source()
    a, b = _spans(src)["Owner"]
    calls = {m.group(1) for m in RAW.finditer(src[a:b])}
    for need in ("cudaMalloc", "cudaHostAlloc", "cudaEventCreateWithFlags", "cudaStreamCreateWithPriority", "cudaFree",
                 "cudaFreeHost", "cudaEventDestroy", "cudaStreamDestroy"):
        assert need in calls, need


def test_objects_hold_an_owner():
    src = _source()
    for obj in ("bw_fold", "bw_smap", "bw_join"):
        a, b = _body(src, rf"^struct {obj} \{{")
        assert re.search(r"^\s*Owner own;", src[a:b], flags=re.M), f"{obj} holds no Owner"
