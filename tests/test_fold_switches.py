"""The window fold reads its environment switches in one place.

`read_switches` in bwgpu.cu reads every `BW_*` variable once, when a fold is created, into fields of `bw_fold`: a
switch then takes effect on every fold, whichever path the fold ends up on.  These are the switches the tests use to
force a path or a kernel configuration that production folds reach through other shapes."""

import os
import re

from tests.test_host_ownership import _body

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bytewax_b200", "csrc")

SWITCHES = {"BW_STREAM", "BW_LATE_SPLIT", "BW_FLUSH", "BW_TIMER_STRIDE", "BW_SC_STG", "BW_SC_EVERY", "BW_SC_STAGES",
            "BW_SEG_SHIFT"}
GETENV = re.compile(r"\bgetenv\s*\(")


def _uncommented(path):
    src = open(path).read()
    # blank out comments, keeping offsets
    return re.sub(r"//[^\n]*|/\*.*?\*/", lambda m: re.sub(r"[^\n]", " ", m.group(0)), src, flags=re.S)


def test_getenv_only_in_the_reader():
    stray = []
    for name in sorted(os.listdir(CSRC)):
        src = _uncommented(os.path.join(CSRC, name))
        a, b = _body(src, r"^static void read_switches\(") if name == "bwgpu.cu" else (0, 0)
        stray += [f"{name} line {src.count(chr(10), 0, m.start()) + 1}" for m in GETENV.finditer(src) if not a <= m.start() < b]
    assert not stray, "getenv outside read_switches:\n" + "\n".join(stray)


def test_reader_reads_exactly_the_switches():
    src = _uncommented(os.path.join(CSRC, "bwgpu.cu"))
    a, b = _body(src, r"^static void read_switches\(")
    body = src[a:b]
    names = re.findall(r"\bgetenv\s*\(\s*\"(\w+)\"\s*\)", body)
    assert len(names) == len(GETENV.findall(body)), "every getenv in read_switches names its variable"
    assert len(names) == len(set(names)), names
    assert set(names) == SWITCHES
