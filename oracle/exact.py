"""Exact accumulators of a windowed fold.  TEST INFRASTRUCTURE ONLY.

``fold(...)`` returns, for every ``(key, window_id)`` an input opens, the
accumulator computed with unbounded precision, so that the value limits of the
device's accumulators (64-bit carries, signed vs unsigned ops, the ordered float
encoding, f32 widening, the pane combine) can be checked independently of any
floating-point summation order.  Which rows are emitted, when and in which order
is NOT restated here: that stays with ``oracle/coracle.py`` (the order never
depends on the values).

Only inputs without late rows are accepted: every row's timestamp must be at
least its key's running maximum minus ``wait``.  A key then never loses its open
windows before EOF, nothing is late, and window membership is just the pane
formula of DESIGN.md section 3: a row at ``d = ts - align`` belongs to windows
``floor((d - length) / offset) + 1 .. floor(d / offset)``
(``SlidingWindower.intersects``, pysrc/bytewax/operators/windowing.py:611-618).

Rules per reduction (paths relative to the bytewax v0.21.1 source tree):

* count: the number of rows (windowing.py:1679-1689).
* integer sum: the Python ``int`` sum reduced mod 2^64 and read back with the
  dtype's signedness -- the documented device contract (DESIGN.md section 10,
  "64-bit integer sums wrap"); the reference's ints would not wrap.
* min / max: ``min(acc, v)`` / ``max(acc, v)`` in arrival order, seeded with the
  first value (``reduce_window``, windowing.py:2268-2285, with ``min`` / ``max``
  as the reducer, :2189 / :2236).  Python's ``min`` and ``max`` return their
  FIRST argument when neither is smaller / larger, so among equal values the one
  that arrived first is kept (this is what distinguishes ``-0.0`` from ``+0.0``).
* float sum and mean: ``FloatSum`` -- ``math.fsum`` of the values as binary64
  (the correctly rounded exact sum), the sum of their magnitudes and their number,
  so that a test can bound the error of f64 summation in any order.
"""

from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Iterable, Optional, Sequence, Tuple

M64 = 1 << 64
U = 2.0 ** -53  # unit roundoff of binary64


@dataclass(frozen=True)
class FloatSum:
    fsum: float     # math.fsum of the values: the exact sum, rounded once
    abs_sum: float  # sum of |x|
    n: int          # number of values (the MEAN divisor)

    def bound(self) -> float:
        """Largest error of ANY order of n - 1 binary64 additions of these values, measured against ``fsum``:
        (n - 1) u sum|x| for the additions (each rounds a partial sum no larger than sum|x|), plus u sum|x| for the
        rounding of ``fsum`` itself.  A single rounding to binary32 anywhere costs ~2^-24 relative: far outside."""
        return self.n * U * self.abs_sum * (1.0 + 2.0 * self.n * U)


def window_ids(ts: int, length_us: int, offset_us: int, align_us: int) -> range:
    d = ts - align_us
    return range((d - length_us) // offset_us + 1, d // offset_us + 1)


def _reduce(reduction: str, dtype: str, vals: Sequence):
    if reduction == "count":
        return len(vals)
    if reduction == "sum" and dtype in ("i64", "u64"):
        s = sum(vals) % M64
        return s - M64 if dtype == "i64" and s >= (1 << 63) else s
    if reduction in ("sum", "mean"):
        fv = [float(v) for v in vals]
        return FloatSum(math.fsum(fv), math.fsum(abs(v) for v in fv), len(fv))
    if reduction in ("min", "max"):
        pick = min if reduction == "min" else max
        acc = vals[0]
        for v in vals[1:]:
            acc = pick(acc, v)  # (returns acc unless v is strictly smaller / larger: the first of equals stays)
        return acc
    raise ValueError(reduction)


def _py_values(vals, n: int, dtype: str) -> list:
    if vals is None:
        return [0] * n
    if dtype in ("f32", "f64"):
        # an f32 value is the binary64 value it widens to (exact)
        return [float(v) for v in (vals.tolist() if hasattr(vals, "tolist") else vals)]
    out = [int(v) for v in (vals.tolist() if hasattr(vals, "tolist") else vals)]
    lo, hi = (-(1 << 63), 1 << 63) if dtype == "i64" else (0, M64)
    for v in out:
        if not lo <= v < hi:
            raise ValueError(f"value {v} does not fit {dtype}")
    return out


def fold(reduction: str, length_us: int, offset_us: Optional[int], align_us: int, wait_us: Optional[int],
         batches: Iterable[Tuple[Sequence[int], Sequence[int], Optional[Sequence]]], dtype: str = "i64") -> Dict[Tuple[int, int], object]:
    """``(key, window_id) -> exact accumulator`` over ``batches`` of ``(keys, ts_us, vals)`` in arrival order.
    ``wait_us=None`` is "wait forever".  Raises ``ValueError`` on a row that might be late."""
    offset_us = offset_us or length_us
    groups: Dict[Tuple[int, int], list] = {}
    max_ts: Dict[int, int] = {}
    for keys, ts, vals in batches:
        keys = [int(k) for k in (keys.tolist() if hasattr(keys, "tolist") else keys)]
        ts = [int(t) for t in (ts.tolist() if hasattr(ts, "tolist") else ts)]
        for k, t, v in zip(keys, ts, _py_values(vals, len(keys), dtype)):
            m = max_ts.get(k)
            if m is not None and wait_us is not None and t < m - wait_us:
                raise ValueError(f"key {k}: ts {t} may be late (key's maximum {m}, wait {wait_us})")
            max_ts[k] = t if m is None else max(m, t)
            for w in window_ids(t, length_us, offset_us, align_us):
                groups.setdefault((k, w), []).append(v)
    return {kw: _reduce(reduction, dtype, vs) for kw, vs in groups.items()}


def final(reduction: str, batches: Iterable[Tuple[Sequence[int], Optional[Sequence]]], dtype: str = "i64") -> Dict[int, object]:
    """``key -> exact accumulator`` of a ``*_final`` fold over ``batches`` of ``(keys, vals)`` in arrival order: what
    ``fold`` gives for window 0 with every row at the align, grouped with a stable numpy sort instead of a loop per row
    (the same ``_reduce`` per key, on the key's values in arrival order)."""
    import numpy as np

    batches = list(batches)
    keys = np.concatenate([np.asarray(k, dtype=np.uint64) for k, _ in batches])
    order = np.argsort(keys, kind="stable")
    vals = None if any(v is None for _, v in batches) else np.concatenate([np.asarray(v) for _, v in batches])[order]
    vals = _py_values(vals, len(keys), dtype)  # grouped by key, each key's in arrival order
    uk, start = np.unique(keys[order], return_index=True)
    ends = np.append(start[1:], len(keys)).tolist()
    return {k: _reduce(reduction, dtype, vals[s:e]) for k, s, e in zip(uk.tolist(), start.tolist(), ends)}
