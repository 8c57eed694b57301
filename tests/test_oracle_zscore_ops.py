"""The correctly rounded twin of the z-score detector (the device's arithmetic) against the reference's arithmetic.

`po.ZScoreDetector(correctly_rounded=True)` squares with `d * d` and takes `math.sqrt`; the reference mapper writes
`** 2` and `** 0.5`, which CPython evaluates with libm `pow`, not always correctly rounded.  The sums are the builtin
`sum` in both, Neumaier-compensated on CPython >= 3.12.  So the mean must agree bit for bit, sigma within one ulp, and a
flag may differ only where z sits within a few ulp of the threshold."""

import math
import random
import sys

import pytest

from oracle import pyoracle as po
from oracle import streams

pytestmark = pytest.mark.skipif(sys.version_info < (3, 12), reason="sum() of floats is Neumaier-compensated from CPython 3.12")


def _drive(keys, vals, window, threshold, correctly_rounded):
    """Per row: (mu, sigma, flag, z), z being the value's distance from the previous mean in previous sigmas (None where the
    mapper's `if self.mu and self.sigma` suppresses the test)."""
    states, out = {}, []
    for k, v in zip(keys, vals):
        st = states.get(k)
        if st is None:
            st = states[k] = po.ZScoreDetector(window, threshold, correctly_rounded)
        z = abs(v - st.mu) / st.sigma if (st.mu and st.sigma) else None
        _, mu, sigma, flag = st.on_value(v)
        out.append((mu, sigma, flag, z))
    return out


def _compare(keys, vals, window, threshold):
    ref = _drive(keys, vals, window, threshold, False)
    twin = _drive(keys, vals, window, threshold, True)
    # run_zscore is the same detector behind the batch interface the GPU tests use
    assert [r[:3] for r in ref] == [tuple(r) for r in po.run_zscore([(keys, vals)], window, threshold)[0]]
    assert [r[:3] for r in twin] == [tuple(r) for r in po.run_zscore([(keys, vals)], window, threshold, correctly_rounded=True)[0]]
    sigma_ulps = flips = 0
    for i, ((mr, sr, fr, zr), (mt, st, ft, zt)) in enumerate(zip(ref, twin)):
        assert math.copysign(1, mr) == math.copysign(1, mt) and mr == mt, (i, mr, mt)
        assert abs(sr - st) <= math.ulp(st), (i, sr, st)
        sigma_ulps += sr != st
        assert (zr is None) == (zt is None), i
        if fr != ft:
            flips += 1
            assert (zr > threshold) != (zt > threshold), (i, zr, zt)
            assert abs(zr - threshold) <= 4 * math.ulp(threshold) and abs(zt - threshold) <= 4 * math.ulp(threshold), (i, zr, zt)
    return sigma_ulps, flips


@pytest.mark.parametrize("window", [1, 2, 3, 10, 31, 32])
@pytest.mark.parametrize("family", streams.ZSCORE_FAMILIES)
def test_twin_agrees_with_reference_arithmetic(family, window):
    rnd = random.Random(f"zscore-{family}-{window}")
    n = 3000
    keys = [rnd.randrange(12) for _ in range(n)]
    vals = [streams.zscore_value(family, rnd) for _ in range(n)]
    for threshold in (0.5, 2.0, 3.0):
        _compare(keys, vals, window, threshold)


def test_twin_sigma_differs_by_one_ulp_somewhere():
    """The two arithmetics are not the same function: over three-decimal windows sigma differs (by one ulp) in some rows."""
    rnd = random.Random(5)
    keys = [rnd.randrange(50) for _ in range(20000)]
    vals = [streams.zscore_value("dec3", rnd) for _ in keys]
    sigma_ulps, _ = _compare(keys, vals, 10, 2.0)
    assert sigma_ulps > 0


def test_flip_sequence():
    """One key's values on which the reference flags the last value anomalous and correctly rounded arithmetic does not:
    sigma differs by one ulp and z is 2.0000000000000004 against exactly 2.0."""
    vals = streams.ZSCORE_FLIP
    keys = [7] * len(vals)
    ref = _drive(keys, vals, 10, 2.0, False)
    twin = _drive(keys, vals, 10, 2.0, True)
    assert ref[-1][2] is True and twin[-1][2] is False
    assert ref[-1][3] == 2.0000000000000004 and twin[-1][3] == 2.0
    assert abs(ref[-2][1] - twin[-2][1]) == math.ulp(twin[-2][1])
    assert _compare(keys, vals, 10, 2.0)[1] == 1
