"""numpy's float32 summation order (oracle/pairwise_sum.py), and the C oracle's copy of it, against np.sum itself.

The reference sums rows of hands with np.sum; for rows of 8 or more float32 elements that is numpy's pairwise order,
not a sequential loop.  The restatements must reproduce np.sum bit for bit, sign of zero included, at every row length
up to past the 128-element block where numpy splits the row in two."""
import ctypes as C

import numpy as np
import pytest

import cfr_c
from pairwise_sum import numpy_sum_f32, pairwise_sum_f32


def _rows(n, rng):
    """Rows of length n: wide exponent range with mixed signs, exact zeros of both signs, subnormals, cancellation,
    all -0.0, and sequences on which the sequential and the pairwise orders round differently."""
    rows = []
    for k in range(40):
        x = (rng.standard_normal(n) * np.exp2(rng.integers(-40, 40, n))).astype(np.float32)
        if k % 5 == 1:
            x[rng.random(n) < 0.4] = 0.0
        if k % 5 == 2:
            x[rng.random(n) < 0.4] = -0.0
        if k % 5 == 3:
            sub = np.float32(1e-42) * rng.integers(-700, 700, n).astype(np.float32)  # subnormals
            m = rng.random(n) < 0.5
            x[m] = sub[m]
        if k % 5 == 4:
            x = np.concatenate([x[: n // 2], -x[: n - n // 2]])  # cancelling halves
        rows.append(x)
    rows.append(np.full(n, -0.0, np.float32))
    rows.append(np.full(n, np.float32(1e-45)))
    rows.append(np.float32(1.0) / np.arange(1, n + 1, dtype=np.float32))
    rows.append(rng.random(n).astype(np.float32) / np.float32(n))  # like a reach row
    return rows


def _bits(v):
    return np.float32(v).view(np.uint32)


@pytest.mark.parametrize("n", range(1, 131))
def test_restatements_equal_np_sum(n):
    rng = np.random.default_rng(n)
    L = cfr_c.lib()
    for x in _rows(n, rng):
        want = _bits(np.sum(x))
        assert _bits(numpy_sum_f32(x)) == want, x
        c = np.float32(L.orc_pairwise_sum(x.ctypes.data_as(C.c_void_p), n))
        assert _bits(np.float32(0.0) + c) == want, x
        assert _bits(c) == _bits(pairwise_sum_f32(x)), x


def test_sequential_order_differs_from_np_sum_on_bigleduc_rows():
    """The reason for the restatement: on rows of 24 hands a plain loop often rounds differently from np.sum, on rows
    of Leduc's 6 hands never."""
    rng = np.random.default_rng(7)

    def seq(x):
        s = np.float32(0.0)
        for v in x:
            s = np.float32(s + v)
        return s

    diff = {6: 0, 24: 0}
    for n in diff:
        for _ in range(500):
            x = rng.random(n).astype(np.float32)
            diff[n] += _bits(seq(x)) != _bits(np.sum(x))
    assert diff[6] == 0 and diff[24] > 100, diff
