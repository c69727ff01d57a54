"""NumPy's float32 summation order, restated.  TEST INFRASTRUCTURE ONLY.

`np.sum` over a contiguous float32 row (and `np.sum(x, axis=-1)` of a C-contiguous array) does not add the elements
in order: it calls `pairwise_sum` (numpy/_core/src/umath/loops_utils.h.src) and adds the result to the reduction's
identity, +0.0.  `pairwise_sum` over n elements
  - n < 8:        adds them in order;
  - 8 <= n <= 128: keeps 8 interleaved partial sums r[j] = x[j] + x[j + 8] + x[j + 16] + ... over the first n - n % 8
                  elements, combines them as ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then adds the last
                  n % 8 elements in order;
  - n > 128:      splits at n2 = n // 2 rounded down to a multiple of 8 and adds the two halves' pairwise sums.

The reference sums rows of RANGE_SIZE hands this way (ValueFiller.py:101, 110, 122).  For Leduc (6 hands) that is the
sequential order; for BigLeduc (24 hands) it is not.  oracle/cfr_oracle.c (`orc_pairwise_sum`) and the one-card CUDA
kernels (`numpy_sum` in pokerrl_b200/csrc/cfr_levels.cu) implement `pairwise_sum_f32`.  They leave out the +0.0
identity, which changes nothing but the sign of a zero total (see `numpy_sum_f32`).
"""
import numpy as np

_F = np.float32


def pairwise_sum_f32(x):
    """numpy's pairwise_sum of a 1-D float32 array, every addition rounded to float32."""
    x = np.asarray(x, dtype=np.float32)
    n = len(x)
    if n < 8:
        s = _F(-0.0)  # -0.0 + x0 == x0 for every x0, so this is "start from x0"
        for v in x:
            s = _F(s + v)
        return s
    if n <= 128:
        r = [_F(v) for v in x[:8]]
        i = 8
        while i < n - n % 8:
            for j in range(8):
                r[j] = _F(r[j] + x[i + j])
            i += 8
        s = _F(_F(_F(r[0] + r[1]) + _F(r[2] + r[3])) + _F(_F(r[4] + r[5]) + _F(r[6] + r[7])))
        for v in x[i:]:
            s = _F(s + v)
        return s
    n2 = n // 2
    n2 -= n2 % 8
    return _F(pairwise_sum_f32(x[:n2]) + pairwise_sum_f32(x[n2:]))


def numpy_sum_f32(x):
    """np.sum of a 1-D float32 array: the identity +0.0 plus the pairwise sum.  The identity only turns a total of
    -0.0 (all elements -0.0) into +0.0."""
    return _F(_F(0.0) + pairwise_sum_f32(x))
