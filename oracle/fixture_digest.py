"""Digests of per-node arrays, and the formula strategy profile.  TEST INFRASTRUCTURE ONLY.

BigLeduc's per-node arrays (12 207 nodes x 2 seats x 24 hands, per snapshot) would make fixtures of ~14 MB, so its
fixtures store SHA-256 digests of them.  The generator (oracle/gen_golden_cfr.py) and the tests hash the same
DFS-ordered arrays with `array_digest`.

A digest compares arrays the way `np.array_equal(a, b, equal_nan=True)` does: the sign of a zero and the payload of a
NaN are canonicalised first.  Dtype and shape are part of the digest.
"""
import hashlib

import numpy as np


def array_digest(a):
    a = np.array(a, copy=True, order="C")
    if a.dtype.kind == "f":
        a[a == 0] = 0
        a[np.isnan(a)] = np.nan
    h = hashlib.sha256()
    h.update(("%s%s" % (a.dtype.str, a.shape)).encode())
    h.update(a.tobytes())
    return h.hexdigest()


def _mix(x):
    """splitmix64 finaliser on python ints"""
    m = (1 << 64) - 1
    x = (x + 0x9E3779B97F4A7C15) & m
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & m
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & m
    return x ^ (x >> 31)


def formula_strategy(dfs_index, n_actions, n_hands):
    """[n_hands, n_actions] float64 strategy of the decision node with DFS pre-order index `dfs_index`.

    Row h is drawn from _mix(dfs_index, h): a quarter of the rows are pure (one action 1.0, the rest exact zeros);
    the others weight action k by an integer 0..3 from _mix(dfs_index, h, k), normalised in float64, so that they
    mix zeros with unequal probabilities."""
    out = np.zeros((n_hands, n_actions), np.float64)
    for h in range(n_hands):
        x = _mix((dfs_index << 8) | h)
        if x % 4 == 0:
            out[h, (x >> 2) % n_actions] = 1.0
            continue
        w = np.array([_mix((x << 8) | k) % 4 for k in range(n_actions)], np.float64)
        if w.sum() == 0:
            w[(x >> 2) % n_actions] = 1.0
        out[h] = w / w.sum()
    return out
