"""Discounted CFR (Brown & Sandholm, "Solving Imperfect-Information Games via Discounted Regret Minimization", AAAI 2019):
the per-iteration factors, and the one place that knows their formula.

Iteration counter i (0-based, the engines' iter_counter), t = i + 1:
    a_t = t^alpha / (t^alpha + 1)   discount of a positive regret sum
    b_t = t^beta / (t^beta + 1)     discount of a negative regret sum
    w_t = t^gamma                   weight of the iteration's strategy in the reach-weighted average sum
each computed in float64 and rounded once to float32.  The kernels read them from a device table float32[n][3] indexed by
the counter (prl_buffers_t.dcfr / prl_board_game_t.dcfr), so a persistent launch over many iterations needs no host step.
DCFR(1, 1, 1) gives R_D(t) = R_L(t) / (t + 1) and the average sums of Linear CFR.

Predictive CFR+ weighs its average sums with the same w_t = t^gamma: its device table is the factor table of
pcfr_params(gamma), of which the kernels read column 2 only.
"""
import math

import numpy as np
import torch

DEFAULT = (1.5, 0.0, 2.0)  # the paper's recommendation


def check_params(alpha, beta, gamma):
    """(alpha, beta, gamma) as floats; ValueError unless all three are finite numbers"""
    try:
        p = tuple(float(x) for x in (alpha, beta, gamma))
    except (TypeError, ValueError):
        raise ValueError("DCFR alpha, beta, gamma must be numbers, got %r" % ((alpha, beta, gamma),)) from None
    if not all(math.isfinite(x) for x in p):
        raise ValueError("DCFR alpha, beta, gamma must be finite, got %r" % (p,))
    return p


def check_gamma(gamma):
    """PCFR+'s gamma as a float; ValueError unless it is a finite number"""
    try:
        g = float(gamma)
    except (TypeError, ValueError):
        raise ValueError("PCFR+ gamma must be a number, got %r" % (gamma,)) from None
    if not math.isfinite(g):
        raise ValueError("PCFR+ gamma must be finite, got %r" % (g,))
    return g


def pcfr_params(gamma):
    """the (alpha, beta, gamma) of PCFR+'s factor table: w_t = t^gamma in column 2 as DCFR's; alpha = beta = 1 fill the
    unread columns 0 and 1"""
    return (1.0, 1.0, check_gamma(gamma))


def factors(alpha, beta, gamma, n):
    """float32 [n, 3]: row i = {a_t, b_t, w_t} of iteration counter i (t = i + 1).  ValueError if a w_t is not finite in
    float32."""
    alpha, beta, gamma = check_params(alpha, beta, gamma)
    t = np.arange(1, int(n) + 1, dtype=np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        def disc(e):
            x = t ** e
            return np.where(np.isinf(x), 1.0, x / (x + 1.0))  # t^e beyond float64: the limit 1

        out = np.stack([disc(alpha), disc(beta), t ** gamma], axis=1).astype(np.float32)
    bad = ~np.isfinite(out[:, 2])
    if bad.any():
        raise ValueError("gamma = %r: the average weight t^gamma of iteration t = %d is not finite in float32"
                         % (gamma, int(np.argmax(bad)) + 1))
    return out


class FactorTable:
    """The device table of one solver, grown on the host before each call that updates with higher counters."""

    def __init__(self, params, device):
        self.params = check_params(*params)
        self.device = device
        self.host = np.zeros((0, 3), np.float32)
        self.t = None

    def ensure(self, n):
        """rows for counters 0 .. n - 1 exist on the device; returns the table's device pointer"""
        if n > self.host.shape[0]:
            try:  # room to grow; a gamma whose weights leave float32 early gets exactly the rows asked for
                self.host = factors(*self.params, max(int(n), 2 * self.host.shape[0], 1024))
            except ValueError:
                self.host = factors(*self.params, int(n))
            self.t = torch.from_numpy(self.host).to(self.device)
        return self.t.data_ptr()

    def w(self, i):
        """w_t of counter i (host float)"""
        self.ensure(i + 1)
        return float(self.host[i, 2])
