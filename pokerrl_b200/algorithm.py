"""The CFR algorithms as every engine runs them on the host (solver, distributed, board_engine, the tabular agents): ABI
codes, parameters, where the average strategy is, the weight of an iteration in the average sums and the checkpoint keys
that name an algorithm.  DCFR's formula, and the t^gamma average weight PCFR+ shares with it, live in pokerrl_b200.dcfr."""
from pokerrl_b200 import _native as nat
from pokerrl_b200 import dcfr as _dcfr

ALGOS = {"VanillaCFR": nat.ALGO_VANILLA, "CFRPlus": nat.ALGO_CFR_PLUS, "LinearCFR": nat.ALGO_LINEAR, "DCFR": nat.ALGO_DCFR}
# Predictive CFR+ (Farina, Kroer & Sandholm, AAAI 2021), registered beside the four: it needs a table of predicted regrets
# on the board engine (allocated for it alone), and its checkpoints carry its own key (`pcfr_gamma`).  Every engine, and
# board_engine.supports / CFRBase, accept the names of ALL.
PREDICTIVE = {"PCFRPlus": nat.ALGO_PCFR_PLUS}
ALL = {**ALGOS, **PREDICTIVE}
PCFR_GAMMA = 2.0  # quadratic averaging, the paper's choice

CURRENT = "current"  # Algorithm.average: CFR+ at t == delay + 1, the current strategy (CFRPlus.py:83-84)
AVERAGE = "average"  # CFR+ after that: the average table
SUMS = "sums"        # the others: the reach-weighted sums, normalised (LinearCFR.py:64-71)


class Algorithm:
    """A CFR algorithm by name, with `delay` for CFR+ only, DCFR's (alpha, beta, gamma) for DCFR only and `pcfr_gamma` for
    PCFR+ only (ignored for the others); owns the factor table of DCFR / PCFR+ on `device` (`factors`: a dcfr.FactorTable,
    None for the others)."""

    def __init__(self, name, delay=0, dcfr=_dcfr.DEFAULT, device=None, pcfr_gamma=PCFR_GAMMA):
        if name not in ALL:
            raise ValueError("unknown algorithm %r (one of %s)" % (name, ", ".join(ALL)))
        self.name, self.code = name, ALL[name]
        self.delay = int(delay) if self.code == nat.ALGO_CFR_PLUS else 0
        self.dcfr = _dcfr.check_params(*dcfr) if self.code == nat.ALGO_DCFR else None
        self.pcfr_gamma = _dcfr.check_gamma(pcfr_gamma) if self.code == nat.ALGO_PCFR_PLUS else None
        params = self.dcfr if self.dcfr else _dcfr.pcfr_params(self.pcfr_gamma) if self.pcfr_gamma is not None else None
        self.factors = _dcfr.FactorTable(params, device) if params else None

    def factor_table(self, n):
        """DCFR / PCFR+: device pointer of the factor table covering iteration counters < n; None for the others"""
        return self.factors.ensure(n) if self.factors is not None else None

    def average(self, t):
        """CURRENT, AVERAGE or SUMS: which table is the average strategy after t iterations"""
        if self.code != nat.ALGO_CFR_PLUS:
            return SUMS
        if t <= self.delay:
            raise RuntimeError("CFR+ has no average strategy before iteration delay+1 (CFRPlus.py:33-35)")
        return CURRENT if t == self.delay + 1 else AVERAGE

    def sum_weight(self, t):
        """weight of iteration counter t's strategy in the average sums (VanillaCFR.py:56-59, LinearCFR.py:55-58, DCFR's w_t);
        None for CFR+, whose average is a running mean (CFRPlus.py:68-73)"""
        if self.code in (nat.ALGO_DCFR, nat.ALGO_PCFR_PLUS):
            return self.factors.w(t)
        return {nat.ALGO_VANILLA: 1.0, nat.ALGO_LINEAR: float(t + 1)}.get(self.code)

    def identity(self):
        """the checkpoint keys that name the algorithm (PCFR+ adds its gamma)"""
        ident = {"algo": self.name, "delay": self.delay, "dcfr": list(self.dcfr) if self.dcfr else None}
        if self.pcfr_gamma is not None:
            ident["pcfr_gamma"] = self.pcfr_gamma
        return ident


def check_identity(state, mine):
    """ValueError unless the checkpoint `state` has every key of `mine` with its value (a missing key reads None)"""
    for k, v in mine.items():
        if state.get(k) != v:
            raise ValueError("checkpoint mismatch on %r: file has %r, this solver %r" % (k, state.get(k), v))


def seat_averaged(expl, ev_normalizer):
    """the two seats' exploitabilities (chips) as one number in the game's unit (_CFRBase.py:198-216)"""
    return sum(float(expl[p]) * ev_normalizer for p in range(2)) / 2
