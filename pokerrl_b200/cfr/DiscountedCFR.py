"""Discounted CFR (Brown & Sandholm, "Solving Imperfect-Information Games via Discounted Regret Minimization", AAAI
2019), which the reference does not implement: Vanilla CFR's regret update followed by a discount of each regret sum,
t^alpha / (t^alpha + 1) where it is positive and t^beta / (t^beta + 1) where it is not, and a reach-weighted strategy sum
with weight t^gamma.  DCFR(1, 1, 1) is Linear CFR up to a positive factor of the regrets.  Same schedule, logging and
`eval_every` as the other three; factors: pokerrl_b200.dcfr, arithmetic: csrc/cfr_levels.cu, cfr_twocard.cu, cfr_board.cu."""
from pokerrl_b200 import dcfr as _dcfr
from pokerrl_b200.cfr._CFRBase import CFRBase as _CFRBase


class DiscountedCFR(_CFRBase):
    _SOLVER_ALGO = "DCFR"

    def __init__(self, name, chief_handle, game_cls, agent_bet_set, starting_stack_sizes=None, alpha=1.5, beta=0.0,
                 gamma=2.0, **engine_kw):
        self.alpha, self.beta, self.gamma = _dcfr.check_params(alpha, beta, gamma)
        super().__init__(name=name, chief_handle=chief_handle, game_cls=game_cls,
                         starting_stack_sizes=starting_stack_sizes, agent_bet_set=agent_bet_set,
                         algo_name="DCFR", dcfr=(self.alpha, self.beta, self.gamma), **engine_kw)
        self.reset()
