"""Predictive CFR+ (Farina, Kroer & Sandholm, "Faster Game Solving via Predictive Blackwell Approachability", AAAI 2021),
which the reference does not implement.  Seat p's update at iteration counter i (t = i + 1), with d = v(child) - v(node):

    R <- max(d + R, 0)          CFR+'s regret
    Q  = max(R + d, 0)          the prediction: the last instantaneous regret added to the new regret
    sigma = regret matching of Q (uniform where Q sums to 0), which the reach update and the next values use
    S += t^gamma * reach_p * sigma

The average strategy is the normalised S (gamma = 2: the paper's quadratic averaging).  The level engines keep sigma in their
strategy table, so Q needs no table of its own there; the board engine, which stores no strategy, keeps Q in a third table
of rows (`BoardCFRSolver.pred`).  Same schedule, logging and `eval_every` as the other algorithms; weights:
pokerrl_b200.dcfr, arithmetic: csrc/cfr_levels.cu, cfr_twocard.cu, cfr_board.cu (the PRED instantiations)."""
from pokerrl_b200 import dcfr as _dcfr
from pokerrl_b200.cfr._CFRBase import CFRBase as _CFRBase


class PredictiveCFRPlus(_CFRBase):
    _SOLVER_ALGO = "PCFRPlus"

    def __init__(self, name, chief_handle, game_cls, agent_bet_set, starting_stack_sizes=None, gamma=2.0, **engine_kw):
        self.gamma = _dcfr.check_gamma(gamma)
        super().__init__(name=name, chief_handle=chief_handle, game_cls=game_cls,
                         starting_stack_sizes=starting_stack_sizes, agent_bet_set=agent_bet_set,
                         algo_name="PCFRPlus", pcfr_gamma=self.gamma, **engine_kw)
        self.reset()
