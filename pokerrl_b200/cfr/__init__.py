from pokerrl_b200.cfr.DiscountedCFR import DiscountedCFR
from pokerrl_b200.cfr.PredictiveCFRPlus import PredictiveCFRPlus

__all__ = ["DiscountedCFR", "PredictiveCFRPlus"]
