from pokerrl_b200.cfr.DiscountedCFR import DiscountedCFR
from pokerrl_b200.cfr.PredictiveCFRPlus import PredictiveCFRPlus
from pokerrl_b200.cfr.RestrictedNashResponse import RestrictedNashResponse

__all__ = ["DiscountedCFR", "PredictiveCFRPlus", "RestrictedNashResponse"]
