from pokerrl_b200.cfr.DiscountedCFR import DiscountedCFR

__all__ = ["DiscountedCFR"]
