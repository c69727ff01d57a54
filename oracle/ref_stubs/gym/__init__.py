"""Minimal stand-in for `gym` (absent in this image) so that the read-only PokerRL
reference checkout can be imported by the golden-vector generators.
Test infrastructure only: PokerRL uses gym.spaces solely to *describe* the observation
space (PokerEnv.py:8, 189-197, 260-261, 329-330)."""
from . import spaces  # noqa: F401
