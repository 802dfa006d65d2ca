"""pips_b200: H100-native (sm_90a) implementation of the PIPs inference hot path.

``from pips_b200 import Pips`` is a drop-in for ``from nets.pips import Pips`` of aharley/pips.
"""
from .pips import Pips  # noqa: F401

__all__ = ["Pips"]
__version__ = "0.1.0"
