"""flashy_b200 -- a Hopper-native (H100) implementation of ``flashy.distrib``.

``flashy_b200.distrib`` exports exactly the reference module's names
(the reference's ``flashy/distrib.py``); see INTEGRATION.md for dropping it into a Flashy
checkout.  ``VirtualWorld`` hosts several virtual ranks on one GPU for rehearsal / testing.
"""
__version__ = "0.1.0"

from . import distrib  # noqa: F401
from .context import VirtualWorld  # noqa: F401
