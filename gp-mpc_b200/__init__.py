"""gp_mpc_b200 -- H100-native (sm_90a) Gaussian-process regression engine behind the
``gp_mpc.GP`` API of helgeanl/GP-MPC.

Import name: ``gp_mpc_b200`` (the directory is ``gp-mpc_b200/``; the repo-root module
``gp_mpc_b200.py`` maps the importable name onto it).  ``GP`` is the drop-in for
``gp_mpc.gp_class.GP`` (reference gp_mpc/__init__.py:9); ``mpc_class.py`` and
``model_class.py`` stay on the host unchanged and are not part of this package.
"""
from . import _lib, optimize, partition            # noqa: F401
from ._lib import Engine, GpmpcError                # noqa: F401
from .comm import Comm                              # noqa: F401
from .gp_class import GP, lqr                       # noqa: F401

__all__ = ['GP', 'lqr', 'Engine', 'Comm', 'GpmpcError', 'optimize', 'partition']
