"""`from nbodykit_b200.lab import *` -- the subset of nbodykit.lab this package implements (lab.py:1-25)."""
import numpy  # noqa: F401

from . import CurrentMPIComm, set_options, setup_logging  # noqa: F401
from .source.catalog import *  # noqa: F401,F403
from .source.mesh import *  # noqa: F401,F403
from .algorithms import *  # noqa: F401,F403
from .binned_statistic import BinnedStatistic  # noqa: F401
from . import cosmology, transform  # noqa: F401
from .hod import HODModel, Hearin15Model, Leauthaud11Model, Zheng07Model  # noqa: F401
