"""pyprob_b200 — H100-native inference-compilation hot path of pyprob (see DESIGN.md).

``import pyprob_b200 as pyprob`` gives the reference's public names for the importance-sampling path:
Model, sample/observe/tag/factor, the enums, and ``pyprob_b200.distributions``.
"""
__version__ = '0.1.0'

from .util import (InferenceEngine, InferenceNetwork, LearningRateScheduler, ObserveEmbedding, Optimizer,  # noqa: F401
                   PriorInflation, TraceMode, seed, set_device, set_verbosity)
from .state import factor, observe, sample, tag, while_loop  # noqa: F401
from .model import Model  # noqa: F401
from . import distributions  # noqa: F401
from . import diagnostics  # noqa: F401
