# -*- coding: utf-8 -*-
"""stoke_b200 -- the H100-native engine behind fidelity/stoke's ``Stoke(...)`` / ``.model`` / ``.loss`` / ``.backward`` /
``.step`` API.  Same export list as the reference package (/root/reference/stoke/__init__.py:17-43)."""
from .configs import *  # noqa: F401,F403
from .configs import __all__ as _config_names
from .data import BucketedDistributedSampler, argsort_lengths
from .optim import LAMB, LARS
from .status import DistributedOptions, FP16Options
from .stoke import Stoke
from .utils import ParamNormalize

__all__ = ["Stoke", "ParamNormalize", "FP16Options", "DistributedOptions", "BucketedDistributedSampler",
           "argsort_lengths", "LAMB", "LARS"] + list(_config_names)
__version__ = "0.1.0"
