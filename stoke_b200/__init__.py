# -*- coding: utf-8 -*-
"""stoke_b200 -- the H100-native engine behind fidelity/stoke's ``Stoke(...)`` / ``.model`` / ``.loss`` / ``.backward`` /
``.step`` API.  Same export list as the reference package (/root/reference/stoke/__init__.py:17-43)."""
from .configs import *  # noqa: F401,F403
from .configs import __all__ as _config_names
from .data import BucketedDistributedSampler, argsort_lengths
from .optim import (LAMB, LARS, Adam8bit, AdamW8bit, AdEMAMix8bit, Adan, AdamWScheduleFree, AdEMAMix, Lion, Lion8bit,
                    MuonWithAuxAdamW, RMSpropTF, SGDScheduleFree, StableAdamW)
from .status import DistributedOptions, FP16Options
from .stoke import Stoke
from .utils import ParamNormalize
from .weight_average import WeightAverage

__all__ = ["Stoke", "ParamNormalize", "FP16Options", "DistributedOptions", "BucketedDistributedSampler",
           "argsort_lengths", "LAMB", "LARS", "Lion", "AdamWScheduleFree", "SGDScheduleFree", "AdEMAMix",
           "RMSpropTF", "Adan", "AdamW8bit", "Adam8bit", "Lion8bit", "AdEMAMix8bit", "StableAdamW", "MuonWithAuxAdamW",
           "WeightAverage"] + list(_config_names)
__version__ = "0.1.0"
