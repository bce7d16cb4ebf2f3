"""Import the REAL reference's `imitation.algorithms.density` through the names-only shim (oracle/refimport.py).

TEST INFRASTRUCTURE; only usable where the reference sources are present (the GPU box has none).  That module needs two
names the shim does not carry: `gymnasium.spaces.utils` (its `flatten` of a Box, the array flattened, and of a
Discrete, one-hot; and the `FlatType` name) and `stable_baselines3.common.base_class.BasePolicy` (a return annotation).
`load()` attaches them to the shim's modules in this process, then imports the reference's module.
"""
import sys
import types
from typing import Any

import numpy as np

from . import refimport


def flatten(space, x):
    """gymnasium.spaces.utils.flatten for the Box and Discrete spaces of the shim."""
    if hasattr(space, "n") and not hasattr(space, "low"):
        onehot = np.zeros(space.n, dtype=space.dtype)
        onehot[int(x) - getattr(space, "start", 0)] = 1
        return onehot
    if hasattr(space, "low"):
        return np.asarray(x, dtype=space.dtype).flatten()
    raise NotImplementedError(f"density oracle: flatten of {type(space).__name__}")


def load():
    refimport.load()
    from gymnasium import spaces
    from stable_baselines3.common import base_class, policies

    if not hasattr(spaces, "utils"):
        utils = types.ModuleType("gymnasium.spaces.utils")
        utils.flatten, utils.FlatType = flatten, Any
        spaces.utils = utils
        sys.modules["gymnasium.spaces.utils"] = utils
    if not hasattr(base_class, "BasePolicy"):
        base_class.BasePolicy = policies.BasePolicy
    from imitation.algorithms import density

    return density
