"""VecEnv type names (the reference's DAgger collector annotates step_wait with VecEnvStepReturn)."""
from typing import Any, Tuple

VecEnvStepReturn = Tuple[Any, Any, Any, Any]
