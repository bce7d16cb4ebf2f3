from .classic import SUPPORTED_ENVS, ClassicVecEnv, make_vec_env  # noqa: F401
from .synth import DeviceVecEnv  # noqa: F401
