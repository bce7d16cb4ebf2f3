"""Classic-control envs on the device: seals/CartPole-v0 and Pendulum-v1, stepped inside the rollout kernels.

Both never terminate and are cut at a fixed horizon (500 and 200 steps), so they run in lock-step like the synthetic
env and every rollout mode (plain, ensemble, exploration, DAgger) carries over.  The kernels step them thread per env in
float64 from the float32 observation, which is the env's whole state (DESIGN.md section 7e); `oracle/classic_env.py` is
their NumPy twin.  Reset draws come from the device's Philox stream, so they follow gymnasium's reset distributions but
not its PCG64 bits.
"""
from typing import Any, Callable, Mapping, Optional, Sequence

import numpy as np

from .. import _lib, spaces
from .synth import DeviceVecEnv

_F32_MAX = float(np.finfo(np.float32).max)

# env id -> (kind, d_obs, d_act, discrete, default horizon, observation space, action space)
_SPECS = {
    "seals/CartPole-v0": (_lib.ENV_CARTPOLE, 4, 2, True, 500,
                          lambda: spaces.Box(-np.array([_F32_MAX, _F32_MAX, np.pi, _F32_MAX]),
                                             np.array([_F32_MAX, _F32_MAX, np.pi, _F32_MAX]), (4,), np.float32),
                          lambda: spaces.Discrete(2)),
    "Pendulum-v1": (_lib.ENV_PENDULUM, 3, 1, False, 200,
                    lambda: spaces.Box(np.array([-1.0, -1.0, -8.0]), np.array([1.0, 1.0, 8.0]), (3,), np.float32),
                    lambda: spaces.Box(-2.0, 2.0, (1,), np.float32)),
}
SUPPORTED_ENVS = tuple(_SPECS)
# envs that end episodes early: the device rollout's closed-form transition order needs every env in lock-step
_TERMINATING = ("CartPole-v0", "CartPole-v1", "MountainCar-v0", "Acrobot-v1", "LunarLander-v2", "LunarLander-v3")


class ClassicVecEnv(DeviceVecEnv):
    """A `DeviceVecEnv` of `num_envs` copies of one classic-control env (`env_name` in SUPPORTED_ENVS), with the env's
    real spaces and horizon.  Env i has global id env_id_offset + i; the reset draws are keyed by `seed`."""

    def __init__(self, env_name: str, num_envs: int, *, horizon: Optional[int] = None, seed: int = 0,
                 env_id_offset: int = 0, device="cuda"):
        kind, d_obs, d_act, discrete, default_horizon, obs_space, act_space = _SPECS[env_name]
        horizon = default_horizon if horizon is None else int(horizon)
        if horizon < 1:
            raise ValueError(f"max_episode_steps must be >= 1, got {horizon}")
        self.env_name = env_name
        self._init_env(kind, d_obs, d_act, num_envs, discrete, horizon, seed, env_id_offset, device, obs_space(),
                       act_space())
        self.params = None  # the kernels read no parameters for these kinds


def make_vec_env(env_name: str, *, rng: np.random.Generator, n_envs: int = 8, parallel: bool = False,
                 log_dir: Optional[str] = None, max_episode_steps: Optional[int] = None,
                 post_wrappers: Optional[Sequence[Callable[[Any, int], Any]]] = None,
                 env_make_kwargs: Optional[Mapping[str, Any]] = None) -> ClassicVecEnv:
    """`imitation.util.util.make_vec_env` for the envs the device steps (util/util.py:80-167).

    Draws make_seeds(rng, n_envs) as the reference does, so a shared `rng` advances identically; the device env is keyed
    by the first seed.  `max_episode_steps` overrides the horizon.  `parallel` has no effect (there are no
    subprocesses: every env steps on the GPU).  `log_dir` (Monitor files), `post_wrappers` (per-env gym wrappers) and
    `env_make_kwargs` have no device counterpart and raise NotImplementedError.
    """
    del parallel
    if env_name not in _SPECS:
        if env_name in _TERMINATING:
            raise ValueError(f"{env_name!r} terminates episodes early; the device rollout steps fixed-horizon envs in "
                             f"lock-step (which gives its flattened transition order a closed form).  Use one of "
                             f"{', '.join(SUPPORTED_ENVS)}")
        raise ValueError(f"no device env {env_name!r}: supported are {', '.join(SUPPORTED_ENVS)}")
    if log_dir is not None:
        raise NotImplementedError("log_dir: the device env writes no Monitor files")
    if post_wrappers:
        raise NotImplementedError("post_wrappers: the device env is stepped inside the rollout kernel, so per-env gym "
                                  "wrappers cannot run")
    if env_make_kwargs:
        raise NotImplementedError(f"env_make_kwargs {dict(env_make_kwargs)!r}: the device envs have fixed constants")
    if n_envs < 1:
        raise ValueError(f"n_envs must be >= 1, got {n_envs}")
    seeds = rng.integers(0, (1 << 31) - 1, (n_envs,)).tolist()  # util.make_seeds(rng, n_envs)
    return ClassicVecEnv(env_name, n_envs, horizon=max_episode_steps, seed=int(seeds[0]))
