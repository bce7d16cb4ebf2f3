"""GPU-resident batched VecEnv: the synthetic MuJoCo-shaped environment (SURVEY.md section 8d).

obs' = tanh(A obs + Bm u + c), reward = w.obs' - 0.1|u|^2 (u = clip(act,-1,1) or one-hot),
fixed horizon with SB3-VecEnv auto-reset semantics; state lives SoA [d_obs][E] in HBM and is
stepped by csrc/imb_rollout.cu.  One slice of the global env index space per rank
(`env_id_offset`) so that N GPUs roll out disjoint environments.
"""
import numpy as np
import torch as th

from .. import _desc, _lib, spaces


class DeviceVecEnv:
    """Duck-types the parts of SB3's VecEnv the reference's trainers read
    (`num_envs`, `observation_space`, `action_space`, `reset`)."""

    def __init__(self, d_obs: int, d_act: int, num_envs: int, *, discrete: bool = False, horizon: int = 1000,
                 seed: int = 0, env_id_offset: int = 0, device="cuda"):
        self._init_env(_lib.ENV_SYNTH, d_obs, d_act, num_envs, discrete, horizon, seed, env_id_offset, device,
                       spaces.Box(-np.inf, np.inf, (d_obs,), np.float32),
                       spaces.Discrete(d_act) if discrete else spaces.Box(-1.0, 1.0, (d_act,), np.float32))
        self.params = th.as_tensor(_desc.synth_env_params(d_obs, d_act, seed)).to(self.device)

    def _init_env(self, kind: int, d_obs: int, d_act: int, num_envs: int, discrete: bool, horizon: int, seed: int,
                  env_id_offset: int, device, observation_space, action_space) -> None:
        """Everything but the env's parameters (`self.params`, the synthetic env's matrices; None for the
        classic-control kinds, whose dynamics are fixed)."""
        self.num_envs = int(num_envs)
        self.kind = kind
        self.d_obs, self.d_act, self.discrete, self.horizon, self.seed = d_obs, d_act, discrete, horizon, seed
        self.observation_space, self.action_space = observation_space, action_space
        self.device = th.device(device)
        self.desc = _lib.EnvDesc(d_obs=d_obs, d_act=d_act, discrete=int(discrete), horizon=horizon, seed=seed,
                                 env_id_offset=env_id_offset, kind=kind)
        self.obs = th.zeros(d_obs, self.num_envs, device=self.device)  # SoA
        self.state = th.zeros(_lib.ST_WORDS, dtype=th.int64, device=self.device)
        self._reset_done = False
        self.host_ep_step = 0  # host mirror of state[ST_EP_STEP] (deterministic; avoids D2H reads)

    def reset(self) -> np.ndarray:
        """(Re)draw the initial observations; returns [E, d_obs] on the host like VecEnv.reset()."""
        if self._reset_done:
            self.state[_lib.ST_EPISODE] += 1
            self.state[_lib.ST_EP_STEP] = 0
            self.host_ep_step = 0
        _lib.env_reset(self.obs, self.num_envs, self.desc, self.state)
        self._reset_done = True
        return self.obs.t().contiguous().cpu().numpy()

    def ensure_reset(self) -> None:
        if not self._reset_done:
            _lib.env_reset(self.obs, self.num_envs, self.desc, self.state)
            self._reset_done = True

    def step_async(self, actions):
        raise NotImplementedError("DeviceVecEnv is stepped by the fused rollout kernel (DevicePPO.learn); "
                                  "host-side per-step stepping is not part of the GPU hot path")

    def step_wait(self):
        raise NotImplementedError("see step_async")

    def close(self):
        pass
