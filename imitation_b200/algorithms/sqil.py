"""Soft Q Imitation Learning (mirror of imitation.algorithms.sqil; https://arxiv.org/abs/1905.11108).

`SQIL` trains a DQN (`algorithms.dqn.DeviceDQN`) whose replay buffer, `SQILReplayBuffer`, gives every learner
transition reward 0 and draws half of each minibatch from the demonstrations, which have reward 1.  Both buffers live
on the device: the learner ring as a feature-major transition table [tw][buffer_size] in SB3's (position, env) order,
the demonstrations as a feature-major table uploaded once.  With Discrete actions the learner is the device DQN and
the action columns are one-hot; with Box actions it is the device SAC (`algorithms.sac.SAC`) and the action columns
are the float actions.  TD3 and DDPG have no device port.

As in the reference, the expert rows hold the demonstrations' actions as recorded (env scale, e.g. [-2, 2] on
Pendulum-v1), while the learner rows hold SAC's buffer actions, scaled to [-1, 1]: `set_demonstrations` adds the
demonstrations unscaled.
"""
from typing import Any, Dict, List, NamedTuple, Optional, Tuple

import numpy as np
import torch as th

from .. import _lib, spaces
from ..data import rollout, types
from ..util import logger as imit_logger
from . import base as algo_base
from . import dqn, sac


def split_in_half(x: int) -> Tuple[int, int]:
    """util.split_in_half: (x // 2, x - x // 2)."""
    half = x // 2
    return half, x - half


class ReplayBufferSamples(NamedTuple):
    observations: th.Tensor
    actions: th.Tensor
    next_observations: th.Tensor
    dones: th.Tensor
    rewards: th.Tensor


class ExpertBuffer:
    """The demonstrations as SB3's ReplayBuffer(n_envs=1) holds them: observations / actions / next_observations
    [n][1][...], dones and rewards [n][1] (NumPy, host)."""

    def __init__(self, obs, acts, next_obs, dones, discrete: bool = True):
        n = len(obs)
        self.buffer_size = n
        self.observations = np.asarray(obs, np.float32).reshape(n, 1, -1)
        self.actions = (np.asarray(acts).astype(np.int64).reshape(n, 1, 1) if discrete
                        else np.asarray(acts, np.float32).reshape(n, 1, -1))
        self.next_observations = np.asarray(next_obs, np.float32).reshape(n, 1, -1)
        self.dones = np.asarray(dones, np.float32).reshape(n, 1)
        self.rewards = np.ones((n, 1), np.float32)
        self.pos, self.full = 0, True

    def size(self) -> int:
        return self.buffer_size


def _transitions(demonstrations) -> types.Transitions:
    """The reference's conversion: a Transitions object, or trajectories flattened; NotImplementedError otherwise."""
    if not isinstance(demonstrations, types.Transitions):
        try:
            items = list(demonstrations)
        except TypeError:
            items = []
        if items and isinstance(items[0], types.Trajectory):
            demonstrations = rollout.flatten_trajectories(items)
    if not isinstance(demonstrations, types.Transitions):
        raise NotImplementedError(f"Unsupported demonstrations type: {demonstrations}")
    return demonstrations


class SQILReplayBuffer:
    """A replay buffer that injects 50% expert demonstrations when sampling (sqil.py SQILReplayBuffer): SB3's
    ReplayBuffer with handle_timeout_termination=False, reward 0 for every added transition, and an expert buffer of
    reward-1 transitions."""

    def __init__(self, buffer_size: int, observation_space, action_space, demonstrations=None, device="auto",
                 n_envs: int = 1, optimize_memory_usage: bool = False):
        if optimize_memory_usage:
            raise NotImplementedError("optimize_memory_usage=True: the device ring stores next_obs beside obs")
        if not (spaces.is_discrete(action_space) or spaces.is_box(action_space)):
            raise NotImplementedError(f"action space {action_space!r}: the device SQIL runs Discrete and Box action "
                                      "spaces")
        self.observation_space, self.action_space = observation_space, action_space
        self.device = th.device("cuda" if device == "auto" else device)
        self.n_envs = int(n_envs)
        self.buffer_size = max(int(buffer_size) // self.n_envs, 1)
        self.discrete = spaces.is_discrete(action_space)
        # action columns: one-hot over n_actions (Discrete) or the d_act floats (Box)
        self.d_obs = spaces.flat_dim(observation_space)
        self.n_actions = int(action_space.n) if self.discrete else spaces.flat_dim(action_space)
        self.tw = 2 * self.d_obs + self.n_actions + 1
        self.capacity = self.buffer_size * self.n_envs
        self.ring = th.zeros(self.tw, self.capacity, device=self.device)
        self.pos, self.full = 0, False  # host mirrors of ring_state, which the device path reads and advances
        self.ring_state = th.zeros(_lib.ST_WORDS, dtype=th.int64, device=self.device)
        self.expert_buffer: Optional[ExpertBuffer] = None
        self.expert_table: Optional[th.Tensor] = None
        self.n_expert = 0
        if demonstrations is not None:
            self.set_demonstrations(demonstrations)

    def set_demonstrations(self, demonstrations) -> None:
        """Set the expert demonstrations to be injected when sampling; uploads them once as a feature-major table."""
        d = _transitions(demonstrations)
        n = len(d)
        self.expert_buffer = ExpertBuffer(d.obs, d.acts, d.next_obs, d.dones, self.discrete)
        table = np.zeros((self.tw, n), np.float32)
        Do, A = self.d_obs, self.n_actions
        table[:Do] = np.asarray(d.obs, np.float32).reshape(n, Do).T
        if self.discrete:
            acts = np.asarray(d.acts).astype(np.int64).reshape(n)
            table[Do + acts, np.arange(n)] = 1.0
        else:  # the recorded actions, unscaled (the reference adds the demonstrations as they are)
            table[Do:Do + A] = np.asarray(d.acts, np.float32).reshape(n, A).T
        table[Do + A:2 * Do + A] = np.asarray(d.next_obs, np.float32).reshape(n, Do).T
        table[2 * Do + A] = np.asarray(d.dones, np.float32).reshape(n)
        self.expert_table = th.as_tensor(table).to(self.device)
        self.n_expert = n

    # -- SB3 ReplayBuffer's host interface (not on the training path, which fills and samples on the device) -----------
    @property
    def observations(self) -> np.ndarray:
        return self._field(0, self.d_obs)

    @property
    def actions(self) -> np.ndarray:
        if not self.discrete:
            return self._field(self.d_obs, self.n_actions)
        return self._field(self.d_obs, self.n_actions).argmax(-1)[..., None].astype(np.int64)

    @property
    def next_observations(self) -> np.ndarray:
        return self._field(self.d_obs + self.n_actions, self.d_obs)

    @property
    def dones(self) -> np.ndarray:
        return self._field(self.tw - 1, 1)[..., 0]

    @property
    def rewards(self) -> np.ndarray:
        return np.zeros((self.buffer_size, self.n_envs), np.float32)

    def _field(self, c0: int, n: int) -> np.ndarray:
        """Rows [c0, c0 + n) of the ring as SB3's [buffer_size][n_envs][n] array."""
        return self.ring[c0:c0 + n].t().reshape(self.buffer_size, self.n_envs, n).cpu().numpy()

    def size(self) -> int:
        return self.buffer_size if self.full else self.pos

    def sync_ring_state(self) -> None:
        """Write the host's position and fill into the device counters (ring_state[RING_IDX], [RING_N])."""
        self.ring_state[_lib.ST_RING_IDX] = self.pos
        self.ring_state[_lib.ST_RING_N] = self.size()

    def add(self, obs, next_obs, action, reward, done, infos: List[Dict[str, Any]]) -> None:
        """Store one VecEnv step at the ring position (the reward is SQIL's 0 whatever is passed)."""
        E, Do, A = self.n_envs, self.d_obs, self.n_actions
        col = np.zeros((self.tw, E), np.float32)
        col[:Do] = np.asarray(obs, np.float32).reshape(E, Do).T
        if self.discrete:
            col[Do + np.asarray(action).astype(np.int64).reshape(E), np.arange(E)] = 1.0
        else:
            col[Do:Do + A] = np.asarray(action, np.float32).reshape(E, A).T
        col[Do + A:2 * Do + A] = np.asarray(next_obs, np.float32).reshape(E, Do).T
        col[2 * Do + A] = np.asarray(done, np.float32).reshape(E)
        self.ring[:, self.pos * E:(self.pos + 1) * E] = th.as_tensor(col).to(self.device)
        self.pos += 1
        if self.pos == self.buffer_size:
            self.full, self.pos = True, 0

    def _gather(self, table: th.Tensor, cols: np.ndarray, reward: float) -> ReplayBufferSamples:
        Do, A = self.d_obs, self.n_actions
        x = table[:, th.as_tensor(cols, device=self.device)].t()
        n = len(cols)
        acts = x[:, Do:Do + A].argmax(1, keepdim=True) if self.discrete else x[:, Do:Do + A]
        return ReplayBufferSamples(x[:, :Do], acts, x[:, Do + A:2 * Do + A],
                                   x[:, 2 * Do + A:], th.full((n, 1), reward, device=self.device))

    def sample(self, batch_size: int, env=None) -> ReplayBufferSamples:
        """Half learner transitions (first), half expert transitions, drawn from the global NumPy RNG as SB3's
        ReplayBuffer.sample draws them."""
        n_l, n_e = split_in_half(batch_size)
        upper = self.buffer_size if self.full else self.pos
        bi = np.random.randint(0, upper, size=n_l)
        ei = np.random.randint(0, self.n_envs, size=(n_l,))
        new = self._gather(self.ring, bi * self.n_envs + ei, 0.0)
        xi = np.random.randint(0, self.n_expert, size=n_e)
        np.random.randint(0, 1, size=(n_e,))
        exp = self._gather(self.expert_table, xi, 1.0)
        return ReplayBufferSamples(*(th.cat((a, b)) for a, b in zip(new, exp)))


class SQIL(algo_base.DemonstrationAlgorithm):
    """Soft Q Imitation Learning (SQIL): a DQN (Discrete actions) or a SAC (Box actions) trained on a buffer that mixes
    reward-0 learner transitions with reward-1 demonstrations."""

    def __init__(self, *, venv, demonstrations, policy, custom_logger: Optional[imit_logger.HierarchicalLogger] = None,
                 rl_algo_class=dqn.DQN, rl_kwargs: Optional[Dict[str, Any]] = None):
        self.venv = venv
        rl_kwargs = dict(rl_kwargs or {})
        if "replay_buffer_class" in rl_kwargs:
            raise ValueError("SQIL uses a custom replay buffer: 'replay_buffer_class' not allowed.")
        if "replay_buffer_kwargs" in rl_kwargs:
            raise ValueError("SQIL uses a custom replay buffer: 'replay_buffer_kwargs' not allowed.")
        if rl_algo_class not in (dqn.DeviceDQN, sac.SAC):
            raise NotImplementedError(f"rl_algo_class {getattr(rl_algo_class, '__name__', rl_algo_class)!r}: the "
                                      "device SQIL trains DQN and SAC (TD3 / DDPG have no device port)")
        self.rl_algo = rl_algo_class(policy=policy, env=venv, replay_buffer_class=SQILReplayBuffer,
                                     replay_buffer_kwargs={"demonstrations": demonstrations}, **rl_kwargs)
        super().__init__(demonstrations=demonstrations, custom_logger=custom_logger)
        self.rl_algo.set_logger(self.logger)

    def set_demonstrations(self, demonstrations) -> None:
        self.rl_algo.replay_buffer.set_demonstrations(demonstrations)

    def train(self, *, total_timesteps: int, tb_log_name: str = "SQIL", **kwargs: Any):
        self.rl_algo.learn(total_timesteps=total_timesteps, tb_log_name=tb_log_name, **kwargs)

    @property
    def policy(self):
        return self.rl_algo.policy
